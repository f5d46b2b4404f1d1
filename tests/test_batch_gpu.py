"""Static batching (aha_b200_generate_batch; SURVEY 8f rank 4 -- the reference serves one request at a time, server/api.rs:117).

The reference's answer for a request does not depend on what else is being served, so every request of a batch is compared with its
OWN fresh oracle run (generate_generic / the restated sampler): ids must be equal, whatever the mix of lengths, samplers, stop
positions and modalities in the batch.  The batched GEMV is also checked on its own against numpy and against the exact SIMT GEMM."""
import os

import numpy as np
import pytest

from conftest import make_model, make_oracle

pytestmark = pytest.mark.gpu


def _ids(n, vocab, seed):
    from aha_b200 import synth
    return synth.synth_text_ids(n, vocab - 8, seed)


def _oracle_generate(o, ids, data, n, **samp):
    from test_prefix_cache_gpu import _oracle_generate as og
    return og(o, ids, data, n, **samp)


@pytest.fixture(scope="module")
def q3():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=2048)
    yield cfg, w, m, make_oracle("qwen3", cfg, w)
    m.close()


# N 4728 / 4736 and 9464 / 9472 sit on either side of gemv_pick_rpw's thresholds (N / 16 >= 296 -> 2 rows per warp, N / 32 >= 296 -> 4);
# the last four are the Qwen3-VL-8B text projections: qkv, o_proj, gate/up, down (K = 12288 stages 48 KB in gemv_kernel, six 2048 passes here)
@pytest.mark.parametrize("M", [1, 3, 4, 5, 8])
@pytest.mark.parametrize("N,K", [(64, 256), (2048, 2048), (4096, 1024), (12288, 2048), (2048, 6144), (1000, 4112),
                                 (4728, 1024), (4736, 1024), (9464, 1024), (9472, 1024),
                                 (6144, 4096), (4096, 4096), (24576, 4096), (4096, 12288)])
def test_batched_gemv_matches_numpy_and_the_simt_gemm(q3, M, N, K):
    """gemv_batch_kernel (impl 5) on M <= 8 activation rows: store / residual / SwiGLU epilogues, K spanning one and several 2048-element
    passes (and a ragged last pass), every rows-per-warp variant (N picks 1 / 2 / 4).  Every row of impl 5 and of its cp.async-ring twin
    (impl 6) is bit-identical to the batch-1 gemv_kernel (impl 4) on that row alone: a batched step reproduces the per-op step."""
    cfg, w, m, o = q3
    rng = np.random.default_rng(N + K + M)
    x = rng.standard_normal((M, K)).astype(np.float32)
    W = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
    bias = rng.standard_normal(N).astype(np.float32)
    resid = rng.standard_normal((M, N)).astype(np.float32)
    ref = x.astype(np.float64) @ W.astype(np.float64).T
    got, _ = m.debug_gemm(x, W, bias=bias, impl=5, epi=0)
    assert np.abs(got - (ref + bias)).max() <= 2e-4 * max(1.0, np.abs(ref).max())
    simt, _ = m.debug_gemm(x, W, bias=bias, impl=1, epi=0)
    assert np.abs(got - simt).max() <= 1e-4 * max(1.0, np.abs(ref).max())
    ring, _ = m.debug_gemm(x, W, bias=bias, impl=6, epi=0)        # weights through the cp.async ring: the same fmas in the same order
    assert np.array_equal(ring, got)
    one, _ = m.debug_gemm(x, W, bias=bias, impl=4, epi=0)
    assert np.array_equal(one, got)
    got, _ = m.debug_gemm(x, W, resid=resid, impl=5, epi=1)
    assert np.abs(got - (ref + resid)).max() <= 2e-4 * max(1.0, np.abs(ref).max())
    assert np.array_equal(m.debug_gemm(x, W, resid=resid, impl=6, epi=1)[0], got)
    assert np.array_equal(m.debug_gemm(x, W, resid=resid, impl=4, epi=1)[0], got)
    if N % 2 == 0:   # SwiGLU on interleaved (gate, up) rows, behind a unit-gain RMSNorm prologue
        xn = x / np.sqrt((x.astype(np.float64) ** 2).mean(-1, keepdims=True) + 1e-6)
        r2 = xn @ W.astype(np.float64).T
        g, u = r2[:, 0::2], r2[:, 1::2]
        want = g / (1 + np.exp(-g)) * u
        got, _ = m.debug_gemm(x, W, impl=5, epi=3)
        assert got.shape == (M, N // 2)
        assert np.abs(got - want).max() <= 2e-4 * max(1.0, np.abs(want).max())
        assert np.array_equal(m.debug_gemm(x, W, impl=6, epi=3)[0], got)
        assert np.array_equal(m.debug_gemm(x, W, impl=4, epi=3)[0], got)


def _requests(V, spec):
    return [dict(input_ids=_ids(S, V, 100 + i), max_tokens=n, **kw) for i, (S, n, kw) in enumerate(spec)]


@pytest.mark.parametrize("twin,graph", [(0, True), (0, False), (1, True), (2, True), (2, False)])
def test_batch_of_greedy_requests_equals_single_requests(q3, twin, graph):
    """8 prompts of different lengths and budgets (page boundaries crossed at different steps, requests leaving the batch one by one):
    every request's ids equal its own oracle run and the library's own single-request generate."""
    cfg, w, m, o = q3
    V = cfg["vocab_size"]
    spec = [(5, 40, {}), (33, 9, {}), (64, 70, {}), (1, 12, {}), (200, 33, {}), (97, 1, {}), (31, 64, {}), (150, 20, {})]
    reqs = _requests(V, spec)
    os.environ["AHA_BATCH_GEMV"] = str(twin)                   # 0 / 2: batched GEMV (weights in registers / through the cp.async ring), 1: exact SIMT GEMM
    os.environ["AHA_BATCH_GRAPH"] = "1" if graph else "0"      # 0: eager launches instead of one CUDA graph per composition of the batch
    try:
        res = m.generate_batch(reqs)
    finally:
        os.environ.pop("AHA_BATCH_GEMV", None)
        os.environ.pop("AHA_BATCH_GRAPH", None)
    for r, (toks, usage) in zip(reqs, res):
        want = _oracle_generate(o, r["input_ids"], None, r["max_tokens"])
        assert toks == want, (len(r["input_ids"]), r["max_tokens"])
        assert usage["prompt_tokens"] == len(r["input_ids"]) and usage["completion_tokens"] == len(want)
        single, _ = m.generate(r["input_ids"], max_tokens=r["max_tokens"])
        assert single == toks
    # the handle is back to the single-request state: prefix reuse, direct trait calls
    a, _ = m.generate(reqs[0]["input_ids"], max_tokens=5, reuse_prefix=True)
    assert a == res[0][0][:5]
    m.clear_cache()


def test_batch_with_samplers_and_partial_batches(q3):
    """Every request carries its own sampler (mode, seed, repeat penalty, RNG stream); batches of 1, 2, 3 and 5 requests."""
    cfg, w, m, o = q3
    V = cfg["vocab_size"]
    samplers = [dict(temperature=0.8, top_p=0.9, top_k=30, repeat_penalty=1.15, repeat_last_n=16, seed=7),
                dict(),
                dict(temperature=1.1, seed=3),
                dict(temperature=0.6, top_p=0.7, seed=11),
                dict(temperature=0.9, top_k=5, seed=5),
                dict(repeat_penalty=1.3, repeat_last_n=8)]
    for n in (1, 2, 3, 5):
        spec = [(20 + 13 * i, 14 + 3 * i, samplers[(i + n) % len(samplers)]) for i in range(n)]
        reqs = _requests(V, spec)
        res = m.generate_batch(reqs)
        for r, (toks, _) in zip(reqs, res):
            kw = {k: v for k, v in r.items() if k not in ("input_ids", "max_tokens")}
            assert toks == _oracle_generate(o, r["input_ids"], None, r["max_tokens"], **kw), (n, kw)


def test_batch_stops_each_request_at_its_own_eos():
    """An EOS token ends only the request that produced it (and is pushed, like generate_generic does); the others run on."""
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=1024)
    o = make_oracle("qwen3", cfg, w)
    V = cfg["vocab_size"]
    probe = [m.generate(_ids(10 + i, V, 300 + i), max_tokens=30)[0] for i in range(4)]
    m.close()
    eos = [probe[1][7], probe[3][15]]            # tokens that requests 1 and 3 produce mid-way become stop ids
    from aha_b200 import B200Model
    m = B200Model("qwen3", cfg, w, eos_ids=eos, max_ctx=1024)
    o2 = type(o)(cfg, w, eos)                     # the oracle with the same stop ids
    reqs = [dict(input_ids=_ids(10 + i, V, 300 + i), max_tokens=30) for i in range(4)]
    res = m.generate_batch(reqs)
    lens = []
    for r, (toks, _) in zip(reqs, res):
        want = _oracle_generate(o2, r["input_ids"], None, 30)
        assert toks == want
        lens.append(len(toks))
    assert min(lens) < 30 and max(lens) >= min(lens)      # at least one request stopped early
    m.close()


def test_batch_capacity_and_argument_errors(q3):
    from aha_b200 import B200Error
    cfg, w, m, o = q3
    V = cfg["vocab_size"]
    with pytest.raises(B200Error, match="1 to 8 requests"):
        m.generate_batch(_requests(V, [(4, 2, {})] * 9))
    with pytest.raises(B200Error, match="KV capacity"):
        m.generate_batch(_requests(V, [(700, 100, {})] * 4))            # 4 x 800 tokens > max_ctx 2048
    ok = m.generate_batch(_requests(V, [(10, 3, {})]))                   # and the handle still works afterwards
    assert ok[0][0] == _oracle_generate(o, _ids(10, V, 100), None, 3)


def test_batch_mixes_image_and_text_requests():
    """Qwen3-VL: a request with an image (M-RoPE positions, rope_delta carried into its decode steps) next to text-only requests."""
    from aha_b200 import synth
    from oracle.qwen3vl import process_image
    cfg, w, m = make_model("qwen3vl", "tiny", max_ctx=2048, max_patches=1024)
    o = make_oracle("qwen3vl", cfg, w)
    V = cfg["text_config"]["vocab_size"]
    pv, grid = process_image(synth.synth_image(256, 320, 1))
    data = [pv, grid, None, None, None]
    pv2, grid2 = process_image(synth.synth_image(128, 192, 2))
    data2 = [pv2, grid2, None, None, None]
    reqs = [dict(input_ids=synth.vl_prompt_ids(cfg, grid, 12), data=data, max_tokens=10),
            dict(input_ids=_ids(40, V, 9), data=[None] * 5, max_tokens=16),
            dict(input_ids=synth.vl_prompt_ids(cfg, grid2, 5), data=data2, max_tokens=12, temperature=0.7, top_p=0.9, seed=4),
            dict(input_ids=_ids(7, V, 10), data=[None] * 5, max_tokens=6)]
    res = m.generate_batch(reqs)
    for r, (toks, usage) in zip(reqs, res):
        kw = {k: v for k, v in r.items() if k not in ("input_ids", "max_tokens", "data")}
        assert toks == _oracle_generate(o, r["input_ids"], r["data"], r["max_tokens"], **kw)
        assert (usage["vision_secs"] > 0) == (r["data"][0] is not None)
    m.close()


# ---- continuous batching: requests join and leave a running batch between steps (aha_b200_batch_open / _add / _step / _close) ----
class _Session:
    def __init__(self, m):
        self.m, self.out, self.running, self.slot_of = m, {}, {}, {}
        m.batch_open()

    def add(self, name, ids, **kw):
        slot, tok, fin = self.m.batch_add(ids, **kw)
        self.out[name] = [tok]
        self.slot_of[name] = slot
        if not fin:
            assert slot not in self.running
            self.running[slot] = name
        return slot

    def step(self, n=1):
        for _ in range(n):
            res = self.m.batch_step()
            assert sorted(res) == sorted(self.running)          # exactly the running requests produce a token
            for slot, (tok, fin) in res.items():
                self.out[self.running[slot]].append(tok)
                if fin:
                    del self.running[slot]

    def drain(self):
        while self.running:
            self.step()


def test_continuous_batching_requests_join_and_leave(q3):
    """Requests are admitted while others are mid-generation and take over the slots (and KV pages) of finished ones; whatever the
    schedule, every request's ids are those of its own oracle run."""
    cfg, w, m, o = q3
    V = cfg["vocab_size"]
    m.clear_cache()
    reqs = {"A": (_ids(40, V, 401), dict(max_tokens=30)),
            "B": (_ids(90, V, 402), dict(max_tokens=12)),
            "C": (_ids(15, V, 403), dict(max_tokens=25, temperature=0.8, top_p=0.9, top_k=20, repeat_penalty=1.1, repeat_last_n=8, seed=9)),
            "D": (_ids(70, V, 404), dict(max_tokens=18)),
            "E": (_ids(33, V, 405), dict(max_tokens=10, temperature=1.0, seed=2)),
            "F": (_ids(5, V, 406), dict(max_tokens=1))}
    s = _Session(m)
    s.add("A", reqs["A"][0], **reqs["A"][1])
    slot_b = s.add("B", reqs["B"][0], **reqs["B"][1])
    s.step(5)
    s.add("C", reqs["C"][0], **reqs["C"][1])                    # joins while A and B are decoding
    while "B" in s.running.values():
        s.step()
    assert s.add("D", reqs["D"][0], **reqs["D"][1]) == slot_b   # takes over B's slot (and its pages)
    s.step(3)
    s.add("E", reqs["E"][0], **reqs["E"][1])
    s.add("F", reqs["F"][0], **reqs["F"][1])                    # a one-token request is finished by its prefill and never occupies a step
    assert "F" not in s.running.values()
    s.drain()
    assert m.batch_step() == {}
    m.batch_close()
    for name, (ids, kw) in reqs.items():
        n = kw["max_tokens"]
        samp = {k: v for k, v in kw.items() if k != "max_tokens"}
        assert s.out[name] == _oracle_generate(o, ids, None, n, **samp), name
    toks, _ = m.generate(reqs["A"][0], max_tokens=30)             # the handle serves single requests again
    assert toks == s.out["A"]


def test_graph_per_running_count(q3):
    """Many join / leave cycles at three running counts: at most one step graph per count, and every request's ids are those of its own
    single-request generate."""
    cfg, w, m, o = q3
    V = cfg["vocab_size"]
    m.clear_cache()
    reqs, counts = {}, set()
    s = _Session(m)
    try:
        k = 0
        for cycle in range(15):
            while len(s.running) < (3, 5, 8)[cycle % 3]:
                kw = dict(max_tokens=2 + k % 5, **(dict(temperature=0.9, top_k=20, seed=k) if k % 3 == 0 else {}))
                reqs[k] = (_ids(10 + 7 * k % 50, V, 5000 + k), kw)
                s.add(k, reqs[k][0], **kw)
                k += 1
            counts.add(len(s.running))
            s.step()
        while s.running:
            counts.add(len(s.running))
            s.step()
        graphs = int(m.debug_read("batch_graphs", 0, 1)[0])
        assert k > 20 and 1 <= graphs <= len(counts), (k, graphs, counts)
    finally:
        m.batch_close()
    for name, (ids, kw) in reqs.items():
        assert s.out[name] == m.generate(ids, **kw)[0], name


def test_batch_session_rules(q3):
    from aha_b200 import B200Error
    cfg, w, m, o = q3
    V = cfg["vocab_size"]
    m.clear_cache()
    with pytest.raises(B200Error, match="no batch session is open"):
        m.batch_add(_ids(4, V, 1), max_tokens=2)
    m.batch_open()
    with pytest.raises(B200Error, match="batch session is open"):
        m.generate(_ids(4, V, 1), max_tokens=2)
    with pytest.raises(B200Error, match="batch session is open"):
        m.forward_initial(_ids(4, V, 1), 0)
    with pytest.raises(B200Error, match="KV capacity"):
        m.batch_add(_ids(1500, V, 2), max_tokens=1000)            # 2500 tokens > max_ctx 2048: refused, session intact
    slots = [m.batch_add(_ids(10 + i, V, 20 + i), max_tokens=40)[0] for i in range(8)]
    assert sorted(slots) == list(range(8))
    with pytest.raises(B200Error, match="all 8 slots"):
        m.batch_add(_ids(4, V, 3), max_tokens=2)
    assert len(m.batch_step()) == 8
    m.clear_cache()                                               # clear_cache ends the session
    toks, _ = m.generate(_ids(10, V, 20), max_tokens=6)
    assert toks == _oracle_generate(o, _ids(10, V, 20), None, 6)
    m.batch_open(); m.batch_close()
    with pytest.raises(B200Error, match="no batch session is open"):
        m.batch_step()
