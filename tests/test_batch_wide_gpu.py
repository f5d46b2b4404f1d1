"""Wide continuous-batching sessions (aha_b200_batch_open_wide / batch_step_n, B200Model.batch_open_wide).

Up to 64 requests decode in lockstep with every projection and the lm_head on the wgmma kernel of gemv_wide.cuh.  Every request must
produce the ids of its own fresh oracle run, and its ids must not depend on its slot, on the requests beside it or on the step it joined at
(the tensor-core sums are fixed by the shape alone).  The kernel itself is checked through debug_gemm(impl=7)."""
import ctypes as C

import numpy as np
import pytest

from conftest import TOL, make_model, make_oracle

pytestmark = pytest.mark.gpu

# the last four are the Qwen3-VL-8B text projections (qkv, o_proj, gate/up, down: wide_plan splits K = 12288 nine ways)
SHAPES = [(64, 256), (1024, 256), (2048, 2048), (4096, 1024), (2048, 6144), (12288, 2048), (6144, 4096), (4096, 4096), (24576, 4096),
          (4096, 12288)]
ROWS = [1, 2, 8, 9, 33, 64]


def _ids(n, vocab, seed):
    from aha_b200 import synth
    return synth.synth_text_ids(n, vocab - 8, seed)


def _samp(r):
    return {k: v for k, v in r.items() if k not in ("input_ids", "max_tokens", "data", "flags")}


def _oracle_generate(o, r):
    from test_prefix_cache_gpu import _oracle_generate as og
    return og(o, r["input_ids"], r.get("data"), r["max_tokens"], **_samp(r))


# ---------------------------------------------------------------------------------------------------------------- the kernel

@pytest.fixture(scope="module")
def tiny():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=1024)
    yield m
    m.close()


def _case(N, K, M, seed):
    rng = np.random.default_rng(seed)
    W = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
    x = rng.standard_normal((M, K)).astype(np.float32)
    return rng, W, x


@pytest.mark.parametrize("N,K", SHAPES)
def test_kernel_against_float64(tiny, N, K):
    m = tiny
    for M in ROWS:
        rng, W, x = _case(N, K, M, N + K + M)
        bias = rng.standard_normal(N).astype(np.float32)
        resid = rng.standard_normal((M, N)).astype(np.float32)
        ref = x.astype(np.float64) @ W.astype(np.float64).T
        tol = 2e-4 * max(1.0, np.abs(ref).max())
        got, _ = m.debug_gemm(x, W, bias=bias, impl=7, epi=0)
        assert np.abs(got - (ref + bias)).max() <= tol, (M, "store")
        got, _ = m.debug_gemm(x, W, resid=resid, impl=7, epi=1)
        assert np.abs(got - (ref + resid)).max() <= tol, (M, "residual")
        xn = x / np.sqrt((x.astype(np.float64) ** 2).mean(-1, keepdims=True) + 1e-6)
        r2 = xn @ W.astype(np.float64).T
        g, u = r2[:, 0::2], r2[:, 1::2]
        want = g / (1 + np.exp(-g)) * u
        got, _ = m.debug_gemm(x, W, impl=7, epi=3)
        assert got.shape == (M, N // 2)
        assert np.abs(got - want).max() <= 2e-4 * max(1.0, np.abs(want).max()), (M, "swiglu")


@pytest.mark.parametrize("N,K", [(1024, 2048), (2048, 6144), (4096, 1024)])   # split-K (o_proj / down shapes) and a single-split shape
@pytest.mark.parametrize("epi", [0, 1, 3])
def test_kernel_column_invariance(tiny, N, K, epi):
    """Row b alone, among 63 others and after a permutation of the rows gives the same bits."""
    m = tiny
    rng, W, x = _case(N, K, 64, 7 * N + K)
    bias = rng.standard_normal(N).astype(np.float32) if epi == 0 else None
    resid = rng.standard_normal((64, N)).astype(np.float32) if epi == 1 else None
    run = lambda rows: m.debug_gemm(x[rows], W, bias=bias, resid=None if resid is None else resid[rows], impl=7, epi=epi)[0]
    every = run(np.arange(64))
    for b in (0, 5, 63):
        assert np.array_equal(run(np.array([b]))[0], every[b]), b
    perm = rng.permutation(64)
    assert np.array_equal(run(perm), every[perm])
    assert np.array_equal(run(np.arange(9))[:9], every[:9])


def test_kernel_refusals(tiny):
    from aha_b200 import B200Error
    m = tiny
    _, W, x = _case(128, 256, 65, 1)
    with pytest.raises(B200Error, match="M <= 64"):
        m.debug_gemm(x, W, impl=7, epi=0)
    for N, K in [(96, 256), (128, 224)]:
        _, W, x = _case(N, K, 4, 2)
        with pytest.raises(B200Error, match="multiples of 64"):
            m.debug_gemm(x, W, impl=7, epi=0)


# ---------------------------------------------------------------------------------------------------------------- sessions

class _Session:
    """Drives a session and records every request's ids by name."""

    def __init__(self, m, width=64):
        self.m, self.out, self.running, self.counts = m, {}, {}, set()
        m.batch_open_wide(width)

    def _admitted(self, name, slot, tok, fin):
        self.out[name] = [tok]
        self.slot = getattr(self, "slot", {})
        self.slot[name] = slot
        if not fin:
            assert slot not in self.running
            self.running[slot] = name

    def add(self, name, r):
        slot, tok, fin = self.m.batch_add(**r)
        self._admitted(name, slot, tok, fin)
        return slot

    def add_many(self, named):
        res = self.m.batch_add_many([r for _, r in named])
        for (name, _), (slot, tok, fin) in zip(named, res):
            self._admitted(name, slot, tok, fin)
        return res

    def step(self, n=1):
        for _ in range(n):
            if not self.running:
                return
            self.counts.add(len(self.running))
            res = self.m.batch_step()
            assert sorted(res) == sorted(self.running)
            for slot, (tok, fin) in res.items():
                self.out[self.running[slot]].append(tok)
                if fin:
                    del self.running[slot]

    def drain(self):
        while self.running:
            self.step()

    def close(self):
        self.m.batch_close()


SAMPLERS = [{}, dict(temperature=0.8), dict(temperature=0.9, top_k=20, repeat_penalty=1.2, repeat_last_n=16),
            dict(temperature=0.7, top_p=0.85, repeat_penalty=1.1, repeat_last_n=8),
            dict(temperature=1.0, top_k=30, top_p=0.9, repeat_penalty=1.3, repeat_last_n=32)]


def _spec64(V, seed, max_budget=70):
    """64 requests: prompts of 1..200 tokens, budgets of 1..max_budget, greedy and the four samplers with their own seeds."""
    rng = np.random.default_rng(seed)
    lens = list(rng.integers(1, 201, 64))
    budgets = list(rng.integers(1, max_budget + 1, 64))
    lens[:4], budgets[:4] = [1, 200, 32, 31], [max_budget, 1, max_budget, max_budget - 3]
    reqs = []
    for i in range(64):
        kw = dict(SAMPLERS[i % len(SAMPLERS)])
        if kw:
            kw["seed"] = 1000 + 17 * i
        reqs.append(dict(input_ids=_ids(int(lens[i]), V, seed * 100 + i), max_tokens=int(budgets[i]), **kw))
    return reqs


def _draw_margin(o, r, k):
    """How close the oracle's draw of token k of request r lies to a decision boundary: for a sampled request the distance of the draw
    u * total from the nearest cumulative weight (relative to the total) or, with top-p, of the nucleus sum from top_p; for a greedy one the
    gap between the two largest logits."""
    from oracle.sample import Sampler, sampling_mode, softmax_blocked, topk_candidates, topp_weights, use_repeat_penalty
    kw = _samp(r)
    ids = np.asarray(r["input_ids"]).reshape(1, -1)
    s = Sampler(kw.get("temperature"), kw.get("top_p"), kw.get("top_k"), kw.get("repeat_penalty", 1.0), kw.get("repeat_last_n", 64),
                seed=kw.get("seed", 299792458))
    o.clear_cache()
    toks = []
    lg = o.forward_initial(ids, 0, r.get("data"))
    for i in range(k):
        t = s.sample_and_push(lg, toks)
        lg = o.forward_step(np.array([[t]]), ids.shape[1] + i)
    logits = use_repeat_penalty(s.repeat_penalty, s.repeat_last_n, np.asarray(lg, np.float32).reshape(-1), toks)
    mode = sampling_mode(s.temperature, s.top_p, s.top_k)
    if mode == "argmax":
        a, b = np.sort(logits)[-2:]
        return float(b - a)
    p = softmax_blocked(logits, s.temperature)
    cut = 1.0
    if mode in ("topp", "topk_topp") and 0.0 < s.top_p < 1.0:   # which tokens enter the nucleus
        cut = float(np.abs(np.cumsum(np.sort(p.astype(np.float64))[::-1][:s.top_k or len(p)]) - s.top_p).min())
    if mode in ("topk", "topk_topp") and s.top_k < len(p):
        w, _ = topk_candidates(p, s.top_k)
        if mode == "topk_topp" and not (s.top_p <= 0.0 or s.top_p >= w.sum()):
            keep = np.concatenate([[0.0], np.cumsum(w, dtype=np.float32)[:-1]]) < np.float32(s.top_p)
            w = np.where(keep, w, 0)
    else:
        w = topp_weights(p, s.top_p) if mode != "all" and 0.0 < s.top_p < 1.0 else p
    cum = np.cumsum(w.astype(np.float64))
    return min(cut, float(np.abs(cum - s.rng.uniform01(s.draws) * cum[-1]).min() / cum[-1]))


def _check_oracle_ids(o, reqs, out):
    """Every request's ids equal its oracle run's.  A request may part from it only at a draw that the oracle itself takes within 5e-5 of
    a decision boundary (the GPU's fp32 sums are ordered differently from numpy's, so the last bits of the logits differ), and at most 2
    of the requests may do so."""
    near = []
    for i, r in enumerate(reqs):
        want = _oracle_generate(o, r)
        if out[i] != want:
            k = next(j for j in range(min(len(want), len(out[i]))) if out[i][j] != want[j])
            margin = _draw_margin(o, r, k)
            assert margin < 5e-5, (i, len(r["input_ids"]), _samp(r), k, margin)
            near.append((i, k, margin))
    assert len(near) <= 2, near


def _wide_oracle_run(kind, preset, max_budget):
    """64 requests on a width-64 session, admitted through several packs, single adds and into freed slots mid-flight, with a request that
    stops on its first token and stop ids inside some budgets: every request yields its own oracle ids."""
    from aha_b200 import B200Model, _lib as L
    cfg, w, m = make_model(kind, preset, max_ctx=256)
    o = make_oracle(kind, cfg, w)
    m.close()
    V = cfg["vocab_size"]
    reqs = _spec64(V, 3, max_budget)
    probe = dict(input_ids=_ids(45, V, 900), max_tokens=1)
    stop_first = _oracle_generate(o, probe)[0]
    mid = _oracle_generate(o, dict(reqs[0], max_tokens=8))[5]      # a token that ends request 0 (and maybe others) inside its budget
    eos = [cfg["eos_token_id"], stop_first, mid]
    o = type(o)(cfg, w, eos)
    reqs.append(dict(probe, max_tokens=20, flags=L.GEN_EOS_ON_FIRST))
    m = B200Model(kind, cfg, w, eos_ids=eos, max_ctx=24576, max_prefill=256)
    try:
        s = _Session(m)
        s.add_many([(i, reqs[i]) for i in range(24)])               # several packs of max_prefill 256
        for i in range(24, 40):
            s.add(i, reqs[i])
        s.add_many([(i, reqs[i]) for i in range(40, 60)])
        s.step(2)
        while 64 - len(s.running) < 5:                              # wait for freed slots, then fill them
            s.step()
        res = s.add_many([(i, reqs[i]) for i in range(60, 65)])
        assert res[-1][2] and res[-1][1] == stop_first              # finished at admission
        assert any(r[0] < 60 for r in res)                          # some took the slot of a finished request
        s.drain()
        s.close()
        assert s.out[64] == [stop_first]
        _check_oracle_ids(o, reqs[:64], s.out)
        assert len(s.out[0]) < reqs[0]["max_tokens"]                # a stop id inside a budget
    finally:
        m.close()


# the mid oracle takes ~0.3 s per token on the host, so its requests generate at most 12 tokens (their prompts still reach 200)
@pytest.mark.parametrize("preset,max_budget", [("tiny", 70), ("tiny-g1", 70), ("tiny-g4", 70), ("mid", 12)])
def test_sixty_four_requests_oracle_ids(preset, max_budget):
    _wide_oracle_run("qwen3", preset, max_budget)


@pytest.fixture(scope="module")
def q3():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=16384, max_prefill=512)
    yield cfg, w, m, make_oracle("qwen3", cfg, w)
    m.close()


def _others(V, n, seed):
    rng = np.random.default_rng(seed)
    return [dict(input_ids=_ids(int(rng.integers(1, 180)), V, seed + i), max_tokens=int(rng.integers(2, 60)),
                 **(dict(temperature=0.9, seed=i) if i % 3 == 0 else {})) for i in range(n)]


def _alone(m, target, many):
    s = _Session(m)
    try:
        if many:
            s.add_many([("X", target)])
        else:
            s.add("X", target)
        s.drain()
    finally:
        s.close()
    return s.out["X"]


def _crowded(m, target, others, many):
    """target among 50 others of mixed lengths: 30 before it (some finish before it), 20 joining after it, in another slot than alone."""
    s = _Session(m)
    try:
        s.add_many([(("o", i), others[i]) for i in range(20)])
        s.step(3)
        if many:   # in the middle of a pack
            s.add_many([(("o", i), others[i]) for i in range(20, 25)] + [("X", target)] + [(("o", i), others[i]) for i in range(25, 30)])
        else:
            for i in range(20, 30):
                s.add(("o", i), others[i])
            s.add("X", target)
        s.step(4)
        s.add_many([(("o", i), others[i]) for i in range(30, 40)])
        s.step(2)
        for i in range(40, 50):
            s.add(("o", i), others[i])
        s.drain()
    finally:
        s.close()
    assert s.slot["X"] != 0
    return s.out["X"], {k: v for k, v in s.out.items() if k != "X"}


@pytest.mark.parametrize("many", [False, True])
def test_composition_invariance(q3, many, monkeypatch):
    cfg, w, m, o = q3
    V = cfg["vocab_size"]
    target = dict(input_ids=_ids(90, V, 4242), max_tokens=45, temperature=0.8, top_k=25, repeat_penalty=1.15, repeat_last_n=16, seed=77)
    others = _others(V, 50, 600)
    alone = _alone(m, target, many)
    assert alone == _oracle_generate(o, target)
    got, rest = _crowded(m, target, others, many)
    assert got == alone
    monkeypatch.setenv("AHA_BATCH_GRAPH", "0")                     # eager launches: the same ids
    got2, rest2 = _crowded(m, target, others, many)
    assert got2 == alone and rest2 == rest


def test_graph_per_running_count(q3):
    """Many composition changes at a few running counts: at most one step graph per count."""
    cfg, w, m, o = q3
    V = cfg["vocab_size"]
    s = _Session(m, 16)
    try:
        k = 0
        for _ in range(6):
            while len(s.running) < 12:
                s.add(("r", k), dict(input_ids=_ids(10 + 7 * k % 50, V, 3000 + k), max_tokens=2 + k % 5)); k += 1
            s.step()
        graphs = int(m.debug_read("batch_graphs", 0, 1)[0])
        assert k > 20 and 1 <= graphs <= len(s.counts), (k, graphs, s.counts)
        s.drain()
    finally:
        s.close()
    assert int(m.debug_read("batch_graphs", 0, 1)[0]) == 0


def test_qwen3vl_image_request_beside_packed_text():
    from aha_b200 import synth
    from oracle.qwen3vl import process_image
    cfg, w, m = make_model("qwen3vl", "tiny", max_ctx=4096, max_patches=1024)
    o = make_oracle("qwen3vl", cfg, w)
    try:
        V = cfg["text_config"]["vocab_size"]
        pv, grid = process_image(synth.synth_image(256, 320, 1))
        reqs = [dict(input_ids=_ids(40, V, 9), data=[None] * 5, max_tokens=16),
                dict(input_ids=synth.vl_prompt_ids(cfg, grid, 12), data=[pv, grid, None, None, None], max_tokens=10),
                dict(input_ids=_ids(7, V, 10), data=[None] * 5, max_tokens=6, temperature=0.7, top_p=0.9, seed=4),
                dict(input_ids=_ids(100, V, 11), data=[None] * 5, max_tokens=12)]
        s = _Session(m, 12)
        try:
            s.add_many([(i, r) for i, r in enumerate(reqs)])
            s.drain()
        finally:
            s.close()
        for i, r in enumerate(reqs):
            assert s.out[i] == _oracle_generate(o, r), i
    finally:
        m.close()


def _raw_step(m, cap, n_fn):
    toks, status, n = (C.c_uint32 * cap)(), (C.c_int32 * cap)(), C.c_size_t(0)
    return n_fn(m, toks, status, cap, n)


def test_errors_and_state(q3):
    from aha_b200 import B200Error, B200Model, synth
    cfg, w, m, o = q3
    V = cfg["vocab_size"]
    for bad in (0, 65):
        with pytest.raises(B200Error, match="1 to 64"):
            m.batch_open_wide(bad)
    m.batch_open()
    with pytest.raises(B200Error, match="a batch session is open"):
        m.batch_open_wide(8)
    m.batch_close()
    bcfg = dict(synth.get_config("qwen3", "tiny"), vocab_size=1000, eos_token_id=999)
    bm = B200Model("qwen3", bcfg, synth.make_weights("qwen3", bcfg, 0), eos_ids=[999], max_ctx=1024)
    try:
        with pytest.raises(B200Error, match="multiples of 64"):
            bm.batch_open_wide(8)
    finally:
        bm.close()

    running = {"A": dict(input_ids=_ids(40, V, 802), max_tokens=24), "B": dict(input_ids=_ids(70, V, 803), max_tokens=20, temperature=0.9, seed=1)}
    ok = dict(input_ids=_ids(20, V, 801), max_tokens=4)
    s = _Session(m, 12)
    try:
        s.add("A", running["A"])
        s.add("B", running["B"])
        lib, h = m._lib, m._h
        with pytest.raises(B200Error, match="batch_step_n"):
            m._check(lib.aha_b200_batch_step(h, (C.c_uint32 * 8)(), (C.c_int32 * 8)(), C.byref(C.c_size_t(0))))
        s.step()
        with pytest.raises(B200Error, match="smaller than the session width"):
            m._check(lib.aha_b200_batch_step_n(h, (C.c_uint32 * 11)(), (C.c_int32 * 11)(), 11, C.byref(C.c_size_t(0))))
        s.step()
        with pytest.raises(B200Error, match="only 10 of the 12 slots are free"):
            m.batch_add_many([ok] * 11)
        s.step()
        with pytest.raises(B200Error, match="KV capacity"):
            m.batch_add_many([ok, dict(input_ids=_ids(900, V, 804), max_tokens=16000)])
        s.step()
        with pytest.raises(B200Error, match="KV capacity"):
            m.batch_add(input_ids=_ids(900, V, 805), max_tokens=16000)
        s.drain()
        for name, r in running.items():
            assert s.out[name] == _oracle_generate(o, r), name
        # nothing leaked: twelve requests of 42 pages each take 504 of the 512 pages
        fill = [dict(input_ids=_ids(200, V, 810 + i), max_tokens=1130) for i in range(12)]
        res = m.batch_add_many(fill)
        assert [r[0] for r in res] == list(range(12))
        with pytest.raises(B200Error, match="slots"):
            m.batch_add(**ok)
        assert len(m.batch_step()) == 12
    finally:
        s.close()
    # the handle serves single requests again, and a narrow session still equals single runs bit for bit
    toks, _ = m.generate(ok["input_ids"], max_tokens=4)
    assert toks == _oracle_generate(o, ok)
    ids = _ids(50, V, 820)
    got = m.forward_initial(ids, 0)[0, 0]
    want = o.forward_initial(ids.reshape(1, -1), 0, None)[0, 0]
    o.clear_cache()
    assert np.abs(got - want).max() <= TOL
    m.clear_cache()
    narrow = _others(V, 6, 900)
    singles = [m.generate(r["input_ids"], max_tokens=r["max_tokens"], **_samp(r))[0] for r in narrow]
    m.batch_open()
    try:
        out, run = {}, {}
        for i, r in enumerate(narrow):
            slot, tok, fin = m.batch_add(**r)
            out[i] = [tok]
            if not fin:
                run[slot] = i
        while run:
            for slot, (tok, fin) in m.batch_step().items():
                out[run[slot]].append(tok)
                if fin:
                    del run[slot]
    finally:
        m.batch_close()
    for i in range(len(narrow)):
        assert out[i] == singles[i], i
