"""Packed admission into a continuous-batching session (aha_b200_batch_add_many / B200Model.batch_add_many).

Several waiting requests enter the session in one call: the text-only ones share packed prefills (each request attends only to itself,
its K/V written straight into its own pages), their first tokens come from one batched lm_head.  Every request must still produce the ids
of its own fresh oracle run, and for prompts of 32 tokens or more (every prompt with the SIMT GEMM) exactly the ids batch_add gives it."""
import numpy as np
import pytest

from conftest import TOL, make_model, make_oracle

pytestmark = pytest.mark.gpu

# prompt lengths across the 32-token page, the 64-token KV tile and the 128-token query tile; budgets and samplers mixed
SPEC = [(1, 12, {}),
        (5, 20, dict(temperature=0.8, top_p=0.9, top_k=30, seed=7)),
        (31, 9, dict(repeat_penalty=1.3, repeat_last_n=8)),
        (32, 16, dict(temperature=1.1, seed=3)),
        (33, 1, {}),
        (64, 25, dict(temperature=0.9, top_k=5, repeat_penalty=1.15, repeat_last_n=4, seed=5)),
        (65, 14, {}),
        (200, 30, dict(temperature=0.6, top_p=0.7, seed=11))]


def _ids(n, vocab, seed):
    from aha_b200 import synth
    return synth.synth_text_ids(n, vocab - 8, seed)


def _requests(V, spec, seed0=100):
    return [dict(input_ids=_ids(S, V, seed0 + i), max_tokens=n, **kw) for i, (S, n, kw) in enumerate(spec)]


def _samp(r):
    return {k: v for k, v in r.items() if k not in ("input_ids", "max_tokens", "data")}


def _oracle_generate(o, r):
    from test_prefix_cache_gpu import _oracle_generate as og
    return og(o, r["input_ids"], r.get("data"), r["max_tokens"], **_samp(r))


class _Session:
    """Drives a session and records every request's ids by name."""

    def __init__(self, m):
        self.m, self.out, self.running = m, {}, {}
        m.batch_open()

    def _admitted(self, name, slot, tok, fin):
        self.out[name] = [tok]
        if not fin:
            assert slot not in self.running
            self.running[slot] = name

    def add(self, name, r):
        slot, tok, fin = self.m.batch_add(**r)
        self._admitted(name, slot, tok, fin)
        return slot

    def add_many(self, named):
        res, usage = self.m.batch_add_many([r for _, r in named], return_usage=True)
        for (name, _), (slot, tok, fin) in zip(named, res):
            self._admitted(name, slot, tok, fin)
        return res, usage

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

    def close(self):
        self.m.batch_close()


def _run_session(m, reqs, many):
    """Admit `reqs` at session start (one batch_add_many, or one batch_add each), drain -> (ids per request, admission results, usage)."""
    s = _Session(m)
    try:
        named = [(i, r) for i, r in enumerate(reqs)]
        if many:
            res, usage = s.add_many(named)
        else:
            res, usage = [], None
            for i, r in named:
                slot = s.add(i, r)
                res.append((slot, s.out[i][0], slot not in s.running))
        s.drain()
    finally:
        s.close()
    return [s.out[i] for i in range(len(reqs))], res, usage


_ORACLE = {}


def _oracle_cached(key, o, r):
    k = (key, tuple(int(t) for t in r["input_ids"]), r["max_tokens"], tuple(sorted(_samp(r).items())))
    if k not in _ORACLE:
        _ORACLE[k] = _oracle_generate(o, r)
    return _ORACLE[k]


@pytest.fixture(scope="module")
def q3():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=2048)
    yield cfg, w, m, make_oracle("qwen3", cfg, w)
    m.close()


def _check_eight(m, cfg, w, o, exact_below_32):
    V = cfg["vocab_size"]
    reqs = _requests(V, SPEC)
    got, res, usage = _run_session(m, reqs, many=True)
    assert [r[0] for r in res] == list(range(8))                # input order, lowest free slot first
    alone, _, _ = _run_session(m, reqs, many=False)
    for r, ids, (slot, tok, fin), u, ref in zip(reqs, got, res, usage, alone):
        n = len(r["input_ids"])
        assert ids == _oracle_cached("qwen3-tiny", o, r), (n, _samp(r))
        if n >= 32 or exact_below_32:
            assert ids == ref, n
        assert tok == ids[0] and fin == (r["max_tokens"] == 1)
        assert u["prompt_tokens"] == n and u["completion_tokens"] == 1
        assert u["prompt_secs"] > 0 and u["vision_secs"] == 0


def test_eight_requests_at_session_start(q3):
    cfg, w, m, o = q3
    _check_eight(m, cfg, w, o, exact_below_32=False)


def test_eight_requests_simt_gemm_exact_for_every_length(q3):
    """With the SIMT GEMM (gemm_impl = 1) for every row count, the packed prefill equals the one-by-one prefill for every prompt length."""
    cfg, w, _, o = q3
    _, _, m = make_model("qwen3", "tiny", max_ctx=2048, gemm_impl=1)
    try:
        _check_eight(m, cfg, w, o, exact_below_32=True)
    finally:
        m.close()


def test_admission_mid_flight():
    """batch_add_many while other requests decode: lowest free slots, slots and pages of finished requests taken over, a one-token request
    and one whose first token is a stop id (AHA_GEN_EOS_ON_FIRST) reported finished at admission."""
    from aha_b200 import B200Model, _lib as L
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=2048)
    o = make_oracle("qwen3", cfg, w)
    V = cfg["vocab_size"]
    probe = dict(input_ids=_ids(45, V, 900), max_tokens=1)
    m.close()
    stop_tok = _oracle_generate(o, probe)[0]                    # the first token of `probe` becomes a stop id
    eos = [cfg["eos_token_id"], stop_tok]
    m = B200Model("qwen3", cfg, w, eos_ids=eos, max_ctx=2048)
    o2 = type(o)(cfg, w, eos)
    try:
        reqs = {"A": dict(input_ids=_ids(40, V, 401), max_tokens=30),
                "B": dict(input_ids=_ids(90, V, 402), max_tokens=8),
                "C": dict(input_ids=_ids(15, V, 403), max_tokens=25, temperature=0.8, top_p=0.9, top_k=20, repeat_penalty=1.1, repeat_last_n=8, seed=9),
                "D": dict(input_ids=_ids(70, V, 404), max_tokens=18),
                "E": dict(input_ids=_ids(129, V, 405), max_tokens=10, temperature=1.0, seed=2),
                "F": dict(input_ids=_ids(33, V, 406), max_tokens=12),
                "G": dict(input_ids=_ids(5, V, 407), max_tokens=1),
                "H": dict(probe, max_tokens=20, flags=L.GEN_EOS_ON_FIRST)}
        s = _Session(m)
        s.add("A", reqs["A"])
        slot_b = s.add("B", reqs["B"])
        s.step(3)
        res, _ = s.add_many([(k, reqs[k]) for k in "CDE"])      # join while A and B decode
        assert [r[0] for r in res] == [2, 3, 4]
        while "B" in s.running.values():
            s.step()
        free = [i for i in range(8) if i not in s.running]
        res, _ = s.add_many([(k, reqs[k]) for k in "FGH"])      # B's slot and pages are taken over
        assert [r[0] for r in res] == free[:3] and slot_b in free[:3]
        assert res[1][2] and res[2][2] and res[2][1] == stop_tok  # G (one token) and H (stop id first) finished at admission
        assert "G" not in s.running.values() and "H" not in s.running.values()
        s.drain()
        assert m.batch_step() == {}
        s.close()
        for name, r in reqs.items():
            if name == "H":
                assert s.out[name] == [stop_tok]
            else:
                assert s.out[name] == _oracle_generate(o2, r), name
    finally:
        m.close()


def test_several_packs_and_a_long_request(q3):
    """max_prefill = 128: six 60-token requests take three packs and give the ids a max_prefill = 2048 handle gives them; a 300-token
    request in the same call is prefilled alone (in chunks) and matches the oracle."""
    cfg, w, big, o = q3
    V = cfg["vocab_size"]
    six = _requests(V, [(60, 10 + i, dict(temperature=0.7, seed=i) if i % 2 else {}) for i in range(6)], seed0=500)
    want, _, _ = _run_session(big, six, many=True)
    long_req = dict(input_ids=_ids(300, V, 599), max_tokens=12)
    _, _, m = make_model("qwen3", "tiny", max_ctx=2048, max_prefill=128)
    try:
        got, res, _ = _run_session(m, six[:3] + [long_req] + six[3:], many=True)
        assert [r[0] for r in res] == list(range(7))
        assert got[:3] + got[4:] == want
        assert got[3] == _oracle_cached("qwen3-tiny", o, long_req)
        for r, ids in zip(six, want):
            assert ids == _oracle_cached("qwen3-tiny", o, r)
    finally:
        m.close()


@pytest.mark.parametrize("attn_impl", [1, 2])
def test_attention_twins(q3, attn_impl):
    """The SIMT (1) and mma.sync (2) attention run one flash_dispatch per packed request."""
    cfg, w, _, o = q3
    _, _, m = make_model("qwen3", "tiny", max_ctx=2048, attn_impl=attn_impl)
    try:
        reqs = _requests(cfg["vocab_size"], SPEC)
        got, _, _ = _run_session(m, reqs, many=True)
        for r, ids in zip(reqs, got):
            assert ids == _oracle_cached("qwen3-tiny", o, r), len(r["input_ids"])
    finally:
        m.close()


def test_qwen3vl_text_requests_packed_beside_an_image_request():
    from aha_b200 import synth
    from oracle.qwen3vl import process_image
    cfg, w, m = make_model("qwen3vl", "tiny", max_ctx=2048, max_patches=1024)
    o = make_oracle("qwen3vl", cfg, w)
    try:
        V = cfg["text_config"]["vocab_size"]
        pv, grid = process_image(synth.synth_image(256, 320, 1))
        reqs = [dict(input_ids=_ids(40, V, 9), data=[None] * 5, max_tokens=16),
                dict(input_ids=synth.vl_prompt_ids(cfg, grid, 12), data=[pv, grid, None, None, None], max_tokens=10),
                dict(input_ids=_ids(7, V, 10), data=[None] * 5, max_tokens=6, temperature=0.7, top_p=0.9, seed=4)]
        got, res, usage = _run_session(m, reqs, many=True)
        assert [r[0] for r in res] == [0, 1, 2]
        for r, ids, u in zip(reqs, got, usage):
            assert ids == _oracle_generate(o, r)
            assert (u["vision_secs"] > 0) == (r["data"][0] is not None)
            assert u["prompt_tokens"] == len(r["input_ids"])
    finally:
        m.close()


def test_packing_launches_fewer_kernels(q3):
    """Eight 64-token requests: one batch_add_many launches fewer than half the kernels of eight batch_add calls (the per-layer prefill
    kernels run once per pack instead of once per request) and gives the same first tokens."""
    cfg, w, m, o = q3
    reqs = _requests(cfg["vocab_size"], [(64, 4, {})] * 8, seed0=700)
    counts, firsts = [], []
    for many in (False, True):
        m.batch_open()
        try:
            m.reset_stats()
            res = m.batch_add_many(reqs) if many else [m.batch_add(**r) for r in reqs]
            counts.append(m.stats()["kernel_launches"])
            firsts.append([t for _, t, _ in res])
        finally:
            m.batch_close()
    assert firsts[0] == firsts[1]
    assert 2 * counts[1] < counts[0], counts


def test_errors_admit_nothing(q3):
    """Every refusal leaves the session as it was: the running requests keep stepping to their oracle ids, and no slot or page leaks."""
    from aha_b200 import B200Error, _lib as L
    cfg, w, m, o = q3
    V = cfg["vocab_size"]
    m.clear_cache()
    ok = dict(input_ids=_ids(20, V, 801), max_tokens=4)
    with pytest.raises(B200Error, match="no batch session is open"):
        m.batch_add_many([ok])
    running = {"A": dict(input_ids=_ids(40, V, 802), max_tokens=24), "B": dict(input_ids=_ids(70, V, 803), max_tokens=20, temperature=0.9, seed=1)}
    s = _Session(m)
    try:
        s.add("A", running["A"])
        s.add("B", running["B"])
        bad = [([], "no requests"),
               ([ok] * 7, "only 6 of the 8 slots are free"),
               ([ok, dict(input_ids=_ids(900, V, 804), max_tokens=100), dict(input_ids=_ids(900, V, 805), max_tokens=100)], "KV capacity"),
               ([ok, dict(input_ids=np.array([1, 2, V], np.uint32), max_tokens=4)], "token id out of range"),
               ([ok, dict(ok, flags=L.GEN_CONTINUE_RNG)], "CONTINUE_RNG"),
               ([dict(ok, flags=L.GEN_REUSE_PREFIX)], "REUSE_PREFIX")]
        for reqs, msg in bad:
            with pytest.raises(B200Error, match=msg):
                m.batch_add_many(reqs)
            s.step()                                            # A and B still run, nobody else
        s.drain()
        for name, r in running.items():
            assert s.out[name] == _oracle_generate(o, r), name
        # nothing leaked: eight requests of 8 pages each exactly fill the 64-page pool (max_ctx 2048)
        fill = _requests(V, [(200, 56, {})] * 8, seed0=810)
        res = m.batch_add_many(fill)
        assert [r[0] for r in res] == list(range(8))
        with pytest.raises(B200Error, match="slots"):
            m.batch_add_many([ok])
        assert len(m.batch_step()) == 8
    finally:
        s.close()
    # the handle serves single requests again
    toks, _ = m.generate(ok["input_ids"], max_tokens=4)
    assert toks == _oracle_generate(o, ok)
    ids = _ids(50, V, 820)
    got = m.forward_initial(ids, 0)[0, 0]
    want = o.forward_initial(ids.reshape(1, -1), 0, None)[0, 0]
    o.clear_cache()
    assert np.abs(got - want).max() <= TOL
    m.clear_cache()
