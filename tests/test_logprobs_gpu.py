"""Token log-probability records (logprobs.cuh) on the GPU: the kernels on given logits against a float64 log-softmax, the single-request
entries (tokens unchanged, records against the oracle's logits, the greedy invariant, streaming), narrow and wide batch sessions (records
bit-identical to the request's own run / whatever runs beside it), the step graphs and every refusal."""
import ctypes as C

import numpy as np
import pytest

import logprob_ref as R
from aha_b200 import B200Error
from aha_b200 import _lib as L
from conftest import make_model, make_oracle
from test_sampling_gpu import MODES

pytestmark = pytest.mark.gpu

ORACLE_TOL = 2e-3      # twice the 1e-3 logit budget


def _key(r):
    """a record, bit for bit"""
    return (r["token"], r["index"], np.float32(r["logprob"]).tobytes(), tuple(r["top_ids"]),
            b"".join(np.float32(v).tobytes() for v in r["top_logprobs"]))


def _ids(n, V, seed):
    return np.random.default_rng(seed).integers(0, min(V, 1000), n).astype(np.uint32)


@pytest.fixture(scope="module")
def q3():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=4096, max_prefill=512)
    yield cfg, w, m
    m.close()


# ------------------------------------------------------------------------------------------------------------- kernel on given logits

def _rows(V, rng):
    yield (rng.standard_normal(V) * 0.3).astype(np.float32)
    yield (rng.standard_normal(V) * 4.0).astype(np.float32)
    yield (rng.standard_normal(V) * 30.0).astype(np.float32)
    x = rng.integers(-3, 4, V).astype(np.float32)           # few distinct values: exact ties everywhere
    yield x
    x = (rng.standard_normal(V) * 0.5).astype(np.float32)
    x[rng.integers(0, V)] = 40.0                             # one dominant entry
    yield x
    x = np.full(V, -1.5, np.float32)                         # every entry tied
    yield x


@pytest.mark.parametrize("V", [1, 7, 1024, 2048, 2049, 4096, 5003, 151936])
def test_kernels_on_given_logits(q3, V):
    cfg, w, m = q3
    rng = np.random.default_rng(V)
    for k, x in enumerate(_rows(V, rng)):
        for n in sorted({0, 1, 2, 5, 19, 20} if V >= 20 else {0, 1, V}):
            tok = int(rng.integers(0, V))
            r = m.debug_logprobs(x, tok, n)
            lp, ids, tops = R.logprobs(x, tok, n)
            assert r["token"] == tok and r["index"] == 0
            assert abs(float(r["logprob"]) - lp) <= 1e-5, (V, k, n)
            assert r["top_ids"] == ids, (V, k, n)
            assert np.max(np.abs(np.asarray(r["top_logprobs"], np.float64) - tops), initial=0.0) <= 1e-5
            if n and tok == ids[0]:
                assert _key(r)[2] == np.float32(r["top_logprobs"][0]).tobytes()
    r1 = m.debug_logprobs(x, 0, 0)
    assert _key(r1) == _key(m.debug_logprobs(x, 0, 0))       # deterministic


def test_debug_refusals(q3):
    cfg, w, m = q3
    x = np.zeros(10, np.float32)
    for tok, n in ((10, 0), (0, 11), (0, 21)):
        with pytest.raises(B200Error):
            m.debug_logprobs(x, tok, n)
    with pytest.raises(B200Error, match="V must be"):
        m.debug_logprobs(np.zeros(128 * 2048 + 1, np.float32), 0, 0)


# ------------------------------------------------------------------------------------------------------------- single request

SAMPLERS = [("greedy", {})] + [(k, dict(temperature=t, top_p=p, top_k=kk)) for k, (t, p, kk) in sorted(MODES.items())]


@pytest.mark.parametrize("decode_impl", [0, 1])
def test_tokens_unchanged_and_greedy_invariant(decode_impl):
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=1024, decode_impl=decode_impl)
    try:
        V = cfg["vocab_size"]
        ids = _ids(37, V, 11)
        for name, kw in SAMPLERS:
            for pen in ({}, dict(repeat_penalty=1.3, repeat_last_n=16)):
                want, _ = m.generate(ids, max_tokens=40, seed=5, **kw, **pen)
                got, usage, recs = m.generate(ids, max_tokens=40, seed=5, logprobs=True, top_logprobs=5, **kw, **pen)
                assert got == want, (name, pen)
                assert usage["completion_tokens"] == len(got) == len(recs)
                assert [r["token"] for r in recs] == got and [r["index"] for r in recs] == list(range(len(got)))
                assert all(len(r["top_ids"]) == 5 for r in recs)
                for r in recs:
                    assert np.isfinite(r["logprob"]) and r["logprob"] <= 0
                if name == "greedy" and not pen:
                    for r in recs:
                        assert r["token"] == r["top_ids"][0]
                        assert np.float32(r["logprob"]).tobytes() == np.float32(r["top_logprobs"][0]).tobytes()
        _, _, r0 = m.generate(ids, max_tokens=6, logprobs=True)                # top_logprobs = 0
        assert all(r["top_ids"] == [] for r in r0)
    finally:
        m.close()


def _check_against_logits(recs, logits_rows):
    """records against the float64 log-softmax of the oracle's logits at each position"""
    for r, lg in zip(recs, logits_rows):
        lg = np.asarray(lg, np.float32).reshape(-1)
        ref = R.log_softmax64(lg)
        assert abs(float(r["logprob"]) - ref[r["token"]]) <= ORACLE_TOL, r["index"]
        got = np.asarray(r["top_logprobs"], np.float64)
        assert np.max(np.abs(got - ref[r["top_ids"]]), initial=0.0) <= ORACLE_TOL
        order = R.top_order(lg, len(r["top_ids"]) + 1)
        for j, i in enumerate(r["top_ids"]):
            # the oracle's order wherever neighbouring oracle logits are apart by more than the tolerance
            sep_prev = j == 0 or lg[order[j - 1]] - lg[order[j]] > ORACLE_TOL
            sep_next = j + 1 >= len(order) or lg[order[j]] - lg[order[j + 1]] > ORACLE_TOL
            if sep_prev and sep_next:
                assert i == order[j], (r["index"], j)


def _teacher_force(o, ids, toks, data=None):
    """the oracle's logits at every generated position, fed the GPU's own tokens"""
    rows = [o.forward_initial(ids.reshape(1, -1), 0, data) if data is not None else o.forward_initial(ids.reshape(1, -1), 0)]
    off = len(ids)
    for t in toks[:-1]:
        rows.append(o.forward_step(np.array([[t]]), off))
        off += 1
    o.clear_cache()
    return rows


@pytest.mark.parametrize("preset", ["tiny", "tiny-g1", "tiny-g4"])
def test_records_against_the_oracle(preset):
    cfg, w, m = make_model("qwen3", preset, max_ctx=1024)
    try:
        o = make_oracle("qwen3", cfg, w)
        ids = _ids(45, cfg["vocab_size"], 21)
        toks, _, recs = m.generate(ids, max_tokens=24, temperature=0.8, top_k=40, seed=3, logprobs=True, top_logprobs=20)
        _check_against_logits(recs, _teacher_force(o, ids, toks))
    finally:
        m.close()


def test_records_against_the_oracle_qwen3vl_image():
    from aha_b200 import synth
    from oracle.qwen3vl import process_image
    cfg, w, m = make_model("qwen3vl", "tiny", max_ctx=2048, max_patches=1024)
    try:
        o = make_oracle("qwen3vl", cfg, w)
        pv, grid = process_image(synth.synth_image(256, 320, 1))
        ids = synth.vl_prompt_ids(cfg, grid, 16)
        data = [pv, grid, None, None, None]
        toks, _, recs = m.generate(ids, data, max_tokens=12, logprobs=True, top_logprobs=8)
        _check_against_logits(recs, _teacher_force(o, np.asarray(ids, np.uint32), toks, data))
    finally:
        m.close()


def test_records_of_a_prefix_reuse_second_turn(q3):
    cfg, w, m = q3
    V = cfg["vocab_size"]
    o = make_oracle("qwen3", cfg, w)
    p1 = _ids(40, V, 31)
    a1, _ = m.generate(p1, max_tokens=9, reuse_prefix=True)
    p2 = np.concatenate([p1, np.asarray(a1[:-1], np.uint32), _ids(7, V, 32)])
    toks, _, recs = m.generate(p2, max_tokens=10, reuse_prefix=True, logprobs=True, top_logprobs=4)
    assert m.last_prefix_hit() > 0
    m.clear_cache()
    _check_against_logits(recs, _teacher_force(o, p2, toks))
    want, _, wrecs = m.generate(p2, max_tokens=10, logprobs=True, top_logprobs=4)      # a cold run: the same tokens
    assert want == toks


def test_stream_equals_non_stream(q3):
    cfg, w, m = q3
    ids = _ids(33, cfg["vocab_size"], 41)
    for kw in ({}, dict(temperature=0.7, top_k=20, top_p=0.8, repeat_penalty=1.1, repeat_last_n=8, seed=5)):
        toks, _, recs = m.generate(ids, max_tokens=21, logprobs=True, top_logprobs=3, **kw)
        seen = []
        m.generate_stream(ids, lambda t, i, r: seen.append((t, i, r)) and False, max_tokens=21, logprobs=True, top_logprobs=3, **kw)
        assert [t for t, _, _ in seen] == toks and [i for _, i, _ in seen] == list(range(len(toks)))
        assert [_key(r) for _, _, r in seen] == [_key(r) for r in recs]
        plain = []
        m.generate_stream(ids, lambda t, i: plain.append(t) and False, max_tokens=21, **kw)   # the two-argument callback is unchanged
        assert plain == toks


# ------------------------------------------------------------------------------------------------------------- batch sessions

class _Sess:
    """drives a session and gathers every request's tokens and (when it asked) records through batch_logprobs"""

    def __init__(self, m, wide=0):
        self.m, self.toks, self.recs, self.running, self.asks, self.slot = m, {}, {}, {}, {}, {}
        m.batch_open_wide(wide) if wide else m.batch_open()

    def _gather(self, names_by_slot):
        lp = self.m.batch_logprobs()
        for slot, name in names_by_slot.items():
            if self.asks[name]:
                assert slot in lp
                self.recs[name].append(_key(lp[slot]))
            else:
                assert slot not in lp

    def add_many(self, named):
        res = self.m.batch_add_many([r for _, r in named])
        by_slot = {}
        for (name, r), (slot, tok, fin) in zip(named, res):
            self.toks[name], self.recs[name], self.asks[name], self.slot[name] = [tok], [], bool(r.get("logprobs")), slot
            by_slot[slot] = name
            if not fin:
                self.running[slot] = name
        self._gather(by_slot)
        return res

    def add(self, name, r):
        slot, tok, fin = self.m.batch_add(**r)
        self.toks[name], self.recs[name], self.asks[name], self.slot[name] = [tok], [], bool(r.get("logprobs")), slot
        self._gather({slot: name})
        if not fin:
            self.running[slot] = name

    def step(self, n=1):
        for _ in range(n):
            if not self.running:
                return
            res = self.m.batch_step()
            assert sorted(res) == sorted(self.running)
            by_slot = {}
            for slot, (tok, fin) in res.items():
                name = self.running[slot]
                self.toks[name].append(tok)
                by_slot[slot] = name
                if fin:
                    del self.running[slot]
            self._gather(by_slot)

    def drain(self):
        while self.running:
            self.step()

    def close(self):
        self.m.batch_close()


def _req(V, id_seed, n_prompt, max_tokens, lp=True, top=5, **kw):
    r = dict(input_ids=_ids(n_prompt, V, id_seed), max_tokens=max_tokens, **kw)
    if lp:
        r.update(logprobs=True, top_logprobs=top)
    return r


def _single(m, r):
    kw = {k: v for k, v in r.items() if k != "input_ids"}
    if not r.get("logprobs"):
        return m.generate(r["input_ids"], **kw)[0], []
    toks, _, recs = m.generate(r["input_ids"], **kw)
    return toks, [_key(x) for x in recs]


@pytest.fixture(scope="module")
def q3_perop():
    # the narrow session mirrors the per-op decode GEMV's summation order, so its logits are those of the per-op single-request step
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=4096, max_prefill=512, decode_impl=1)
    yield cfg, w, m
    m.close()


@pytest.mark.parametrize("many", [False, True])
def test_narrow_session_records_equal_single_requests(q3_perop, many):
    cfg, w, m = q3_perop
    V = cfg["vocab_size"]
    reqs = [("a", _req(V, 1, 40, 14)), ("b", _req(V, 2, 64, 9, temperature=0.8, top_k=30, seed=4)),
            ("c", _req(V, 3, 35, 20, lp=False)), ("d", _req(V, 4, 50, 1, top=20)),
            ("e", _req(V, 5, 33, 12, top=0, temperature=0.7, top_p=0.9, repeat_penalty=1.2, repeat_last_n=8, seed=9))]
    late = [("f", _req(V, 6, 48, 8, top=3)), ("g", _req(V, 7, 36, 6, lp=False)), ("h", _req(V, 8, 70, 10, top=7, temperature=0.9, seed=2))]
    want = {name: _single(m, r) for name, r in reqs + late}
    s = _Sess(m)
    try:
        if many:
            s.add_many(reqs)
        else:
            for name, r in reqs:
                s.add(name, r)
        s.step(3)
        if many:
            s.add_many(late[:2])
            s.step(2)
            s.add_many(late[2:])
        else:
            for name, r in late:
                s.add(name, r)
                s.step()
        s.drain()
    finally:
        s.close()
    for name, _ in reqs + late:
        toks, recs = want[name]
        assert s.toks[name] == toks, name
        assert s.recs[name] == (recs if s.asks[name] else []), name


def _wide_target(V):
    return _req(V, 4242, 90, 30, top=20, temperature=0.8, top_k=25, repeat_penalty=1.15, repeat_last_n=16, seed=77)


def _others(V, n, seed):
    rng = np.random.default_rng(seed)
    return [_req(V, seed + i, int(rng.integers(1, 150)), int(rng.integers(2, 40)), lp=i % 2 == 0, top=i % 21,
                 **(dict(temperature=0.9, seed=i) if i % 3 == 0 else {})) for i in range(n)]


def _wide_alone(m, target):
    s = _Sess(m, 64)
    try:
        s.add_many([("X", target)])
        s.drain()
    finally:
        s.close()
    return s.toks["X"], s.recs["X"]


def _wide_crowded(m, target, others):
    s = _Sess(m, 64)
    try:
        s.add_many([(("o", i), others[i]) for i in range(20)])
        s.step(3)
        s.add_many([(("o", i), others[i]) for i in range(20, 25)] + [("X", target)] + [(("o", i), others[i]) for i in range(25, 30)])
        s.step(4)
        s.add_many([(("o", i), others[i]) for i in range(30, 40)])
        s.drain()
    finally:
        s.close()
    assert s.slot["X"] != 0
    return s.toks["X"], s.recs["X"], {k: v for k, v in s.recs.items() if k != "X"}


def test_wide_session_records_invariant_and_against_the_oracle(q3, monkeypatch):
    cfg, w, m = q3
    V = cfg["vocab_size"]
    target = _wide_target(V)
    toks, recs = _wide_alone(m, target)
    got_toks, got_recs, rest = _wide_crowded(m, target, _others(V, 40, 900))
    assert got_toks == toks and got_recs == recs
    monkeypatch.setenv("AHA_BATCH_GRAPH", "0")                    # eager launches: the same records
    t2, r2, rest2 = _wide_crowded(m, target, _others(V, 40, 900))
    assert t2 == toks and r2 == recs and rest2 == rest
    o = make_oracle("qwen3", cfg, w)
    rows = _teacher_force(o, target["input_ids"], toks)
    decoded = [dict(token=k[0], index=k[1], logprob=np.frombuffer(k[2], np.float32)[0], top_ids=list(k[3]),
                    top_logprobs=list(np.frombuffer(k[4], np.float32))) for k in recs]
    assert [d["token"] for d in decoded] == toks and [d["index"] for d in decoded] == list(range(len(toks)))
    _check_against_logits(decoded, rows)


def test_graphs_and_launches(q3):
    cfg, w, m = q3
    V = cfg["vocab_size"]
    graphs = lambda: int(m.debug_read("batch_graphs", 0, 1)[0])
    for wide in (0, 16):
        s = _Sess(m, wide)
        try:
            # no request asks: at most one graph per running count
            s.add_many([(("p", i), _req(V, 100 + i, 20 + i, 30, lp=False)) for i in range(3)])
            s.step(2)
            assert graphs() == 1
            m.reset_stats()
            s.step()
            base = m.stats()["kernel_launches"]
            # a request that asks joins: one more graph for the same count with the two extra launches
            s.add("q", _req(V, 200, 25, 3, top=2))
            s.step(2)
            assert graphs() <= 3
            assert "q" not in s.running.values()
            s.step()                                              # the asking request has left: the plain graph of 3 again
            m.reset_stats()
            s.step()
            assert m.stats()["kernel_launches"] == base
            counts = {3, 4}
            k = 0
            while len(s.running) < 6:
                s.add(("r", k), _req(V, 300 + k, 10 + k, 4 + k % 3, lp=k % 2 == 0, top=k)); k += 1
            while s.running:
                counts.add(len(s.running))
                s.step()
            assert graphs() <= 2 * len(counts)
        finally:
            s.close()
        assert graphs() == 0


def _raw(m, fn, ids, flags, *tail):
    """a single-request C entry called with exactly `flags` (the Python wrappers add AHA_GEN_LOGPROBS themselves)"""
    p = m._gen_params(3, 0.0, None, None, 1.0, 64, 1, flags)
    return m._check(fn(m._h, ids.ctypes.data_as(C.POINTER(C.c_uint32)), ids.size, None, C.byref(p), *tail))


def test_refusals_leave_the_session_usable(q3):
    cfg, w, m = q3
    V = cfg["vocab_size"]
    ids = _ids(20, V, 5)
    bad_flags = [L.GEN_LOGPROBS | L.gen_top_logprobs(21), L.gen_top_logprobs(3), L.GEN_LOGPROBS | L.gen_top_logprobs(300)]
    # single-request entries
    for n in (21, 300):
        with pytest.raises(B200Error, match="at most 20"):
            m.generate(ids, max_tokens=3, logprobs=True, flags=L.gen_top_logprobs(n))
    toks, recs, n_out = (C.c_uint32 * 3)(), (L.Logprobs * 3)(), C.c_size_t(0)
    with pytest.raises(B200Error, match="needs AHA_GEN_LOGPROBS"):
        _raw(m, m._lib.aha_b200_generate_logprobs, ids, L.gen_top_logprobs(2), toks, recs, 3, C.byref(n_out), None)
    with pytest.raises(B200Error, match="must carry AHA_GEN_LOGPROBS"):
        _raw(m, m._lib.aha_b200_generate_logprobs, ids, 0, toks, recs, 3, C.byref(n_out), None)
    for f in (L.GEN_LOGPROBS, L.gen_top_logprobs(2)):
        with pytest.raises(B200Error, match="use aha_b200_generate_logprobs"):
            m.generate(ids, max_tokens=3, flags=f)
        with pytest.raises(B200Error, match="use aha_b200_generate_stream_logprobs"):
            _raw(m, m._lib.aha_b200_generate_stream, ids, f, L.TOKEN_CALLBACK(lambda u, t, i: 0), None, None)
    with pytest.raises(B200Error, match="batch session"):
        m.generate_batch([dict(input_ids=ids, max_tokens=3, logprobs=True)])
    greedy, _ = m.generate(ids, max_tokens=5)
    assert m.generate(ids, max_tokens=5, logprobs=True)[0] == greedy
    # batch sessions
    with pytest.raises(B200Error, match="no batch session"):
        m.batch_logprobs()
    s = _Sess(m)
    try:
        s.add("a", _req(V, 1, 30, 6))
        running = dict(s.running)
        for f in bad_flags:
            with pytest.raises(B200Error):
                m.batch_add(ids, max_tokens=3, flags=f)
            with pytest.raises(B200Error):
                m.batch_add_many([dict(input_ids=ids, max_tokens=3), dict(input_ids=ids, max_tokens=3, flags=f)])
        recs = (L.Logprobs * 8)()
        with pytest.raises(B200Error, match="smaller than the session width"):
            m._check(m._lib.aha_b200_batch_logprobs(m._h, recs, 7))
        with pytest.raises(B200Error, match="out"):
            m._check(m._lib.aha_b200_batch_logprobs(m._h, None, 8))
        assert s.running == running
        s.add("b", _req(V, 2, 25, 4, top=20))
        s.drain()
        assert len(s.toks["a"]) == 6 and len(s.toks["b"]) == 4
        # every slot is free again: eight requests fit
        s.add_many([(("c", i), _req(V, 10 + i, 12, 2, lp=i % 2 == 0)) for i in range(8)])
        s.drain()
    finally:
        s.close()
    with pytest.raises(B200Error, match="no batch session"):
        m.batch_logprobs()


def test_asr_generate_refuses_the_flag():
    cfg, w, m = make_model("qwen3_asr", "tiny", max_ctx=512, max_frames=400)
    try:
        ids = _ids(8, 1000, 1)
        ch = L.AsrChunk()
        ch.ids, ch.seq_len = ids.ctypes.data_as(C.POINTER(C.c_uint32)), ids.size
        p = m._gen_params(3, 0.0, None, None, 1.0, 64, 1, L.GEN_LOGPROBS | L.gen_top_logprobs(2))
        out, n = (C.c_uint32 * 3)(), C.c_size_t(0)
        with pytest.raises(B200Error, match="asr_generate returns no log-probabilities"):
            m._check(m._lib.aha_b200_asr_generate(m._h, C.byref(ch), 1, C.byref(p), out, 3, C.byref(n), L.TOKEN_CALLBACK(0), None, None))
    finally:
        m.close()
