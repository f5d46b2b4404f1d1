"""Several choices of one request (OpenAI `n`): aha_b200_batch_add_n / aha_b200_generate_n and B200Model.batch_add_n / generate_n.

The prompt is prefilled once, its K/V pages are copied into every other choice's own pages by kv_fork_kernel, and every choice draws its
first token from the same prefill logits with its own sampler.  Choice i must yield, bit for bit, what a fresh session's batch_add yields
for the request with seed i (and generate() for a narrow session), with the same log-probability records."""
import numpy as np
import pytest

from conftest import make_model, make_oracle

pytestmark = pytest.mark.gpu

SEED = 299792458


def _ids(n, vocab, seed):
    from aha_b200 import synth
    return synth.synth_text_ids(n, vocab - 8, seed)


def _samp(r):
    return {k: v for k, v in r.items() if k not in ("input_ids", "max_tokens", "data", "flags")}


def _oracle_generate(o, r):
    from test_prefix_cache_gpu import _oracle_generate as og
    return og(o, r["input_ids"], r.get("data"), r["max_tokens"], **_samp(r))


def _seeds_of(r, n, seeds):
    return list(seeds) if seeds is not None else [r.get("seed", SEED) + i for i in range(n)]


class _Session:
    """Drives an open session: ids (and records) per name; wide = 0 opens a narrow session."""

    def __init__(self, m, wide=0, records=False):
        self.m, self.out, self.rec, self.running, self.records = m, {}, {}, {}, records
        self.counts = set()
        m.batch_open_wide(wide) if wide else m.batch_open()

    def _admitted(self, name, slot, tok, fin):
        self.out[name] = [tok]
        if self.records:
            self.rec[name] = [self.m.batch_logprobs()[slot]]
        if not fin:
            assert slot not in self.running
            self.running[slot] = name

    def add(self, name, r):
        res = self.m.batch_add(**r)
        self._admitted(name, *res)
        return res

    def add_n(self, names, r, seeds=None):
        res = self.m.batch_add_n(n=len(names), seeds=seeds, **r)
        for name, (slot, tok, fin) in zip(names, res):
            self._admitted(name, slot, tok, fin)
        return res

    def step(self, n=1):
        for _ in range(n):
            self.counts.add(len(self.running))
            res = self.m.batch_step()
            assert sorted(res) == sorted(self.running)
            recs = self.m.batch_logprobs() if self.records else None
            for slot, (tok, fin) in res.items():
                name = self.running[slot]
                self.out[name].append(tok)
                if self.records:
                    self.rec[name].append(recs[slot])
                if fin:
                    del self.running[slot]

    def drain(self):
        while self.running:
            self.step()

    def close(self):
        self.m.batch_close()


def _forked(m, r, n, seeds=None, wide=0, records=False):
    """one batch_add_n at session start, drained -> (ids per choice, records per choice, admission results)"""
    s = _Session(m, wide, records)
    try:
        res = s.add_n(list(range(n)), r, seeds)
        s.drain()
    finally:
        s.close()
    return [s.out[i] for i in range(n)], [s.rec.get(i) for i in range(n)], res


def _alone(m, r, wide=0, records=False):
    """the request alone in a fresh session (batch_add) -> (ids, records)"""
    s = _Session(m, wide, records)
    try:
        s.add("X", r)
        s.drain()
    finally:
        s.close()
    return s.out["X"], s.rec.get("X")


@pytest.fixture(scope="module")
def q3():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=8192)
    yield cfg, w, m, make_oracle("qwen3", cfg, w)
    m.close()


# prompts across the 32-token page (a partial last page, exactly one page, one token past it); samplers mixed, one greedy with a penalty
SAMPLERS = {1: dict(temperature=0.8, top_p=0.9, top_k=30, seed=5),
            31: dict(temperature=1.0, repeat_penalty=1.3, repeat_last_n=8, seed=6),
            32: dict(temperature=0.7, top_k=5, seed=7),
            33: dict(repeat_penalty=1.2, repeat_last_n=16),
            200: dict(temperature=0.9, top_p=0.8, repeat_penalty=1.1, repeat_last_n=16, seed=8)}
_ORACLE = {}


@pytest.mark.parametrize("n,given", [(1, False), (3, True), (8, False)])
@pytest.mark.parametrize("S", sorted(SAMPLERS))
def test_narrow_choices_exact(q3, S, n, given):
    cfg, w, m, o = q3
    V = cfg["vocab_size"]
    r = dict(input_ids=_ids(S, V, 40 + S), max_tokens=14, **SAMPLERS[S])
    seeds = [1000 + 31 * i for i in range(n)] if given else None
    got, _, res = _forked(m, r, n, seeds)
    assert [x[0] for x in res] == list(range(n))
    per_seed = _seeds_of(r, n, seeds)
    for i, sd in enumerate(per_seed):
        one = dict(r, seed=sd)
        assert got[i] == _alone(m, one)[0], (S, n, i)
        assert got[i] == m.generate(**one)[0], (S, n, i)
    if "temperature" in r and n == 8:
        assert len({tuple(g) for g in got}) > 1                      # the seeds really differ
    if "temperature" not in r:
        assert all(g == got[0] for g in got)                         # greedy choices are identical
    k = (S, per_seed[0])
    if k not in _ORACLE:
        _ORACLE[k] = _oracle_generate(o, dict(r, seed=per_seed[0]))
    assert got[0] == _ORACLE[k]
    gen = m.generate_n(n=n, seeds=seeds, **r)
    assert [g[0] for g in gen] == got
    for g in gen:
        assert g[1]["prompt_tokens"] == S and g[1]["completion_tokens"] == len(g[0])


@pytest.mark.parametrize("n", [16, 64])
def test_wide_choices_exact(n):
    from test_batch_wide_gpu import _check_oracle_ids
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=16384, max_prefill=512)
    o = make_oracle("qwen3", cfg, w)
    try:
        V = cfg["vocab_size"]
        r = dict(input_ids=_ids(77, V, 4040), max_tokens=10, temperature=0.9, top_k=40, repeat_penalty=1.1, repeat_last_n=8, seed=21)
        got, _, res = _forked(m, r, n, wide=64)
        assert [x[0] for x in res] == list(range(n))
        seeds = _seeds_of(r, n, None)
        for i, sd in enumerate(seeds):
            assert got[i] == _alone(m, dict(r, seed=sd), wide=64)[0], i
        sub = [0, 5, n - 1]
        _check_oracle_ids(o, [dict(r, seed=seeds[i]) for i in sub], [got[i] for i in sub])
    finally:
        m.close()


def test_mid_flight():
    """Choices forked into a session that already decodes: the running requests keep their ids; one choice stops early on a stop id that
    only it emits, a new request takes its slot and pages, and the other choices still match their own runs."""
    from aha_b200 import B200Model
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=4096)
    V = cfg["vocab_size"]
    X = dict(input_ids=_ids(70, V, 77), max_tokens=20, temperature=1.1, top_k=50, seed=3)
    n = 4
    first = [g[0] for g in m.generate_n(n=n, **X)]
    m.close()
    stop, early = None, None
    for j in range(n):                                               # a token choice j emits early and no other choice emits at all
        for k in range(2, min(8, len(first[j]))):
            t = first[j][k]
            if t not in first[j][:k] and all(t not in first[i] for i in range(n) if i != j) and t != cfg["eos_token_id"]:
                stop, early = t, j
                break
        if stop is not None:
            break
    assert stop is not None, first
    m = B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"], stop], max_ctx=4096)
    try:
        running = {"A": dict(input_ids=_ids(40, V, 78), max_tokens=30),
                   "B": dict(input_ids=_ids(90, V, 79), max_tokens=28, temperature=0.8, top_p=0.9, seed=4)}
        late = dict(input_ids=_ids(33, V, 80), max_tokens=12, temperature=0.7, seed=9)
        s = _Session(m)
        s.add("A", running["A"])
        s.add("B", running["B"])
        s.step(3)
        names = [("X", i) for i in range(n)]
        res = s.add_n(names, X)
        assert [x[0] for x in res] == [2, 3, 4, 5]
        slot_early = res[early][0]
        while ("X", early) in s.running.values():
            s.step()
        assert s.out[("X", early)][-1] == stop
        assert len(s.running) >= 3                                   # the others still decode
        slot, _, _ = s.add("late", late)
        assert slot == slot_early                                    # the lowest free slot, with the pages the choice released
        s.drain()
        s.close()
        for name, r in running.items():
            assert s.out[name] == _alone(m, r)[0], name
        for i, sd in enumerate(_seeds_of(X, n, None)):
            assert s.out[("X", i)] == _alone(m, dict(X, seed=sd))[0], i
        assert s.out["late"] == _alone(m, late)[0]
    finally:
        m.close()


def test_qwen3vl_image_prompt():
    """An image prompt with n = 4: the vision tower and the prefill run once, so batch_add_n launches fewer kernels than four batch_add
    calls, and every choice equals batch_add with its seed."""
    from aha_b200 import synth
    from oracle.qwen3vl import process_image
    cfg, w, m = make_model("qwen3vl", "tiny", max_ctx=4096, max_patches=1024)
    o = make_oracle("qwen3vl", cfg, w)
    try:
        pv, grid = process_image(synth.synth_image(256, 320, 1))
        r = dict(input_ids=synth.vl_prompt_ids(cfg, grid, 12), data=[pv, grid, None, None, None], max_tokens=10, temperature=0.8, top_k=20, seed=2)
        n = 4
        counts = []
        for fork in (True, False):
            m.batch_open()
            try:
                m.reset_stats()
                if fork:
                    res, usage = m.batch_add_n(n=n, return_usage=True, **r)
                    assert all(u["prompt_tokens"] == len(r["input_ids"]) and u["vision_secs"] > 0 for u in usage)
                else:
                    for sd in _seeds_of(r, n, None):
                        m.batch_add(**dict(r, seed=sd))
                counts.append(m.stats()["kernel_launches"])
            finally:
                m.batch_close()
        assert counts[0] < counts[1], counts
        got, _, _ = _forked(m, r, n)
        for i, sd in enumerate(_seeds_of(r, n, None)):
            assert got[i] == _alone(m, dict(r, seed=sd))[0], i
        assert got[0] == _oracle_generate(o, r)
    finally:
        m.close()


def test_prompt_longer_than_max_prefill(q3):
    cfg, w, _, o = q3
    _, _, m = make_model("qwen3", "tiny", max_ctx=4096, max_prefill=128)
    try:
        r = dict(input_ids=_ids(300, cfg["vocab_size"], 301), max_tokens=12, temperature=0.9, top_p=0.9, seed=12)
        got, _, _ = _forked(m, r, 3)
        for i, sd in enumerate(_seeds_of(r, 3, None)):
            assert got[i] == _alone(m, dict(r, seed=sd))[0], i
        assert got[0] == _oracle_generate(o, r)
    finally:
        m.close()


@pytest.fixture(scope="module")
def q3_perop():
    # the narrow session mirrors the per-op decode GEMV's summation order, so its records are those of the per-op single-request step
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=4096, decode_impl=1)
    yield cfg, m
    m.close()


@pytest.mark.parametrize("wide", [0, 8])
def test_logprobs(q3_perop, wide):
    cfg, m = q3_perop
    r = dict(input_ids=_ids(45, cfg["vocab_size"], 451), max_tokens=12, temperature=0.9, top_k=30, seed=17, logprobs=True, top_logprobs=3)
    seeds = [5, 6, 7]
    got, recs, _ = _forked(m, r, 3, seeds, wide=wide, records=True)
    for i, sd in enumerate(seeds):
        ids, rec = _alone(m, dict(r, seed=sd), wide=wide, records=True)
        assert got[i] == ids and recs[i] == rec, i
        if not wide:
            ids1, _, rec1 = m.generate(**dict(r, seed=sd))
            assert got[i] == ids1 and recs[i] == rec1, i
    if not wide:
        gen = m.generate_n(n=3, seeds=seeds, **r)
        assert [g[0] for g in gen] == got and [g[2] for g in gen] == recs


def test_refusals_change_nothing(q3):
    """Every refusal comes before device work: the running requests keep their ids, and the admissions that fit still fit."""
    from aha_b200 import B200Error, _lib as L
    cfg, w, m, o = q3
    V = cfg["vocab_size"]
    ok = dict(input_ids=_ids(20, V, 801), max_tokens=4, temperature=0.9, seed=1)
    with pytest.raises(B200Error, match="no batch session is open"):
        m.batch_add_n(n=2, **ok)
    with pytest.raises(B200Error, match="1 to 8"):
        m.generate_n(n=9, **ok)
    with pytest.raises(B200Error, match="1 to 8"):
        m.generate_n(n=0, **ok)
    running = {"A": dict(input_ids=_ids(40, V, 802), max_tokens=24), "B": dict(input_ids=_ids(70, V, 803), max_tokens=20, temperature=0.9, seed=1)}
    # 256 pages; A and B hold 5, so 251 are free: six choices of 44 pages do not fit, five do
    big = dict(input_ids=_ids(1400, V, 804), max_tokens=4)
    s = _Session(m)
    try:
        s.add("A", running["A"])
        s.add("B", running["B"])
        bad = [(0, ok, "at least 1"),
               (7, ok, "only 6 of the 8 slots are free"),
               (6, big, "KV capacity"),
               (2, dict(ok, flags=L.GEN_CONTINUE_RNG), "CONTINUE_RNG"),
               (2, dict(ok, flags=L.GEN_REUSE_PREFIX), "REUSE_PREFIX"),
               (2, dict(ok, input_ids=np.array([1, 2, V], np.uint32)), "token id out of range")]
        for n, r, msg in bad:
            with pytest.raises(B200Error, match=msg):
                m.batch_add_n(n=n, **r)
            s.step()
        with pytest.raises(B200Error, match="batch session is open"):
            m.generate_n(n=2, **ok)
        res = s.add_n([("big", i) for i in range(5)], big)
        assert [x[0] for x in res] == [2, 3, 4, 5, 6]
        s.add_n([("ok", 0)], ok)
        with pytest.raises(B200Error, match="slots"):
            m.batch_add_n(n=1, **ok)
        s.drain()
    finally:
        s.close()
    for name, r in running.items():
        assert s.out[name] == _alone(m, r)[0], name
    assert s.out[("ok", 0)] == _alone(m, ok)[0]


@pytest.mark.parametrize("graph", ["0", "1"])
def test_graphs_per_running_count(q3, graph, monkeypatch):
    cfg, w, m, o = q3
    monkeypatch.setenv("AHA_BATCH_GRAPH", graph)
    V = cfg["vocab_size"]
    s = _Session(m)
    try:
        for k in range(4):
            r = dict(input_ids=_ids(10 + 9 * k, V, 900 + k), max_tokens=3 + 2 * k, temperature=0.8, seed=k)
            s.add_n([(k, i) for i in range(min(8 - len(s.running), 3))], r)
            s.step(2)
        graphs = int(m.debug_read("batch_graphs", 0, 1)[0])
        assert graphs <= len(s.counts), (graphs, s.counts)
        if graph == "1":
            assert graphs >= 1
        s.drain()
    finally:
        s.close()
