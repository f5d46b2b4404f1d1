"""Cancel, suspend and resume requests of a batch session (aha_b200_batch_cancel / _suspend / _resume / _discard / _swap_space).

  - the page copies alone: a round trip between scattered pool pages and scattered host pages, bytes equal, other pages untouched;
  - exactness: requests suspended after admission, mid-generation and one step before their budget, at pos = 0, 1 and 31 (mod 32), then
    resumed into another slot, yield exactly what they yield uninterrupted (narrow: generate()'s ids and records; wide: an uninterrupted
    wide run), for greedy, sampled, penalised, logit-rules, constrained, top-20 log-probability and Qwen3-VL image requests;
  - oversubscription: four requests through a pool that holds two, rotated through suspend / resume;
  - prefix-cache pages evicted while their request is suspended, cancel, step graphs, eager launches and refusals."""
import numpy as np
import pytest

import constrain_ref as CR
from conftest import make_model

pytestmark = pytest.mark.gpu


def _ids(n, V, seed):
    from aha_b200 import synth
    return [int(t) for t in synth.synth_text_ids(n, V - 8, seed)]


def _key(r):
    """a record, bit for bit"""
    return (r["token"], r["index"], np.float32(r["logprob"]).tobytes(), tuple(r["top_ids"]),
            b"".join(np.float32(v).tobytes() for v in r["top_logprobs"]))


def _pages(n_tokens):
    return -(-n_tokens // 32)


# ------------------------------------------------------------------------------------------------------------ the page copies alone

@pytest.mark.parametrize("page_floats", [1, 1024, 16384, 65536])
def test_kv_swap_round_trip(page_floats):
    _, _, m = make_model("qwen3", "tiny", max_ctx=256)
    try:
        rng = np.random.default_rng(page_floats)
        layers, n_pool, n_host = 3, 12, 7
        table_out, host_pages, table_in = [7, 2, 9, 4, 0], [5, 0, 3, 1, 6], [10, 1, 11, 6, 3]
        pool = np.full((layers, n_pool, page_floats), np.nan, np.float32)
        for p in table_out:
            pool[:, p] = rng.standard_normal((layers, page_floats)).astype(np.float32)
        host, back = m.debug_kv_swap(pool, table_out, table_in, host_pages, n_host)
        bits = lambda a: a.view(np.uint32)
        for p, h in zip(table_out, host_pages):
            assert np.array_equal(bits(host[h]), bits(pool[:, p]))
        for h in set(range(n_host)) - set(host_pages):
            assert np.isnan(host[h]).all()
        for p, q in zip(table_out, table_in):
            assert np.array_equal(bits(back[:, q]), bits(pool[:, p]))
        for q in set(range(n_pool)) - set(table_in):
            assert np.array_equal(bits(back[:, q]), bits(pool[:, q]))
    finally:
        m.close()


# ------------------------------------------------------------------------------------------------------------ sessions

class _Drive:
    """a session: every request's tokens and (when it asked) records, by name; suspended requests by name"""

    def __init__(self, m, wide=0):
        self.m, self.width = m, wide or 8
        self.toks, self.recs, self.asks, self.slot, self.budget, self.plen = {}, {}, {}, {}, {}, {}
        self.running, self.susp = {}, {}
        m.batch_open_wide(wide) if wide else m.batch_open()

    def _gather(self, by_slot):
        lp = self.m.batch_logprobs()
        for slot, name in by_slot.items():
            if self.asks[name]:
                self.recs[name].append(_key(lp[slot]))
            else:
                assert slot not in lp

    def add(self, name, r):
        slot, tok, fin = self.m.batch_add(**r)
        self.toks[name], self.recs[name], self.asks[name], self.slot[name] = [tok], [], bool(r.get("logprobs")), slot
        self.budget[name], self.plen[name] = r["max_tokens"], len(r["input_ids"])
        self._gather({slot: name})
        if not fin:
            self.running[slot] = name
        return slot

    def pos(self, name):   # the request's DecodeState pos: tokens whose K/V are written
        return self.plen[name] + len(self.toks[name]) - 1

    def step(self, n=1):
        for _ in range(n):
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

    def free(self):
        return [i for i in range(self.width) if i not in self.running]

    def suspend(self, name):
        slot = self.slot[name]
        self.susp[name] = self.m.batch_suspend(slot)
        del self.running[slot]
        assert slot not in self.m.batch_logprobs()
        return slot

    def resume(self, name):
        slot = self.m.batch_resume(self.susp.pop(name))
        assert slot not in self.running
        self.running[slot], self.slot[name] = name, slot
        assert slot not in self.m.batch_logprobs()      # no token delivered: no record until the next step
        return slot

    def cancel(self, name):
        slot = self.slot[name]
        self.m.batch_cancel(slot)
        del self.running[slot]
        return slot


def _filler(V, k, **kw):
    return dict(input_ids=_ids(20 + 9 * k % 40, V, 900 + k), max_tokens=3 + k % 4, **kw)


def _run_plan(m, V, wide, reqs, plan, **filler_kw):
    """Admit reqs ([(name, request)]) with batch_add and step them to the end.  plan {name: [predicate(pos, produced, budget), ...]}: after
    admission and after every step a running request whose next predicate holds is suspended; fillers take the lowest free slot while it
    is the request's own, and the request is resumed after the next step, into another slot.
    -> (tokens by name, records by name, every request by name (fillers included), positions it was suspended at by name)"""
    d = _Drive(m, wide)
    pending = {k: list(v) for k, v in plan.items()}
    allreq, at, due = dict(reqs), {}, []
    try:
        m.batch_swap_space(1 << 14)

        def check():
            for name in list(d.running.values()):
                preds = pending.get(name)
                if preds and preds[0](d.pos(name), len(d.toks[name]), d.budget[name]):
                    preds.pop(0)
                    at.setdefault(name, []).append(d.pos(name))
                    old = d.suspend(name)
                    while min(d.free()) == old:
                        k = len(allreq)
                        allreq[f"f{k}"] = _filler(V, k, **filler_kw)
                        d.add(f"f{k}", allreq[f"f{k}"])
                    due.append((name, old))

        for name, r in reqs:
            d.add(name, r)
        check()
        while d.running or due:
            d.step()
            for name, old in due:
                assert d.resume(name) != old
            due.clear()
            check()
        assert not any(pending.values()), pending
        st = m.batch_swap_stats()
        assert st["suspended"] == 0 and st["free_host_pages"] == st["host_pages"] == (1 << 14) // 32
        return d.toks, d.recs, allreq, at
    finally:
        m.batch_close()


def _uninterrupted(m, wide, named):
    d = _Drive(m, wide)
    try:
        for name, r in named.items():
            d.add(name, r)
        while d.running:
            d.step()
        return d.toks, d.recs
    finally:
        m.batch_close()


def _single(m, r):
    kw = {k: v for k, v in r.items() if k != "input_ids"}
    if not r.get("logprobs"):
        return m.generate(r["input_ids"], **kw)[0], []
    toks, _, recs = m.generate(r["input_ids"], **kw)
    return toks, [_key(x) for x in recs]


def _check_exact(m, wide, toks, recs, allreq):
    if wide:
        wt, wr = _uninterrupted(m, wide, allreq)
        assert toks == wt
        assert recs == wr
    else:
        for name, r in allreq.items():
            want = _single(m, r)
            assert toks[name] == want[0], name
            assert recs[name] == want[1], name


@pytest.fixture(scope="module")
def q3():
    # decode_impl 1: the narrow session's records are those of the per-op single-request step (test_logprobs_gpu.py)
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=2048, decode_impl=1)
    V = cfg["vocab_size"]
    f = m.fsm_create(*CR.random_fsm(V, 5, 77))
    rl = m.rules_create(presence_penalty=0.5, frequency_penalty=0.3, logit_bias={3: 2.0, 11: -5.0})
    kinds = {"greedy": dict(),
             "sampled": dict(temperature=0.8, top_p=0.9, top_k=40, seed=7),
             "repeat_penalty": dict(temperature=0.7, repeat_penalty=1.3, repeat_last_n=16, seed=8),
             "rules": dict(temperature=0.9, seed=5, rules=rl),
             "constrained": dict(temperature=0.7, seed=3, fsm=f),
             "logprobs": dict(temperature=0.6, seed=9, logprobs=True, top_logprobs=20)}
    yield cfg, m, kinds
    m.close()


AT_ADMISSION = lambda pos, produced, budget: True
MOD1 = lambda pos, produced, budget: pos % 32 == 1
LAST_STEP = lambda pos, produced, budget: produced == budget - 1


@pytest.mark.parametrize("wide", [0, 16])
@pytest.mark.parametrize("kind", ["greedy", "sampled", "repeat_penalty", "rules", "constrained", "logprobs"])
def test_resumed_requests_are_exact(q3, kind, wide):
    cfg, m, kinds = q3
    V = cfg["vocab_size"]
    kw = kinds[kind]
    reqs = [("a", dict(input_ids=_ids(64, V, 1), max_tokens=12, **kw)),       # suspended at admission, pos 64
            ("b", dict(input_ids=_ids(40, V, 2), max_tokens=30, **kw)),       # mid-generation at pos 65
            ("c", dict(input_ids=_ids(50, V, 3), max_tokens=15, **kw)),       # one step before its budget, at pos 63
            ("d", dict(input_ids=_ids(33, V, 4), max_tokens=20))]             # a neighbour that is never suspended
    toks, recs, allreq, at = _run_plan(m, V, wide, reqs, {"a": [AT_ADMISSION, MOD1], "b": [MOD1], "c": [LAST_STEP]})
    assert at == {"a": [64, 65], "b": [65], "c": [63]}
    assert len(toks["c"]) == 15 and len(toks["b"]) == 30
    _check_exact(m, wide, toks, recs, allreq)


@pytest.mark.parametrize("wide", [0, 8])
def test_resumed_image_request_is_exact(wide):
    """Qwen3-VL: an image request carries a non-zero rope_delta in its DecodeState through three suspensions."""
    from aha_b200 import synth
    from oracle.qwen3vl import process_image
    cfg, _, m = make_model("qwen3vl", "tiny", max_ctx=2048, max_patches=1024, decode_impl=1)
    try:
        V = cfg["text_config"]["vocab_size"]
        pv, grid = process_image(synth.synth_image(256, 320, 1))
        img = dict(input_ids=[int(t) for t in synth.vl_prompt_ids(cfg, grid, 12)], data=[pv, grid, None, None, None], max_tokens=40)
        text = dict(input_ids=_ids(40, V, 9), data=[None] * 5, max_tokens=30, temperature=0.7, top_p=0.9, seed=4)
        m.batch_open()
        m.batch_add(**img)
        assert m.debug_read("rope_delta", 0, 1)[0] != 0
        m.batch_close()
        toks, recs, allreq, at = _run_plan(m, V, wide, [("img", img), ("text", text)],
                                           {"img": [AT_ADMISSION, MOD1, LAST_STEP], "text": [MOD1]}, data=[None] * 5)
        assert len(at["img"]) == 3
        _check_exact(m, wide, toks, recs, allreq)
    finally:
        m.close()


def test_oversubscribed_pool_rotates_four_requests():
    """max_ctx holds two requests' pages: four run to completion by taking turns.  Whenever one is suspended another takes its pages and
    writes its own K/V there before it comes back."""
    cfg, _, m = make_model("qwen3", "tiny", max_ctx=256, decode_impl=1)       # 8 pages; each request needs 4
    try:
        V = cfg["vocab_size"]
        named = {f"r{i}": dict(input_ids=_ids(n, V, 30 + i), max_tokens=b, **kw)
                 for i, (n, b, kw) in enumerate([(70, 50, {}), (75, 45, dict(temperature=0.8, top_k=20, seed=2)), (80, 40, {}),
                                                 (72, 48, dict(temperature=0.7, repeat_penalty=1.2, repeat_last_n=8, seed=3))])}
        need = {k: _pages(len(r["input_ids"]) + r["max_tokens"]) for k, r in named.items()}
        assert set(need.values()) == {4}
        d = _Drive(m)
        waiting, suspended, rotations = list(named), [], 0
        free_pages = lambda: m.batch_prefix_stats()[0]["free_pages"]
        try:
            m.batch_swap_space(512)                                 # up to three requests suspended at once
            while waiting or suspended or d.running:
                # new requests first, then the suspended ones, while pages last
                while (waiting or suspended) and free_pages() >= 4:
                    if waiting:
                        name = waiting.pop(0)
                        d.add(name, named[name])
                    else:
                        d.resume(suspended.pop(0))
                    if free_pages() == 0:
                        assert len(d.running) == 2          # the pages a suspended request left are all in use again
                if d.running:
                    d.step(3)
                if len(d.running) == 2 and (waiting or suspended):
                    # a request is waiting: preempt the running request with the most tokens left
                    name = max(d.running.values(), key=lambda k: d.budget[k] - len(d.toks[k]))
                    d.suspend(name)
                    suspended.append(name)
                    rotations += 1
            assert rotations >= 4
            st = m.batch_swap_stats()
            page_bytes = cfg["num_hidden_layers"] * 2 * cfg["num_key_value_heads"] * 32 * cfg["head_dim"] * 4
            assert st["suspended"] == 0 and st["pages_out"] == st["pages_in"] > 0
            assert st["bytes_out"] == st["pages_out"] * page_bytes and st["bytes_in"] == st["bytes_out"]
        finally:
            m.batch_close()
        for name, r in named.items():
            assert d.toks[name] == _single(m, r)[0], name
    finally:
        m.close()


def test_prefix_pages_evicted_while_suspended():
    cfg, _, m = make_model("qwen3", "tiny", max_ctx=2048, decode_impl=1)
    try:
        V = cfg["vocab_size"]
        n_pages = 2048 // 32
        system = _ids(96, V, 51)
        r = dict(input_ids=system + _ids(40, V, 52), max_tokens=12, temperature=0.8, seed=6)
        d = _Drive(m)
        try:
            m.batch_prefix_cache(4096)
            m.batch_swap_space(2048)
            d.add("warm", dict(input_ids=system + _ids(20, V, 53), max_tokens=2))
            d.step()
            slot = d.add("r", r)
            st, hits = m.batch_prefix_stats()
            # the 3 system pages shared with the index, r's own 4th full page inserted
            assert hits == {slot: 96} and st["cached_pages"] == 4 and st["shared_pages"] == 4
            d.step(3)
            d.suspend("r")
            st, hits = m.batch_prefix_stats()
            assert hits == {} and st["cached_pages"] == 4 and st["shared_pages"] == 0 and st["free_pages"] == n_pages - 4
            m.batch_prefix_cache(32)                               # evict leaves down to the first system page
            st, _ = m.batch_prefix_stats()
            assert st["cached_pages"] == 1 and st["free_pages"] == n_pages - 1
            d.add("other", dict(input_ids=_ids(300, V, 54), max_tokens=4))   # takes the freed pages and writes over them
            d.step()
            # other's insert evicted the last system page and cached its own first page (its table holds it too)
            st, _ = m.batch_prefix_stats()
            assert st["cached_pages"] == 1 and st["shared_pages"] == 1 and st["free_pages"] == n_pages - _pages(304)
            slot = d.resume("r")
            st, hits = m.batch_prefix_stats()
            # restored as r's own 5 pages; the index is not touched
            assert hits == {slot: 96} and st["cached_pages"] == 1 and st["shared_pages"] == 1
            assert st["free_pages"] == n_pages - _pages(304) - _pages(136 + 12)
            while d.running:
                d.step()
            st, _ = m.batch_prefix_stats()
            assert st["free_pages"] == n_pages - st["cached_pages"]
        finally:
            m.batch_close()
        assert d.toks["r"] == _single(m, r)[0]
    finally:
        m.close()


def test_cancel(q3):
    cfg, m, kinds = q3
    V = cfg["vocab_size"]
    reqs = {"a": dict(input_ids=_ids(50, V, 61), max_tokens=20),
            "b": dict(input_ids=_ids(70, V, 62), max_tokens=40, logprobs=True, top_logprobs=5, temperature=0.8, seed=1),
            "c": dict(input_ids=_ids(45, V, 63), max_tokens=25, **kinds["rules"]),
            "d": dict(input_ids=_ids(33, V, 64), max_tokens=10, **kinds["sampled"])}
    d = _Drive(m)
    try:
        for name in "abc":
            d.add(name, reqs[name])
        d.step(2)
        before = m.batch_prefix_stats()[0]["free_pages"]
        slot = d.cancel("b")
        assert m.batch_prefix_stats()[0]["free_pages"] == before + _pages(70 + 40)
        assert slot not in m.batch_logprobs()
        assert d.add("d", reqs["d"]) == slot                   # the slot is taken again in the same step loop
        while d.running:
            d.step()
    finally:
        m.batch_close()
    for name in "acd":
        assert d.toks[name] == _single(m, reqs[name])[0], name


def test_cancel_speculative_slot(q3):
    cfg, m, _ = q3
    V = cfg["vocab_size"]
    plain = dict(input_ids=_ids(40, V, 71), max_tokens=20)
    ids = _ids(60, V, 72)

    def run(cancel):
        m.batch_open_wide(8)
        try:
            s0, t0, _ = m.batch_add(**plain)
            out = [t0]
            s1, _, _ = m.batch_add_speculative(ids, prediction=ids[10:40], max_draft=3, max_tokens=30, logprobs=True)
            for _ in range(2):
                st = m.batch_step_spec()
                out += st[s0][0]
            if cancel:
                before = m.batch_prefix_stats()[0]["free_pages"]
                stats = m.batch_spec_stats()
                m.batch_cancel(s1)
                assert m.batch_prefix_stats()[0]["free_pages"] == before + _pages(60 + 30 + 3)
                assert m.batch_spec_stats() == stats and stats[s1]["passes"] == 2
                assert s1 not in m.batch_logprobs() and s1 not in m.batch_logprobs_spec()
            while True:
                st = m.batch_step_spec()
                if s0 not in st:
                    break
                out += st[s0][0]
                if st[s0][1]:
                    break
            return out
        finally:
            m.batch_close()
    assert run(True) == run(False)


def test_graphs_and_eager_launches(q3, monkeypatch):
    cfg, m, kinds = q3
    V = cfg["vocab_size"]
    reqs = {f"r{i}": dict(input_ids=_ids(30 + 5 * i, V, 80 + i), max_tokens=60, **(kinds["sampled"] if i % 2 else {})) for i in range(4)}

    def run():
        d = _Drive(m)
        graphs = []
        try:
            m.batch_swap_space(4096)
            for name, r in reqs.items():
                d.add(name, r)
            for cycle in range(6):
                d.suspend("r1")             # 3 running
                d.step()
                d.resume("r1")              # 4 running again
                d.step()
                graphs.append(int(m.debug_read("batch_graphs", 0, 1)[0]))
            while d.running:
                d.step()
            return d.toks, graphs
        finally:
            m.batch_close()

    toks, graphs = run()
    assert graphs[0] == 2 and all(g == 2 for g in graphs)     # one graph per running count, none added by later cycles
    monkeypatch.setenv("AHA_BATCH_GRAPH", "0")
    eager, eg = run()
    assert eager == toks and all(g == 0 for g in eg)
    for name, r in reqs.items():
        assert toks[name] == _single(m, r)[0], name


def test_refusals_change_nothing():
    cfg, _, m = make_model("qwen3", "tiny", max_ctx=256)             # 8 pages
    try:
        V = cfg["vocab_size"]
        for call, args in ((m.batch_suspend, (0,)), (m.batch_cancel, (0,)), (m.batch_resume, (1,)), (m.batch_discard, (1,))):
            with pytest.raises(RuntimeError, match="no batch session is open"):
                call(*args)
        m.batch_swap_space(0)                                            # works without a session
        f = m.fsm_create(*CR.random_fsm(V, 4, 5))
        rl = m.rules_create(frequency_penalty=0.5)
        a = dict(input_ids=_ids(40, V, 91), max_tokens=20, temperature=0.8, seed=3)
        d = _Drive(m)
        try:
            sa = d.add("a", a)
            d.add("e", dict(input_ids=_ids(10, V, 92), max_tokens=20, temperature=0.5, seed=1, fsm=f))
            d.add("g", dict(input_ids=_ids(12, V, 93), max_tokens=20, rules=rl))
            with pytest.raises(RuntimeError, match="outside the session's 8 slots"):
                m.batch_suspend(8)
            with pytest.raises(RuntimeError, match="runs no request"):
                m.batch_suspend(5)
            with pytest.raises(RuntimeError, match="runs no request"):
                m.batch_cancel(5)
            with pytest.raises(RuntimeError, match="no swap space"):
                m.batch_suspend(sa)
            m.batch_swap_space(32)                                       # one host page; a has written 2 pages
            with pytest.raises(RuntimeError, match="host pages are free"):
                m.batch_suspend(sa)
            assert m.batch_swap_stats()["suspended"] == 0
            d.step()
            m.batch_swap_space(256)
            d.suspend("a")
            d.suspend("e")
            d.suspend("g")
            ids_g = d.susp["g"]
            with pytest.raises(RuntimeError, match="requests are suspended"):
                m.batch_swap_space(512)
            with pytest.raises(RuntimeError, match="constrains suspended request"):
                m.fsm_destroy(f)
            with pytest.raises(RuntimeError, match="applies to suspended request"):
                m.rules_destroy(rl)
            with pytest.raises(RuntimeError, match="no suspended request of this session has id 999"):
                m.batch_resume(999)
            with pytest.raises(RuntimeError, match="no suspended request"):
                m.batch_discard(999)
            m.batch_discard(d.susp.pop("g"))
            with pytest.raises(RuntimeError, match="no suspended request"):
                m.batch_resume(ids_g)
            st = m.batch_swap_stats()
            assert st["suspended"] == 2 and st["host_pages"] == 8
            # no free slot: 8 one-page requests
            for i in range(8):
                d.add(f"s{i}", dict(input_ids=_ids(10, V, 100 + i), max_tokens=3))
            with pytest.raises(RuntimeError, match="all 8 slots are decoding"):
                m.batch_resume(d.susp["a"])
            while d.running:
                d.step()
            # no pages: one request holds 7 of the 8, a needs 2
            big = d.add("big", dict(input_ids=_ids(100, V, 110), max_tokens=100))
            with pytest.raises(RuntimeError, match="tokens of KV capacity"):
                m.batch_resume(d.susp["a"])
            assert m.batch_swap_stats() == st
            d.cancel("big")
            assert big not in m.batch_logprobs()
            d.resume("a")
            while d.running:
                d.step()
            assert m.batch_swap_stats()["suspended"] == 1
        finally:
            m.batch_close()
        st = m.batch_swap_stats()                                        # batch_close discarded e
        assert st["suspended"] == 0 and st["free_host_pages"] == st["host_pages"] == 8
        m.fsm_destroy(f)
        m.rules_destroy(rl)
        assert d.toks["a"] == _single(m, a)[0]
        # a speculative slot cannot be suspended
        m.batch_open_wide(4)
        try:
            ids = _ids(40, V, 120)
            s, _, _ = m.batch_add_speculative(ids, prediction=ids[:20], max_draft=3, max_tokens=10)
            with pytest.raises(RuntimeError, match="speculative request, which cannot be suspended"):
                m.batch_suspend(s)
            m.batch_cancel(s)
        finally:
            m.batch_close()
        m.batch_swap_space(0)
        assert m.batch_swap_stats()["host_pages"] == 0
    finally:
        m.close()
