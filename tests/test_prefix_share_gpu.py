"""The batch-session prefix cache (aha_b200_batch_prefix_cache / _stats): requests share the KV pages of cached prompt prefixes and packed
admission prefills only what follows.

  - the prefixed varlen attention (wgmma kernel and both twins) against float64, and each segment bit for bit against the single-segment
    continuation launch;
  - a request admitted with a hit yields exactly the ids and records it yields admitted cold through the same entry, in narrow and wide
    sessions, for greedy, sampled, constrained, logit-rules and top-logprobs requests, and with the SIMT GEMM;
  - sharing among running requests, page accounting, eviction, refusals, off-means-off and the scope edges."""
import numpy as np
import pytest

import constrain_ref as CR
import prefix_share_ref as R
from conftest import make_model, make_oracle

pytestmark = pytest.mark.gpu
HD = 128
# max |kernel - reference| / max |V|: the fp32 SIMT twin at the grade of test_attention_gpu.py; the split-fp16 tensor-core kernels at 4x the
# largest bound that file sets for them (these prefixes put up to 2348 keys in a row)
BOUND = {0: 8e-5, 1: 1e-5, 2: 8e-5}


def _ids(n, V, seed):
    from aha_b200 import synth
    return [int(t) for t in synth.synth_text_ids(n, V - 8, seed)]


# ------------------------------------------------------------------------------------------------------------ kernel against float64

def _qkv(rng, segs, nh, nkv, regime):
    Sq, Skv = sum(n for _, n in segs), sum(p + n for p, n in segs)
    q = rng.standard_normal((Sq, nh, HD))
    k = rng.standard_normal((Skv, nkv, HD))
    v = rng.standard_normal((Skv, nkv, HD))
    if regime == "peaked":   # every query aimed at one visible key of its segment (prefix keys included)
        q0 = k0 = 0
        G = nh // nkv
        for p, n in segs:
            for i in range(n):
                j = k0 + rng.integers(0, p + i + 1)
                for h in range(nh):
                    q[q0 + i, h] = 6.0 * k[j, h // G] / np.linalg.norm(k[j, h // G]) * np.sqrt(HD) / 4
            q0, k0 = q0 + n, k0 + p + n
    return q.astype(np.float32), k.astype(np.float32), v.astype(np.float32)


SEGS = [
    [(32, 32)],
    [(0, 48), (32, 64), (96, 160), (2048, 300)],        # prefixes 0 / 32 / 96 / 2048, suffixes across 64-key and 128-query tiles
    [(96, 144), (0, 48), (64, 200)],                    # keys start at 0, 240, 288: on 16-row but not 32-row boundaries
]


@pytest.fixture(scope="module")
def tiny():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=2048)
    yield cfg, w, m
    m.close()


@pytest.mark.parametrize("impl", [0, 1, 2])
@pytest.mark.parametrize("regime", ["flat", "peaked"])
@pytest.mark.parametrize("case", range(len(SEGS)))
@pytest.mark.parametrize("heads", [(8, 8), (16, 2)])
def test_prefixed_segments_against_float64(tiny, impl, regime, case, heads):
    _, _, m = tiny
    nh, nkv = heads
    segs = SEGS[case]
    rng = np.random.default_rng(100 * case + nh)
    q, k, v = _qkv(rng, segs, nh, nkv, regime)
    n_pages = -(-k.shape[0] // 32)
    order = rng.permutation(n_pages) + 3                 # scattered pages; pages 0..2 and the slack are NaN
    got = m.debug_prefix_attention(q, k, v, impl, segs, page_order=order)
    ref = R.prefix_attention(q, k, v, segs)
    assert np.isfinite(got).all()
    err = np.abs(got - ref).max() / np.abs(v).max()
    assert err <= BOUND[impl], err
    # each segment's rows are bit-equal to the single-segment continuation launch (causal, sq < skv)
    q0 = k0 = 0
    for p, n in segs:
        alone = m.debug_attention(q[q0:q0 + n], k[k0:k0 + p + n], v[k0:k0 + p + n], impl, True)
        assert np.array_equal(got[q0:q0 + n], alone), (p, n)
        q0, k0 = q0 + n, k0 + p + n


def test_packed_without_prefix_matches_packed_segments(tiny):
    """No prefixes: the generalised work list computes what the packed-segment entry computes, bit for bit."""
    _, _, m = tiny
    rng = np.random.default_rng(5)
    lens = [64, 96, 200]
    segs = [(0, n) for n in lens]
    q, k, v = _qkv(rng, segs, 16, 8, "flat")
    starts = np.cumsum([0] + lens)[:-1]
    for impl in (0, 1, 2):
        a = m.debug_prefix_attention(q, k, v, impl, segs)
        b = m.debug_attention(q, k, v, impl, True, segments=[(int(s), n) for s, n in zip(starts, lens)])
        assert np.array_equal(a, b), impl


# ------------------------------------------------------------------------------------------------------------ sessions

def _drive(m, admit, n_steps_max=400):
    """admit() -> [(slot, tok, fin), ...]; step until they finish -> (ids per request, records per request or None)"""
    res = admit()
    lp = m.batch_logprobs()
    out = [[tok] for _, tok, _ in res]
    recs = [[lp[s]] if s in lp else None for s, _, _ in res]
    running = {s: i for i, (s, _, fin) in enumerate(res) if not fin}
    for _ in range(n_steps_max):
        if not running:
            break
        st = m.batch_step()
        lp = m.batch_logprobs()
        for s, (tok, fin) in st.items():
            i = running[s]
            out[i].append(tok)
            if recs[i] is not None:
                recs[i].append(lp[s])
            if fin:
                del running[s]
    assert not running
    return out, recs


def _open(m, wide):
    if wide:
        m.batch_open_wide(16)
    else:
        m.batch_open()


def _admit_fn(m, entry, reqs):
    if entry == "add":
        return lambda: [m.batch_add(**r) for r in reqs]
    return lambda: m.batch_add_many(reqs)


def _warm_then(m, wide, entry, warm, reqs, cache=1 << 16):
    """session with the cache on: admit `warm` and let it finish, then admit reqs -> (ids, records, per-request hits, stats)"""
    _open(m, wide)
    try:
        m.batch_prefix_cache(cache)
        _drive(m, _admit_fn(m, entry, warm))
        hits = []

        def admit():
            res = _admit_fn(m, entry, reqs)()
            st, h = m.batch_prefix_stats()
            hits.extend(h.get(s, 0) for s, _, _ in res)
            return res
        out, recs = _drive(m, admit)
        return out, recs, hits, m.batch_prefix_stats()[0]
    finally:
        m.batch_close()


def _cold(m, wide, entry, reqs):
    _open(m, wide)
    try:
        return _drive(m, _admit_fn(m, entry, reqs))
    finally:
        m.batch_close()


def _kinds(m, V):
    f = m.fsm_create(*CR.random_fsm(V, 5, 77))
    rl = m.rules_create(presence_penalty=0.5, frequency_penalty=0.3, logit_bias={3: 2.0, 11: -5.0})
    return {"greedy": dict(),
            "sampled": dict(temperature=0.8, top_p=0.9, top_k=40, repeat_penalty=1.1, repeat_last_n=16, seed=7),
            "constrained": dict(temperature=0.7, seed=3, fsm=f),
            "rules": dict(temperature=0.9, seed=5, rules=rl),
            "logprobs": dict(temperature=0.6, seed=9, logprobs=True, top_logprobs=3)}


@pytest.mark.parametrize("wide", [False, True])
@pytest.mark.parametrize("entry", ["add", "many"])
def test_hit_is_exact(tiny, wide, entry):
    cfg, _, m = tiny
    V = cfg["vocab_size"]
    system = _ids(100, V, 1)
    a = system + _ids(30, V, 2)
    warm = [dict(input_ids=a, max_tokens=3)]
    for name, kw in _kinds(m, V).items():
        reqs = [dict(input_ids=system + _ids(50, V, 3), max_tokens=12, **kw),
                dict(input_ids=_ids(70, V, 4), max_tokens=6),                    # no hit, in the same call
                dict(input_ids=a[:96] + _ids(40, V, 5), max_tokens=9, **kw)]
        got, grec, hits, st = _warm_then(m, wide, entry, warm, reqs)
        want, wrec = _cold(m, wide, entry, reqs)
        expect = [R.hit_tokens(R.cached_pages([a], r["input_ids"]), len(r["input_ids"])) for r in reqs]
        assert hits == expect and expect[0] == 96 and expect[2] == 96, (name, hits)
        assert st["hit_tokens"] == sum(expect) and st["lookups"] == 1 + len(reqs)
        assert got == want, name
        assert grec == wrec, name


def test_hit_is_exact_simt_gemm():
    """gemm_impl = 1: the hit may leave fewer than 32 prompt tokens to run."""
    cfg, _, m = make_model("qwen3", "tiny", max_ctx=1024, gemm_impl=1)
    try:
        V = cfg["vocab_size"]
        a = _ids(128, V, 11)
        reqs = [dict(input_ids=a[:96] + _ids(7, V, 12), max_tokens=10, temperature=0.8, seed=4),
                dict(input_ids=a[:64] + _ids(1, V, 13), max_tokens=10)]
        for entry in ("add", "many"):
            got, _, hits, _ = _warm_then(m, False, entry, [dict(input_ids=a, max_tokens=2)], reqs)
            assert hits == [96, 64]
            assert got == _cold(m, False, entry, reqs)[0]
    finally:
        m.close()


def test_eight_requests_share_one_system_prompt(tiny):
    cfg, w, m = tiny
    V = cfg["vocab_size"]
    o = make_oracle("qwen3", cfg, w)
    from test_prefix_cache_gpu import _oracle_generate
    system = _ids(256, V, 21)
    warm = dict(input_ids=system + _ids(40, V, 22), max_tokens=2)
    reqs = [dict(input_ids=system + _ids(40, V, 30 + i), max_tokens=4 + 3 * i) for i in range(8)]
    n_pages = 2048 // 32
    m.batch_open()
    try:
        m.batch_prefix_cache(4096)
        _drive(m, lambda: [m.batch_add(**warm)])
        st, _ = m.batch_prefix_stats()
        assert st["cached_pages"] == 9 and st["shared_pages"] == 0 and st["free_pages"] == n_pages - 9
        res = m.batch_add_many(reqs)
        st, hits = m.batch_prefix_stats()
        assert hits == {s: 256 for s, _, _ in res}
        # the 8 system pages are held once; each request adds its own 9th full page to the index
        assert st["cached_pages"] == 9 + 8 and st["shared_pages"] == 8 + 8
        own = sum(-(-(296 + r["max_tokens"]) // 32) - 8 for r in reqs)
        assert st["free_pages"] == n_pages - 9 - own
        out = [[t] for _, t, _ in res]
        running = {s: i for i, (s, _, _) in enumerate(res)}
        while running:
            for s, (t, fin) in m.batch_step().items():
                out[running[s]].append(t)
                if fin:
                    del running[s]
            st, _ = m.batch_prefix_stats()
            # finished requests free only their own unindexed pages; the shared ones stay for the others
            assert st["cached_pages"] == 17
        st, _ = m.batch_prefix_stats()
        assert st["shared_pages"] == 0 and st["free_pages"] == n_pages - 17
        for r, ids in zip(reqs, out):
            assert ids == _oracle_generate(o, r["input_ids"], None, r["max_tokens"])
    finally:
        m.batch_close()
    m.batch_open()
    try:
        assert m.batch_prefix_stats()[0]["free_pages"] == n_pages and m.batch_prefix_stats()[0]["cached_pages"] == 0
    finally:
        m.batch_close()


def test_eviction_and_refusal():
    cfg, _, m = make_model("qwen3", "tiny", max_ctx=512)      # 16 pages
    try:
        V = cfg["vocab_size"]
        A, B = _ids(100, V, 41), _ids(100, V, 42)
        m.batch_open()
        m.batch_prefix_cache(512)
        _drive(m, lambda: [m.batch_add(input_ids=A, max_tokens=4)])
        _drive(m, lambda: [m.batch_add(input_ids=B, max_tokens=4)])
        st, _ = m.batch_prefix_stats()
        assert st["cached_pages"] == 6 and st["free_pages"] == 10 and st["evicted_pages"] == 0
        # a request that needs more than free + evictable is refused, and nothing changes
        with pytest.raises(RuntimeError, match="KV capacity"):          # 12 + 5 pages > 10 free + 6 evictable
            m.batch_add_many([dict(input_ids=_ids(300, V, 43), max_tokens=60), dict(input_ids=_ids(100, V, 46), max_tokens=30)])
        assert m.batch_prefix_stats()[0] == st
        # 12 pages: free 10 + 2 evicted, least recently used leaves first (A's last two pages)
        C = _ids(300, V, 44)
        _drive(m, lambda: [m.batch_add(input_ids=C, max_tokens=60)])
        st, _ = m.batch_prefix_stats()
        assert st["evicted_pages"] == 2
        slot, _, _ = m.batch_add(input_ids=A[:64] + _ids(40, V, 45), max_tokens=2)
        assert m.batch_prefix_stats()[1] == {slot: 32}     # A's first page survived, its second did not
        _drive(m, lambda: [])
        while m.batch_step():
            pass
        # max_tokens 0 releases every page only the index holds
        m.batch_prefix_cache(0)
        st, _ = m.batch_prefix_stats()
        assert st["cached_pages"] == 0 and st["free_pages"] == 16
        m.batch_close()
    finally:
        m.close()


def test_off_means_off(tiny):
    """A session that never turns the cache on, and one that turns it off again, launch the same kernels and keep the same pages."""
    cfg, _, m = tiny
    V = cfg["vocab_size"]
    system = _ids(100, V, 51)
    reqs = [dict(input_ids=system + _ids(40 + i, V, 52 + i), max_tokens=5) for i in range(3)]

    def run(toggle):
        m.batch_open()
        try:
            if toggle:
                m.batch_prefix_cache(4096)
                m.batch_prefix_cache(0)
            m.reset_stats()
            out, _ = _drive(m, lambda: m.batch_add_many(reqs))
            out2, _ = _drive(m, lambda: [m.batch_add(**reqs[0])])
            st, hits = m.batch_prefix_stats()
            return out + out2, m.stats()["kernel_launches"], st
        finally:
            m.batch_close()
    a, ka, sa = run(False)
    b, kb, sb = run(True)
    assert a == b and ka == kb
    assert sa["cached_pages"] == sb["cached_pages"] == 0 and sa["lookups"] == 0 and sa["free_pages"] == sb["free_pages"] == 2048 // 32


def test_long_prompt_hits_and_matches_oracle():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=1024, max_prefill=128)
    try:
        o = make_oracle("qwen3", cfg, w)
        from test_prefix_cache_gpu import _oracle_generate
        V = cfg["vocab_size"]
        system = _ids(200, V, 61)
        m.batch_open()
        m.batch_prefix_cache(1024)
        _drive(m, lambda: [m.batch_add(input_ids=system + _ids(10, V, 62), max_tokens=2)])
        r = dict(input_ids=system + _ids(150, V, 63), max_tokens=8)
        got, _ = _drive(m, lambda: m.batch_add_many([r]))
        assert m.batch_prefix_stats()[0]["hit_tokens"] == 192
        m.batch_close()
        assert got[0] == _oracle_generate(o, r["input_ids"], None, 8)
    finally:
        m.close()


def test_add_n_with_a_hit(tiny):
    cfg, _, m = tiny
    V = cfg["vocab_size"]
    system = _ids(128, V, 71)
    ids = system + _ids(40, V, 72)
    kw = dict(max_tokens=10, temperature=0.9, top_k=20, seed=100)
    m.batch_open()
    try:
        m.batch_prefix_cache(4096)
        _drive(m, lambda: [m.batch_add(input_ids=system + _ids(5, V, 73), max_tokens=2)])
        got, _ = _drive(m, lambda: m.batch_add_n(ids, 3, **kw))
        assert m.batch_prefix_stats()[0]["hit_tokens"] == 128
        single = []
        for i in range(3):
            single.append(_drive(m, lambda: [m.batch_add(ids, **dict(kw, seed=100 + i))])[0][0])
        assert got == single
    finally:
        m.batch_close()


def test_vl_images_never_hit_or_insert():
    from aha_b200 import synth
    from oracle.qwen3vl import process_image
    cfg, _, m = make_model("qwen3vl", "tiny", max_ctx=2048, max_patches=1024)
    try:
        V = cfg["text_config"]["vocab_size"]
        pv, grid = process_image(synth.synth_image(128, 192, 2))
        data = [pv, grid, None, None, None]
        img = [int(t) for t in synth.vl_prompt_ids(cfg, grid, 80)]
        text = _ids(120, V, 81)
        none = [None] * 5
        m.batch_open()
        m.batch_prefix_cache(4096)
        _drive(m, lambda: [m.batch_add(img, data=data, max_tokens=2)])
        assert m.batch_prefix_stats()[0]["cached_pages"] == 0
        _drive(m, lambda: [m.batch_add(img, data=data, max_tokens=2)])
        assert m.batch_prefix_stats()[0]["hit_tokens"] == 0
        _drive(m, lambda: [m.batch_add(text, data=none, max_tokens=2)])
        assert m.batch_prefix_stats()[0]["cached_pages"] == 3
        r = dict(input_ids=text[:96] + _ids(50, V, 82), data=none, max_tokens=8)
        got, _ = _drive(m, lambda: m.batch_add_many([r]))
        assert m.batch_prefix_stats()[0]["hit_tokens"] == 96
        m.batch_close()
        want = _cold(m, False, "many", [r])[0]
        assert got == want
    finally:
        m.close()
