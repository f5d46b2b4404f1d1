"""The device sampler (sampling.cuh: sample_kernel and sample_rows_kernel) at the vocabularies the models ship with and at the edges of
its blocked arithmetic, through aha_b200_debug_sample on host logits.

 * token for token against oracle/sample.py for V from 1 to 262144 (ragged last chunks, up to 1024 chunk owners), in six logit regimes
   (scaled normal, peaked with underflowed probabilities, a coarse grid with exact ties, all equal, masked -inf, and tie groups built to
   straddle chunk boundaries at the k-th value and at the top-p threshold), every mode, top_k / top_p / draw index / seed edges, and the
   repeat penalty over long contexts;
 * the two kernels agree, and a row's token does not depend on its slot, the other rows or rows that do not sample;
 * the DecodeState a call leaves (n_draws, the overwritten ArgMax token);
 * drawn frequencies against float64 truncated probabilities built with candle's rule, independently of the oracle;
 * refusals (sampler error, bad shapes) that leave the handle usable.
Each case asserts on the oracle side the property it was built for (ties at the cut, zero probabilities, V % 256), so a regime that
stops exercising its branch fails instead of passing quietly."""
import numpy as np
import pytest
from scipy.stats import chisquare

from conftest import make_model
from oracle import sample as S

pytestmark = pytest.mark.gpu

F32 = np.float32
QWEN3_V = 151936                       # = 593 * 256 + 128: the last chunk holds 128 entries
TOP_K = (1, 2, 255, 256, 257, 513, 1000, 1024)
TOP_P = (1e-4, 0.3, 0.9, 0.999999, 1.0, 1.5)
DRAWS = (0, 15, 16, 17, 2**32 - 1)      # both sides of a ChaCha block (16 words), and the last index
SEEDS = (0, 2**64 - 1, 1234)
NONE = 0xFFFFFFFF


@pytest.fixture(scope="module")
def tiny():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=512)
    yield m
    m.close()


def _f32(x):
    return None if x is None else float(F32(x))


def _want(lg, q, ctx=(), draw=0, overwrite=False):
    """the oracle's token for one row; the parameters are rounded to the float32 the device reads"""
    ctx = [int(t) for t in ctx]
    if overwrite:
        ctx = ctx[:-1]
    pl = S.use_repeat_penalty(_f32(q.get("repeat_penalty", 1.0)), q.get("repeat_last_n", 64), lg, ctx)
    return S.sample(pl, _f32(q.get("temperature", 0.0)), _f32(q.get("top_p")), q.get("top_k"), S.StdRng(q.get("seed", 299792458)), int(draw))


def _imp(V):
    """ids where chunk bugs show: the first, both sides of the first boundary, and the ragged last chunk"""
    last0 = (V - 1) // 256 * 256
    return sorted({i for i in (0, 255, 256, last0, (last0 + V - 1) // 2, V - 1) if i < V})


def _tie_group(V):
    """ids of a tie group that crosses chunk boundaries: 250..261, both sides of up to 40 later boundaries, and the last chunk"""
    g = set(range(250, 262))
    nch = (V + 255) // 256
    for c in range(2, nch, max(1, nch // 40)):
        g |= {c * 256 - 2, c * 256 + 1}
    g |= {V - 3, V - 2}
    return np.array(sorted(i for i in g if i < V and i not in _imp(V)))


def _kth_ties(p, k):
    """number of entries equal to the k-th largest probability"""
    return int(np.count_nonzero(p == np.sort(p)[::-1][k - 1]))


def _case(V, regime):
    """-> (logits [V], temperature, extra rows) with the regime's property asserted on the oracle's probabilities"""
    rng = np.random.default_rng(V * 7 + len(regime))
    imp = _imp(V)
    extra = []
    if regime == "normal":
        t = 0.9
        lg = (rng.standard_normal(V) * 2.5).astype(F32)
        lg[imp] = lg.max() + np.linspace(0.5, 0.1, len(imp), dtype=F32)
    elif regime == "peaked":                 # at t = 0.05 everything 8 below the head underflows to exactly 0
        t = 0.05
        lg = rng.standard_normal(V).astype(F32)
        lg[imp] = F32(12) - F32(0.05) * np.arange(len(imp), dtype=F32)
        lg[rng.integers(0, V, 5)] = F32(12 - 5.1)           # and a few land on denormals
        extra = [dict(temperature=t, top_k=50), dict(temperature=t, top_k=50, top_p=0.9), dict(temperature=t, top_k=50, top_p=1.0)]
    elif regime == "grid":                   # a 0.5 grid: exact ties at every k and at every threshold
        t = 1.0
        lg = (np.round(rng.standard_normal(V) * 4) / 2).astype(F32)
    elif regime == "equal":
        t = 0.7
        lg = np.zeros(V, F32)
    elif regime == "masked":                 # -inf at id 0, across the first boundary, in 30 % of the rest and in the last chunk
        t = 0.8
        lg = (rng.standard_normal(V) * 2).astype(F32)
        lg[rng.random(V) < 0.3] = -np.inf
        lg[[0, *range(250, min(V, 262))]] = -np.inf
        last0 = (V - 1) // 256 * 256
        lg[last0:last0 + (V - last0) // 2] = -np.inf
        lg[V - 1] = 1.0
    elif regime == "straddle":               # a head of distinct values over a tie group that crosses chunk boundaries
        t = 1.0
        lg = (rng.standard_normal(V) - 8).astype(F32)
        lg[imp] = F32(4) - F32(0.2) * np.arange(len(imp), dtype=F32)
        G = _tie_group(V)
        lg[G] = 2.0
        m, g = len(imp), len(G)
        p = S.softmax_blocked(lg, t)
        k_cut = m + g // 2
        assert k_cut <= 1024 and _kth_ties(p, k_cut) == g
        A = S.blocked_sum(np.where(p > p[G[0]], p, F32(0)))
        top_p = float(F32(A + (g // 2 + 0.5) * float(p[G[0]])))          # the threshold cuts the group in the middle
        w = S.topp_weights(p, top_p)
        kept = G[w[G] > 0]
        assert len(kept) == g // 2 + 1
        if V >= 1000:                        # kept and dropped ties on both sides of chunk boundaries
            assert kept[-1] // 256 > kept[0] // 256 and G[-1] // 256 > kept[-1] // 256
        extra = [dict(temperature=t, top_k=k_cut), dict(temperature=t, top_k=k_cut - 1), dict(temperature=t, top_k=m + g - 1),
                 dict(temperature=t, top_p=top_p), dict(temperature=t, top_k=V, top_p=top_p),
                 dict(temperature=t, top_k=min(1024, m + g), top_p=top_p)]
    p = S.softmax_blocked(lg, t)
    if regime == "peaked" and V > 64:
        assert np.count_nonzero(p == 0) > V // 2 and np.count_nonzero(p) < 50
    if regime == "grid" and V >= 1000:
        assert sum(_kth_ties(p, k) > 1 for k in TOP_K if k < V) >= 4
    if regime == "masked" and V > 2:
        assert p[0] == 0 and np.count_nonzero(p == 0) > 0.25 * V
    return lg, t, extra


def _rows(V, t, imp, extra, penalise):
    ks = [k for k in (*TOP_K, V - 1, V, V + 1, 2**31 - 1) if k >= 1 and (k <= 1024 or k >= V)]
    rows = [dict(temperature=t), dict(temperature=t)]
    rows += [dict(temperature=t, top_p=p) for p in TOP_P]
    rows += [dict(temperature=t, top_k=k) for k in ks]
    rows += [dict(temperature=t, top_k=k, top_p=TOP_P[i % len(TOP_P)]) for i, k in enumerate(ks)]
    rows += [dict(temperature=t, top_k=k, top_p=p) for k in (V, 2**31 - 1) for p in (0.9, 1.0, 1.5)]
    rows += [dict(temperature=0.0, repeat_penalty=pen) for pen in (1.3, 3.0)] + extra
    assert len(rows) <= 64
    ctxs, draws = [], []
    for i, q in enumerate(rows):
        q["seed"] = SEEDS[i % len(SEEDS)]
        if penalise and i % 4 == 1 and "repeat_penalty" not in q:
            q["repeat_penalty"] = 1.3
        ctxs.append([imp[0], imp[0], V + 5, imp[-1]])       # a duplicate and an id past the vocabulary
        draws.append(DRAWS[i % len(DRAWS)])
    return rows, ctxs, draws


CASES = [(V, r) for V in (1, 2) for r in ("normal", "equal", "masked") if not (V == 1 and r == "masked")]
CASES += [(V, r) for V in (255, 256, 257, 1000, 4097, QWEN3_V, 262144) for r in ("normal", "peaked", "grid", "equal", "masked", "straddle")]


@pytest.mark.parametrize("V,regime", CASES)
def test_tokens_match_the_oracle(tiny, V, regime):
    lg, t, extra = _case(V, regime)
    rows, ctxs, draws = _rows(V, t, _imp(V), extra, penalise=regime not in ("straddle", "peaked"))
    want = [_want(lg, q, c, d) for q, c, d in zip(rows, ctxs, draws)]
    n = len(rows)
    for kernel, act in ((0, None), (1, np.arange(n)[::-1] + (64 - n))):
        got = tiny.debug_sample_rows(lg, rows, ctxs, draws, kernel=kernel, act=act)["token"]
        bad = [(i, rows[i], draws[i], int(got[i]), want[i]) for i in range(n) if got[i] != want[i]]
        assert not bad, f"kernel {kernel}: {len(bad)} of {n} rows differ from the oracle (row, params, draw, got, want): {bad[:4]}"


def test_topk_over_the_vocabulary_with_top_p_1_is_a_nucleus(tiny):
    """candle's sample_topk_topp with k >= V runs sample_topp even at p = 1; at this row its fp32 sum reaches 1 and the pick moves
    (the premise is pinned on CPU in test_oracle_sample.py).  TopP alone and TopK with k >= V keep the plain multinomial."""
    lg = (np.random.default_rng(7).standard_normal(QWEN3_V) * 1.5).astype(F32)
    q = dict(temperature=0.9, top_p=1.0, top_k=QWEN3_V, seed=77)
    rows = [q, q, dict(q, top_k=2**31 - 1), dict(q, top_k=None), dict(q, top_p=None)]
    for kernel in (0, 1):
        got = tiny.debug_sample_rows(lg, rows, draw_index=[90, 384, 90, 90, 384], kernel=kernel)["token"]
        assert got.tolist() == [106616, 57439, 106616, 106615, 57440]


@pytest.mark.parametrize("V", [1000, QWEN3_V])
def test_repeat_penalty_contexts(tiny, V):
    """contexts of 0 to 4000 tokens with duplicates and ids >= V, last_n 1 / 64 / 5000, penalties 0.5 / 1.3 / 3.0 on rows whose head is
    positive and rows where every logit is negative; ArgMax with the penalty, then sampling"""
    rng = np.random.default_rng(V + 3)
    pos = (rng.standard_normal(V) * 0.5).astype(F32)
    top = rng.choice(V, 3, replace=False)
    pos[top] = [3.0, 2.9, 2.6]
    neg = (pos - 10).astype(F32)
    rows, ctxs, lgs = [], [], []
    for n in (0, 1, 63, 64, 65, 4000):
        for last_n in (1, 64, 5000):
            for pen in (0.5, 1.3, 3.0):
                c = rng.integers(0, V + 50, n).astype(np.int64)
                c[1::7] = V + rng.integers(0, 1000, len(c[1::7]))
                if n >= 3:
                    c[0], c[n // 2], c[-1], c[-2] = top[0], top[1], top[1], top[2]
                elif n == 1:
                    c[0] = top[0]
                rows.append(dict(repeat_penalty=pen, repeat_last_n=last_n))
                ctxs.append(c)
                lgs.append(pos if len(rows) % 2 else neg)
    lg = np.stack(lgs)
    moved = sum(int(np.argmax(S.use_repeat_penalty(_f32(q["repeat_penalty"]), q["repeat_last_n"], l, list(c))) != top[0])
                for q, c, l in zip(rows, ctxs, lgs))
    assert moved >= 10
    for t in (0.0, 0.7):
        qs = [dict(q, temperature=t, seed=SEEDS[i % 3]) for i, q in enumerate(rows)]
        draws = [DRAWS[i % len(DRAWS)] for i in range(len(qs))]
        want = [_want(l, q, c, d) for l, q, c, d in zip(lgs, qs, ctxs, draws)]
        for kernel in (0, 1):
            r = tiny.debug_sample_rows(lg, qs, ctxs, draws, kernel=kernel)
            assert r["token"].tolist() == want, f"t {t} kernel {kernel}"
            assert r["n_draws"].tolist() == [(d + (t > 0)) & NONE for d in draws]
            assert r["n_hist"].tolist() == [len(c) for c in ctxs]


def _mixed_rows(rng, n, V):
    modes = (dict(temperature=0.8), dict(temperature=0.7, top_p=0.9), dict(temperature=0.9, top_k=40),
             dict(temperature=0.6, top_k=300, top_p=0.95), dict(temperature=0.0, repeat_penalty=1.3),
             dict(temperature=1.1, top_k=V, top_p=1.0))
    rows = [dict(modes[i % len(modes)], seed=int(rng.integers(0, 2**63)), repeat_penalty=modes[i % len(modes)].get("repeat_penalty", 1.2))
            for i in range(n)]
    ctxs = [rng.integers(0, V, int(rng.integers(0, 100))) for _ in range(n)]
    draws = rng.integers(0, 2**32, n)
    return rows, ctxs, draws


def test_rows_do_not_depend_on_slot_neighbours_or_kernel(tiny):
    V = QWEN3_V
    rng = np.random.default_rng(21)
    lg = (rng.standard_normal((64, V)) * rng.uniform(1, 3, (64, 1))).astype(F32)
    rows, ctxs, draws = _mixed_rows(rng, 64, V)
    ref = tiny.debug_sample_rows(lg, rows, ctxs, draws, kernel=0)
    assert ref["token"].tolist() == [_want(lg[i], rows[i], ctxs[i], draws[i]) for i in range(64)]
    sampling = np.array([q["temperature"] > 0 for q in rows])
    assert np.array_equal(ref["n_draws"], (draws + sampling).astype(np.uint32))
    r1 = tiny.debug_sample_rows(lg, rows, ctxs, draws, kernel=1)
    for k in ref:
        assert np.array_equal(r1[k], ref[k]), k
    act = rng.permutation(64)
    on = (rng.random(64) < 0.5).astype(np.int32)
    r2 = tiny.debug_sample_rows(lg, rows, ctxs, draws, kernel=1, act=act, on=on)
    runs = on[act] == 1
    assert 10 < runs.sum() < 54
    for k in ref:
        assert np.array_equal(r2[k][runs], ref[k][runs]), k
    off = ~runs                                       # rows that do not sample keep what the call set up
    assert np.all(r2["token"][off] == NONE)
    assert r2["state_token"][off].tolist() == [int(c[-1]) if len(c) else 0 for c, o in zip(ctxs, off) if o]
    assert r2["last_hist"][off].tolist() == [int(c[-1]) if len(c) else NONE for c, o in zip(ctxs, off) if o]
    assert np.array_equal(r2["n_draws"][off], draws[off].astype(np.uint32))
    assert r2["n_hist"][off].tolist() == [len(c) for c, o in zip(ctxs, off) if o]
    for i in (0, 7, 31, 63):                          # alone, in another slot, with other rows' logits absent
        r = tiny.debug_sample_rows(lg[i:i + 1], rows[i:i + 1], ctxs[i:i + 1], draws[i:i + 1], kernel=1, act=[63 - i])
        assert int(r["token"][0]) == int(ref["token"][i])


def test_overwrite_replaces_the_pushed_token(tiny):
    """overwrite: the last context token is the ArgMax token the step pushed; it is not part of the penalty context and the sampled
    token replaces it in the history and in the state.  Without overwrite the history and state token stay."""
    V = 4097
    rng = np.random.default_rng(8)
    lg = rng.standard_normal(V).astype(F32)
    a = int(np.argmax(lg))
    lg[a] = lg.max() + 0.5
    c = [int(x) for x in rng.integers(0, V, 30) if x != a] + [a]
    rows = [dict(temperature=0.0, repeat_penalty=3.0, seed=1), dict(temperature=0.3, top_k=5, repeat_penalty=3.0, seed=2),
            dict(temperature=0.5, top_p=0.5, repeat_penalty=3.0, seed=3)]
    ctxs, draws = [c] * 3, [4, 16, 2**32 - 1]
    assert _want(lg, rows[0], c, 4, overwrite=True) == a != _want(lg, rows[0], c, 4)
    for overwrite in (True, False):
        want = [_want(lg, q, cc, d, overwrite) for q, cc, d in zip(rows, ctxs, draws)]
        for kernel in (0, 1):
            r = tiny.debug_sample_rows(lg, rows, ctxs, draws, overwrite=overwrite, kernel=kernel)
            assert r["token"].tolist() == want
            assert r["n_draws"].tolist() == [4, 17, 0]
            assert r["n_hist"].tolist() == [len(c)] * 3
            assert r["state_token"].tolist() == (want if overwrite else [a] * 3)
            assert r["last_hist"].tolist() == (want if overwrite else [a] * 3)


def _kept_f64(p64, mode):
    """candle's truncation in float64: keep in descending order while the sum of those kept before is < p (top_k first)"""
    order = np.argsort(-p64, kind="stable")
    name, k, top_p = mode
    cand = order[:k] if k else order
    if top_p is None:
        return cand
    before = np.concatenate([[0.0], np.cumsum(p64[cand])[:-1]])
    assert np.min(np.abs(np.cumsum(p64[cand]) - top_p)) > 1e-4       # fp32 and float64 keep the same set
    return cand[before < top_p]


@pytest.mark.parametrize("mode", [("all", None, None), ("topk", 20, None), ("topp", None, 0.8), ("topk_topp", 30, 0.85)],
                         ids=lambda m: m[0])
def test_draw_frequencies_follow_float64_truncated_probabilities(tiny, mode):
    V, t, n_calls = QWEN3_V, 0.8, 128
    rng = np.random.default_rng(99)
    lg = rng.standard_normal(V).astype(F32)
    head = rng.choice(V, 40, replace=False)           # scattered over the chunks
    lg[head] = (9.0 + rng.standard_normal(40)).astype(F32)
    x = lg.astype(np.float64) / t
    p64 = np.exp(x - x.max())
    p64 /= p64.sum()
    kept = _kept_f64(p64, mode)
    if mode[1]:
        s = np.sort(p64)[::-1]
        assert s[mode[1] - 1] > s[mode[1]] * (1 + 1e-4)
    q = dict(temperature=t, top_k=mode[1], top_p=mode[2], seed=2024)
    toks = []
    for c in range(n_calls):
        r = tiny.debug_sample_rows(lg, [q] * 64, draw_index=c * 64 + np.arange(64), kernel=c % 2)
        toks.append(r["token"])
    toks = np.concatenate(toks)
    assert np.isin(toks, kept).all(), f"{np.count_nonzero(~np.isin(toks, kept))} draws outside the kept set"
    w = p64[kept] / p64[kept].sum()
    exp = w * len(toks)
    big = exp >= 5
    obs = np.array([np.count_nonzero(toks == i) for i in kept[big]] + [np.count_nonzero(np.isin(toks, kept[~big]))])
    ex = np.append(exp[big], exp[~big].sum())
    if ex[-1] < 5:                                      # too small for its own bin: fold into the smallest one
        obs, ex = np.append(obs[:-2], obs[-2] + obs[-1]), np.append(ex[:-2], ex[-2] + ex[-1])
    assert len(ex) >= 10
    pv = chisquare(obs, ex).pvalue
    assert pv > 1e-6, f"chi-square p = {pv:.3g} over {len(ex)} bins"


def test_refusals_leave_the_handle_usable(tiny):
    from aha_b200 import B200Error
    V = 4097
    lg = (np.random.default_rng(4).standard_normal(V) * 2).astype(F32)
    good = [dict(temperature=0.8, top_k=40, top_p=0.9, seed=3)]
    want = _want(lg, good[0], (), 5)

    def samples_correctly():
        for kernel in (0, 1):
            assert int(tiny.debug_sample_rows(lg, good, draw_index=5, kernel=kernel)["token"][0]) == want

    samples_correctly()
    nan = lg.copy()
    nan[4000] = np.nan
    modes = (dict(temperature=0.8), dict(temperature=0.8, top_p=0.9), dict(temperature=0.8, top_k=40),
             dict(temperature=0.8, top_k=40, top_p=0.9), dict(temperature=0.8, top_k=V, top_p=1.0))
    for bad in (nan, np.full(V, -np.inf, F32)):
        for q in modes:
            for kernel in (0, 1):
                with pytest.raises(B200Error, match="WeightedIndex"):
                    tiny.debug_sample_rows(bad, [q, good[0]], kernel=kernel)
        samples_correctly()
    with pytest.raises(B200Error, match="top_k > 1024"):
        tiny.debug_sample_rows(lg, [dict(temperature=0.8, top_k=1025)])
    with pytest.raises(B200Error, match="V must be 1 to 262144"):
        tiny.debug_sample_rows(np.zeros(262145, F32), good)
    with pytest.raises(B200Error, match="rows must be 1 to 64"):
        tiny.debug_sample_rows(lg, good * 65)
    samples_correctly()
