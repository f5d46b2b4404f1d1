"""Every attention kernel against the float64 reference (tests/attn_ref.py) on host data, through aha_b200_debug_attention (prefill: the
wgmma, SIMT and mma.sync kernels behind the models' dispatch) and aha_b200_debug_decode_attn (decode_attn_kernel, decode_attn_batch_kernel).

Every shape runs in four score regimes, each checked on the reference to have the property it is named for:
  flat    q, k ~ N(0, 1): near-uniform rows, as in the synthetic models;
  peaked  each query aimed at one visible key: most rows put > 0.99 of their mass on it;
  rising  scores grow along the keys: every 64-key tile raises the row max, so every tile rescales the running sums;
  sink    the first visible key dominates every row, and V spans four decades.
The pools are NaN outside what the page tables own (debug entries), so a read of unowned memory, even under a mask, shows.
Errors are max |kernel - reference| / max |V|."""
import numpy as np
import pytest

import attn_ref

pytestmark = pytest.mark.gpu

REGIMES = ("flat", "peaked", "rising", "sink")
HD = 128

# Bounds on max |kernel - reference| / max |V| over every case of a test.  The fp32 SIMT kernels (the prefill twin, decode) keep the 1e-5
# grade of the verify attention.  The split-fp16 tensor-core kernels: 4x the largest error measured over this file's cases, per kernel and
# regime, on an H100 80GB HBM3 (700 W power limit); the measured value is in the comment.  (The SIMT twin measured 3.2e-7, 8.7e-7, 3.5e-6
# and 1.7e-6.)
SIMT_BOUND = 1e-5
TC_BOUND = {
    0: {"flat": 2.7e-6,     # wgmma: 6.95e-7
        "peaked": 1.1e-5,   # 2.78e-6
        "rising": 7.9e-6,   # 1.99e-6
        "sink": 2.0e-5},    # 5.18e-6
    2: {"flat": 3.2e-6,     # mma.sync: 8.06e-7
        "peaked": 1.0e-5,   # 2.74e-6
        "rising": 8.3e-6,   # 2.10e-6
        "sink": 2.0e-5},    # 5.10e-6
}
DECODE_BOUND = 1e-5   # measured on the same H100: flat 1.3e-7, peaked 2.1e-7, rising 5.0e-7, sink 3.8e-7


def bound(impl, regime):
    return SIMT_BOUND if impl == 1 else TC_BOUND[impl][regime]


# ------------------------------------------------------------------------------------------------------------ inputs and regimes

def _first_visible(vis):
    return np.argmax(vis, axis=1)


def _unit(rng, n):
    u = rng.standard_normal(n)
    return u / np.linalg.norm(u)


def _ramp(n, hd, noise, u):
    """keys 0 .. n - 1 along u with length slope * j * sqrt(hd) / |q| for |q| = sqrt(hd) (score slope * j: +3.2 per 64-key tile, at
    most ~150), plus `noise` projected orthogonal to u"""
    slope = min(0.05, 150.0 / max(n, 1))
    noise = 0.3 * (noise - (noise @ u)[..., None] * u)
    return slope * np.arange(n)[:, None, None] * u + noise


def prefill_inputs(regime, Sq, Skv, nh, nkv, hd, vis, rng):
    """q [Sq][nh][hd], k / v [Skv][nkv][hd] float32 in `regime` (vis: [Sq][Skv] keys each query sees)."""
    G = nh // nkv
    kvh = np.arange(nh) // G
    q = rng.standard_normal((Sq, nh, hd))
    k = rng.standard_normal((Skv, nkv, hd))
    v = rng.standard_normal((Skv, nkv, hd))
    rows = np.flatnonzero(vis.any(axis=1))
    if regime == "peaked":
        for i in rows:
            t = rng.choice(np.flatnonzero(vis[i]), size=nh)
            q[i] = 2.5 * k[t, kvh] + 0.3 * q[i]
    elif regime == "rising":   # every q along u, key j = slope * j along u plus noise orthogonal to u: score slope * j
        u = _unit(rng, hd)
        q = np.broadcast_to(np.sqrt(hd) * u, q.shape).copy()
        k = _ramp(Skv, hd, k, u)
    elif regime == "sink":
        j0 = _first_visible(vis)
        q[rows] = 16 / np.sqrt(hd) * k[j0[rows]][:, kvh] + q[rows]   # score ~16 on the first key
        v *= 10.0 ** rng.uniform(-2, 2, (Skv, 1, 1))
    return q.astype(np.float32), k.astype(np.float32), v.astype(np.float32)


def assert_regime(regime, s, vis, vis_rising=None):
    """s: [nh][Sq][Skv] float64 scores; vis: [Sq][Skv].  The regime has the property it is named for."""
    rows = np.flatnonzero(vis.any(axis=1))
    sm = np.where(vis[None], s, -np.inf)[:, rows]
    p = np.exp(sm - sm.max(axis=-1, keepdims=True))
    p /= p.sum(axis=-1, keepdims=True)
    pmax = p.max(axis=-1)
    nvis = vis[rows].sum(axis=1)
    if regime == "flat":   # rows of 64 keys or more: no key near 1, a typical top key well under 1 / 4
        wide = pmax[:, nvis >= 64]
        assert wide.size == 0 or ((wide < 0.75).all() and wide.mean() < 0.2), wide.max()
    elif regime == "peaked":
        assert (pmax > 0.99).mean() >= 0.9, (pmax > 0.99).mean()
    elif regime == "sink":
        j0 = _first_visible(vis)[rows]
        assert (p[:, np.arange(len(rows)), j0] > 0.5).all()
    elif regime == "rising":   # 64-key tiles counted from each row's first visible key
        vr = vis if vis_rising is None else vis_rising
        j = np.arange(vr.shape[1])[None, :]
        tile = np.where(vr, (j - _first_visible(vr)[:, None]) // 64, -1)
        prev = None
        for t in range(tile.max() + 1):
            on = tile == t
            cur = np.where(on[None], s, -np.inf).max(axis=-1)
            if prev is not None:
                has = on.any(axis=1)
                assert (cur[:, has] > prev[:, has]).all(), t
            prev = np.where(on.any(axis=1)[None], cur, prev) if prev is not None else cur


# ------------------------------------------------------------------------------------------------------------ prefill

@pytest.fixture(scope="module")
def model():
    from conftest import make_model
    _, _, m = make_model("qwen3", "tiny", max_ctx=2048)
    yield m
    m.close()


def _page_order(Skv, rng):
    """distinct physical pages, shuffled and sparse: half the pool is referenced by no table"""
    n = -(-Skv // 32)
    return rng.permutation(2 * n)[:n]


def run_prefill(m, impl, regime, Sq, Skv, nh, nkv, hd, causal, segments=None, seed=0, split_out=False):
    """-> (error / max|V|, kernel output, reference) of one case"""
    rng = np.random.default_rng(seed)
    vis = attn_ref.visible(Sq, Skv, causal, segments)
    q, k, v = prefill_inputs(regime, Sq, Skv, nh, nkv, hd, vis, rng)
    assert_regime(regime, attn_ref.scores(q, k), vis)
    po = _page_order(Skv, rng) if causal else None
    got = m.debug_attention(q, k, v, impl, causal, segments=segments, page_order=po, split_out=split_out)
    want = attn_ref.attention(q, k, v, causal, segments)
    covered = vis.any(axis=1)
    assert np.isnan(got[~covered]).all()                  # rows outside every segment are never written
    assert np.isfinite(got[covered]).all(), "NaN / inf in the output: a read of unowned memory"
    err = float(np.abs(got[covered] - want[covered]).max() / np.abs(v).max())
    return err, got, want


CAUSAL_POS0 = (0, 1, 31, 64, 127, 300)
CAUSAL_S = (1, 15, 16, 17, 63, 64, 65, 127, 128, 129, 257)


def causal_cases():
    """(Sq, Skv, nh, nkv): every pos0 x S, with G cycling through 1, 2, 4, 6 (2 kv heads)"""
    out = []
    for a, pos0 in enumerate(CAUSAL_POS0):
        for b, S in enumerate(CAUSAL_S):
            G = (1, 2, 4, 6)[(a + b) % 4]
            out.append((S, pos0 + S, 2 * G, 2))
    return out


def prefill_errors(m, impl, regime):
    """errors of every causal paged case of one impl and regime"""
    return [(c, run_prefill(m, impl, regime, *c, HD, True, seed=i)[0]) for i, c in enumerate(causal_cases())]


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("impl", [0, 1, 2])
def test_causal_paged_prefill(model, impl, regime):
    errs = prefill_errors(model, impl, regime)
    worst = max(errs, key=lambda e: e[1])
    assert worst[1] <= bound(impl, regime), worst


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("impl", [0, 1, 2])
def test_causal_prefill_long_context(model, impl, regime):
    """a 300-token chunk behind 3796 cached tokens (Skv = 4096), G = 6"""
    err = run_prefill(model, impl, regime, 300, 4096, 6, 1, HD, True, seed=7)[0]
    assert err <= bound(impl, regime), err


# not tile multiples, a 1-token segment, segments straddling the 64 / 128 tiles, and rows 129 .. 139 in no segment (never written)
ENCODER_SEGMENTS = [(0, 1), (1, 63), (64, 65), (140, 189), (329, 17)]


def encoder_errors(m, impl, regime):
    out = []
    for i, (hd, G) in enumerate([(64, 1), (128, 1), (64, 2), (128, 2)]):
        out.append((("segments", hd, G), run_prefill(m, impl, regime, 346, 346, 4 * G, 4, hd, False, ENCODER_SEGMENTS, seed=10 + i)[0]))
    out.append((("cross", 64), run_prefill(m, impl, regime, 100, 300, 4, 2, 64, False, seed=20)[0]))
    return out


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("impl", [0, 1, 2])
def test_noncausal_segments(model, impl, regime):
    worst = max(encoder_errors(model, impl, regime), key=lambda e: e[1])
    assert worst[1] <= bound(impl, regime), worst


def pack_segments(lens, align=16):
    """(start, len) of texts packed as plan_pack packs them: each on the next multiple of `align`, the filler joining the text before it"""
    starts = [0]
    for n in lens[:-1]:
        starts.append(-(-(starts[-1] + n) // align) * align)
    ends = starts[1:] + [starts[-1] + lens[-1]]
    return [(s, e - s) for s, e in zip(starts, ends)]


VARLEN_PACKS = [pack_segments(lens) for lens in ([37, 1, 130, 129, 300], [128], [1, 1, 1], [200, 64, 15])]
VARLEN_PACKS.append([(0, 20), (48, 30), (96, 129)])   # rows 20 .. 47 and 78 .. 95 in no segment (never written)


def varlen_errors(m, impl, regime):
    out = []
    for i, segs in enumerate(VARLEN_PACKS):
        T = segs[-1][0] + segs[-1][1]
        G = (1, 2, 4, 6, 2)[i]
        out.append((tuple(segs), run_prefill(m, impl, regime, T, T, 2 * G, 2, HD, True, segs, seed=30 + i)[0]))
    return out


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("impl", [0, 1, 2])
def test_causal_varlen_packs(model, impl, regime):
    worst = max(varlen_errors(model, impl, regime), key=lambda e: e[1])
    assert worst[1] <= bound(impl, regime), worst


@pytest.mark.parametrize("regime", REGIMES)
def test_wgmma_split_output_is_the_fp32_output_rounded(model, regime):
    """out_hi + out_lo (the o_proj operand) is the fp32 output up to the rounding of lo to fp16"""
    for case in [(129, 429, 12, 2, HD, True), (346, 346, 8, 4, 64, False, ENCODER_SEGMENTS)]:
        _, f32, _ = run_prefill(model, 0, regime, *case, seed=40)
        _, hilo, _ = run_prefill(model, 0, regime, *case, seed=40, split_out=True)
        ok = np.isfinite(f32)
        assert np.isfinite(hilo[ok]).all()
        assert (np.abs(hilo[ok] - f32[ok]) <= np.abs(f32[ok]) * 2.0 ** -22 + 2.0 ** -25).all()


# ------------------------------------------------------------------------------------------------------------ decode

def decode_weights(regime, rng):
    """non-unit q / k RMSNorm weights; peaked rows come from q_norm ~ 3 (|q| ~ 3 sqrt(hd))"""
    return (rng.uniform(0.5, 1.5, HD) * (3.0 if regime == "peaked" else 1.0)).astype(np.float32), rng.uniform(0.5, 1.5, HD).astype(np.float32)


def decode_inputs(regime, pos, rope_delta, nh, nkv, qw, rng, theta=1e6):
    """(qkv raw row, k_cache, v_cache) of one sequence at cache index pos in `regime`: the raw q is chosen so that after the kernel's
    RMSNorm (weights qw) and RoPE it points where the regime needs it."""
    G = nh // nkv
    kvh = np.arange(nh) // G
    kc = rng.standard_normal((pos, nkv, HD))
    vc = rng.standard_normal((pos, nkv, HD))
    raw = rng.standard_normal((nh + 2 * nkv, HD))
    d = None
    if regime == "peaked" and pos:
        d = kc[rng.integers(0, pos, nh), kvh]
    elif regime == "sink" and pos:
        kc[0] *= 1.5
        d = kc[0, kvh] / np.linalg.norm(kc[0, kvh], axis=-1, keepdims=True) + 0.5 * rng.standard_normal((nh, HD)) / np.sqrt(HD)
        vc *= 10.0 ** rng.uniform(-2, 2, (pos, 1, 1))
    elif regime == "rising" and pos:
        u = _unit(rng, HD)
        kc = _ramp(pos, HD, kc, u)
        d = np.tile(u, (nh, 1))
    if d is not None:   # RMSNorm keeps the direction of raw * qw, RoPE then rotates it to d
        raw[:nh] = attn_ref.rope(d, pos + rope_delta, theta, inverse=True) / qw
    f = lambda x: np.ascontiguousarray(x, np.float32)
    return f(raw.reshape(-1)), f(kc), f(vc)


def _interleaved_tables(ctxs, rng, spare=3):
    """page tables of sequences whose pages interleave in one pool (plus `spare` pages no table references), shuffled"""
    need = [-(-c // 32) for c in ctxs]
    order = [b for p in range(max(need)) for b in range(len(ctxs)) if p < need[b]]
    phys = rng.permutation(len(order) + spare)
    tables = [[] for _ in ctxs]
    for i, b in enumerate(order):
        tables[b].append(int(phys[i]))
    return tables, len(order) + spare


def _expected_pool(n_pages, nkv, seqs, tables):
    pool = np.full((n_pages, 2, nkv, 32, HD), np.nan, np.float32)
    for (_, kc, vc), t in zip(seqs, tables):
        for j in range(kc.shape[0]):
            pool[t[j // 32], 0, :, j % 32] = kc[j]
            pool[t[j // 32], 1, :, j % 32] = vc[j]
    return pool


def run_decode(m, regime, ctxs, nh, nkv, rope_delta=0, seed=0, eps=1e-6, theta=1e6):
    """B = len(ctxs) sequences (context ctx = pos + 1 each, pages interleaved in one pool) through one call; checks the output, the
    appended K / V and the untouched pool.  The output checked is that of a run on the pool as a decode step finds it (the new tokens'
    slots not yet written); a second run on the same partials and counters, over the pool the first left, must give the same bits.
    -> dict(err = worst error / max|V|, out, pool, seqs, qw, kw)"""
    rng = np.random.default_rng(seed)
    qw, kw = decode_weights(regime, rng)
    seqs = [decode_inputs(regime, c - 1, rope_delta, nh, nkv, qw, rng, theta) for c in ctxs]
    tables, n_pages = _interleaved_tables(ctxs, rng)
    pos = [c - 1 for c in ctxs]
    out, again, pool = m.debug_decode_attn(np.stack([s[0] for s in seqs]), pos, [rope_delta] * len(ctxs), [s[1] for s in seqs],
                                           [s[2] for s in seqs], tables, n_pages, qw, kw, nh, nkv, eps, theta)
    want_pool = _expected_pool(n_pages, nkv, seqs, tables)
    written = np.zeros(want_pool.shape, bool)
    worst = 0.0
    for b, (qkv, kc, vc) in enumerate(seqs):
        p = pos[b]
        want, k_new, v_new = attn_ref.decode_attention(qkv, kc, vc, p, rope_delta, qw, kw, eps, theta, nh, nkv)
        q, _, _ = attn_ref.decode_prologue(qkv, nh, nkv, qw, kw, eps, p + rope_delta, theta)
        vis = np.ones((1, p + 1), bool)
        ramp = vis.copy()
        ramp[0, p] = False   # the new key is not part of the rising ramp
        assert_regime(regime, attn_ref.scores(q[None], np.concatenate([kc.astype(np.float64), k_new[None]])), vis, ramp)
        assert np.isfinite(out[b]).all(), (b, "NaN in the output: a read of unowned memory or a counter that did not reset")
        vmax = max(np.abs(vc).max() if p else 0.0, np.abs(v_new).max())
        worst = max(worst, float(np.abs(out[b] - want).max() / vmax))
        page, slot = tables[b][p // 32], p % 32
        assert np.abs(pool[page, 0, :, slot] - k_new).max() <= 1e-5 * np.abs(k_new).max(), b   # the new K, normalised and rotated
        assert np.array_equal(pool[page, 1, :, slot], v_new.astype(np.float32)), b
        written[page, :, :, slot] = True
    u = lambda x: x.view(np.uint32)
    assert np.array_equal(u(again), u(out)), "the second run differs: a split counter did not reset, or the output depends on the new slot"
    assert np.array_equal(u(pool)[~written], u(want_pool)[~written]), "the call changed pool words outside the new tokens' slots"
    return dict(err=worst, out=out, pool=pool, seqs=seqs, qw=qw, kw=kw)


DECODE_CTX = (1, 2, 15, 16, 17, 32, 33, 256, 257, 2049)


def decode_errors(m, regime, G):
    out = []
    for i, ctx in enumerate(DECODE_CTX):
        for j, nkv in enumerate((1, 2, 8)):
            rd = (0, -1980)[(i + j) % 2]
            out.append(((ctx, nkv, rd), run_decode(m, regime, [ctx], G * nkv, nkv, rd, seed=100 * i + j)["err"]))
    return out


@pytest.mark.parametrize("G", [1, 2, 4, 6])
@pytest.mark.parametrize("regime", REGIMES)
def test_decode_attention(model, regime, G):
    worst = max(decode_errors(model, regime, G), key=lambda e: e[1])
    assert worst[1] <= DECODE_BOUND, worst


@pytest.mark.parametrize("regime", REGIMES)
def test_decode_attention_long_context(model, regime):
    """32800 tokens: 2050 per split"""
    for G, rd in ((6, -1980), (2, 0)):
        err = run_decode(model, regime, [32800], 2 * G, 2, rd, seed=G)["err"]
        assert err <= DECODE_BOUND, (G, err)


@pytest.mark.parametrize("G", [1, 6])
def test_decode_is_deterministic_and_batch_rows_match_single_calls(model, G):
    """two identical calls give identical bits; each sequence of a B = 5 batch (pages interleaved in one pool) gives the bits of its
    own B = 1 call"""
    ctxs = [1, 17, 300, 2049, 64]
    nkv = 2
    a = run_decode(model, "peaked", ctxs, G * nkv, nkv, -1980, seed=5)
    b = run_decode(model, "peaked", ctxs, G * nkv, nkv, -1980, seed=5)
    assert np.array_equal(a["out"], b["out"]) and np.array_equal(a["pool"].view(np.uint32), b["pool"].view(np.uint32))
    for i, (c, (qkv, kc, vc)) in enumerate(zip(ctxs, a["seqs"])):
        n = -(-c // 32)
        out, _, _ = model.debug_decode_attn(qkv[None], [c - 1], [-1980], [kc], [vc], [list(range(n))[::-1]], n + 1, a["qw"], a["kw"],
                                            G * nkv, nkv)
        assert np.array_equal(out[0], a["out"][i]), (i, c)
