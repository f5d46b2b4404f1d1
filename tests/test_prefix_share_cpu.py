"""Host-side checks of the batch-session prefix cache: the ctypes layout of aha_prefix_stats against the header, and the restated hit rule
and prefixed-segment attention (tests/prefix_share_ref.py) against the plain references they stand for."""
import ctypes
import os
import re

import numpy as np

import attn_ref
import prefix_share_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_prefix_stats_layout_matches_header():
    from aha_b200 import _lib as L
    h = open(os.path.join(ROOT, "include", "aha_b200.h")).read()
    body = re.search(r"typedef struct aha_prefix_stats \{(.*?)\} aha_prefix_stats;", h, re.S).group(1)
    fields = re.findall(r"uint64_t (\w+);", body)
    assert fields == [n for n, _ in L.PrefixStats._fields_]
    assert ctypes.sizeof(L.PrefixStats) == 8 * len(fields)


def test_hit_rule():
    # whole pages only, at least 32 prompt tokens run (wgmma GEMM) unless gemm_impl is 1, never the whole prompt
    assert R.hit_tokens(3, 130) == 96
    assert R.hit_tokens(3, 100) == 64          # 100 - 32 = 68 -> two pages
    assert R.hit_tokens(3, 96) == 64
    assert R.hit_tokens(3, 96, gemm_impl=1) == 64   # 95 -> two pages
    assert R.hit_tokens(3, 97, gemm_impl=1) == 96   # one prompt token left to run
    assert R.hit_tokens(5, 31) == 0 and R.hit_tokens(5, 31, gemm_impl=1) == 0
    assert R.hit_tokens(0, 4096) == 0
    for n in range(1, 300):
        for g in (0, 1):
            h = R.hit_tokens(100, n, g)
            assert h % 32 == 0 and h <= n - 1 and (g == 1 or n - h >= 32 or h == 0)


def test_cached_pages():
    a = list(range(100))
    assert R.cached_pages([a], a[:96] + [7] * 40) == 3
    assert R.cached_pages([a], a[:95] + [7] * 40) == 2        # page 2 differs in its last token
    assert R.cached_pages([a[:70]], a) == 2                    # only full pages of the earlier prompt are cached
    assert R.cached_pages([], a) == 0
    assert R.cached_pages([a[:40], a], a + [1]) == 3


def test_prefix_attention_is_the_continuation_per_segment():
    rng = np.random.default_rng(0)
    segs = [(0, 40), (32, 8), (96, 33)]
    nh, nkv, hd = 4, 2, 16
    Sq, Skv = sum(n for _, n in segs), sum(p + n for p, n in segs)
    q, k, v = rng.standard_normal((Sq, nh, hd)), rng.standard_normal((Skv, nkv, hd)), rng.standard_normal((Skv, nkv, hd))
    got = R.prefix_attention(q, k, v, segs)
    # no prefixes: the packed-segment reference
    plain = [(0, n) for _, n in segs]
    starts = np.cumsum([0] + [n for _, n in segs])[:-1]
    qp = q
    kp = np.concatenate([k[sum(p + n for p, n in segs[:j]) + p:][:n] for j, (p, n) in enumerate(segs)])
    vp = np.concatenate([v[sum(p + n for p, n in segs[:j]) + p:][:n] for j, (p, n) in enumerate(segs)])
    ref = attn_ref.attention(qp, kp, vp, True, [(int(s), n) for s, (_, n) in zip(starts, segs)])
    assert np.allclose(R.prefix_attention(qp, kp, vp, plain), ref)
    # a prefixed segment: its rows are the last rows of causal attention over its prefix and rows together
    p, n = segs[2]
    k0 = sum(pp + nn for pp, nn in segs[:2])
    qq = np.concatenate([rng.standard_normal((p, nh, hd)), q[-n:]])
    assert np.allclose(got[-n:], attn_ref.attention(qq, k[k0:], v[k0:], True)[p:])
