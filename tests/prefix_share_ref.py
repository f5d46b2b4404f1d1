"""Restatements behind the batch-session prefix cache (aha_b200_batch_prefix_cache): the float64 attention of a pack whose segments have
cached prefixes, and the hit rule."""
import numpy as np

import attn_ref

PAGE = 32


def prefix_attention(q, k, v, segments):
    """segments [(prefix, rows), ...]: segment j has `rows` query rows, laid after the previous segment's, and prefix + rows keys, laid after
    the previous segment's keys; query i of segment j sees its keys 0 .. prefix + i.  q [sum rows][nh][hd], k / v [sum (prefix + rows)]
    [nkv][hd] -> [sum rows][nh][hd] float64."""
    out, q0, k0 = [], 0, 0
    for p, n in segments:
        out.append(attn_ref.attention(q[q0:q0 + n], k[k0:k0 + p + n], v[k0:k0 + p + n], causal=True))
        q0, k0 = q0 + n, k0 + p + n
    return np.concatenate(out)


def cached_pages(earlier, ids):
    """Full pages of `ids` that an index filled by the prompts `earlier` (nothing evicted) holds in a row from the start: page k is cached
    when an earlier prompt has at least k + 1 full pages and shares the first (k + 1) * 32 tokens."""
    best = 0
    for e in earlier:
        lcp = 0
        for a, b in zip(e, ids):
            if int(a) != int(b):
                break
            lcp += 1
        best = max(best, min(lcp, len(e) // PAGE * PAGE) // PAGE)
    return best


def hit_tokens(chain_pages, seq_len, gemm_impl=0):
    """The hit rule: the cached chain, at most seq_len - 1 tokens and, unless gemm_impl is 1 (SIMT everywhere), at most seq_len - 32 so that
    at least 32 prompt tokens run on the wgmma GEMM; always a multiple of 32."""
    cap = seq_len - 1 if gemm_impl == 1 else max(seq_len - PAGE, 0)
    return min(chain_pages, cap // PAGE) * PAGE
