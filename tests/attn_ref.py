"""float64 reference of the attention kernels (prefill, decode, speculative verify), tied to the oracle by tests/test_attn_ref.py.

softmax(q k^T / sqrt(hd) + mask) v per query head, query head h reading kv head h // (nh // nkv) (oracle/qwen3.py repeat_kv).  The decode
prologue is the oracle's QKNormAttention before the attention: per-head RMSNorm, then RoPE (x cos + rotate_half(x) sin) whose angle is
rounded to float32 as float32(pos + rope_delta) * inv_freq, like oracle/rope.py and the kernels; cos and sin are taken in float64."""
import numpy as np

from oracle.rope import compute_default_rope_parameters


def visible(Sq, Skv, causal, segments=None):
    """[Sq][Skv] bool: which keys each query sees.  causal: query i sees keys j <= i + Skv - Sq.  segments [(start, len)] (Sq == Skv):
    a query sees only keys of its own segment (causally if causal); rows outside every segment see nothing."""
    i = np.arange(Sq)[:, None]
    j = np.arange(Skv)[None, :]
    if segments is None:
        return (j <= i + Skv - Sq) if causal else np.ones((Sq, Skv), bool)
    vis = np.zeros((Sq, Skv), bool)
    for s0, n in segments:
        blk = np.tril(np.ones((n, n), bool)) if causal else np.ones((n, n), bool)
        vis[s0:s0 + n, s0:s0 + n] = blk
    return vis


def scores(q, k, nkv_of_head=None):
    """[nh][Sq][Skv] float64 scaled scores q k^T / sqrt(hd)."""
    q = np.asarray(q, np.float64)
    k = np.asarray(k, np.float64)
    nh, hd = q.shape[1], q.shape[2]
    G = nh // k.shape[1]
    return np.stack([q[:, h] @ k[:, h // G].T for h in range(nh)]) / np.sqrt(hd)


def probs(q, k, causal, segments=None):
    """[nh][Sq][Skv] float64 attention probabilities (zero where masked; rows that see no key are all zero)."""
    s = scores(q, k)
    vis = visible(q.shape[0], k.shape[0], causal, segments)[None]
    s = np.where(vis, s, -np.inf)
    m = s.max(axis=-1, keepdims=True)
    m = np.where(np.isfinite(m), m, 0.0)
    e = np.where(vis, np.exp(s - m), 0.0)
    l = e.sum(axis=-1, keepdims=True)
    return e / np.where(l > 0, l, 1.0)


def attention(q, k, v, causal, segments=None):
    """q [Sq][nh][hd], k / v [Skv][nkv][hd] -> [Sq][nh][hd] float64; rows outside every segment are NaN."""
    p = probs(q, k, causal, segments)
    v = np.asarray(v, np.float64)
    G = q.shape[1] // k.shape[1]
    out = np.stack([p[h] @ v[:, h // G] for h in range(q.shape[1])], axis=1)
    if segments is not None:
        covered = visible(q.shape[0], k.shape[0], causal, segments).any(axis=1)
        out[~covered] = np.nan
    return out


def rope_angles(pos, hd, theta):
    """float32(pos) * inv_freq (float32, like the kernels and oracle.rope.RoPE), repeated over both halves, as float64."""
    inv = compute_default_rope_parameters(hd, theta)
    a = (np.float32(pos) * inv).astype(np.float32)
    return np.concatenate([a, a]).astype(np.float64)


def rope(x, pos, theta, inverse=False):
    """x [..., hd] rotated to position pos (or back from it) in float64."""
    x = np.asarray(x, np.float64)
    hd = x.shape[-1]
    a = rope_angles(pos, hd, theta)
    c, s = np.cos(a), np.sin(a)
    if inverse:
        s = -s
    rot = np.concatenate([-x[..., hd // 2:], x[..., :hd // 2]], axis=-1)
    return x * c + rot * s


def rms_norm(x, w, eps):
    x = np.asarray(x, np.float64)
    return x / np.sqrt(np.mean(x * x, axis=-1, keepdims=True) + eps) * np.asarray(w, np.float64)


def decode_prologue(qkv, nh, nkv, q_norm, k_norm, eps, rope_pos, theta, hd=128):
    """one raw projection row [(nh + 2 nkv) * hd] -> (q [nh][hd], k [nkv][hd], v [nkv][hd]) in float64: q and k RMS-normalised per head
    and rotated to rope_pos, v as given."""
    x = np.asarray(qkv, np.float64).reshape(nh + 2 * nkv, hd)
    q = rope(rms_norm(x[:nh], q_norm, eps), rope_pos, theta)
    k = rope(rms_norm(x[nh:nh + nkv], k_norm, eps), rope_pos, theta)
    return q, k, x[nh + nkv:]


def decode_attention(qkv, k_cache, v_cache, pos, rope_delta, q_norm, k_norm, eps, theta, nh, nkv, hd=128):
    """one decode step: the new token at cache index pos (RoPE position pos + rope_delta) attends to k_cache / v_cache [pos][nkv][hd]
    and itself -> (out [nh][hd], k_new [nkv][hd], v_new [nkv][hd]) in float64."""
    q, k_new, v_new = decode_prologue(qkv, nh, nkv, q_norm, k_norm, eps, pos + rope_delta, theta, hd)
    K = np.concatenate([np.asarray(k_cache, np.float64).reshape(-1, nkv, hd), k_new[None]])
    V = np.concatenate([np.asarray(v_cache, np.float64).reshape(-1, nkv, hd), v_new[None]])
    return attention(q[None], K, V, causal=True)[0], k_new, v_new
