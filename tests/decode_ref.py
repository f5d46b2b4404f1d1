"""float64 reference of the Qwen3 text decoder, tied to the float32 oracle by tests/test_decode_ref.py.

A whole token sequence in, the hidden state (after the final RMSNorm) and the logits at every position out: a teacher-forced decode of n
steps is one causal pass, so no KV cache is needed.  The fp16 weights and gains are widened to float64 and everything is computed in
float64: RMSNorm x / sqrt(mean(x^2) + eps) * w, per-head q / k RMSNorm, RoPE, grouped-query attention softmax(q k^T / sqrt(hd)) v (query
head h reads kv head h // (nh / nkv)), SwiGLU down(silu(gate) * up), the final norm and the tied or untied lm_head.  The rotary angle is
what the model defines: the float32 inv_freq of oracle/rope.py times float32(pos), rounded to float32; its cos and sin are taken in
float64.  The reference then differs from the kernels only by their rounding.

Several sequences go through one call, their rows stacked for every projection (each weight matrix is widened once per call)."""
import numpy as np

from oracle.rope import compute_default_rope_parameters

F64 = np.float64


def rms_norm(x, w, eps):
    x = np.asarray(x, F64)
    return x / np.sqrt(np.mean(x * x, axis=-1, keepdims=True) + eps) * np.asarray(w, F64)


def silu(x):
    return x / (1.0 + np.exp(-x))


def log_softmax(logits):
    """float64 log-softmax over the last axis."""
    l = np.asarray(logits, F64)
    m = l.max(axis=-1, keepdims=True)
    return l - (m + np.log(np.exp(l - m).sum(axis=-1, keepdims=True)))


def rope_tables(n, hd, theta):
    """(cos, sin) [n][hd] float64 for positions 0..n-1: angle float32(float32(pos) * inv_freq), both halves."""
    inv = compute_default_rope_parameters(hd, theta)
    a = (np.arange(n, dtype=np.float32)[:, None] * inv[None, :]).astype(np.float32).astype(F64)
    a = np.concatenate([a, a], axis=-1)
    return np.cos(a), np.sin(a)


def rotate(x, cos, sin):
    """x [S][heads][hd] rotated row by row (NeoX half split: x cos + rotate_half(x) sin)."""
    h = x.shape[-1] // 2
    rot = np.concatenate([-x[..., h:], x[..., :h]], axis=-1)
    return x * cos[:, None, :] + rot * sin[:, None, :]


def _linear(x, w):
    return x @ np.asarray(w, F64).T


def _prefix(w):
    return "model." if "model.embed_tokens.weight" in w else ""


def hidden(cfg, w, seqs):
    """token sequences -> [len(seq)][H] float64 hidden states after the final RMSNorm, one array per sequence."""
    p = _prefix(w)
    H, nh, nkv, hd = cfg["hidden_size"], cfg["num_attention_heads"], cfg["num_key_value_heads"], cfg["head_dim"]
    eps, G = cfg["rms_norm_eps"], nh // nkv
    seqs = [np.asarray(s, np.int64).reshape(-1) for s in seqs]
    lens = [len(s) for s in seqs]
    starts = np.concatenate([[0], np.cumsum(lens)])
    x = np.asarray(w[p + "embed_tokens.weight"], F64)[np.concatenate(seqs)]
    cos, sin = rope_tables(max(lens), hd, cfg["rope_theta"])
    cos = np.concatenate([cos[:n] for n in lens])
    sin = np.concatenate([sin[:n] for n in lens])
    scale = 1.0 / np.sqrt(F64(hd))
    for i in range(cfg["num_hidden_layers"]):
        lp = f"{p}layers.{i}."
        xn = rms_norm(x, w[lp + "input_layernorm.weight"], eps)
        q = _linear(xn, w[lp + "self_attn.q_proj.weight"]).reshape(-1, nh, hd)
        k = _linear(xn, w[lp + "self_attn.k_proj.weight"]).reshape(-1, nkv, hd)
        v = _linear(xn, w[lp + "self_attn.v_proj.weight"]).reshape(-1, nkv, hd)
        q = rotate(rms_norm(q, w[lp + "self_attn.q_norm.weight"], eps), cos, sin)
        k = rotate(rms_norm(k, w[lp + "self_attn.k_norm.weight"], eps), cos, sin)
        o = np.empty_like(q)
        for s, n in zip(starts[:-1], lens):
            qs, ks, vs = q[s:s + n], k[s:s + n], v[s:s + n]
            causal = np.tril(np.ones((n, n), bool))
            for h in range(nh):
                sc = (qs[:, h] @ ks[:, h // G].T) * scale
                sc = np.where(causal, sc, -np.inf)
                e = np.exp(sc - sc.max(axis=-1, keepdims=True))
                o[s:s + n, h] = (e / e.sum(axis=-1, keepdims=True)) @ vs[:, h // G]
        x = x + _linear(o.reshape(-1, nh * hd), w[lp + "self_attn.o_proj.weight"])
        xn = rms_norm(x, w[lp + "post_attention_layernorm.weight"], eps)
        g = _linear(xn, w[lp + "mlp.gate_proj.weight"])
        u = _linear(xn, w[lp + "mlp.up_proj.weight"])
        x = x + _linear(silu(g) * u, w[lp + "mlp.down_proj.weight"])
    x = rms_norm(x, w[p + "norm.weight"], eps)
    return [x[s:s + n] for s, n in zip(starts[:-1], lens)]


def lm_head(cfg, w):
    """the lm_head matrix [V][H] (fp16, as stored): the embedding table when tied."""
    return w[_prefix(w) + "embed_tokens.weight"] if cfg.get("tie_word_embeddings", False) else w["lm_head.weight"]


def logits_of(hid, head, chunk=16384):
    """hidden [S][H] float64 x lm_head [V][H] -> [S][V] float64, the vocabulary widened a chunk at a time."""
    hid = np.asarray(hid, F64)
    out = np.empty((hid.shape[0], head.shape[0]), F64)
    for r in range(0, head.shape[0], chunk):
        out[:, r:r + chunk] = hid @ np.asarray(head[r:r + chunk], F64).T
    return out


def logits(cfg, w, seqs):
    """token sequences -> [len(seq)][V] float64 logits at every position, one array per sequence."""
    hs = hidden(cfg, w, seqs)
    n = [len(h) for h in hs]
    l = logits_of(np.concatenate(hs), lm_head(cfg, w))
    return np.split(l, np.cumsum(n)[:-1])
