"""RoPE family -- restates src/position_embed/{rope.rs,sinusoidal_pe.rs}."""
import numpy as np

F32 = np.float32


def compute_default_rope_parameters(dim, base):
    """rope.rs:7-13: inv_freq[i] = 1 / base.powf(i / dim) for even i, all in f32.  f32::powf calls the C library's powf, as the library's
    rope_inv_freq does.  numpy's float32 power can differ from it by 1 ulp (at 15 of the 64 frequencies of base 1e6, dim 128); the power
    taken in f64 and rounded to f32 matches the C powf (tests/test_attn_ref.py checks it)."""
    i = np.arange(0, dim, 2, dtype=F32)
    p = np.power(np.float64(F32(base)), (i / F32(dim)).astype(np.float64)).astype(F32)
    return (F32(1.0) / p).astype(F32)


def rotate_half(x):
    """rope.rs:15-22: cat(-x2, x1) over the last dim (NeoX half-split)."""
    h = x.shape[-1] // 2
    return np.concatenate([-x[..., h:], x[..., :h]], axis=-1)


def apply_rotary_pos_emb(q, k, cos, sin):
    """rope.rs:96-132 with tof32=false: x*cos + rotate_half(x)*sin.
    q/k: (b, heads, S, hd); cos/sin (S, hd) or (b, S, hd)."""
    if cos.ndim == 2:
        cos = cos[None, None]
        sin = sin[None, None]
    elif cos.ndim == 3:
        cos = cos[:, None]
        sin = sin[:, None]
    cos = cos.astype(q.dtype)
    sin = sin.astype(q.dtype)
    return q * cos + rotate_half(q) * sin, k * cos + rotate_half(k) * sin


def apply_rotary_pos_emb_vision(q, k, cos, sin):
    """rope.rs:75-94: q,k (S, heads, hd); cos,sin (S, hd)."""
    cos = cos[:, None, :].astype(q.dtype)
    sin = sin[:, None, :].astype(q.dtype)
    return q * cos + rotate_half(q) * sin, k * cos + rotate_half(k) * sin


class RoPE:
    """rope.rs:583-612: 1-D RoPE tables for positions [offset, offset+S)."""

    def __init__(self, dim, theta):
        self.inv_freq = compute_default_rope_parameters(dim, theta)[None, :]

    def forward(self, seqlen_offset, seq_len):
        pos = np.arange(seqlen_offset, seqlen_offset + seq_len, dtype=F32).reshape(seq_len, 1)
        freqs = np.matmul(pos, self.inv_freq).astype(F32)
        emb = np.concatenate([freqs, freqs], axis=-1)
        return np.cos(emb).astype(F32), np.sin(emb).astype(F32)


class Qwen3VLTextRotaryEmbedding:
    """rope.rs:444-580: interleaved M-RoPE (VL variant `forward`, ASR variant `forward_asr`)."""

    def __init__(self, dim, theta):
        self.inv_freq = compute_default_rope_parameters(dim, theta)

    @staticmethod
    def apply_interleaved_mrope(freqs, mrope_section):
        """rope.rs:454-476: start from the T row; for dim in (1,2) overwrite indices
        dim, dim+3, ... < 3*section[dim] with that row."""
        out = freqs[0].copy()
        for dim in (1, 2):
            length = mrope_section[dim] * 3
            idx = np.arange(dim, length, 3)
            out[..., idx] = freqs[dim][..., idx]
        return out

    @staticmethod
    def apply_interleaved_mrope_asr(freqs, mrope_section):
        """rope.rs:478-500: as above but `length = mrope_section[dim]` (not x3)."""
        out = freqs[0].copy()
        for dim in (1, 2):
            length = mrope_section[dim]
            idx = np.arange(dim, length, 3)
            out[..., idx] = freqs[dim][..., idx]
        return out

    def _freqs(self, position_ids):
        position_ids = np.asarray(position_ids)
        if position_ids.ndim == 2:
            position_ids = np.broadcast_to(position_ids[None], (3,) + position_ids.shape)
        pos = position_ids.astype(F32)  # (3, b, S)
        # (3,b,hd/2,1) @ (3,b,1,S) -> transpose -> (3,b,S,hd/2)
        return (pos[..., None] * self.inv_freq[None, None, None, :]).astype(F32)

    def forward(self, position_ids, mrope_section):
        f = self.apply_interleaved_mrope(self._freqs(position_ids), mrope_section)
        emb = np.concatenate([f, f], axis=-1)
        return np.cos(emb).astype(F32), np.sin(emb).astype(F32)

    def forward_asr(self, position_ids, mrope_section):
        f = self.apply_interleaved_mrope_asr(self._freqs(position_ids), mrope_section)
        emb = np.concatenate([f, f], axis=-1)
        return np.cos(emb).astype(F32), np.sin(emb).astype(F32)


class Qwen2_5VisionRotaryEmbedding:
    """rope.rs:424-441: freq table (seqlen, dim/2) = p * inv_freq(dim, 1e4)."""

    def __init__(self, dim, theta=10000.0):
        self.inv_freq = compute_default_rope_parameters(dim, theta)

    def forward(self, seqlen):
        seq = np.arange(0, seqlen, dtype=F32).reshape(seqlen, 1)
        return np.matmul(seq, self.inv_freq[None, :]).astype(F32)


class SinusoidalPositionEncoderCat:
    """sinusoidal_pe.rs:6-58: [sin | cos] of p * inv_freq(dim, 1e4), added to xs (b, S, dim)."""

    def __init__(self, dim):
        self.inv_freq = compute_default_rope_parameters(dim, 10000.0)[None, :]

    def encode(self, seqlen_offset, seq_len):
        pos = np.arange(seqlen_offset, seqlen_offset + seq_len, dtype=F32).reshape(seq_len, 1)
        freqs = np.matmul(pos, self.inv_freq).astype(F32)
        return np.concatenate([np.sin(freqs), np.cos(freqs)], axis=-1).astype(F32)

    def forward(self, xs, seqlen_offset=0):
        return xs + self.encode(seqlen_offset, xs.shape[1])[None]
