"""The float64 attention reference (tests/attn_ref.py) against the oracle's own eager path (oracle/qwen3.py, oracle/rope.py), so that the
reference the kernel tests use cannot drift from the model's semantics.  No GPU."""
import ctypes
import ctypes.util

import numpy as np
import pytest

import attn_ref
from oracle import nn
from oracle.qwen3 import QKNormAttention, eager_attention_forward, prepare_causal_attention_mask
from oracle.rope import RoPE, compute_default_rope_parameters

F32 = np.float32


def _oracle_attention(q, k, v, causal):
    """q [Sq][nh][hd], k / v [Skv][nkv][hd] through eager_attention_forward -> [Sq][nh][hd]"""
    Sq, nh, hd = q.shape
    Skv, nkv = k.shape[:2]
    mask = prepare_causal_attention_mask(1, Sq, Skv - Sq) if causal else None
    t = lambda x: np.ascontiguousarray(np.swapaxes(x, 0, 1)[None])
    return eager_attention_forward(t(q), t(k), t(v), nh // nkv, mask, 1.0 / np.sqrt(np.float64(hd)))[0]


@pytest.mark.parametrize("G", [1, 2, 6])
@pytest.mark.parametrize("Sq,Skv,causal", [(1, 1, True), (5, 5, True), (3, 40, True), (7, 19, False)])
def test_attention_matches_oracle_eager_path(G, Sq, Skv, causal):
    rng = np.random.default_rng(Sq * 31 + Skv + G)
    nkv, hd = 2, 64
    q = rng.standard_normal((Sq, G * nkv, hd)).astype(F32) * 2
    k = rng.standard_normal((Skv, nkv, hd)).astype(F32)
    v = rng.standard_normal((Skv, nkv, hd)).astype(F32)
    want = _oracle_attention(q, k, v, causal)
    got = attn_ref.attention(q, k, v, causal)
    assert np.abs(got - want).max() <= 2e-5


def test_segments_are_independent_sequences():
    rng = np.random.default_rng(3)
    segs = [(0, 5), (8, 1), (16, 9)]
    q = rng.standard_normal((25, 4, 64)).astype(F32)
    k = rng.standard_normal((25, 2, 64)).astype(F32)
    v = rng.standard_normal((25, 2, 64)).astype(F32)
    for causal in (True, False):
        got = attn_ref.attention(q, k, v, causal, segments=segs)
        for s0, n in segs:
            sl = slice(s0, s0 + n)
            assert np.abs(got[sl] - _oracle_attention(q[sl], k[sl], v[sl], causal)).max() <= 2e-5
        assert np.isnan(got[5:8]).all() and np.isnan(got[9:16]).all()   # rows no segment covers


@pytest.mark.parametrize("theta", [1e4, 1e6, 5e6, 1e7])
@pytest.mark.parametrize("dim", [64, 80, 128])
def test_rope_frequencies_are_the_c_library_powf(dim, theta):
    """the oracle's inv_freq equals 1 / powf(theta, i / dim) from the C library, the powf rope.rs (f32::powf) and the library's
    rope_inv_freq call, bit for bit"""
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    libm.powf.restype = ctypes.c_float
    libm.powf.argtypes = [ctypes.c_float, ctypes.c_float]
    e = np.arange(0, dim, 2, dtype=F32) / F32(dim)
    want = np.array([F32(1.0) / F32(libm.powf(F32(theta), float(x))) for x in e], F32)
    assert np.array_equal(compute_default_rope_parameters(dim, theta), want)


@pytest.mark.parametrize("pos", [0, 1, 31, 2049, 33000])
def test_rope_angle_is_the_oracle_float32_product(pos):
    """float32(pos) * inv_freq, the oracle's RoPE table argument, bit for bit; cos / sin within float32 rounding of the oracle's"""
    hd, theta = 128, 1e6
    ro = RoPE(hd, theta)
    freqs = np.matmul(np.arange(pos, pos + 1, dtype=F32).reshape(1, 1), ro.inv_freq).astype(F32)[0]
    a = attn_ref.rope_angles(pos, hd, theta)
    assert np.array_equal(a[:hd // 2].astype(F32), freqs) and np.array_equal(a[:hd // 2], a[hd // 2:])
    cos, sin = ro.forward(pos, 1)
    assert np.abs(np.cos(a) - cos[0]).max() <= 1e-6 and np.abs(np.sin(a) - sin[0]).max() <= 1e-6
    x = np.random.default_rng(pos).standard_normal(hd)
    assert np.allclose(attn_ref.rope(attn_ref.rope(x, pos, theta), pos, theta, inverse=True), x, atol=1e-12)


@pytest.mark.parametrize("nh,nkv", [(2, 2), (4, 1), (12, 2)])
def test_decode_step_matches_oracle_attention_layer(nh, nkv):
    """A whole QKNormAttention of the oracle (prefill of `pos` tokens, then one step), with o_proj the identity so that its output is
    the attention rows: the reference's prologue + attention on the raw projections of the step gives the same rows."""
    rng = np.random.default_rng(nh * 10 + nkv)
    hd, H, pos, eps, theta = 128, 64, 37, 1e-6, 1e6
    w = {"a.q_proj.weight": rng.standard_normal((nh * hd, H)).astype(F32) / 8,
         "a.k_proj.weight": rng.standard_normal((nkv * hd, H)).astype(F32) / 8,
         "a.v_proj.weight": rng.standard_normal((nkv * hd, H)).astype(F32) / 8,
         "a.o_proj.weight": np.eye(nh * hd, dtype=F32),
         "a.q_norm.weight": rng.uniform(0.5, 3.0, hd).astype(F32),
         "a.k_norm.weight": rng.uniform(0.5, 3.0, hd).astype(F32)}
    att = QKNormAttention(w, "a.", nh, hd, nkv, eps)
    x = rng.standard_normal((1, pos + 1, H)).astype(F32)
    rope = RoPE(hd, theta)
    cos, sin = rope.forward(0, pos)
    att.forward(x[:, :pos], cos, sin, prepare_causal_attention_mask(1, pos))
    cos, sin = rope.forward(pos, 1)
    want = att.forward(x[:, pos:], cos, sin, None)[0, 0].reshape(nh, hd)
    # the cache as the oracle holds it (rotated K, V), and the raw projections of the new token
    k_cache = np.swapaxes(att.kv_cache[0][0, :, :pos], 0, 1)
    v_cache = np.swapaxes(att.kv_cache[1][0, :, :pos], 0, 1)
    qkv = np.concatenate([nn.linear(x[0, pos], w[f"a.{n}_proj.weight"]) for n in "qkv"])
    got, k_new, v_new = attn_ref.decode_attention(qkv, k_cache, v_cache, pos, 0, w["a.q_norm.weight"], w["a.k_norm.weight"], eps, theta, nh, nkv)
    assert np.abs(got - want).max() <= 2e-5 * max(1.0, np.abs(v_cache).max())
    assert np.abs(k_new - att.kv_cache[0][0, :, pos]).max() <= 1e-5 * np.abs(k_new).max()
    assert np.array_equal(v_new, att.kv_cache[1][0, :, pos])
