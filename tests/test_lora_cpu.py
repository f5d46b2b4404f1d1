"""The float64 LoRA reference (tests/lora_ref.py) against the unmerged form, and the declarations of the LoRA entries in the C header, the
ctypes bindings and the C++ wrapper."""
import os

import numpy as np

import decode_ref
import lora_ref
from conftest import ROOT

CFG = dict(hidden_size=128, intermediate_size=192, num_attention_heads=4, num_key_value_heads=2, head_dim=32, num_hidden_layers=2,
           vocab_size=96, rms_norm_eps=1e-6, rope_theta=1e6, tie_word_embeddings=True)


def _weights(seed):
    rng = np.random.default_rng(seed)
    H, I, hd, L = CFG["hidden_size"], CFG["intermediate_size"], CFG["head_dim"], CFG["num_hidden_layers"]
    w = {"model.embed_tokens.weight": (rng.standard_normal((CFG["vocab_size"], H)) * 0.3).astype(np.float16),
         "model.norm.weight": (1 + 0.02 * rng.standard_normal(H)).astype(np.float16)}
    for l in range(L):
        p = f"model.layers.{l}."
        for t in lora_ref.TARGETS:
            N, K = lora_ref.target_shape(CFG, t)
            w[p + lora_ref.TARGETS[t] + ".weight"] = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
        for n, d in (("input_layernorm", H), ("post_attention_layernorm", H), ("self_attn.q_norm", hd), ("self_attn.k_norm", hd)):
            w[p + n + ".weight"] = (1 + 0.02 * rng.standard_normal(d)).astype(np.float16)
    return w


def test_merged_equals_unmerged_projection():
    rng = np.random.default_rng(3)
    for t in lora_ref.TARGETS:
        N, K = lora_ref.target_shape(CFG, t)
        W = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
        ad = lora_ref.make_adapter(CFG, 5, 8, targets=(t,), layers=[0])
        (name, (A, B)), = lora_ref._pairs(ad).items()
        x = rng.standard_normal((7, K))
        merged = lora_ref.merged({name: W}, ad, 0.75)[name]
        np.testing.assert_allclose(x @ merged.T, lora_ref.unmerged_linear(x, W, A, B, 0.75), rtol=1e-12, atol=1e-12)


def test_reference_decoder_under_an_adapter():
    """the merged decoder changes the logits, a zero-B adapter does not, and base_model.model. names merge the same weights"""
    w = _weights(0)
    seqs = [np.arange(11) % CFG["vocab_size"]]
    base = decode_ref.logits(CFG, w, seqs)[0]
    ad = lora_ref.make_adapter(CFG, 1, 4)
    got = lora_ref.logits(CFG, w, ad, 2.0, seqs)[0]
    assert np.abs(got - base).max() > 1e-3
    peft = {"base_model.model." + k: v for k, v in ad.items()}
    np.testing.assert_array_equal(lora_ref.logits(CFG, w, peft, 2.0, seqs)[0], got)
    zero = lora_ref.make_adapter(CFG, 1, 4, zero_b=True)
    np.testing.assert_array_equal(lora_ref.logits(CFG, w, zero, 2.0, seqs)[0], base)


def test_step_bytes_at_the_0_6b_shape():
    """a rank-16 adapter on all seven targets of Qwen3-0.6B (28 layers): about 2 % of the base weight stream per step"""
    from aha_b200 import synth
    cfg = synth.get_config("qwen3", "q0.6")
    b = lora_ref.step_bytes(cfg, 16)
    H, I, L, hd = cfg["hidden_size"], cfg["intermediate_size"], cfg["num_hidden_layers"], cfg["head_dim"]
    q, kv = cfg["num_attention_heads"] * hd, cfg["num_key_value_heads"] * hd
    base = 2 * L * ((q + 2 * kv) * H + H * q + 2 * I * H + H * I) + 2 * cfg["vocab_size"] * H
    assert 0.01 < b / base < 0.03, b / base


def test_lora_entries_are_declared():
    with open(os.path.join(ROOT, "include", "aha_b200.h")) as f:
        h = f.read()
    with open(os.path.join(ROOT, "include", "aha_b200.hpp")) as f:
        hpp = f.read()
    from aha_b200 import _lib
    for fn in ("aha_b200_lora_create", "aha_b200_lora_destroy", "aha_b200_batch_add_lora"):
        assert fn + "(" in h, fn
        assert fn in _lib.SYMBOLS, fn
        assert fn + "(" in hpp, fn
    from aha_b200 import B200Model
    for m in ("lora_create", "lora_destroy", "batch_add_lora"):
        assert callable(getattr(B200Model, m))
