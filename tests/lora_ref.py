"""float64 LoRA reference on tests/decode_ref.py, and synthetic adapters from a seed.

An adapter changes a projection y = W x into y = W x + s B (A x).  The reference merges it, W' = W + s B A in float64, and runs the float64
decoder on the merged weights; tests/test_lora_cpu.py checks that the merged form equals the unmerged one."""
import numpy as np

import decode_ref

F64 = np.float64
# PEFT target -> the base projection it names
TARGETS = {"q": "self_attn.q_proj", "k": "self_attn.k_proj", "v": "self_attn.v_proj", "o": "self_attn.o_proj",
           "gate": "mlp.gate_proj", "up": "mlp.up_proj", "down": "mlp.down_proj"}


def target_shape(cfg, t):
    """(N, K) of the base projection of target t"""
    H, I, hd = cfg["hidden_size"], cfg["intermediate_size"], cfg["head_dim"]
    q, kv = cfg["num_attention_heads"] * hd, cfg["num_key_value_heads"] * hd
    return {"q": (q, H), "k": (kv, H), "v": (kv, H), "o": (H, q), "gate": (I, H), "up": (I, H), "down": (H, I)}[t]


def make_adapter(cfg, seed, r, targets=tuple(TARGETS), layers=None, b_std=0.1, zero_b=False, prefix="model.", peft_prefix=""):
    """a synthetic adapter -> {PEFT name: fp16 array}: A [r, K] ~ N(0, 1 / K), B [N, r] ~ N(0, b_std) (zeros with zero_b), for every
    target in every layer of `layers` (None: all)"""
    rng = np.random.default_rng(seed)
    out = {}
    for l in (range(cfg["num_hidden_layers"]) if layers is None else layers):
        for t in targets:
            N, K = target_shape(cfg, t)
            base = f"{peft_prefix}{prefix}layers.{l}.{TARGETS[t]}"
            out[base + ".lora_A.weight"] = (rng.standard_normal((r, K), dtype=np.float32) / np.sqrt(K)).astype(np.float16)
            b = np.zeros((N, r), np.float32) if zero_b else rng.standard_normal((N, r), dtype=np.float32) * b_std
            out[base + ".lora_B.weight"] = b.astype(np.float16)
    return out


def _pairs(adapter):
    """{base weight name (without any base_model.model. prefix): (A, B)}"""
    pairs = {}
    for name, a in adapter.items():
        n = name[len("base_model.model."):] if name.startswith("base_model.model.") else name
        for which in ("A", "B"):
            suf = f".lora_{which}.weight"
            if n.endswith(suf):
                pairs.setdefault(n[: -len(suf)] + ".weight", {})[which] = a
    return {k: (v["A"], v["B"]) for k, v in pairs.items()}


def merged(w, adapter, scale):
    """the base weights with W' = W + scale B A (float64) for every target of the adapter"""
    out = dict(w)
    for name, (A, B) in _pairs(adapter).items():
        out[name] = np.asarray(w[name], F64) + F64(scale) * (np.asarray(B, F64) @ np.asarray(A, F64))
    return out


def unmerged_linear(x, W, A, B, scale):
    """y = W x + s B (A x) over rows of x, float64"""
    x = np.asarray(x, F64)
    return x @ np.asarray(W, F64).T + F64(scale) * ((x @ np.asarray(A, F64).T) @ np.asarray(B, F64).T)


def logits(cfg, w, adapter, scale, seqs):
    """float64 logits at every position of every sequence under the adapter (None: the base model)"""
    return decode_ref.logits(cfg, merged(w, adapter, scale) if adapter else w, seqs)


def step_bytes(cfg, r, targets=tuple(TARGETS)):
    """bytes one adapter adds to a decode step, from shapes: per layer and projection group, (N + K) x its 16-aligned columns x 2 bytes
    (the B columns the tail streams and the A rows the shrink reads).  A lower bound: the tail streams whole 64-column k-blocks, and the
    shrink reads A once per row that runs the adapter."""
    H, I, hd = cfg["hidden_size"], cfg["intermediate_size"], cfg["head_dim"]
    q, kv = cfg["num_attention_heads"] * hd, cfg["num_key_value_heads"] * hd
    groups = [(("q", "k", "v"), q + 2 * kv, H), (("o",), H, q), (("gate", "up"), 2 * I, H), (("down",), H, I)]
    b = 0
    for subs, N, K in groups:
        n = sum(1 for s in subs if s in targets)
        b += 2 * (N + K) * ((n * r + 15) // 16 * 16)
    return b * cfg["num_hidden_layers"]
