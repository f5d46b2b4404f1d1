"""LoRA adapters in a wide batch session (B200Model.batch_add_lora) at the Qwen3-0.6B and Qwen3-VL-2B text shapes (the `q0.6` preset and
the VL2 text rows as a qwen3 model, seed-0 synthetic weights, synthetic ids and adapters on all seven targets).

  python profiles/run_lora.py [--layers L] [--reps R] [--out FILE.json]

Per shape and rank r in {16, 64}, a 64-request wide session (64-token prompts, greedy) is stepped with
  0 adapters, 1 adapter on every row, 8 adapters (8 rows each), 64 distinct adapters (one per row),
and each row reports the decode step's time (host clock around STEPS steps ending in a synchronise, best of R) next to the tail bytes the
adapters add per step, computed from shapes (tests/lora_ref.py step_bytes: per layer and projection group, (N + K) x the adapter's
16-aligned columns x 2 bytes; a lower bound of what the step streams, BASELINE §4) and the base weight bytes of the step.  Then the time
to the first tokens of 8 packed 256-token prompts: batch_add_many (base) against batch_add_lora with 8 distinct adapters.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch

import lora_ref
from aha_b200 import B200Model, synth

STEPS, PROMPT, WIDTH = 16, 64, 64


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown (nvidia-smi unavailable)"


def timed(f):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = f()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def shape_cfg(name, layers):
    cfg = synth.get_config("qwen3", "q0.6")
    if name == "vl2":
        cfg.update(hidden_size=2048, intermediate_size=6144, rope_theta=5000000.0)
    if layers:
        cfg.update(num_hidden_layers=layers)
    return cfg


def base_bytes(cfg):
    H, I, L, hd = cfg["hidden_size"], cfg["intermediate_size"], cfg["num_hidden_layers"], cfg["head_dim"]
    q, kv = cfg["num_attention_heads"] * hd, cfg["num_key_value_heads"] * hd
    return 2 * L * ((q + 2 * kv) * H + H * q + 2 * I * H + H * I) + 2 * cfg["vocab_size"] * H


def step_ms(m, rows_adapters, reps):
    """a 64-request session, request j running rows_adapters[j] -> best ms per step"""
    best = None
    for _ in range(reps):
        m.batch_open_wide(WIDTH)
        try:
            reqs = [dict(input_ids=synth.synth_text_ids(PROMPT, m.vocab_size, 1000 + j), max_tokens=4 * STEPS + 8) for j in range(WIDTH)]
            m.batch_add_lora(reqs, rows_adapters)
            for _ in range(4):   # warm-up: the step graph of 64 rows
                m.batch_step()
            t, _ = timed(lambda: [m.batch_step() for _ in range(STEPS)])
        finally:
            m.batch_close()
        best = t if best is None else min(best, t)
    return 1e3 * best / STEPS


def admit_ms(m, adapters, reps):
    best = None
    for _ in range(reps):
        m.batch_open_wide(WIDTH)
        try:
            reqs = [dict(input_ids=synth.synth_text_ids(256, m.vocab_size, 2000 + j), max_tokens=2) for j in range(8)]
            t, _ = timed(lambda: m.batch_add_lora(reqs, adapters))
        finally:
            m.batch_close()
        best = t if best is None else min(best, t)
    return 1e3 * best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=0, help="layers of each shape (0: the preset's 28)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_lora.py needs the GPU")
    name, limit = card()
    rows = []
    for shape in ("0.6b", "vl2"):
        cfg = shape_cfg(shape, args.layers)
        w = synth.make_weights("qwen3", cfg, 0)
        m = B200Model("qwen3", cfg, w, eos_ids=[], max_ctx=WIDTH * 256 + 4096)
        try:
            base_ms = step_ms(m, [0] * WIDTH, args.reps)
            rows.append(dict(shape=shape, r=0, adapters=0, step_ms=base_ms, tail_bytes=0, base_bytes=base_bytes(cfg)))
            for r in (16, 64):
                ids = [m.lora_create(lora_ref.make_adapter(cfg, 3000 + i, r), 1.0) for i in range(WIDTH)]
                for n_ad, ad in ((1, [ids[0]] * WIDTH), (8, [ids[j % 8] for j in range(WIDTH)]), (64, ids)):
                    ms = step_ms(m, ad, args.reps)
                    tail = n_ad * lora_ref.step_bytes(cfg, r)
                    rows.append(dict(shape=shape, r=r, adapters=n_ad, step_ms=ms, tail_bytes=tail, base_bytes=base_bytes(cfg),
                                     tail_share=tail / base_bytes(cfg), vs_base=ms / base_ms))
                rows.append(dict(shape=shape, r=r, admit8_base_ms=admit_ms(m, [0] * 8, args.reps), admit8_lora_ms=admit_ms(m, ids[:8], args.reps)))
                for i in ids:
                    m.lora_destroy(i)
        finally:
            m.close()
        for row in rows:
            if row["shape"] == shape:
                print(json.dumps(row))
    out = dict(card=name, power_limit=limit, layers=args.layers or "preset", rows=rows)
    print(json.dumps(dict(card=name, power_limit=limit)))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
