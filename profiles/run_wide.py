"""Wide batch sessions (batch_open_wide, tensor-core projections) against the narrow 8-slot session (CUDA-core batched GEMV): decode
throughput per running count.  Synthetic seed-0 weights at the VL2 text-stack shape (AHA_SHAPE=vl2, the default: H 2048, I 6144) or the
Qwen3-0.6B shape (AHA_SHAPE=q0.6), as in run_batch.py.

  AHA_SHAPE=vl2|q0.6 python profiles/run_wide.py [--reps R] [--out FILE.json]

Series: the narrow session at 8 requests, the wide session (width 64) at 8, 16, 32 and 64.  Every request has a 128-token prompt and
generates 64 tokens (no stop ids).  A run admits the requests with one batch_add_many (not timed), then times the 63 lockstep steps on a host
clock that ends in a device synchronise (every batch_step synchronises to deliver its tokens).  Every series is warmed once, then the
series are run alternately R times; the best of R is reported as aggregate decode tokens/s and ms per step.  `weight_share` is the fp16
weight bytes one step streams (every projection and the lm_head once) over the step time, as a share of the data-sheet 3.35 TB/s: a
whole-step rate, not a kernel's.  `ids_equal_single` counts the requests whose 64 ids equal their single-request generate ids (a wide
session promises oracle ids and composition invariance, not bit equality with the CUDA-core GEMV).  The card's name and power limit are
read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from aha_b200 import B200Model, synth

PROMPT, GEN = 128, 64
SERIES = [("narrow", 8), ("wide", 8), ("wide", 16), ("wide", 32), ("wide", 64)]
HBM = 3.35e12


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown (nvidia-smi unavailable)"


def weight_bytes(cfg):
    H, I, L, V = cfg["hidden_size"], cfg["intermediate_size"], cfg["num_hidden_layers"], cfg["vocab_size"]
    q, kv = cfg["num_attention_heads"] * cfg["head_dim"], cfg["num_key_value_heads"] * cfg["head_dim"]
    per_layer = (q + 2 * kv) * H + H * q + 2 * I * H + H * I
    return 2 * (L * per_layer + V * H)


def run(m, reqs, mode):
    """-> (seconds for the GEN - 1 steps, ids per request)"""
    m.batch_open() if mode == "narrow" else m.batch_open_wide(64)
    try:
        res = m.batch_add_many(reqs)
        out = {slot: [tok] for slot, tok, _ in res}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(GEN - 1):
            for slot, (tok, _) in m.batch_step().items():
                out[slot].append(tok)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, [out[slot] for slot, _, _ in res]
    finally:
        m.batch_close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_wide.py needs the GPU")
    name, limit = card()
    shape = os.environ.get("AHA_SHAPE", "vl2")
    cfg = synth.get_config("qwen3", "q0.6")
    if shape == "vl2":
        cfg.update(hidden_size=2048, intermediate_size=6144, rope_theta=5e6)
    w = synth.make_weights("qwen3", cfg, 0)
    m = B200Model("qwen3", cfg, w, eos_ids=[], max_ctx=64 * (PROMPT + GEN + 64), max_prefill=2048)
    del w
    reqs = [dict(input_ids=synth.synth_text_ids(PROMPT, 151000, 500 + i), max_tokens=GEN) for i in range(64)]
    for mode, n in SERIES:   # warm-up: module loads, step graphs of every width
        run(m, reqs[:n], mode)
    best, ids = {}, {}
    for _ in range(args.reps):
        for mode, n in SERIES:
            dt, got = run(m, reqs[:n], mode)
            best[(mode, n)] = min(best.get((mode, n), 1e30), dt)
            ids[(mode, n)] = got
    singles = [m.generate(r["input_ids"], max_tokens=GEN)[0] for r in reqs]
    wb = weight_bytes(cfg)
    rows = []
    for mode, n in SERIES:
        step = best[(mode, n)] / (GEN - 1)
        r = dict(mode=mode, requests=n, ms_per_step=1e3 * step, tokens_per_s=n / step, weight_share=wb / step / HBM,
                 ids_equal_single=sum(a == b for a, b in zip(ids[(mode, n)], singles)))
        rows.append(r)
        print(f"{mode:6s} {n:2d} requests: {r['ms_per_step']:7.3f} ms/step  {r['tokens_per_s']:8.1f} tok/s  weights {100 * r['weight_share']:5.1f}% of 3.35 TB/s"
              f"  ids equal to single runs {r['ids_equal_single']}/{n}", flush=True)
    m.close()
    res = dict(card=name, power_limit=limit, shape=shape, prompt=PROMPT, generated=GEN, reps=args.reps, weight_bytes_per_step=wb, series=rows)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
