"""Packed embeddings against one prefill per text: Qwen3-0.6B shape (the `q0.6` preset, seed-0 synthetic weights, synthetic ids).

  python profiles/run_embed.py [--reps R] [--out FILE.json]

Three workloads: 256 texts x 16 tokens, 64 x 256 and 8 x 2048 (one pack of 16384 tokens: nothing to share, the no-regression side).
Per workload, after one warm-up call of each path, the loop of B200Model.embed and one B200Model.embed_batch are timed alternately, R
times each, every timing ending in a device synchronise; the best of R is reported as texts/s.  max_abs_diff: the largest |difference|
between the two paths' vectors.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from aha_b200 import B200Model, synth

WORKLOADS = [(256, 16), (64, 256), (8, 2048)]


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown (nvidia-smi unavailable)"


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_embed.py needs the GPU")
    name, limit = card()
    cfg = synth.get_config("qwen3", "q0.6")
    w = synth.make_weights("qwen3", cfg, 0)
    cap = max(n * s for n, s in WORKLOADS)
    m = B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"]], max_ctx=cap, max_prefill=cap)
    del w
    rows = []
    for k, (n, s) in enumerate(WORKLOADS):
        texts = [synth.synth_text_ids(s, cfg["vocab_size"], 1000 * k + i) for i in range(n)]
        one = lambda: np.stack([m.embed(t) for t in texts])
        packed = lambda: m.embed_batch(texts)
        one(); packed()   # warm-up: module loads, workspace growth
        t_one, t_packed = [], []
        for _ in range(args.reps):
            dt, a = timed(one); t_one.append(dt)
            dt, b = timed(packed); t_packed.append(dt)
        r = dict(texts=n, tokens_per_text=s, embed_texts_per_s=n / min(t_one), embed_batch_texts_per_s=n / min(t_packed),
                 speedup=min(t_one) / min(t_packed), max_abs_diff=float(np.abs(a - b).max()))
        rows.append(r)
        print(f"{n:4d} x {s:5d} tokens: embed {r['embed_texts_per_s']:10.1f} texts/s   embed_batch {r['embed_batch_texts_per_s']:10.1f} texts/s"
              f"   x{r['speedup']:.2f}   max|d| {r['max_abs_diff']:.2e}", flush=True)
    m.close()
    res = dict(card=name, power_limit=limit, preset="q0.6", reps=args.reps, workloads=rows)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
