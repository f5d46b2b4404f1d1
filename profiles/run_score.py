"""Scoring given text (aha_b200_score / _score_batch): the fused score_head_kernel and the packed path, on synthetic seed-0 weights.

  python profiles/run_score.py [--reps R] [--out FILE.json]

Workloads:
  1. Qwen3-0.6B shape (28 layers, V 151936): one 2048-token text, every position scored with 0 / 5 / 20 alternatives, against `embed` of
     the same text (the same prefill without a head over every row: the prefill-only floor).  head share = (score - embed) / score.
  2. The head alone (aha_b200_bench_kernel) over M = 128 / 512 / 2048 rows of that prefill, score_head_kernel against its twin (gemm_tc
     into a logits block + logprob_partial_rows_kernel), each with its final RMSNorm and stage 2, 0 and 20 alternatives.  Useful work
     2 M V H FLOP (the split-fp16 operands issue twice that); achieved TFLOP/s over the 989 TFLOP/s dense FP16 data-sheet figure is a
     kernel share, not a whole-program one.
  3. lm-eval style: 512 texts of 192 context + 16 continuation tokens, start = 192: one `score_batch` against `score` text by text.
  4. Workload 1 at the Qwen3-VL-2B text-stack shape (H 2048, I 6144, 28 layers, V 151936).
Every path gets one warm-up call; the paths are then timed alternately R times, each timing ending in a device synchronise, best of R.
The card's name and power limit are read in the same run."""
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

PEAK_TFLOPS = 989.0


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


def best_alternated(fns, reps):
    for f in fns.values():
        f()
    t = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            t[k].append(timed(f)[0])
    return {k: min(v) for k, v in t.items()}


def one_text(m, cfg, reps):
    ids = synth.synth_text_ids(2048, cfg["vocab_size"], 1)
    fns = {"embed": lambda: m.embed(ids)}
    for n in (0, 5, 20):
        fns[f"score_top{n}"] = (lambda n=n: m.score(ids, top=n))
    t = best_alternated(fns, reps)
    r = {k + "_ms": v * 1e3 for k, v in t.items()}
    for n in (0, 5, 20):
        r[f"head_share_top{n}"] = (t[f"score_top{n}"] - t["embed"]) / t[f"score_top{n}"]
    return r


def head_alone(m, cfg, reps):
    V, H = cfg["vocab_size"], cfg["hidden_size"]
    rows = []
    for M in (128, 512, 2048):
        for n in (0, 20):
            ms = {}
            for _ in range(reps):
                for impl in ("head", "twin"):
                    v, _ = m.bench_kernel(f"score_{impl}:{M}:{n}", 20)
                    ms[impl] = min(ms.get(impl, 1e30), v)
            useful = 2.0 * M * V * H
            r = dict(M=M, top=n, fused_ms=ms["head"], twin_ms=ms["twin"], speedup=ms["twin"] / ms["head"],
                     fused_tflops=useful / ms["head"] / 1e9, twin_tflops=useful / ms["twin"] / 1e9)
            r["fused_kernel_share"] = r["fused_tflops"] / PEAK_TFLOPS
            r["fused_issued_share"] = 2 * r["fused_kernel_share"]
            rows.append(r)
            print(f"  head M {M:5d} top {n:2d}: fused {r['fused_ms']:.3f} ms ({r['fused_tflops']:.0f} TFLOP/s useful, "
                  f"{100 * r['fused_kernel_share']:.1f} % of {PEAK_TFLOPS:.0f})   twin {r['twin_ms']:.3f} ms   x{r['speedup']:.2f}", flush=True)
    return rows


def lm_eval(m, cfg, reps):
    texts = [synth.synth_text_ids(208, cfg["vocab_size"], 100 + i) for i in range(512)]
    starts = [192] * len(texts)
    one = lambda: [m.score(t, start=192) for t in texts]
    packed = lambda: m.score_batch(texts, starts=starts)
    t = best_alternated({"score": one, "score_batch": packed}, reps)
    a, b = one(), packed()
    diff = max(float(np.abs(x["logprobs"] - y["logprobs"]).max()) for x, y in zip(a, b))
    return dict(texts=len(texts), score_texts_per_s=len(texts) / t["score"], score_batch_texts_per_s=len(texts) / t["score_batch"],
                speedup=t["score"] / t["score_batch"], max_abs_logprob_diff=diff)


def model(cfg):
    w = synth.make_weights("qwen3", cfg, 0)
    m = B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"]], max_ctx=2048, max_prefill=2048)
    del w
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_score.py needs the GPU")
    name, limit = card()
    res = dict(card=name, power_limit=limit, reps=args.reps)
    cfg = synth.get_config("qwen3", "q0.6")
    m = model(cfg)
    res["q0.6_one_text"] = one_text(m, cfg, args.reps)
    print("q0.6 one 2048-token text:", json.dumps(res["q0.6_one_text"]), flush=True)
    res["q0.6_head_alone"] = head_alone(m, cfg, args.reps)
    res["q0.6_lm_eval"] = lm_eval(m, cfg, args.reps)
    print("q0.6 lm-eval:", json.dumps(res["q0.6_lm_eval"]), flush=True)
    m.close()
    vl2 = dict(cfg, hidden_size=2048, intermediate_size=6144, rope_theta=5000000.0)
    m = model(vl2)
    res["vl2_one_text"] = one_text(m, vl2, args.reps)
    print("vl2 one 2048-token text:", json.dumps(res["vl2_one_text"]), flush=True)
    m.close()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
