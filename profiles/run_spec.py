"""What speculative decoding of one request buys.  Synthetic seed-0 weights at the VL2 text-stack shape (Qwen3-0.6B config with H 2048,
I 6144, V 151936, as in run_wide.py) and at the Qwen3-0.6B shape itself.

  python profiles/run_spec.py [--reps R] [--out FILE.json]

Per shape: a 512-token prompt and 256 greedy tokens (no stop ids, so every call emits all 256).  Timed: `generate` on the fused decode
kernel, and `generate_speculative` with an exact prediction (the output of a draftless speculative call), a 50 %-edited one (half of
its positions replaced by random ids), prompt lookup only, and no draft source, at max_draft 7 (R = 8 rows); and, with no draft source,
one call per R in {2, 4, 8, 16} for the time of one pass (R = 1 is not a configuration: max_draft is at least 1).  Every series is
alternated R times, best of R, on usage.completion_secs (the decode loop, which ends in a device synchronise); tok/s counts the 255
tokens after the first.  Kernel times: torch.profiler (CUDA activities) over one more exact-prediction call, by kernel name.  The
card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from aha_b200 import B200Model, synth

PROMPT, GEN = 512, 256


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown (nvidia-smi unavailable)"


def kernel_times(m, ids, pred):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.generate_speculative(ids, prediction=pred, max_draft=7, max_tokens=GEN)
        torch.cuda.synchronize()
    us = {}
    for e in prof.key_averages():
        if "spec_" in e.key or "gemv_wide" in e.key:
            us[e.key.split("(")[0].split("<")[0].split("::")[-1]] = dict(count=e.count, avg_us=e.device_time_total / max(e.count, 1))
    return us


def run_shape(label, cfg, reps):
    w = synth.make_weights("qwen3", cfg, 0)
    m = B200Model("qwen3", cfg, w, eos_ids=[], max_ctx=1024, max_prefill=1024)
    del w
    V = cfg["vocab_size"]
    ids = synth.synth_text_ids(PROMPT, V - 8, 7)
    exact = m.generate_speculative(ids, max_draft=1, max_tokens=GEN)[0]
    rng = np.random.default_rng(1)
    edited = list(exact)
    for i in rng.choice(GEN, GEN // 2, replace=False):
        edited[i] = int(rng.integers(0, V))
    series = {
        "generate": lambda: m.generate(ids, max_tokens=GEN),
        "exact prediction": lambda: m.generate_speculative(ids, prediction=exact, max_draft=7, max_tokens=GEN),
        "50 % edited prediction": lambda: m.generate_speculative(ids, prediction=edited, max_draft=7, max_tokens=GEN),
        "prompt lookup": lambda: m.generate_speculative(ids, prompt_lookup=True, max_draft=7, max_tokens=GEN),
        "no draft source": lambda: m.generate_speculative(ids, max_draft=7, max_tokens=GEN),
    }
    for R in (2, 4, 8, 16):
        series[f"pass R={R}"] = (lambda R=R: m.generate_speculative(ids, max_draft=R - 1, max_tokens=GEN))
    for f in series.values():
        f()
    best, stats, outs = {}, {}, {}
    for _ in range(reps):
        for k, f in series.items():
            r = f()
            best[k] = min(best.get(k, 1e30), r[1]["completion_secs"])
            outs[k] = r[0]
            if len(r) > 2:
                stats[k] = r[2]
    rows = []
    for k in series:
        row = dict(series=k, completion_ms=1e3 * best[k], tok_s=(GEN - 1) / best[k], speedup=best["generate"] / best[k])
        if k in stats:
            row.update(stats[k])
            row["ms_per_pass"] = 1e3 * best[k] / max(stats[k]["passes"], 1)
        rows.append(row)
        print(f"{label} {k:24s} {row['completion_ms']:9.2f} ms  {row['tok_s']:8.1f} tok/s  x{row['speedup']:5.2f}"
              + (f"  passes {row['passes']:4d} drafted {row['drafted']:5d} accepted {row['accepted']:5d}  {row['ms_per_pass']:6.3f} ms/pass" if k in stats else ""),
              flush=True)
    same = all(outs[k] == exact for k in series if k != "generate")
    first_same = outs["generate"][0] == exact[0]
    kt = kernel_times(m, ids, exact)
    print(label, "kernels", json.dumps(kt), flush=True)
    m.close()
    return dict(shape=label, rows=rows, spec_ids_identical=same, first_token_equals_generate=first_same,
                ids_equal_generate=outs["generate"] == exact, kernels=kt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_spec.py needs the GPU")
    name, limit = card()
    vl2 = synth.get_config("qwen3", "q0.6")
    vl2.update(hidden_size=2048, intermediate_size=6144, rope_theta=5e6)
    res = dict(card=name, power_limit=limit, prompt=PROMPT, generated=GEN, reps=args.reps,
               shapes=[run_shape("vl2", vl2, args.reps), run_shape("q0.6", synth.get_config("qwen3", "q0.6"), args.reps)])
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
