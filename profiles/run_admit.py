"""Packed admission into a batch session against one batch_add per request: Qwen3-0.6B shape (the `q0.6` preset, seed-0 synthetic
weights, synthetic ids).

  python profiles/run_admit.py [--reps R] [--out FILE.json]

Three workloads: 8 requests of 16, 128 and 512 prompt tokens (greedy, 17 tokens each).  Per workload, after one warm-up of each path, the
two paths are timed alternately, R times each: a fresh session, then either eight B200Model.batch_add calls or one batch_add_many, the timing
ending in a device synchronise.  The time is the time to all first tokens; the best of R is reported.  Each run then steps the session 16
times: first_equal / ids_equal say whether the two paths gave the same first tokens and the same 17 ids per request.  The card's name and
power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from aha_b200 import B200Model, synth

WORKLOADS = [(8, 16), (8, 128), (8, 512)]
STEPS = 16


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown (nvidia-smi unavailable)"


def run(m, reqs, many):
    """-> (seconds to all first tokens, ids per request after STEPS steps)"""
    m.batch_open()
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = m.batch_add_many(reqs) if many else [m.batch_add(**r) for r in reqs]
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        out = {slot: [tok] for slot, tok, _ in res}
        for _ in range(STEPS):
            for slot, (tok, _) in m.batch_step().items():
                out[slot].append(tok)
        return dt, [out[slot] for slot, _, _ in res]
    finally:
        m.batch_close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_admit.py needs the GPU")
    name, limit = card()
    cfg = synth.get_config("qwen3", "q0.6")
    w = synth.make_weights("qwen3", cfg, 0)
    m = B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"]], max_ctx=8192, max_prefill=4096)
    del w
    rows = []
    for k, (n, s) in enumerate(WORKLOADS):
        reqs = [dict(input_ids=synth.synth_text_ids(s, cfg["vocab_size"], 1000 * k + i), max_tokens=STEPS + 1) for i in range(n)]
        run(m, reqs, False); run(m, reqs, True)   # warm-up: module loads, workspace growth, step graphs
        t_one, t_many, first_equal, ids_equal = [], [], True, True
        for _ in range(args.reps):
            dt, a = run(m, reqs, False); t_one.append(dt)
            dt, b = run(m, reqs, True); t_many.append(dt)
            first_equal = first_equal and [x[0] for x in a] == [x[0] for x in b]
            ids_equal = ids_equal and a == b
        r = dict(requests=n, prompt_tokens=s, batch_add_ms=1e3 * min(t_one), batch_add_many_ms=1e3 * min(t_many),
                 speedup=min(t_one) / min(t_many), first_equal=first_equal, ids_equal=ids_equal)
        rows.append(r)
        print(f"{n} x {s:4d} tokens: batch_add {r['batch_add_ms']:8.2f} ms   batch_add_many {r['batch_add_many_ms']:8.2f} ms   x{r['speedup']:.2f}"
              f"   first tokens equal {first_equal}   ids equal {ids_equal}", flush=True)
    m.close()
    res = dict(card=name, power_limit=limit, preset="q0.6", reps=args.reps, steps=STEPS, workloads=rows)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
