"""Prefix cache of a batch session (B200Model.batch_prefix_cache): admission of requests that share a system prompt, cold against warm,
on the Qwen3-0.6B shape (the `q0.6` preset, seed-0 synthetic weights, synthetic ids).

  python profiles/run_prefix_share.py [--reps R] [--out FILE.json]

Two workloads: 8 requests on a narrow session and 64 on a wide one.  Every request is a 2048-token system prompt followed by its own
64-token tail (greedy, 17 tokens each).  Per workload, after a warm-up, the paths are timed alternately, R times each, and the best of R is
reported:
  cold    a fresh session, one batch_add_many of all requests (the cache off);
  warm    a fresh session with the cache on, one request with the system prompt admitted and finished first (untimed), then the same
          batch_add_many, which finds 2048 tokens of every prompt cached and prefills only the tails;
  decode  16 batch_step calls after each admission, per step: with shared pages the steps read as many KV pages as without.
Admission time ends in a device synchronise.  ids_equal says whether both paths gave every request the same 17 ids.  The card's name and
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

SYSTEM, TAIL, STEPS = 2048, 64, 16
WORKLOADS = [("narrow", 8), ("wide", 64)]


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown (nvidia-smi unavailable)"


def run(m, kind, n, reqs, warm_req):
    """-> (seconds to all first tokens, seconds per decode step, ids per request, tokens the requests took from the cache)"""
    if kind == "narrow":
        m.batch_open()
    else:
        m.batch_open_wide(n)
    try:
        if warm_req is not None:
            m.batch_prefix_cache(SYSTEM + 4 * TAIL)
            m.batch_add(**warm_req)
            while m.batch_step():
                pass
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = m.batch_add_many(reqs)
        torch.cuda.synchronize()
        t_admit = time.perf_counter() - t0
        hit = sum(m.batch_prefix_stats()[1].values()) if warm_req is not None else 0
        out = {slot: [tok] for slot, tok, _ in res}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(STEPS):
            for slot, (tok, _) in m.batch_step().items():
                out[slot].append(tok)
        torch.cuda.synchronize()
        t_step = (time.perf_counter() - t0) / STEPS
        return t_admit, t_step, [out[slot] for slot, _, _ in res], hit
    finally:
        m.batch_close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_prefix_share.py needs the GPU")
    name, limit = card()
    cfg = synth.get_config("qwen3", "q0.6")
    w = synth.make_weights("qwen3", cfg, 0)
    V = cfg["vocab_size"]
    # 64 requests of 2048 + 64 + 17 tokens: 68 pages each
    m = B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"]], max_ctx=72 * 68 * 32, max_prefill=8192)
    del w
    system = [int(t) for t in synth.synth_text_ids(SYSTEM, V - 8, 1)]
    warm_req = dict(input_ids=system + [int(t) for t in synth.synth_text_ids(TAIL, V - 8, 2)], max_tokens=1)
    rows = []
    for kind, n in WORKLOADS:
        reqs = [dict(input_ids=system + [int(t) for t in synth.synth_text_ids(TAIL, V - 8, 100 + i)], max_tokens=STEPS + 1) for i in range(n)]
        run(m, kind, n, reqs, None); run(m, kind, n, reqs, warm_req)   # warm-up: module loads, workspace growth, step graphs
        cold, warm, step_cold, step_warm, ids_equal, hit = [], [], [], [], True, 0
        for _ in range(args.reps):
            ta, ts, a, _ = run(m, kind, n, reqs, None); cold.append(ta); step_cold.append(ts)
            ta, ts, b, hit = run(m, kind, n, reqs, warm_req); warm.append(ta); step_warm.append(ts)
            ids_equal = ids_equal and a == b
        r = dict(session=kind, requests=n, system_tokens=SYSTEM, tail_tokens=TAIL, hit_tokens=hit, cold_admit_ms=1e3 * min(cold),
                 warm_admit_ms=1e3 * min(warm), speedup=min(cold) / min(warm), step_ms_cold=1e3 * min(step_cold),
                 step_ms_warm=1e3 * min(step_warm), ids_equal=ids_equal)
        rows.append(r)
        print(f"{kind:6s} {n:2d} x ({SYSTEM} + {TAIL}): cold {r['cold_admit_ms']:8.2f} ms   warm {r['warm_admit_ms']:8.2f} ms   x{r['speedup']:.2f}"
              f"   step {r['step_ms_cold']:.3f} / {r['step_ms_warm']:.3f} ms   hit {hit}   ids equal {ids_equal}", flush=True)
    m.close()
    res = dict(card=name, power_limit=limit, preset="q0.6", reps=args.reps, steps=STEPS, workloads=rows)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
