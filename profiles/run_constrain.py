"""What constrained decoding (AHA_GEN_CONSTRAINED) costs.  Synthetic seed-0 weights at the Qwen3-0.6B shape (H 1024, 28 layers,
V 151936), CUDA graphs on.

  python profiles/run_constrain.py [--reps R] [--out FILE.json]

Automata (16 states, seeded random successors): all-allowed (one state, every token), sparse (8 tokens per state) and dense (all but 8
tokens per state).  Single request: a 512-token prompt, 128 greedy tokens (no stop ids), unconstrained against each automaton, alternated R
times, best of R on a host clock around the whole call (it ends in a device synchronise); per token = call time / 128.  Wide x 64
session: 64 requests of 128-token prompts, 64 tokens each, every request constrained by the same automaton (greedy), the 63 lockstep
steps timed, alternated, best of R.  Kernel times: torch.profiler (CUDA activities) over one more single request and one more wide session
per automaton, by kernel name (sample_kernel, sample_rows_kernel).  HBM footprint of each automaton: offsets (8 bytes per state + 8) and
tokens + successors (8 bytes per transition), one allocation.  The card's name and power limit are read in the same run."""
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

PROMPT, GEN = 512, 128
W_PROMPT, W_GEN = 128, 64
STATES = 16


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown (nvidia-smi unavailable)"


def automata(V):
    """name -> (offsets, tokens, next, start)"""
    rng = np.random.default_rng(0)
    out = {"all-allowed": (np.array([0, V], np.uint64), np.arange(V, dtype=np.uint32), np.zeros(V, np.uint32), 0)}
    for name, k in (("sparse", 8), ("dense", V - 8)):
        off, tok, nxt = [0], [], []
        for _ in range(STATES):
            t = np.sort(rng.choice(V, size=8, replace=False)) if k == 8 else np.setdiff1d(np.arange(V), rng.choice(V, size=8, replace=False))
            tok.append(t.astype(np.uint32))
            nxt.append(rng.integers(0, STATES, t.size).astype(np.uint32))
            off.append(off[-1] + t.size)
        out[name] = (np.array(off, np.uint64), np.concatenate(tok), np.concatenate(nxt), 0)
    return out


def hbm_bytes(fsm):
    return 8 * len(fsm[0]) + 8 * len(fsm[1])


def single(m, ids, fsm):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = m.generate(ids, max_tokens=GEN, fsm=fsm)[0]
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def wide(m, reqs, fsm):
    m.batch_open_wide(64)
    try:
        m.batch_add_many([dict(r, fsm=fsm) for r in reqs])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(W_GEN - 1):
            m.batch_step()
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    finally:
        m.batch_close()


def kernel_times(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    us = {}
    for e in prof.key_averages():
        if "sample_" in e.key and "kernel" in e.key:
            us[e.key.split("(")[0].split("::")[-1]] = dict(count=e.count, avg_us=e.device_time_total / max(e.count, 1))
    return us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_constrain.py needs the GPU")
    name, limit = card()
    cfg = synth.get_config("qwen3", "q0.6")
    w = synth.make_weights("qwen3", cfg, 0)
    m = B200Model("qwen3", cfg, w, eos_ids=[], max_ctx=64 * (W_PROMPT + W_GEN + 64), max_prefill=2048)
    del w
    V = cfg["vocab_size"]
    fs = automata(V)
    ids_of = {k: m.fsm_create(*f) for k, f in fs.items()}
    modes = [None] + list(fs)
    fid = lambda md: None if md is None else ids_of[md]
    ids = synth.synth_text_ids(PROMPT, 151000, 7)
    for md in modes:
        single(m, ids, fid(md))
    best, outs = {}, {}
    for _ in range(args.reps):
        for md in modes:
            dt, out = single(m, ids, fid(md))
            best[md] = min(best.get(md, 1e30), dt)
            outs[md] = out
    srows = []
    base = best[None]
    for md in modes:
        r = dict(automaton=md or "unconstrained", ms_per_token=1e3 * best[md] / GEN, overhead_us_per_token=1e6 * (best[md] - base) / GEN,
                 overhead_pct=100 * (best[md] - base) / base)
        if md:
            r["hbm_bytes"] = hbm_bytes(fs[md])
            r["kernels"] = kernel_times(lambda: single(m, ids, fid(md)))
        srows.append(r)
        print(f"single {r['automaton']:14s} {r['ms_per_token']:7.3f} ms/token  overhead {r['overhead_us_per_token']:6.1f} us/token "
              f"({r['overhead_pct']:+.2f} %)", flush=True)
    same_ids = outs["all-allowed"] == outs[None]
    reqs = [dict(input_ids=synth.synth_text_ids(W_PROMPT, 151000, 500 + i), max_tokens=W_GEN) for i in range(64)]
    for md in modes:
        wide(m, reqs, fid(md))
    wbest = {}
    for _ in range(args.reps):
        for md in modes:
            wbest[md] = min(wbest.get(md, 1e30), wide(m, reqs, fid(md)))
    wrows = []
    base = wbest[None]
    for md in modes:
        r = dict(automaton=md or "unconstrained", ms_per_step=1e3 * wbest[md] / (W_GEN - 1), overhead_pct=100 * (wbest[md] - base) / base)
        if md:
            r["kernels"] = kernel_times(lambda: wide(m, reqs, fid(md)))
        wrows.append(r)
        print(f"wide x 64 {r['automaton']:14s} {r['ms_per_step']:7.3f} ms/step ({r['overhead_pct']:+.2f} %)", flush=True)
    for f in ids_of.values():
        m.fsm_destroy(f)
    m.close()
    res = dict(card=name, power_limit=limit, shape="q0.6", prompt=PROMPT, generated=GEN, reps=args.reps, all_allowed_same_ids=same_ids,
               single=srows, wide64=wrows)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
