"""What frequency / presence penalties and logit bias (AHA_GEN_LOGIT_RULES) cost.  Synthetic seed-0 weights at the Qwen3-0.6B shape
(H 1024, 28 layers, V 151936), CUDA graphs on.

  python profiles/run_penalties.py [--reps R] [--out FILE.json]

Variants: no rules; zero rules (both penalties 0, no bias: the request only moves to the device sampler); typical rules (frequency 0.5,
presence 0.5, 300 bias entries); heavy bias (every token but 8 biased by -100).  Single request: a 512-token prompt, 128 greedy tokens (no
stop ids), the variants alternated R times, best of R on a host clock around the whole call (it ends in a device synchronise); per token =
call time / 128.  Wide x 64 session: 64 requests of 128-token prompts, 64 tokens each, every request with the same rules (greedy), the 63
lockstep steps timed, alternated, best of R.  Kernel times: torch.profiler (CUDA activities) over one more single request and one more
wide session per variant, by kernel name (sample_kernel, sample_rows_kernel).  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch

from aha_b200 import B200Model, synth
from run_constrain import PROMPT, GEN, W_PROMPT, W_GEN, card, kernel_times


def variants(V):
    """name -> rules_create keywords"""
    rng = np.random.default_rng(0)
    typical = rng.choice(V, size=300, replace=False)
    keep = set(int(t) for t in rng.choice(V, size=8, replace=False))
    return {"zero": dict(),
            "typical": dict(frequency_penalty=0.5, presence_penalty=0.5,
                            logit_bias={int(t): float(v) for t, v in zip(typical, rng.uniform(-5, 5, typical.size))}),
            "heavy-bias": dict(logit_bias={t: -100.0 for t in range(V) if t not in keep})}


def single(m, ids, rules):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = m.generate(ids, max_tokens=GEN, rules=rules)[0]
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def wide(m, reqs, rules):
    m.batch_open_wide(64)
    try:
        m.batch_add_many([dict(r, rules=rules) for r in reqs])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(W_GEN - 1):
            m.batch_step()
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    finally:
        m.batch_close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_penalties.py needs the GPU")
    name, limit = card()
    cfg = synth.get_config("qwen3", "q0.6")
    w = synth.make_weights("qwen3", cfg, 0)
    m = B200Model("qwen3", cfg, w, eos_ids=[], max_ctx=64 * (W_PROMPT + W_GEN + 64), max_prefill=2048)
    del w
    V = cfg["vocab_size"]
    vs = variants(V)
    ids_of = {k: m.rules_create(**v) for k, v in vs.items()}
    modes = [None] + list(vs)
    rid = lambda md: None if md is None else ids_of[md]
    ids = synth.synth_text_ids(PROMPT, 151000, 7)
    for md in modes:
        single(m, ids, rid(md))
    best, outs = {}, {}
    for _ in range(args.reps):
        for md in modes:
            dt, out = single(m, ids, rid(md))
            best[md] = min(best.get(md, 1e30), dt)
            outs[md] = out
    srows = []
    base = best[None]
    for md in modes:
        r = dict(rules=md or "none", ms_per_token=1e3 * best[md] / GEN, overhead_us_per_token=1e6 * (best[md] - base) / GEN,
                 overhead_pct=100 * (best[md] - base) / base)
        if md:
            r["kernels"] = kernel_times(lambda: single(m, ids, rid(md)))
        srows.append(r)
        print(f"single {r['rules']:10s} {r['ms_per_token']:7.3f} ms/token  overhead {r['overhead_us_per_token']:6.1f} us/token "
              f"({r['overhead_pct']:+.2f} %)", flush=True)
    same_ids = outs["zero"] == outs[None]
    reqs = [dict(input_ids=synth.synth_text_ids(W_PROMPT, 151000, 500 + i), max_tokens=W_GEN) for i in range(64)]
    for md in modes:
        wide(m, reqs, rid(md))
    wbest = {}
    for _ in range(args.reps):
        for md in modes:
            wbest[md] = min(wbest.get(md, 1e30), wide(m, reqs, rid(md)))
    wrows = []
    base = wbest[None]
    for md in modes:
        r = dict(rules=md or "none", ms_per_step=1e3 * wbest[md] / (W_GEN - 1), overhead_pct=100 * (wbest[md] - base) / base)
        r["kernels"] = kernel_times(lambda: wide(m, reqs, rid(md)))
        wrows.append(r)
        print(f"wide x 64 {r['rules']:10s} {r['ms_per_step']:7.3f} ms/step ({r['overhead_pct']:+.2f} %)", flush=True)
    for i in ids_of.values():
        m.rules_destroy(i)
    m.close()
    res = dict(card=name, power_limit=limit, shape="q0.6", prompt=PROMPT, generated=GEN, reps=args.reps, zero_rules_same_ids=same_ids,
               single=srows, wide64=wrows)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
