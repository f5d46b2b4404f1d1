"""What token log-probability records cost.  Synthetic seed-0 weights at the VL2 text-stack shape (Qwen3-0.6B config with H 2048, I 6144,
V 151936), as in run_wide.py.

  python profiles/run_logprobs.py [--reps R] [--out FILE.json]

Single request: a 512-token prompt, 128 greedy tokens (no stop ids), `generate` against `generate(logprobs=True)` with top_logprobs 0 and
20, alternated R times, best of R on a host clock around the whole call (it ends in a device synchronise).  The per-step figure is
(call time - the plain call's) / 128.  Wide x 64 session: 64 requests of 128-token prompts, 64 tokens each, the 63 lockstep steps timed
with no request asking, with every request asking top_logprobs 20, and the same with the 64 records copied out after every step
(through the C entry into one buffer), alternated, best of R.  Kernel times: torch.profiler (CUDA activities) over one more generate_logprobs call with top_logprobs 20, by kernel name
(logprob_partial_rows_kernel, logprob_final_rows_kernel).  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from aha_b200 import B200Model, synth
from aha_b200 import _lib as L

PROMPT, GEN = 512, 128
W_PROMPT, W_GEN = 128, 64


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown (nvidia-smi unavailable)"


def single(m, ids, mode):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if mode is None:
        out = m.generate(ids, max_tokens=GEN)[0]
    else:
        out = m.generate(ids, max_tokens=GEN, logprobs=True, top_logprobs=mode)[0]
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def wide(m, reqs, lp, read):
    """read: after every step the 64 records are copied out through the C entry into one buffer (what a server does; the Python
    dicts of batch_logprobs() would cost more host time than the step)"""
    m.batch_open_wide(64)
    recs = (L.Logprobs * 64)()
    try:
        m.batch_add_many([dict(r, logprobs=True, top_logprobs=20) if lp else r for r in reqs])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(W_GEN - 1):
            m.batch_step()
            if read:
                m._check(m._lib.aha_b200_batch_logprobs(m._h, recs, 64))
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    finally:
        m.batch_close()


def kernel_times(m, ids):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.generate(ids, max_tokens=GEN, logprobs=True, top_logprobs=20)
        torch.cuda.synchronize()
    us = {}
    for e in prof.key_averages():
        if "logprob_" in e.key:
            us[e.key.split("(")[0].split("::")[-1]] = dict(count=e.count, avg_us=e.device_time_total / max(e.count, 1))
    return us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_logprobs.py needs the GPU")
    name, limit = card()
    cfg = synth.get_config("qwen3", "q0.6")
    cfg.update(hidden_size=2048, intermediate_size=6144, rope_theta=5e6)
    w = synth.make_weights("qwen3", cfg, 0)
    m = B200Model("qwen3", cfg, w, eos_ids=[], max_ctx=64 * (W_PROMPT + W_GEN + 64), max_prefill=2048)
    del w
    ids = synth.synth_text_ids(PROMPT, 151000, 7)
    modes = [None, 0, 20]
    for md in modes:
        single(m, ids, md)
    best, outs = {}, {}
    for _ in range(args.reps):
        for md in modes:
            dt, out = single(m, ids, md)
            best[md] = min(best.get(md, 1e30), dt)
            outs[md] = out
    same_tokens = outs[0] == outs[None] and outs[20] == outs[None]
    base = best[None]
    srows = []
    for md in modes:
        r = dict(mode="generate" if md is None else f"generate_logprobs n={md}", call_ms=1e3 * best[md],
                 per_step_ms=1e3 * best[md] / GEN, overhead_per_step_us=1e6 * (best[md] - base) / GEN,
                 overhead_pct=100 * (best[md] - base) / base)
        srows.append(r)
        print(f"single {r['mode']:26s} {r['call_ms']:8.2f} ms/call  {r['per_step_ms']:6.3f} ms/token  overhead {r['overhead_per_step_us']:6.1f} us/step "
              f"({r['overhead_pct']:+.2f} %)", flush=True)
    kt = kernel_times(m, ids)
    print("kernels", kt, flush=True)
    reqs = [dict(input_ids=synth.synth_text_ids(W_PROMPT, 151000, 500 + i), max_tokens=W_GEN) for i in range(64)]
    series = [("no request asks", False, False), ("every request n=20", True, False), ("every request n=20, records read", True, True)]
    for _, lp, rd in series:
        wide(m, reqs, lp, rd)
    wbest = {}
    for _ in range(args.reps):
        for label, lp, rd in series:
            wbest[label] = min(wbest.get(label, 1e30), wide(m, reqs, lp, rd))
    wrows = []
    base = wbest[series[0][0]]
    for label, _, _ in series:
        step = wbest[label] / (W_GEN - 1)
        r = dict(series=label, ms_per_step=1e3 * step, overhead_pct=100 * (wbest[label] - base) / base)
        wrows.append(r)
        print(f"wide x 64 {label:32s} {r['ms_per_step']:7.3f} ms/step ({r['overhead_pct']:+.2f} %)", flush=True)
    m.close()
    res = dict(card=name, power_limit=limit, shape="vl2", prompt=PROMPT, generated=GEN, reps=args.reps, same_tokens=same_tokens,
               single=srows, kernels=kt, wide64=wrows)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
