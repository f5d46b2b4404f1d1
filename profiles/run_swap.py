"""Swap preemption of a batch session (B200Model.batch_suspend / batch_resume) on the Qwen3-0.6B shape (the `q0.6` preset, seed-0
synthetic weights, synthetic ids).

  python profiles/run_swap.py [--reps R] [--out FILE.json]

One wide session holds 8 neighbours (64-token prompts) and a target request whose prompt is 128 / 512 / 2048 / 8192 tokens.  Per context:
  admit      batch_add of the target's prompt: what recomputing its K/V would cost at least (and recompute would not be exact);
  suspend    batch_suspend of the target 16 steps after admission: the KV pages it has written to the pinned arena (one strided
             copy-engine copy per page, kv_swap.cuh);
  resume     batch_resume of it;
  ce_d2h / ce_h2d  the copy engine on the same byte count in one piece: torch copies of one device tensor to / from one pinned host tensor;
  step_before / step_after  a decode step of the 9 running requests before the first and after the last suspend / resume cycle.
Suspend and resume end in a stream synchronise, and are timed by the host clock around the call (best of R, alternating); the copy-engine
copies by the host clock around copy + synchronise.  GB/s = bytes / time (1 GB = 1e9 B).  The card's name and power limit are read in the
same run."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from aha_b200 import B200Model, synth

CONTEXTS = [128, 512, 2048, 8192]
NEIGHBOURS, NEIGHBOUR_PROMPT, STEPS = 8, 64, 8


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


def step_ms(m):
    t, _ = timed(lambda: [m.batch_step() for _ in range(STEPS)])
    return 1e3 * t / STEPS


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_swap.py needs the GPU")
    name, limit = card()
    cfg = synth.get_config("qwen3", "q0.6")
    w = synth.make_weights("qwen3", cfg, 0)
    V = cfg["vocab_size"]
    page_bytes = cfg["num_hidden_layers"] * 2 * cfg["num_key_value_heads"] * 32 * cfg["head_dim"] * 4
    budget = STEPS * (2 * args.reps + 4) + 8
    per_neighbour = -(-(NEIGHBOUR_PROMPT + budget) // 32) * 32
    max_ctx = -(-(max(CONTEXTS) + budget + NEIGHBOURS * per_neighbour) // 32) * 32
    m = B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"]], max_ctx=max_ctx, max_prefill=8192)
    del w
    m.batch_swap_space(max(CONTEXTS) + budget)
    rows = []
    for ctx in CONTEXTS:
        target = dict(input_ids=[int(t) for t in synth.synth_text_ids(ctx, V - 8, ctx)], max_tokens=budget)
        m.batch_open_wide(16)
        try:
            for i in range(NEIGHBOURS):
                m.batch_add([int(t) for t in synth.synth_text_ids(NEIGHBOUR_PROMPT, V - 8, 10 + i)], max_tokens=budget)
            slot, _, _ = m.batch_add(**target)                          # warm-up: the prefill shapes of this prompt
            m.batch_cancel(slot)
            admit, (slot, _, _) = timed(lambda: m.batch_add(**target))
            step_ms(m)                                                  # warm-up: the 9-request step graph
            before = step_ms(m)
            out0 = m.batch_swap_stats()["pages_out"]
            sus, res = [], []
            for _ in range(args.reps + 1):                              # the first cycle warms up
                t, sid = timed(lambda: m.batch_suspend(slot))
                sus.append(t)
                t, slot = timed(lambda: m.batch_resume(sid))
                res.append(t)
            after = step_ms(m)
            st = m.batch_swap_stats()
            pages = (st["pages_out"] - out0) // (args.reps + 1)       # the pages the target has written, every cycle
            nbytes = pages * page_bytes
        finally:
            m.batch_close()
        dev = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        d2h, h2d = [], []
        for _ in range(args.reps + 1):
            d2h.append(timed(lambda: host.copy_(dev, non_blocking=True))[0])
            h2d.append(timed(lambda: dev.copy_(host, non_blocking=True))[0])
        del dev, host
        best = lambda xs: min(xs[1:])
        r = dict(ctx=ctx, pages=pages, bytes=nbytes, admit_ms=1e3 * admit,
                 suspend_ms=1e3 * best(sus), suspend_gbps=nbytes / best(sus) / 1e9, resume_ms=1e3 * best(res), resume_gbps=nbytes / best(res) / 1e9,
                 ce_d2h_ms=1e3 * best(d2h), ce_d2h_gbps=nbytes / best(d2h) / 1e9, ce_h2d_ms=1e3 * best(h2d), ce_h2d_gbps=nbytes / best(h2d) / 1e9,
                 step_ms_before=before, step_ms_after=after, pages_out=st["pages_out"], pages_in=st["pages_in"])
        rows.append(r)
        print(f"ctx {ctx:5d} ({nbytes / 1e6:7.1f} MB): admit {r['admit_ms']:8.2f} ms | suspend {r['suspend_ms']:7.2f} ms {r['suspend_gbps']:5.1f} GB/s"
              f" | resume {r['resume_ms']:7.2f} ms {r['resume_gbps']:5.1f} GB/s | copy engine d2h {r['ce_d2h_ms']:7.2f} ms {r['ce_d2h_gbps']:5.1f} GB/s"
              f" h2d {r['ce_h2d_ms']:7.2f} ms {r['ce_h2d_gbps']:5.1f} GB/s | step {before:.3f} / {after:.3f} ms", flush=True)
    m.batch_swap_space(0)
    m.close()
    res = dict(card=name, power_limit=limit, preset="q0.6", reps=args.reps, neighbours=NEIGHBOURS, contexts=rows)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
