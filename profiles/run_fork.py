"""Several choices of one request (OpenAI `n`): one batch_add_n (one prefill, the prompt's KV pages copied by kv_fork_kernel) against n
batch_add calls (n prefills) and, for text, one batch_add_many of n copies (packed prefills).  Synthetic seed-0 weights, synthetic ids.

  python profiles/run_fork.py [--reps R] [--out FILE.json] [--quick]

Workloads: the Qwen3-0.6B shape (`q0.6`) with prompts of 128, 512 and 2048 tokens, and the Qwen3-VL-2B shape (`vl2`) with one 448 x 448
image plus 128 text tokens; 32 generated tokens per choice; n = 4 and 8 in a narrow session, n = 16 and 64 in a wide session of 64 slots.
Requests alternate greedy (n = 4, 16) and sampled (n = 8, 64: temperature 0.8, top-k 50).  max_ctx holds n full copies.  Per workload,
after one warm-up of each path, the paths are timed alternately, R times each: a fresh session, the admission, a device synchronise; the
time is the time to all first tokens, the best of R is reported.  Each run then steps the session to the end: ids_equal says whether
batch_add_n gave every choice exactly the ids of n batch_add calls with the same seeds.  Then kv_fork_kernel alone through bench_kernel
("kv_fork:P:n", P = prompt pages) as achieved GB/s of algorithmic bytes (P read, (n - 1) P written) and its share of 3.35 TB/s.  The card's
name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from aha_b200 import B200Model, synth

GEN = 32
NS = [(4, 0), (8, 0), (16, 64), (64, 64)]          # (n, session width: 0 = narrow)
HBM_GBS = 3350.0


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown (nvidia-smi unavailable)"


def run(m, req, n, width, path):
    """-> (seconds to all first tokens, ids per choice at the end)"""
    m.batch_open_wide(width) if width else m.batch_open()
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if path == "fork":
            res = m.batch_add_n(n=n, **req)
        elif path == "add":
            res = [m.batch_add(**dict(req, seed=req["seed"] + i)) for i in range(n)]
        else:
            res = m.batch_add_many([dict(req, seed=req["seed"] + i) for i in range(n)])
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        out = {slot: [tok] for slot, tok, _ in res}
        running = {slot for slot, _, fin in res if not fin}
        while running:
            for slot, (tok, fin) in m.batch_step().items():
                out[slot].append(tok)
                if fin:
                    running.discard(slot)
        return dt, [out[slot] for slot, _, _ in res]
    finally:
        m.batch_close()


def workload(m, name, req, n, width, reps, text):
    paths = ["fork", "add"] + (["many"] if text else [])
    for p in paths:
        run(m, req, n, width, p)   # warm-up: module loads, workspace growth, step graphs
    best = {p: float("inf") for p in paths}
    ids_equal = True
    for _ in range(reps):
        got = {}
        for p in paths:
            dt, got[p] = run(m, req, n, width, p)
            best[p] = min(best[p], dt)
        ids_equal = ids_equal and got["fork"] == got["add"]
    r = dict(model=name, prompt_tokens=len(req["input_ids"]), n=n, session="wide" if width else "narrow",
             sampled=req.get("temperature", 0.0) > 0, ids_equal=ids_equal, **{f"{p}_ms": 1e3 * best[p] for p in paths})
    r["speedup_vs_add"] = best["add"] / best["fork"]
    if text:
        r["speedup_vs_many"] = best["many"] / best["fork"]
    print(f"{name:5s} S={r['prompt_tokens']:5d} n={n:2d} {r['session']:6s}: batch_add_n {r['fork_ms']:9.2f} ms   n x batch_add {r['add_ms']:9.2f} ms"
          + (f"   batch_add_many {r['many_ms']:9.2f} ms" if text else "") + f"   ids equal {ids_equal}", flush=True)
    return r


def fork_kernel(m, pages, n, iters=50):
    ms, nbytes = m.bench_kernel(f"kv_fork:{pages}:{n}", iters)
    gbs = nbytes / (ms * 1e-3) / 1e9
    r = dict(pages=pages, n=n, ms=ms, bytes=nbytes, gb_per_s=gbs, share_of_hbm=gbs / HBM_GBS)
    print(f"kv_fork P={pages:3d} n={n:2d}: {ms * 1e3:8.1f} us  {nbytes / 1e6:9.1f} MB  {gbs:7.0f} GB/s  ({100 * gbs / HBM_GBS:.0f} % of 3.35 TB/s)", flush=True)
    return r


def sampler(n):
    return dict(temperature=0.8, top_k=50) if n in (8, 64) else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="the 128-token text prompt and the image prompt only")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_fork.py needs the GPU")
    name, limit = card()
    rows, kern = [], []
    cfg = synth.get_config("qwen3", "q0.6")
    w = synth.make_weights("qwen3", cfg, 0)
    lens = [128] if args.quick else [128, 512, 2048]
    m = B200Model("qwen3", cfg, w, eos_ids=[], max_ctx=64 * (max(lens) + GEN), max_prefill=4096)
    del w
    for S in lens:
        ids = synth.synth_text_ids(S, cfg["vocab_size"], S)
        for n, width in NS:
            rows.append(workload(m, "q0.6", dict(input_ids=ids, max_tokens=GEN, seed=1, **sampler(n)), n, width, args.reps, True))
        for n, _ in NS:
            kern.append(dict(model="q0.6", **fork_kernel(m, (S + 31) // 32, n)))
    m.close()
    cfg = synth.get_config("qwen3vl", "vl2")
    w = synth.make_weights("qwen3vl", cfg, 0)
    m = B200Model("qwen3vl", cfg, w, eos_ids=[], max_ctx=64 * 512, max_prefill=4096, max_patches=4096)
    del w
    pv, grid = m.image_patchify(synth.synth_image(448, 448, 1))
    ids = synth.vl_prompt_ids(cfg, grid, 128)
    for n, width in NS:
        req = dict(input_ids=ids, data=[pv, grid, None, None, None], max_tokens=GEN, seed=1, **sampler(n))
        rows.append(workload(m, "vl2", req, n, width, args.reps, False))
    m.close()
    res = dict(card=name, power_limit=limit, reps=args.reps, generated=GEN, workloads=rows, kv_fork=kern)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
