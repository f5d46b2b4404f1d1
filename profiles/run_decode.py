"""Driver for timing experiments on the decode step: text stack only (VL2 or Q0.6 shape), synthetic KV (no ViT).

  python profiles/run_decode.py [steps]              one configuration from the environment (AHA_DECODE_IMPL, AHA_FUSED_DBG, ...)
  python profiles/run_decode.py [steps] --sweep SPEC one process, many configurations (weights generated once):
      SPEC = ';'-separated runs, each ','-separated key=value with keys impl, dbg, stages, ctx, tl (1 = print the phase
      timeline), st (1 = dump the per-stage trace of an AHA_STAGE_TRACE build to profile_out/stage_trace_<tag>.npy and print, per phase
      boundary, how long the CTA had no copy in flight and how long its producer was held back)
      e.g. --sweep "impl=0;impl=0,dbg=3;impl=3,tl=1"
      key inflight=N runs the spec on variants/inflight<N>.so, a build of the library with the producer's in-flight cap set to
      N KB (decode_fused.cuh), loaded side by side with the other builds in this process (same weights, so repeated specs
      alternate builds without process-to-process noise):
        nvcc <aha_b200/build.py NVCC_FLAGS> -DAHA_FUSED_INFLIGHT_KB=N -o variants/inflightN.so aha_b200/csrc/api.cu -ldl
      e.g. --sweep "inflight=48;inflight=64;impl=0;inflight=48;inflight=64;impl=0"
      key trace=1 does the same with an AHA_STAGE_TRACE build (what st=1 / sy=1 read); the keys combine
      (variants/inflight48_trace.so), and a variant that is missing is built first
      key lib=PATH runs the spec on the library at PATH the same way, e.g. a build of the parent commit against this tree's:
        --sweep "lib=/tmp/parent.so,tl=1;impl=0,tl=1;lib=/tmp/parent.so;impl=0"
AHA_SHAPE = vl2 (default) | q0.6; AHA_LIB = path of an alternative libaha_b200.so, loaded instead of the in-tree one."""
import os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from aha_b200 import B200Model, _lib, synth
DEFAULT_LIB = os.path.abspath(os.environ["AHA_LIB"]) if os.environ.get("AHA_LIB") else _lib.LIB_PATH


def torch_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


argv = [a for a in sys.argv[1:]]
sweep = None
if "--sweep" in argv:
    i = argv.index("--sweep")
    sweep = argv[i + 1]
    del argv[i:i + 2]
steps = int(argv[0]) if argv else 8
shape = os.environ.get("AHA_SHAPE", "vl2")
cfg = synth.get_config("qwen3", "q0.6")
if shape == "vl2":
    cfg.update(hidden_size=2048, intermediate_size=6144, rope_theta=5e6)   # Qwen3-VL-2B text stack shape (else: Qwen3-0.6B / ASR-0.6B)
w = synth.make_weights("qwen3", cfg, 0)
# "P1 bar" is empty where qkv goes to the attention as packets (every mode): the hand-off wait is the start of "P2 attn"
NAMES = ["P1 load_x", "P1 gemv", "P1 bar", "P2 -", "P2 attn", "P2 bar", "P3 load_x", "P3 gemv", "P3 bar", "P4 load_x", "P4 gemv", "P4 bar", "P5 load_x", "P5 gemv", "P5 bar"]


def timeline(m, ctx):
    m.decode_steps(5, ctx, 1)
    c = m.debug_read("fused_trace", 0, 4096); p = m.debug_read("fused_trace", 1, 4096)
    print("  consumer stamps", len(c), "producer stamps", len(p), "total us", c[-1] / 1e3, p[-1] / 1e3)
    d = np.diff(c)[: 15 * 28].reshape(28, 15)
    for n, v in zip(NAMES, d[2:].mean(0)):
        print(f"    consumer {n:10s} {v/1e3:7.2f} us")
    print("    consumer per layer", d[2:].sum(1).mean() / 1e3, "us; lm_head phase", (c[-1] - c[15 * 28]) / 1e3)
    dp = np.diff(p)[: 5 * 28].reshape(28, 5)
    for n, v in zip(["qkv", "attn", "o", "gate_up", "down"], dp[2:].mean(0)):
        print(f"    producer {n:8s} {v/1e3:7.2f} us")
    Lx = 10
    cb = c[1 + 15 * Lx: 1 + 15 * (Lx + 1)] / 1e3
    pb = p[1 + 5 * Lx: 1 + 5 * (Lx + 1)] / 1e3
    t0 = c[15 * Lx] / 1e3
    print(f"    layer {Lx} starts at {t0:.1f} us; consumer events (rel):", " ".join(f"{n.replace(' ', '')}@{v - t0:.1f}" for n, v in zip(NAMES, cb)))
    print(f"    producer finished issuing (rel): ", " ".join(f"{n}@{v - t0:.1f}" for n, v in zip(["qkv", "attn", "o", "gate_up", "down"], pb)))


VARIANT_KEYS = (("inflight", "-DAHA_FUSED_INFLIGHT_KB="),)


def variant_lib(conf):
    """variants/<name>.so for the build keys of a spec (None: none given), built from this tree when it is missing"""
    keys = [k for k, _ in VARIANT_KEYS if k in conf]
    if not keys and not int(conf.get("trace", 0)):
        return None
    name = "_".join(f"{k}{conf[k]}" for k in keys) + ("_trace" if int(conf.get("trace", 0)) else "")
    path = os.path.join(ROOT, "variants", name.strip("_") + ".so")
    if not os.path.exists(path):
        from aha_b200 import build
        os.makedirs(os.path.dirname(path), exist_ok=True)
        defs = [d + conf[k] for k, d in VARIANT_KEYS if k in conf] + (["-DAHA_STAGE_TRACE"] if int(conf.get("trace", 0)) else [])
        subprocess.run([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")] + build.NVCC_FLAGS + defs + ["-o", path] + build.SOURCES + ["-ldl"], check=True)
    return path


def rows_per_stage(K, N, grid):   # decode_fused.cuh
    r = max(1, min(8, 16384 // (2 * K)))
    if r > 1:
        r &= ~1
    while r > 2 and N // grid < r * 5:
        r >>= 1
    return r


def n_stages(j0, j1, R, ends=()):
    n, j = 0, j0
    while j < j1:
        end = min([e for e in ends if e > j] + [j1])
        j += min(R, end - j)
        n += 1
    return n


def layer_phases(cta, grid, ctx):
    """stages per phase [qkv, attn, o_proj, gate/up, down] of one layer of CTA `cta` (Producer's schedule in decode_fused.cuh)"""
    H, I, hd, nh, nkv = cfg["hidden_size"], cfg["intermediate_size"], 128, cfg["num_attention_heads"], cfg["num_key_value_heads"]
    nsplit, G, qkv_dim = max(1, min(32, grid // nkv)), nh // nkv, (nh + 2 * nkv) * hd
    rows = lambda N, unit: ((N // unit * cta) // grid * unit, (N // unit * (cta + 1)) // grid * unit)
    out = [0, 0]
    if cta < nkv * nsplit:
        n, split = (G + 2) * hd, cta % nsplit
        out[0] = n_stages(n * split // nsplit, n * (split + 1) // nsplit, rows_per_stage(H, qkv_dim, grid), (G * hd, (G + 1) * hd))
        nhp = (ctx + 1 + 15) // 16
        per = (nhp + nsplit - 1) // nsplit
        out[1] = max(0, min(nhp, split * per + per) - split * per)
    out.append(n_stages(*rows(H, 1), rows_per_stage(nh * hd, H, grid)))
    out.append(n_stages(*rows(2 * I, 2), rows_per_stage(H, 2 * I, grid)))
    out.append(n_stages(*rows(H, 1), rows_per_stage(I, H, grid)))
    return out


def overlap(a0, a1, iv):   # total length of the intervals iv (sorted, disjoint) inside [a0, a1)
    return sum(max(0.0, min(a1, e) - max(a0, b)) for b, e in iv)


def union(iv):
    out = []
    for b, e in sorted(iv):
        if out and b <= out[-1][1]:
            out[-1][1] = max(out[-1][1], e)
        else:
            out.append([b, e])
    return out


def stage_gaps(t, cta, grid, ctx, ns):
    """Per phase boundary of layers 2 .. L-2: the window from the CTA's last slot release of a phase to its first wait of the
    next, how much of it the CTA had no copy in flight, and how long the producer was held back in it (able to issue -- the
    previous stage issued and the slot free -- but not issuing: the in-flight cap, or the run-ahead gate of earlier builds).  A copy is in flight
    from its issue to its landing; the landing is stamped only when the owner warp was already waiting, so for the other
    copies it is taken as issue + the median issue-to-landing time of the waited-for ones (an estimate)."""
    ph = layer_phases(cta, grid, ctx)
    n = int((t[:, 0] > 0).sum())
    t = t[:n].astype(np.float64) / 1e3   # us
    per = sum(ph)
    waited = t[:, 2] - t[:, 1] > 0.1
    lat = np.median(t[waited, 2] - t[waited, 0]) if waited.any() else 0.0
    land = np.where(waited, t[:, 2], np.minimum(t[:, 2], t[:, 0] + lat))
    busy = union([[a, b] for a, b in zip(t[:, 0], land)])
    idle = union([[b1, a2] for (_, b1), (a2, _) in zip(busy[:-1], busy[1:]) if a2 > b1])
    hold = []
    for i in range(1, n):
        free = max(t[i - 1, 0], t[i - ns, 3] if i >= ns else 0.0)
        if t[i, 0] > free:
            hold.append([free, t[i, 0]])
    hold = union(hold)
    names = ["qkv>attn", "attn>o", "o>gate/up", "gate/up>down", "down>qkv"]
    acc = np.zeros((5, 3))
    layers = range(2, cfg["num_hidden_layers"] - 1)
    for l in layers:
        s0 = l * per
        b = np.cumsum([0] + ph) + s0
        for k in range(5):
            cur, nxt = (b[k], b[k + 1]), (b[k + 1], b[k + 2]) if k < 4 else (b[5], b[5] + ph[0])
            if cur[1] == cur[0] or nxt[1] == nxt[0]:
                continue
            w0, w1 = t[cur[0]:cur[1], 3].max(), t[nxt[0]:nxt[1], 1].min()
            acc[k] += [max(0.0, w1 - w0), overlap(w0, w1, idle), overlap(w0, w1, hold)]
    acc /= len(layers)
    lay = (t[(layers[-1] + 1) * per, 0] - t[layers[0] * per, 0]) / len(layers)
    tot_idle = overlap(t[layers[0] * per, 0], t[(layers[-1] + 1) * per, 0], idle) / len(layers)
    tot_hold = overlap(t[layers[0] * per, 0], t[(layers[-1] + 1) * per, 0], hold) / len(layers)
    print(f"  cta {cta} stages/layer {ph}; per layer {lay:.1f} us, no copy in flight {tot_idle:.1f} us, producer held {tot_hold:.1f} us; "
          f"median issue-to-landing {lat:.2f} us")
    for k in range(5):
        print(f"    boundary {names[k]:13s} window {acc[k, 0]:5.2f} us  no copy in flight {acc[k, 1]:5.2f} us  producer held {acc[k, 2]:5.2f} us")


def run(conf, models):
    impl = int(conf.get("impl", os.environ.get("AHA_DECODE_IMPL", "0")))
    ctx = int(conf.get("ctx", os.environ.get("AHA_CTX", "2554")))
    dbg = int(conf.get("dbg", os.environ.get("AHA_FUSED_DBG", "0")))
    if "stages" in conf:
        os.environ["AHA_FUSED_STAGES"] = str(conf["stages"])
    else:
        os.environ.pop("AHA_FUSED_STAGES", None)
    lib = variant_lib(conf) or DEFAULT_LIB
    lib = os.path.abspath(conf["lib"]) if "lib" in conf else lib
    lib_tag = os.path.basename(lib)
    if (lib, impl) not in models:
        _lib._lib, _lib.LIB_PATH = None, lib   # every model keeps the library it was created on
        m = B200Model("qwen3", cfg, w, max_ctx=4096, max_prefill=64, decode_impl=impl)
        m.forward_initial(synth.synth_text_ids(8, 1000, 1), 0, want_logits=False)
        models[(lib, impl)] = m
    m = models[(lib, impl)]
    os.environ["AHA_FUSED_DBG"] = str(dbg)
    # decode at offset ctx: KV pages below ctx hold whatever is in the pool (timing only)
    m.decode_steps(5, ctx, steps, timed=True)
    best = 1e9
    for _ in range(3):
        toks, ms = m.decode_steps(5, ctx, steps, timed=True)
        best = min(best, ms)
    print(f"lib={lib_tag} shape={shape} impl={impl} dbg={dbg} stages={conf.get('stages', '-')} ctx={ctx} steps={steps} ms/step={best/steps:.4f} tok/s={1e3*steps/best:.1f}", flush=True)
    if int(conf.get("tl", 0)) or (sweep is None and dbg & 4):
        os.environ["AHA_FUSED_DBG"] = str(dbg | 4)
        timeline(m, ctx)
    if int(conf.get("st", 0)):
        os.makedirs("profile_out", exist_ok=True)
        for cta in (0, 77, 147):
            os.environ["AHA_FUSED_DBG"] = str(dbg | 128 | (cta << 16))
            m.debug_read("fused_stage_trace", 0, 4 * 8192)   # clears the region
            m.decode_steps(5, ctx, 1)
            t = m.debug_read("fused_stage_trace", 0, 4 * 8192).reshape(8192, 4)
            tag = f"{shape}_{lib_tag[:-3]}_impl{impl}_dbg{dbg}_cta{cta}"
            np.save(f"profile_out/stage_trace_{tag}.npy", t)
            print(f"  saved profile_out/stage_trace_{tag}.npy ({int((t[:, 0] > 0).sum())} stages)")
            if cta < torch_sms() and (t[:, 0] > 0).any():
                stage_gaps(t, cta, torch_sms(), ctx, int(conf.get("stages", conf.get("ns", 11))))
    if int(conf.get("sy", 0)):   # sync anatomy (AHA_STAGE_TRACE build): barrier sub-steps and activation-load sub-steps of 3 CTAs
        os.makedirs("profile_out", exist_ok=True)
        for cta in (0, 77, 147):
            os.environ["AHA_FUSED_DBG"] = str(dbg | 1024 | (cta << 16))
            m.debug_read("fused_sync_trace", 0, 8192)
            m.decode_steps(5, ctx, 1)
            t = m.debug_read("fused_sync_trace", 0, 8192)
            tag = f"{shape}_{lib_tag[:-3]}_impl{impl}_dbg{dbg}_cta{cta}"
            np.save(f"profile_out/sync_trace_{tag}.npy", t)
            b = t[:4096].reshape(512, 8)[:112]
            l = t[4096:].reshape(1024, 4)[:112]
            d = np.diff(b[8:, :6], axis=1)
            print(f"  cta {cta} barrier anatomy (us, mean over barriers 8..111): bar.sync {d[:,0].mean()/1e3:.2f} red.release {d[:,1].mean()/1e3:.2f} poll {d[:,2].mean()/1e3:.2f} fence {d[:,3].mean()/1e3:.2f} bar.sync {d[:,4].mean()/1e3:.2f}; polls/barrier {b[8:,6].mean():.1f}")
            dl = np.diff(l[8:], axis=1)
            print(f"  cta {cta} load_x anatomy: loads+sumsq {dl[:,0].mean()/1e3:.2f} bar.sync {dl[:,1].mean()/1e3:.2f} scale+sts+bar {dl[:,2].mean()/1e3:.2f}")
    if dbg & 64:
        m.decode_steps(5, ctx, 1)
        arr = np.stack([m.debug_read("fused_cta_trace", i, 256) for i in range(torch_sms())])
        os.makedirs("profile_out", exist_ok=True)
        np.save("profile_out/cta_trace.npy", arr)
        print("saved profile_out/cta_trace.npy", arr.shape)
        # arrival skew at each grid barrier of layers 2.. (mode 0: 4 per layer; qkv reaches the attention as packets inside each
        # kv-head group): last CTA against the median and the first
        b = arr[:, 8:4 * 28]
        last, med, first = b.max(0), np.median(b, 0), b.min(0)
        for k, n in enumerate(["attn", "o", "gate_up", "down"]):
            print(f"    arrival skew after {n:8s} last-median {(last - med)[k::4].mean()/1e3:6.2f} us  last-first {(last - first)[k::4].mean()/1e3:6.2f} us")
    os.environ["AHA_FUSED_DBG"] = "0"


models = {}
if sweep is None:
    run({}, models)
else:
    for spec in sweep.split(";"):
        spec = spec.strip()
        if not spec:
            continue
        conf = dict(kv.split("=") for kv in spec.split(","))
        try:
            run(conf, models)
        except Exception as e:   # an experimental variant must not end the sweep
            print(f"shape={shape} {spec}: FAILED {type(e).__name__}: {e}", flush=True)
for m in models.values():
    m.close()
