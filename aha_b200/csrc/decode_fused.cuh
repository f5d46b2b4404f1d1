// decode_fused.cuh -- the whole per-token decode step as ONE persistent, warp-specialised kernel.
//
// Why: at batch 1 the step is pure HBM streaming (3.4 GB of fp16 weights + the KV cache per token for
// Qwen3-VL-2B, ~1 FLOP/byte) cut into ~140 dependent pieces of 8-50 MB; as separate launches every piece pays
// launch + pipeline ramp and the memory system idles between them.  Here one CTA per SM stays resident for
// the whole step:
//   * the last warp (one elected lane) is the PRODUCER: it walks this CTA's static schedule of transfers for all
//     layers -- weight row slabs and paged-KV half pages -- and issues TMA bulk copies
//     (cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes, SASS UBLKCP, L2 evict-first policy) into
//     a ring of 16 KB shared-memory stages guarded by full/empty mbarriers.  It never waits for activations, so
//     weights for the next phase keep streaming while the consumers sit in a grid barrier -- but only up to a run-ahead
//     budget past the end of the consumers' current phase (kFusedAheadBytes), so that the traffic of a phase end
//     (barrier, activation loads) does not queue behind a full ring of next-phase copies from every SM;
//   * the other 11 warps are CONSUMERS: per phase they stage the activation vector in shared memory (RMSNorm
//     fused), and each warp consumes the ring slots it owns: a whole stage of weight rows is reduced by one warp
//     with fp32 dot products (fp16 weights converted exactly) and the fused epilogue (residual add from the rows
//     of the residual stream the CTA keeps on chip, SwiGLU, argmax) is applied by its lanes; attention is split-KV
//     with per-warp online softmax over the half pages the warp owns, q/k RMSNorm + RoPE + KV append fused in, and
//     the merge of the splits folded into the o_proj input load;
//   * some phase outputs travel through L2 as TAGGED PACKETS {value, tag}: the producer of a value stores 8 bytes --
//     single-copy atomic, so the tag validates the value -- and the consumer of a vector polls the packets it needs until
//     their tags carry this step's layer tag.  No fence, no counter, no separate load after a barrier: one store -> one
//     (re)load per dependency instead of the four dependent L2 round trips of store-ack / release / poll / load that a grid
//     barrier costs (measured: red.release 1.0 us + poll 0.7 us + fence.acq_rel 0.4 us + activation load 1.1 us per phase
//     boundary; profiles/README.md).
// The qkv -> attention exchange is packets in both modes of the kernel, but only inside each kv-head group: the nsplit CTAs
// that compute a group's q / k / v rows (qkv_slab) are the ones that run its attention, so that boundary costs one L2 round
// trip to data that is already there instead of a grid barrier + reload.  The other four boundaries per layer depend on the
// template flag PACKET_RESID:
//   * false (the default on one GPU, and decode_impl = 3): grid barriers (one counter in L2, release/acquire); the residual
//     stream lives in global memory, each CTA keeping on chip the rows it updates;
//   * true (the default under tensor parallelism, and decode_impl = 4 on one GPU): every CTA keeps the whole residual
//     stream in shared memory, and its two updates per layer -- the o_proj and down partial sums -- travel as packets.
//     Under tensor parallelism they are stored straight into every peer GPU's packet buffer over NVLink (8-byte stores are
//     atomic there too) and summed in rank order by the reader -- a one-shot all-reduce with no collective call and no
//     cross-GPU barrier.  The boundaries after the attention and after gate/up stay grid barriers: as packets their
//     exchanges are large or need an extra hop (measured slower).
// Phases per layer: [rmsnorm+qkv] -> [attention] -> [o_proj+residual] -> [rmsnorm+gate/up+SwiGLU] ->
// [down+residual]; then [final norm + lm_head + argmax] and the on-device token feedback.
//
// Reference semantics are those of Qwen3DecoderLayer::forward / QKNormAttention::forward / GateUpDownMLP
// (src/models/qwen3/model.rs:71-87, src/models/common/modules.rs:81-87,530-579,757-813)
// with seq_len = 1; arithmetic is fp32 throughout, identical to the per-op kernels in gemv.cuh/attention.cuh.
#pragma once
#include <cooperative_groups.h>

#include "attention.cuh"
#include "common.cuh"
#include "kernels_common.cuh"

namespace aha {

constexpr int kFusedStages = 11;                         // ring slots (all in use by default: one per consumer warp)
constexpr int kFusedStageBytes = 16384;
constexpr int kFusedConsumers = 11;                      // consumer warps (+1 producer = 12 warps: register allocation granularity)
constexpr int kFusedThreads = (kFusedConsumers + 1) * 32;
constexpr int kFusedMaxRows = 8;                         // weight rows per stage (<= 16 KB)
constexpr int kFusedMaxK = 8192;                         // activation vector staged in shared memory (32 KB)
constexpr int kHalfPage = 16;                            // tokens per attention stage (K 8 KB + V 8 KB)
constexpr int kFusedTraceWords = 2 * 4096 + 256 * 256;     // timing traces: CTA 0 consumer/producer stamps + [cta][256] barrier arrivals
constexpr int kFusedMaxOwnRows = 64;                     // residual-stream rows owned by one CTA (H / grid, rounded up)
constexpr int kFusedPartialStride = 128 + 4;             // floats per (head, split) attention partial: acc[128], m, l, pad (16-byte rows)
constexpr int kFusedMergeChunk = 20;                     // splits merged per pass when the o_proj input is assembled
constexpr int kFusedMaxPages = 1024;                     // page-table entries staged in shared memory as uint16 (32K tokens; physical page ids < 65536)
constexpr int kFusedMaxH = 4096;                         // residual stream kept per CTA in shared memory (PACKET_RESID)
constexpr int kFusedMaxTp = 8;                           // tensor-parallel ranks on one NVSwitch domain
// Run-ahead budget of the producer: stages of a phase the consumers have not entered yet may be issued only while they end at
// most this many bytes past the end of the consumers' current phase (stages of the current phase are never held back).  Without
// it every CTA keeps a full ring (176 KB) of the next phases' copies queued in the memory system while it sits in a phase end,
// and the phase end's own traffic -- the barrier arrival and poll, the activation loads -- waits behind them.  96 KB is the
// fastest of 0 / 16 / 32 / 48 / 64 / 96 / 128 / 176 KB on an H100 SXM (700 W) at the Qwen3-VL-2B decode shape (DESIGN §4.1):
// less starves the next phase's first stages, more brings the queueing back.  -DAHA_FUSED_AHEAD_KB=N builds the sweep.
#ifndef AHA_FUSED_AHEAD_KB
#define AHA_FUSED_AHEAD_KB 96
#endif
constexpr uint32_t kFusedAheadBytes = AHA_FUSED_AHEAD_KB * 1024u;
constexpr int kFusedGateWord = 28;                       // the gate's word in the `red` scratch ([0, 11) sums / argmax values, [16, 27) argmax indices, [31] last-CTA flag)

struct __align__(8) LLPk { float v; uint32_t tag; };     // one tagged packet: 8-byte stores / loads are single-copy atomic
struct LLPeerTab {                                       // device-resident table of the symmetric blocks of every tensor-parallel rank
    LLPk* xp[2][kFusedMaxTp];                            // [o_proj | down][destination rank] -> that rank's [tp_world][H] block of partial sums
    LLPk* cand[kFusedMaxTp];                             // [destination rank] -> that rank's [tp_world][2] argmax candidates (value, index)
    uint32_t* flag_xp[2][kFusedMaxTp];                   // [o_proj | down][destination rank] -> that rank's [tp_world][256] "data is out" flags
};

struct FusedLayer {
    const __half *qkv, *o, *gu, *down;
    const float *qkv_b, *o_b;
    const float *ln1, *ln2, *qn, *kn;
};

struct FusedArgs {
    const FusedLayer* layers;   // device array [L]
    int L, H, I, nh, nkv, hd, V, qkv_dim;
    float eps, scaling;
    const __half* embed;
    const __half* lm_head;
    const float* final_norm;
    const float* inv_freq;
    DecodeState* st;
    float* x;          // [H]   residual stream
    float* h1;         // [I]
    float* logits;     // [V]
    float* partial;    // [nh][nsplit][kFusedPartialStride]
    unsigned* sync;    // [2] grid-barrier counter, final ticket   (zeroed by the host before launch)
    float* pmax; int* pidx;  // [grid] per-CTA argmax candidates
    uint32_t* argmax_out;
    uint32_t* history; int hist_cap;
    float* kv_pool; size_t layer_stride, page_stride;
    const int* page_table;
    int nsplit;
    int stages;        // ring slots in use (<= kFusedStages)
    int dbg;           // timing experiments only: bit0 = skip grid barriers, bit1 = skip the GEMV math, bit2 = timestamps, bit3 = old full-fence grid barrier, bit6 = per-CTA barrier arrival stamps, bit4 / bit5 = drop the L2 evict-first hint on weight / KV copies, bit7 = per-stage trace of CTA (dbg >> 16) & 0xff (AHA_STAGE_TRACE builds), bit8 = skip the activation / partial loads (streaming-rate experiments; results are garbage), bit9 = sync only (no weight stream, no math), bit10 = sync anatomy stamps of the traced CTA (AHA_STAGE_TRACE builds)
    unsigned long long* trace;  // [2][4096] globaltimer stamps of CTA 0 (consumer thread 0 / producer), dbg bit2
    // ---- packet buffers (device memory, zero-initialised once; tags make every step's data self-validating).  ll_qkv, ll_tag and
    // ll_abort serve both modes (the qkv -> attention hand-off is always packets); the rest only PACKET_RESID.
    LLPk* ll_qkv;      // [qkv_dim]
    // Per-peer pointers live in a DEVICE table, not in this struct: indexing a kernel-parameter array with a runtime value makes the
    // compiler copy the whole parameter block to local memory, and then every `a.field` of the hot loops is a local load (measured:
    // all phases of the packet modes 1.5-4 us slower until this was moved out).
    const struct LLPeerTab* ll_peers;
    LLPk* ll_xp_local[2];          // this rank's own [tp_world][H] blocks of o_proj | down partial sums
    LLPk* ll_cand_local;           // this rank's own [tp_world][2] argmax candidates
    // "data is out" flags, one word per producing CTA and vector kind: written (relaxed, after the CTA's packets) by thread 0,
    // polled by ONE warp of a consumer that found packets missing -- the other 320 threads of every waiting CTA stay off the
    // memory system (every thread polling its own packets slows the weight stream of the CTAs still working: measured).
    uint32_t* ll_flag_xp_local[2]; // this rank's own [tp_world][256] flags of the o_proj | down partial sums
    uint32_t ll_tag;   // tag of layer 0 of this launch; layer l uses ll_tag + l, the final phase ll_tag + L (never 0, never reused)
    int tp_rank, tp_world;
    int v0, V_l;       // vocabulary shard [v0, v0 + V_l) of the lm_head this rank multiplies (tp_world == 1: the whole of it)
    int* ll_abort;     // set by any thread whose wait timed out (a peer died): every later wait returns at once
};

// ------------------------------------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {}
}
// TMA bulk copy global -> shared, completion signalled on an mbarrier (bytes % 16 == 0, 16-byte aligned).
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
#define AHA_STAMP(a, who, idx) do { if (((a).dbg & 4) && blockIdx.x == 0 && (idx) < 4096) (a).trace[(who) * 4096 + (idx)++] = gtime(); } while (0)
// Per-stage trace (compiled only with -DAHA_STAGE_TRACE, a profiling build: variants/trace.so): for ring stage i of the
// traced CTA, word 4i+0 = producer acquired the slot and issued the copy, 4i+1 = the owner warp started waiting for it,
// 4i+2 = the data had landed, 4i+3 = the warp released the slot.  Lives in the [cta][256] arrival region of the trace buffer.
#ifdef AHA_STAGE_TRACE
#define AHA_STAGE_STAMP(tr, i, k) do { if ((tr) && (i) < 8192u) (tr)[(size_t)(i) * 4 + (k)] = gtime(); } while (0)
// sync anatomy (dbg bit10, traced CTA, thread 0): 8 stamps per grid barrier at trace[8192 + 32768 + 8 * seq + k] and 4 per
// activation load at trace[8192 + 32768 + 2048 + 4 * n + k]
#define AHA_SYNC_STAMP(tr, idx, k, per) do { if ((tr) && (idx) < 400u) (tr)[(size_t)(idx) * (per) + (k)] = gtime(); } while (0)
#else
#define AHA_STAGE_STAMP(tr, i, k) do { } while (0)
#define AHA_SYNC_STAMP(tr, idx, k, per) do { } while (0)
#endif
// Same copy with an L2 evict-first policy: weights are read exactly once per step, so they should not displace the
// activations / partials / barrier words that every CTA re-reads from L2.
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void tma_bulk_g2s_hint(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar, uint64_t policy) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
                 : "memory");
}
__device__ __forceinline__ void consumer_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kFusedConsumers * 32) : "memory"); }
__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// ---- tagged packets.  Stores and loads are relaxed (strong) accesses, so polling them is race-free without fences; the
// .sys forms are used for buffers that a peer GPU writes or reads over NVLink.
template <bool SYS>
__device__ __forceinline__ void ll_store(LLPk* p, float v, uint32_t tag) {
    if (SYS) asm volatile("st.relaxed.sys.global.v2.b32 [%0], {%1, %2};" ::"l"(p), "r"(__float_as_uint(v)), "r"(tag) : "memory");
    else asm volatile("st.relaxed.gpu.global.v2.b32 [%0], {%1, %2};" ::"l"(p), "r"(__float_as_uint(v)), "r"(tag) : "memory");
}
template <bool SYS>
__device__ __forceinline__ uint4 ll_load2(const LLPk* p) {   // two packets (16-byte aligned): {v0, tag0, v1, tag1}
    uint4 r;
    if (SYS) asm volatile("ld.relaxed.sys.global.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    else asm volatile("ld.relaxed.gpu.global.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    return r;
}
template <bool SYS>
__device__ __forceinline__ uint2 ll_load1(const LLPk* p) {
    uint2 r;
    if (SYS) asm volatile("ld.relaxed.sys.global.v2.b32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p) : "memory");
    else asm volatile("ld.relaxed.gpu.global.v2.b32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p) : "memory");
    return r;
}
// Bounded wait: a missing packet means a peer CTA / GPU died.  After ~2 s of polling the waiter raises the abort flag
// and every wait in the grid (and, through the host, the request) ends instead of hanging the GPU.
struct LLWait {
    int* abort_flag;
    long long t0 = 0;
    unsigned n = 0;
    bool dead = false;
    __device__ __forceinline__ bool giveup() {
        if ((++n & 1023u) != 0) return dead;
        if (t0 == 0) t0 = clock64();
        if (*reinterpret_cast<volatile int*>(abort_flag) != 0) dead = true;
        else if (clock64() - t0 > 4000000000ll) { *reinterpret_cast<volatile int*>(abort_flag) = 1; dead = true; }
        return dead;
    }
};
// The polling loops live out of line: the fast path (packet already there) is a load and four compares in the caller, and
// the rare slow path must not cost the callers any registers.
template <bool SYS>
__device__ __noinline__ float ll_spin1(const LLPk* p, uint32_t tag, int* abort_flag) {
    LLWait w{abort_flag};
    uint2 r;
    do { r = ll_load1<SYS>(p); } while (r.y != tag && !w.giveup());
    return __uint_as_float(r.x);
}
template <bool SYS>
__device__ __forceinline__ float ll_wait1(const LLPk* p, uint32_t tag, int* abort_flag) {
    const uint2 r = ll_load1<SYS>(p);
    return r.y == tag ? __uint_as_float(r.x) : ll_spin1<SYS>(p, tag, abort_flag);
}
// four consecutive packets (32-byte aligned) -> float4
template <bool SYS>
__device__ __noinline__ float4 ll_spin4(const LLPk* p, uint32_t tag, int* abort_flag) {
    LLWait w{abort_flag};
    uint4 a, b;
    bool ok;
    do {
        a = ll_load2<SYS>(p); b = ll_load2<SYS>(p + 2);
        ok = a.y == tag && a.w == tag && b.y == tag && b.w == tag;
    } while (!ok && !w.giveup());
    return make_float4(__uint_as_float(a.x), __uint_as_float(a.z), __uint_as_float(b.x), __uint_as_float(b.z));
}
template <bool SYS>
__device__ __forceinline__ float4 ll_wait4(const LLPk* p, uint32_t tag, int* abort_flag) {
    const uint4 a = ll_load2<SYS>(p), b = ll_load2<SYS>(p + 2);
    if (a.y == tag && a.w == tag && b.y == tag && b.w == tag)
        return make_float4(__uint_as_float(a.x), __uint_as_float(a.z), __uint_as_float(b.x), __uint_as_float(b.z));
    return ll_spin4<SYS>(p, tag, abort_flag);
}

template <bool SYS>
__device__ __forceinline__ void ll_flag_store(uint32_t* p, uint32_t tag) {
    if (SYS) asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(tag) : "memory");
    else asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(tag) : "memory");
}
template <bool SYS>
__device__ __forceinline__ uint32_t ll_flag_load(const uint32_t* p) {
    uint32_t v;
    if (SYS) asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    else asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// AND of a predicate over the consumer threads of the CTA (named barrier 1)
__device__ __forceinline__ bool consumer_all(bool ok) {
    uint32_t r;
    asm volatile(
        "{\n\t.reg .pred p, q;\n\t"
        "setp.ne.u32 p, %1, 0;\n\t"
        "bar.red.and.pred q, 1, %2, p;\n\t"
        "selp.u32 %0, 1, 0, q;\n\t}"
        : "=r"(r)
        : "r"((uint32_t)ok), "n"(kFusedConsumers * 32)
        : "memory");
    return r != 0;
}
// Warp 0 polls `rows` x `n` flags (row stride `stride`) until each carries `tag`; everybody meets at the CTA barrier after.
// Every caller passes one row; the two arguments stay because dropping them moves the register allocation around the call
// sites (CUDA 12.9: 40 more bytes of spill stores in decode_step_fused_kernel<2, true>).
template <bool SYS>
__device__ __noinline__ void ll_wait_flags(const uint32_t* f, int rows, int stride, int n, uint32_t tag, int* abort_flag) {
    if (threadIdx.x < 32) {
        LLWait w{abort_flag};
        for (int i = threadIdx.x; i < rows * n; i += 32) {
            const uint32_t* q = f + (size_t)(i / n) * stride + (i % n);
            while (ll_flag_load<SYS>(q) != tag && !w.giveup()) __nanosleep(40);
        }
    }
    consumer_bar_sync();
}

// Lighter synchronisation primitives than __threadfence() (= MEMBAR.SC.GPU + CCTL.IVALL per call): a release
// reduction / acq_rel atomic issued by ONE thread after a CTA barrier publishes the whole CTA's writes (release is
// cumulative over the bar.sync), and a relaxed poll + fence.acq_rel is the matching acquire.  Cross-CTA data is always
// read with ld.global.cg, so no L1 line can be stale.
__device__ __forceinline__ void red_release_add(unsigned* p, unsigned v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned atom_acq_rel_add(unsigned* p, unsigned v) {
    unsigned old;
    asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
    return old;
}
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// Grid barrier joined by the consumer threads only: one arrival counter in L2 (zeroed by the host before every
// launch), polled by consumer thread 0 with relaxed loads; activations are always read with ld.global.cg.
__device__ __forceinline__ void grid_barrier(unsigned* counter, unsigned& seq, int dbg = 0, unsigned long long* trace = nullptr, unsigned long long* sy = nullptr) {
    if (dbg & 1) { consumer_bar_sync(); return; }
    if (threadIdx.x == 0) AHA_SYNC_STAMP(sy, seq, 0, 8);
    consumer_bar_sync();                       // every consumer thread of this CTA has issued its writes
    if (threadIdx.x == 0) {
        AHA_SYNC_STAMP(sy, seq, 1, 8);
        if ((dbg & 64) && seq < 255) trace[8192 + blockIdx.x * 256 + seq] = gtime();   // per-CTA arrival times (skew analysis)
        if (dbg & 8) {                         // A/B: the old full-fence barrier
            __threadfence();
            atomicAdd(counter, 1u);
            const unsigned target = (seq + 1u) * gridDim.x;
            while (ld_relaxed_u32(counter) < target) {}
            __threadfence();
        } else {
            red_release_add(counter, 1u);      // publish the CTA's writes at gpu scope (cumulative through the bar.sync)
            AHA_SYNC_STAMP(sy, seq, 2, 8);
            const unsigned target = (seq + 1u) * gridDim.x;
            unsigned polls = 0;
#ifndef AHA_BARRIER_FENCE
            // acquire loads in the poll (release by the arriving CTAs' reductions -> acquire here -> bar.sync to the other threads)
            // instead of a relaxed poll + fence.acq_rel: the fence alone was 0.4 us of every barrier in the anatomy trace; measured
            // 793.8 vs 768.6 tok/s on the Qwen3-VL-2B stack (profiles/README.md)
            while (ld_acquire_u32(counter) < target) { ++polls; }
            AHA_SYNC_STAMP(sy, seq, 3, 8);
#else
            while (ld_relaxed_u32(counter) < target) { ++polls; }
            AHA_SYNC_STAMP(sy, seq, 3, 8);
            fence_acq_rel_gpu();
#endif
            AHA_SYNC_STAMP(sy, seq, 4, 8);
#ifdef AHA_STAGE_TRACE
            if (sy && seq < 400u) sy[(size_t)seq * 8 + 6] = polls;
#endif
        }
    }
    consumer_bar_sync();
    if (threadIdx.x == 0) AHA_SYNC_STAMP(sy, seq, 5, 8);
    seq += 1u;
}

// ------------------------------------------------------------------------------------------------ schedule
// Row slab of a [N,K] fp16 matrix owned by this CTA: contiguous rows [r0, r1); `unit` = 2 keeps SwiGLU pairs together.
__device__ __forceinline__ void cta_rows(int N, int unit, int& r0, int& r1) {
    const long long units = N / unit;
    r0 = (int)((units * blockIdx.x) / gridDim.x) * unit;
    r1 = (int)((units * (blockIdx.x + 1)) / gridDim.x) * unit;
}
// The rows of one GEMV phase this CTA owns, as the share [j0, j1) of a sequence of rows made of up to three segments of
// contiguous matrix rows (ends e0, e1; sequence position j sits at matrix row j + b[segment]).  The producer and the consumers
// both walk it with Slab::stage, so a stage never straddles two segments and both sides cut the same stages.
struct Slab {
    int j0, j1;
    int e0 = 0x7fffffff, e1 = 0x7fffffff;
    int b0 = 0, b1 = 0, b2 = 0;
    // the stage that starts at position j: its first matrix row and its row count (at most R)
    __device__ __forceinline__ int stage(int j, int R, int& nr) const {
        const int end = j < e0 ? e0 : (j < e1 ? e1 : 0x7fffffff);
        nr = min(R, min(j1, end) - j);
        return j + (j < e0 ? b0 : (j < e1 ? b1 : b2));
    }
};
__device__ __forceinline__ Slab cta_slab(int N, int unit) {
    Slab s;
    cta_rows(N, unit, s.j0, s.j1);
    return s;
}
// qkv rows by kv-head group: group g's sequence is the q rows of its heads gG .. gG+G-1, then the k rows and the v rows of kv
// head g, (G + 2) * hd rows shared evenly by the group's nsplit attention CTAs (attn_item), so that the CTA (g, split) waits only
// for the packets of its own group's CTAs before its attention.  CTAs past nkv * nsplit own no qkv rows.
__device__ __forceinline__ Slab qkv_slab(int nh, int nkv, int hd, int nsplit) {
    Slab s;
    s.j0 = s.j1 = 0;
    if ((int)blockIdx.x >= nkv * nsplit) return s;
    const int g = blockIdx.x / nsplit, split = blockIdx.x % nsplit, G = nh / nkv;
    const int n = (G + 2) * hd;
    s.j0 = (n * split) / nsplit;
    s.j1 = (n * (split + 1)) / nsplit;
    s.e0 = G * hd;
    s.e1 = (G + 1) * hd;
    s.b0 = g * G * hd;
    s.b1 = (nh + g) * hd - s.e0;
    s.b2 = (nh + nkv + g) * hd - s.e1;
    return s;
}
// Rows per ring stage.  Short phases (few rows per CTA) use smaller stages so that the slab spreads over more consumer
// warps -- the per-stage latency of one warp is on the critical path of every phase.
__host__ __device__ __forceinline__ int rows_per_stage(int K, int N, int grid) {
    int r = kFusedStageBytes / (2 * K);
    r = r > kFusedMaxRows ? kFusedMaxRows : (r < 1 ? 1 : r);
    if (r > 1) r &= ~1;            // even, so interleaved gate/up pairs never straddle a stage
    const int per_cta = N / grid;
    while (r > 2 && per_cta < r * 5) r >>= 1;
    return r;
}
// attention work item of this CTA: (kv head, [hp0, hp1) half pages); empty when the CTA has no item
__device__ __forceinline__ bool attn_item(const FusedArgs& a, int ctx, int& kvh, int& split, int& hp0, int& hp1) {
    const int items = a.nkv * a.nsplit;
    if ((int)blockIdx.x >= items) { kvh = 0; split = 0; hp0 = hp1 = 0; return false; }
    kvh = blockIdx.x / a.nsplit;
    split = blockIdx.x % a.nsplit;
    const int nhp = (ctx + kHalfPage - 1) / kHalfPage;
    const int per = (nhp + a.nsplit - 1) / a.nsplit;
    hp0 = split * per;
    hp1 = min(nhp, hp0 + per);
    if (hp1 < hp0) hp1 = hp0;
    return true;
}

struct Ring {
    uint8_t* buf;
    uint64_t* full;
    uint64_t* empty;
};

// ------------------------------------------------------------------------------------------------ producer
// The run-ahead gate: `gate` holds (schedule bytes up to the end of the consumers' current phase) + kFusedAheadBytes, `issued`
// counts the schedule bytes this producer has issued including the stage being acquired; the stage waits while it would end
// past the gate.  No deadlock: consumers enter a phase (and raise the gate) without waiting on any ring slot -- they need only
// the activations, which come from the other CTAs' consumers under the same rule -- and the stages of the phase they are in
// always end below the gate.  Wrapping differences: a step's schedule is far below 2 GB per CTA.
__device__ __forceinline__ uint32_t ld_volatile_shared_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
    return v;
}
struct Producer {
    Ring ring;
    unsigned it = 0;
    unsigned ns = kFusedStages;
    bool use_hint = false, hint_kv = false;
    uint64_t policy = 0;
    unsigned long long* st_trace = nullptr;
    const uint32_t* gate = nullptr;
    uint32_t issued = 0, limit = 0;   // limit: the last value read from the gate (it only grows)
    __device__ __forceinline__ void acquire(int& slot, uint32_t bytes) {
        issued += bytes;
        if ((int)(limit - issued) < 0)
            while ((int)((limit = ld_volatile_shared_u32(gate)) - issued) < 0) __nanosleep(32);
        slot = it % ns;
        mbar_wait(&ring.empty[slot], ((it / ns) & 1u) ^ 1u);
        AHA_STAGE_STAMP(st_trace, it, 0);
    }
    __device__ void rows(const __half* W, int N, int K, const Slab& s) {
        const int R = rows_per_stage(K, N, gridDim.x);
        for (int j = s.j0, nr; j < s.j1; j += nr) {
            const int r = s.stage(j, R, nr);
            const uint32_t bytes = (uint32_t)nr * K * 2u;
            int slot;
            acquire(slot, bytes);
            mbar_expect_tx(&ring.full[slot], bytes);
            if (use_hint) tma_bulk_g2s_hint(ring.buf + (size_t)slot * kFusedStageBytes, W + (size_t)r * K, bytes, &ring.full[slot], policy);
            else tma_bulk_g2s(ring.buf + (size_t)slot * kFusedStageBytes, W + (size_t)r * K, bytes, &ring.full[slot]);
            ++it;
        }
    }
    const uint16_t* pages = nullptr;   // page table staged in shared memory
    __device__ void attn(const FusedArgs& a, int layer, int ctx) {
        int kvh, split, hp0, hp1;
        if (!attn_item(a, ctx, kvh, split, hp0, hp1)) return;
        const float* kbase = a.kv_pool + (size_t)layer * a.layer_stride;
        const size_t vofs = (size_t)a.nkv * kPage * a.hd;
        const uint32_t half_bytes = kHalfPage * a.hd * 4u;  // 8 KB for hd = 128
        for (int hp = hp0; hp < hp1; ++hp) {
            int slot;
            acquire(slot, 2u * half_bytes);
            const int page = pages[(hp * kHalfPage) >> kPageShift];
            const size_t off = (size_t)page * a.page_stride + (size_t)kvh * kPage * a.hd + (size_t)((hp * kHalfPage) & (kPage - 1)) * a.hd;
            uint8_t* dst = ring.buf + (size_t)slot * kFusedStageBytes;
            mbar_expect_tx(&ring.full[slot], 2u * half_bytes);
            if (hint_kv) {
                tma_bulk_g2s_hint(dst, kbase + off, half_bytes, &ring.full[slot], policy);
                tma_bulk_g2s_hint(dst + half_bytes, kbase + vofs + off, half_bytes, &ring.full[slot], policy);
            } else {
                tma_bulk_g2s(dst, kbase + off, half_bytes, &ring.full[slot]);
                tma_bulk_g2s(dst + half_bytes, kbase + vofs + off, half_bytes, &ring.full[slot]);
            }
            ++it;
        }
    }
};

// ------------------------------------------------------------------------------------------------ consumer
// Ring slots are OWNED by consumer warps: slot s is only ever consumed by warp s % kFusedConsumers, so each warp sees the
// uses of its slots strictly in order (no cross-warp mbarrier phase hazards) and up to kFusedConsumers stages are processed
// concurrently.
// A GEMV stage (R rows x K fp16) is reduced entirely by its owner warp against the activation vector staged in
// shared memory; the epilogue is applied by the lanes of that warp -- no cross-warp partial sums.
enum FusedEpi { FE_QKV = 0, FE_RESID = 1, FE_SWIGLU = 2, FE_LOGITS = 3 };

struct Consumer {
    Ring ring;
    unsigned it = 0;    // global stage counter (same sequence as the producer's)
    float* xs;          // [K] activation vector (shared), also aliased by the attention scratch
    float* red;         // [32] scratch
    float* xown;        // [kFusedMaxOwnRows] this CTA's rows of the residual stream (never re-read from global memory; barrier mode)
    float* xres = nullptr;   // [H] PACKET_RESID: the whole residual stream, kept by every CTA (thread t always touches the same elements)
    int* ll_abort = nullptr;
    int warp, lane;

    unsigned ns = kFusedStages;
    unsigned long long* st_trace = nullptr;
    bool skip_loads = false;   // dbg bit8: timing experiments only
    bool sync_only = false;    // dbg bit9: no weight stream and no math, only the barriers and activation loads
    unsigned long long* sy_trace = nullptr;   // sync anatomy stamps (AHA_STAGE_TRACE builds, dbg bit10)
    unsigned n_loads = 0;
    // Called once the phase's activations are staged, before its first wait_full: the producer may now run
    // kFusedAheadBytes past the end of this phase.  A phase without stages leaves the gate where it is.  Only thread 0
    // writes the gate word (no register of the hot loops holds it).
    __device__ __forceinline__ void enter(uint32_t bytes) const {
        if (threadIdx.x == 0) reinterpret_cast<volatile uint32_t*>(red)[kFusedGateWord] += bytes;
    }
    __device__ __forceinline__ bool owns(unsigned i) const { return (int)((i % ns) % kFusedConsumers) == warp; }
    __device__ __forceinline__ const uint8_t* wait_full(unsigned i) {
        const int slot = i % ns;
        if (lane == 0) AHA_STAGE_STAMP(st_trace, i, 1);
        mbar_wait(&ring.full[slot], (i / ns) & 1u);
        if (lane == 0) AHA_STAGE_STAMP(st_trace, i, 2);
        return ring.buf + (size_t)slot * kFusedStageBytes;
    }
    __device__ __forceinline__ void release(unsigned i) {
        __syncwarp();
        if (lane == 0) { AHA_STAGE_STAMP(st_trace, i, 3); mbar_arrive(&ring.empty[i % ns]); }
    }

    // Shared-memory layout of the activation vector: element e = 8c + j sits at 4c + j (j < 4) or K/2 + 4c + (j - 4), so
    // the two float4 halves of chunk c are read by lane c at a 16-byte lane stride -- conflict-free LDS.128 (a plain
    // [K] layout puts the lanes 32 bytes apart and every x read pays a 2-way bank conflict).
    static __device__ __forceinline__ int xs_pos(int e, int K) { return ((e >> 2) & 1) * (K >> 1) + (e >> 3) * 4; }
    // Stage the activation vector of a GEMV in shared memory (all consumer threads), optional RMSNorm.
    // src is fp32 global written by other CTAs (ld.global.cg) or an fp16 embedding row.
    __device__ void load_x(int K, const float* src32, const __half* src16, const float* norm_w, float eps, bool capture = false) {
        const int tid = threadIdx.x;
        constexpr int kPer = (kFusedMaxK + kFusedConsumers * 32 * 4 - 1) / (kFusedConsumers * 32 * 4);   // float4 per thread
        float4 v[kPer], w[kPer];
        float ss = 0.f;
        if (tid == 0) AHA_SYNC_STAMP(sy_trace ? sy_trace + 4096 : nullptr, n_loads, 0, 4);
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
            const int e = (tid + j * kFusedConsumers * 32) * 4;
            v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            w[j] = v[j];
            if (e < K && !skip_loads) {
                if (norm_w) w[j] = *reinterpret_cast<const float4*>(norm_w + e);   // static data: in flight with x
                if (src16) {
                    const uint2 u = *reinterpret_cast<const uint2*>(src16 + e);
                    const float2 a = h2_to_f2(u.x), b = h2_to_f2(u.y);
                    v[j] = make_float4(a.x, a.y, b.x, b.y);
                } else {
                    v[j] = __ldcg(reinterpret_cast<const float4*>(src32 + e));
                }
            }
        }
        if (capture) {
#pragma unroll
            for (int j = 0; j < kPer; ++j) {
                const int e = (tid + j * kFusedConsumers * 32) * 4;
                if (e < K) *reinterpret_cast<float4*>(xres + e) = v[j];
            }
        }
        if (norm_w) {
#pragma unroll
            for (int j = 0; j < kPer; ++j) ss += v[j].x * v[j].x + v[j].y * v[j].y + v[j].z * v[j].z + v[j].w * v[j].w;
            ss = warp_sum(ss);
            if (lane == 0) red[warp] = ss;
            if (tid == 0) AHA_SYNC_STAMP(sy_trace ? sy_trace + 4096 : nullptr, n_loads, 1, 4);
            consumer_bar_sync();
            if (tid == 0) AHA_SYNC_STAMP(sy_trace ? sy_trace + 4096 : nullptr, n_loads, 2, 4);
            float tot = 0.f;
#pragma unroll
            for (int q = 0; q < kFusedConsumers; ++q) tot += red[q];
            const float inv = 1.0f / sqrtf(tot / (float)K + eps);
#pragma unroll
            for (int j = 0; j < kPer; ++j) { v[j].x *= inv * w[j].x; v[j].y *= inv * w[j].y; v[j].z *= inv * w[j].z; v[j].w *= inv * w[j].w; }
        }
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
            const int e = (tid + j * kFusedConsumers * 32) * 4;
            if (e < K) *reinterpret_cast<float4*>(xs + xs_pos(e, K)) = v[j];
        }
        consumer_bar_sync();
        if (tid == 0) AHA_SYNC_STAMP(sy_trace ? sy_trace + 4096 : nullptr, n_loads, 3, 4);
        ++n_loads;
    }

    // PACKET_RESID: x = residual + sum_r packets[r * vstride + e] is added into the residual stream this CTA keeps in shared
    // memory, and RMSNorm(x) is staged in xs.  The packets are polled until they carry `tag`; all loads of a vector are issued
    // before the first tag is looked at, and the common case (data already there) costs one L2 round trip.  Fixed rank order
    // r = 0, 1, ... -> every CTA of every GPU forms bit-identical sums.
    // flags / nflag: the "data is out" words of the CTAs that produce vector r (row r of `flags`, row stride 256).
    template <bool SYS>
    __device__ __forceinline__ void load_ll(int K, const LLPk* pk, int nvec, size_t vstride, uint32_t tag, const float* norm_w, float eps, const uint32_t* flags, int nflag) {
        constexpr int kChunk = kFusedConsumers * 32 * 4;   // elements one pass of the consumer threads covers
        if (K <= 2 * kChunk) load_ll_n<SYS, 2>(K, pk, nvec, vstride, tag, norm_w, eps, flags, nflag);
        else if (K <= 3 * kChunk) load_ll_n<SYS, 3>(K, pk, nvec, vstride, tag, norm_w, eps, flags, nflag);
        else load_ll_n<SYS, (kFusedMaxK + kChunk - 1) / kChunk>(K, pk, nvec, vstride, tag, norm_w, eps, flags, nflag);
    }
    template <bool SYS, int kPer>
    __device__ void load_ll_n(int K, const LLPk* pk, int nvec, size_t vstride, uint32_t tag, const float* norm_w, float eps, const uint32_t* flags, int nflag) {
        const int tid = threadIdx.x;
        float4 v[kPer], w[kPer];
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
            const int e = (tid + j * kFusedConsumers * 32) * 4;
            v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            w[j] = v[j];
            if (e < K) {
                w[j] = *reinterpret_cast<const float4*>(norm_w + e);
                v[j] = *reinterpret_cast<const float4*>(xres + e);
            }
        }
        for (int r = 0; r < nvec; ++r) {
            const LLPk* base = pk + (size_t)r * vstride;
            uint4 pa[kPer], pb[kPer];
#pragma unroll
            for (int j = 0; j < kPer; ++j) {
                const int e = (tid + j * kFusedConsumers * 32) * 4;
                if (e < K) { pa[j] = ll_load2<SYS>(base + e); pb[j] = ll_load2<SYS>(base + e + 2); }
            }
            bool ok = true;
#pragma unroll
            for (int j = 0; j < kPer; ++j) {
                const int e = (tid + j * kFusedConsumers * 32) * 4;
                if (e < K) ok = ok && pa[j].y == tag && pa[j].w == tag && pb[j].y == tag && pb[j].w == tag;
            }
            // fast path: every packet of every thread was there (one L2 round trip).  Otherwise ONE warp waits for the producers'
            // flags and the stale packets are read again (a flag can overtake its packets: the re-read still checks the tags).
            const bool all_ok = consumer_all(ok);
            if (!all_ok) ll_wait_flags<SYS>(flags + (size_t)r * 256, 1, 0, nflag, tag, ll_abort);
#pragma unroll
            for (int j = 0; j < kPer; ++j) {
                const int e = (tid + j * kFusedConsumers * 32) * 4;
                if (e < K) {
                    float4 t;
                    if (pa[j].y == tag && pa[j].w == tag && pb[j].y == tag && pb[j].w == tag)
                        t = make_float4(__uint_as_float(pa[j].x), __uint_as_float(pa[j].z), __uint_as_float(pb[j].x), __uint_as_float(pb[j].z));
                    else t = ll_spin4<SYS>(base + e, tag, ll_abort);
                    v[j].x += t.x; v[j].y += t.y; v[j].z += t.z; v[j].w += t.w;
                }
            }
        }
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
            const int e = (tid + j * kFusedConsumers * 32) * 4;
            if (e < K) *reinterpret_cast<float4*>(xres + e) = v[j];
        }
        float ss = 0.f;
#pragma unroll
        for (int j = 0; j < kPer; ++j) ss += v[j].x * v[j].x + v[j].y * v[j].y + v[j].z * v[j].z + v[j].w * v[j].w;
        ss = warp_sum(ss);
        if (lane == 0) red[warp] = ss;
        consumer_bar_sync();
        float tot = 0.f;
#pragma unroll
        for (int q = 0; q < kFusedConsumers; ++q) tot += red[q];
        const float inv = 1.0f / sqrtf(tot / (float)K + eps);
#pragma unroll
        for (int j = 0; j < kPer; ++j) { v[j].x *= inv * w[j].x; v[j].y *= inv * w[j].y; v[j].z *= inv * w[j].z; v[j].w *= inv * w[j].w; }
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
            const int e = (tid + j * kFusedConsumers * 32) * 4;
            if (e < K) *reinterpret_cast<float4*>(xs + xs_pos(e, K)) = v[j];
        }
        consumer_bar_sync();
    }

    // Input of o_proj: merge the split-KV attention partials of every head straight into xs -- each CTA does the (tiny)
    // merge redundantly from L2 instead of one "last" CTA per kv head publishing it behind a fence + atomic + two more
    // dependent L2 round trips.  One warp per head; all loads of a pass are in flight at once.
    __device__ void load_attn(const FusedArgs& a) {
        constexpr int HD = 128, PS = kFusedPartialStride, CH = kFusedMergeChunk;
        const int K = a.nh * HD;
        for (int h0 = warp; h0 < a.nh && !skip_loads; h0 += kFusedConsumers) {
            const int h = (h0 + (int)blockIdx.x) % a.nh;   // all CTAs read the same lines: rotate the head order so they spread over the L2 slices
            const float* pb = a.partial + (size_t)h * a.nsplit * PS;
            float M = -INFINITY, L = 0.f;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int s0 = 0; s0 < a.nsplit; s0 += CH) {
                float4 v[CH];
#pragma unroll
                for (int j = 0; j < CH; ++j)
                    v[j] = (s0 + j < a.nsplit) ? __ldcg(reinterpret_cast<const float4*>(pb + (size_t)(s0 + j) * PS) + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
                float m = -INFINITY, l = 0.f;
                if (lane < CH && s0 + lane < a.nsplit) {
                    const float2 ml = __ldcg(reinterpret_cast<const float2*>(pb + (size_t)(s0 + lane) * PS + HD));
                    m = ml.x; l = ml.y;
                }
                float cm = m;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, o));
                const float Mn = fmaxf(M, cm);
                const float so = (M == -INFINITY) ? 0.f : expf(M - Mn);
                const float e = (m == -INFINITY) ? 0.f : expf(m - Mn);
                L = L * so + warp_sum(l * e);
                acc.x *= so; acc.y *= so; acc.z *= so; acc.w *= so;
#pragma unroll
                for (int j = 0; j < CH; ++j) {
                    const float ej = __shfl_sync(0xffffffffu, e, j);
                    acc.x += v[j].x * ej; acc.y += v[j].y * ej; acc.z += v[j].z * ej; acc.w += v[j].w * ej;
                }
                M = Mn;
            }
            *reinterpret_cast<float4*>(xs + xs_pos(h * HD + 4 * lane, K)) = make_float4(acc.x / L, acc.y / L, acc.z / L, acc.w / L);
        }
        consumer_bar_sync();
    }

    // dot products of a FULL stage of R rows against xs; NA independent accumulators per row break the FMA chain
    template <int R, int NA>
    __device__ __forceinline__ void stage_dots(const uint8_t* st, int K, float (&v)[kFusedMaxRows]) const {
        float acc[R][NA];
#pragma unroll
        for (int q = 0; q < R; ++q)
#pragma unroll
            for (int n = 0; n < NA; ++n) acc[q][n] = 0.f;
        const int nchunk = K >> 3;
        int c = lane;
        for (; c + 32 * (NA - 1) < nchunk; c += 32 * NA) {
#pragma unroll
            for (int n = 0; n < NA; ++n) {
                const int cc = c + 32 * n;
                const float4 x0 = *reinterpret_cast<const float4*>(xs + cc * 4);
                const float4 x1 = *reinterpret_cast<const float4*>(xs + (K >> 1) + cc * 4);
#pragma unroll
                for (int q = 0; q < R; ++q)
                    acc[q][n] = dot8(*reinterpret_cast<const uint4*>(st + (size_t)cc * 16 + (size_t)q * K * 2), x0, x1, acc[q][n]);
            }
        }
        for (; c < nchunk; c += 32) {
            const float4 x0 = *reinterpret_cast<const float4*>(xs + c * 4);
            const float4 x1 = *reinterpret_cast<const float4*>(xs + (K >> 1) + c * 4);
#pragma unroll
            for (int q = 0; q < R; ++q) acc[q][0] = dot8(*reinterpret_cast<const uint4*>(st + (size_t)c * 16 + (size_t)q * K * 2), x0, x1, acc[q][0]);
        }
#pragma unroll
        for (int q = 0; q < R; ++q) {
            float t = 0.f;
#pragma unroll
            for (int n = 0; n < NA; ++n) t += acc[q][n];
            v[q] = t;
        }
    }

    // One GEMV phase: y[r0:r1) = W[r0:r1, :] . xs  with the fused epilogue.  Ends with a consumer barrier so
    // that xs may be overwritten by the next phase.
    // LL: the outputs leave as tagged packets (qkv -> ll_qkv, o_proj / down partial sums -> the [rank][H] block `par` of every
    // tensor-parallel peer, WITHOUT the residual: readers add it from their own copy of the stream).
    template <int EPI, bool LL = false>
    __device__ void gemv(const FusedArgs& a, int N, int K, const float* bias, float* out, float& best, int& bi, uint32_t tag = 0, int par = 0, int row_off = 0) {
        const Slab s = EPI == FE_QKV ? qkv_slab(a.nh, a.nkv, a.hd, a.nsplit) : cta_slab(N, EPI == FE_SWIGLU ? 2 : 1);
        const int r0 = s.j0;
        const int R = rows_per_stage(K, N, gridDim.x);
        enter((uint32_t)(s.j1 - s.j0) * K * 2u);
        if (sync_only) { consumer_bar_sync(); return; }
        unsigned i = it;
        for (int j = s.j0, nr; j < s.j1; j += nr, ++i) {
            const int r = s.stage(j, R, nr);
            if (!owns(i)) continue;
            const uint8_t* st = wait_full(i);
            float v[kFusedMaxRows];
#pragma unroll
            for (int q = 0; q < kFusedMaxRows; ++q) v[q] = 0.f;
            if (!(a.dbg & 2)) {
                if (nr == R) {
                    switch (R) {
                        case 8: stage_dots<8, 1>(st, K, v); break;
                        case 4: stage_dots<4, 2>(st, K, v); break;
                        case 2: stage_dots<2, 2>(st, K, v); break;
                        default: stage_dots<1, 4>(st, K, v); break;
                    }
                } else {   // tail stage of the slab: row by row
                    for (int q = 0; q < nr; ++q) {
                        float t[kFusedMaxRows];
                        // a qkv row takes the accumulators of a full stage (NA 1 at R 8, else 2): its sum must not depend on where
                        // the shares of its kv group end
                        if (EPI == FE_QKV && R == 8) stage_dots<1, 1>(st + (size_t)q * K * 2, K, t);
                        else if (EPI == FE_QKV) stage_dots<1, 2>(st + (size_t)q * K * 2, K, t);
                        else stage_dots<1, 4>(st + (size_t)q * K * 2, K, t);
#pragma unroll
                        for (int z = 0; z < kFusedMaxRows; ++z) if (z == q) v[z] = t[0];
                    }
                }
            }
            release(i);   // every shared-memory read of the stage fed v[] above; __syncwarp orders the lanes
            float mine = 0.f, mate = 0.f;   // lane q keeps row q (and row q^1 for the SwiGLU pair)
#pragma unroll
            for (int q = 0; q < kFusedMaxRows; ++q) {
                if (q < nr) {
                    const float t = warp_sum(v[q]);
                    if (lane == q) mine = t;
                    if (lane == (q ^ 1)) mate = t;
                }
            }
            if (lane < nr) {
                const int row = r + lane;
                if (EPI == FE_SWIGLU) {
                    if ((lane & 1) == 0) out[row >> 1] = silu_f(mine) * mate;   // rows (2i, 2i+1) = (gate_i, up_i)
                } else {
                    float y = mine;
                    if (bias) y += bias[row];
                    if (LL && EPI == FE_RESID) {
                        if (a.tp_world == 1) ll_store<false>(a.ll_xp_local[par] + row, y, tag);   // one GPU: gpu-scope store, no pointer table
                        else for (int w = 0; w < a.tp_world; ++w) ll_store<true>(a.ll_peers->xp[par][w] + (size_t)a.tp_rank * a.H + row, y, tag);
                    } else if (LL && EPI == FE_QKV) {
                        ll_store<false>(a.ll_qkv + row, y, tag);
                    } else {
                        if (EPI == FE_RESID) { y += xown[row - r0]; xown[row - r0] = y; }   // o_proj and down own the same rows of x
                        out[row] = y;
                        if (EPI == FE_LOGITS && (y > best || (y == best && row + row_off < bi))) { best = y; bi = row + row_off; }
                    }
                }
            }
        }
        it = i;
        consumer_bar_sync();
        if (LL && EPI == FE_RESID && threadIdx.x == 0) {   // every packet store of this CTA has been issued: raise its "data is out" flag
            if (a.tp_world == 1) ll_flag_store<false>(a.ll_flag_xp_local[par] + blockIdx.x, tag);
            else for (int w = 0; w < a.tp_world; ++w) ll_flag_store<true>(a.ll_peers->flag_xp[par][w] + (size_t)a.tp_rank * 256 + blockIdx.x, tag);
        }
    }
};

// Attention scratch in shared memory (consumer side; aliases the xs region, unused during this phase)
template <int G>
struct AttnSmem {
    alignas(16) float qs[G][128];
    alignas(16) float knew[128];
    alignas(16) float vnew[128];
    float m[kFusedConsumers][G];
    float l[kFusedConsumers][G];
    alignas(16) float acc[kFusedConsumers][G][128];   // float4 stores: for G = 1 the two arrays above end on an 8-byte boundary

};

template <int G>
__device__ void fused_attention(const FusedArgs& a, Consumer& c, AttnSmem<G>& s, const float* cs, const uint16_t* spages, int layer, const FusedLayer& Ly, int t_new, uint32_t tag) {
    constexpr int HD = 128;
    const int ctx = t_new + 1;
    const int lane = c.lane, warp = c.warp, tid = threadIdx.x;
    int kvh, split, hp0, hp1;
    const bool has_item = attn_item(a, ctx, kvh, split, hp0, hp1);
    if (!has_item || c.sync_only) return;  // this CTA's producer issued nothing for the phase either
    // ---- prologue: q heads (warps 0..G-1) and the new k (warp G): RMSNorm over hd then RoPE; v copy (warp G+1)
    // Warps 0..G+1 each poll the 128 packets of their own row of q / k / v until they carry this layer's tag: one L2 round trip
    // once the group's CTAs (qkv_slab) have stored them.  No "data is out" flag here: the flag poll, the CTA barrier after it and
    // the re-read of the packets were three more dependent round trips (measured: 1.82 -> 1.75 ms per VL2 step on an H100 when
    // dropped), and 512 polled floats per CTA are too little traffic to slow the weight streams of the CTAs still in qkv.
    if (warp <= G) {
        const bool is_q = warp < G;
        const size_t src_off = (size_t)(is_q ? (kvh * G + warp) : (a.nh + kvh)) * HD + lane * 4;
        const float4 x = ll_wait4<false>(a.ll_qkv + src_off, tag, c.ll_abort);
        float ss = x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
        ss = warp_sum(ss);
        const float inv = 1.0f / sqrtf(ss / (float)HD + a.eps);
        const float4 w = *reinterpret_cast<const float4*>((is_q ? Ly.qn : Ly.kn) + lane * 4);
        const float n[4] = {x.x * inv * w.x, x.y * inv * w.y, x.z * inv * w.z, x.w * inv * w.w};
        float o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float partner = __shfl_xor_sync(0xffffffffu, n[e], 16);
            const int d = lane * 4 + e, j = d & (HD / 2 - 1);
            const float rot = (d < HD / 2) ? -partner : partner;
            o[e] = n[e] * cs[j] + rot * cs[HD / 2 + j];
        }
        float* dst = is_q ? s.qs[warp] : s.knew;
#ifdef AHA_KV_ROUND_FP16
        if (!is_q) { for (int e = 0; e < 4; ++e) o[e] = kv_store_round(o[e]); }
#endif
        *reinterpret_cast<float4*>(dst + lane * 4) = make_float4(o[0], o[1], o[2], o[3]);
    } else if (warp == G + 1) {
        const size_t src_off = (size_t)(a.nh + a.nkv + kvh) * HD + lane * 4;
        float4 v = ll_wait4<false>(a.ll_qkv + src_off, tag, c.ll_abort);
#ifdef AHA_KV_ROUND_FP16
        v = make_float4(kv_store_round(v.x), kv_store_round(v.y), kv_store_round(v.z), kv_store_round(v.w));
#endif
        *reinterpret_cast<float4*>(s.vnew + lane * 4) = v;
    }
    consumer_bar_sync();
    c.enter((uint32_t)(hp1 - hp0) * 2u * kHalfPage * HD * 4u);   // (a CTA without an item has no stages: its gate stays put)
    const int hp_new = t_new / kHalfPage;
    if (hp_new >= hp0 && hp_new < hp1 && tid < HD) {  // append K,V of the current token to the paged cache
        const int page = spages[t_new >> kPageShift];
        const size_t off = (size_t)layer * a.layer_stride + (size_t)page * a.page_stride + (size_t)kvh * kPage * HD + (size_t)(t_new & (kPage - 1)) * HD + tid;
        a.kv_pool[off] = s.knew[tid];
        a.kv_pool[off + (size_t)a.nkv * kPage * HD] = s.vnew[tid];
    }
    // Lane layout inside the owner warp: group = lane / 8 handles token (4*itr + group) of the half page,
    // sub = lane % 8 handles dims {4*sub + 32*e + 0..3 : e = 0..3} (conflict-free 128-byte rows per quarter warp).
    const int grp = lane >> 3, sub = lane & 7;
    float4 q[G][4];
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
        for (int e = 0; e < 4; ++e) q[g][e] = *reinterpret_cast<const float4*>(s.qs[g] + 4 * sub + 32 * e);
    float m[G], l[G];
    float4 acc[G][4];
#pragma unroll
    for (int g = 0; g < G; ++g) {
        m[g] = -INFINITY; l[g] = 0.f;
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[g][e] = make_float4(0.f, 0.f, 0.f, 0.f);
    }

    unsigned i = c.it;
    for (int hp = hp0; hp < hp1; ++hp, ++i) {
        if (!c.owns(i)) continue;
        const uint8_t* st = c.wait_full(i);
        const float* ks = reinterpret_cast<const float*>(st);
        const float* vs = reinterpret_cast<const float*>(st + kHalfPage * HD * 4);
        const int tbase = hp * kHalfPage;
#pragma unroll
        for (int itr = 0; itr < kHalfPage / 4; ++itr) {
            const int tl = 4 * itr + grp;          // token inside the half page
            const int t = tbase + tl;
            const bool valid = t < ctx;
            const float* kr = (t == t_new) ? s.knew : ks + tl * HD;
            const float* vr = (t == t_new) ? s.vnew : vs + tl * HD;
            float4 kk[4], vv[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                kk[e] = *reinterpret_cast<const float4*>(kr + 4 * sub + 32 * e);
                vv[e] = *reinterpret_cast<const float4*>(vr + 4 * sub + 32 * e);
                if (!valid) vv[e] = make_float4(0.f, 0.f, 0.f, 0.f);   // slots past ctx hold stale data: 0 * x must stay 0
            }
#pragma unroll
            for (int g = 0; g < G; ++g) {
                float sc = 0.f;
#pragma unroll
                for (int e = 0; e < 4; ++e) sc += q[g][e].x * kk[e].x + q[g][e].y * kk[e].y + q[g][e].z * kk[e].z + q[g][e].w * kk[e].w;
                sc += __shfl_xor_sync(0xffffffffu, sc, 1);
                sc += __shfl_xor_sync(0xffffffffu, sc, 2);
                sc += __shfl_xor_sync(0xffffffffu, sc, 4);
                sc = valid ? sc * a.scaling : -INFINITY;
                const float mnew = fmaxf(m[g], sc);
                const float muse = (mnew == -INFINITY) ? 0.f : mnew;
                const float alpha = expf(m[g] - muse);
                const float pp = expf(sc - muse);
                l[g] = l[g] * alpha + pp;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    acc[g][e].x = acc[g][e].x * alpha + pp * vv[e].x;
                    acc[g][e].y = acc[g][e].y * alpha + pp * vv[e].y;
                    acc[g][e].z = acc[g][e].z * alpha + pp * vv[e].z;
                    acc[g][e].w = acc[g][e].w * alpha + pp * vv[e].w;
                }
                m[g] = mnew;
            }
        }
        c.release(i);  // after the math: every shared-memory read of this stage has been consumed
    }
    c.it = i;
    // merge the 4 token groups of the warp (lanes differing in bits 3,4), then publish the per-warp state
#pragma unroll
    for (int g = 0; g < G; ++g) {
        float M = fmaxf(m[g], __shfl_xor_sync(0xffffffffu, m[g], 8));
        M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, 16));
        const float sc = (m[g] == -INFINITY) ? 0.f : expf(m[g] - M);
        float L = l[g] * sc;
        L += __shfl_xor_sync(0xffffffffu, L, 8);
        L += __shfl_xor_sync(0xffffffffu, L, 16);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float4 t = make_float4(acc[g][e].x * sc, acc[g][e].y * sc, acc[g][e].z * sc, acc[g][e].w * sc);
            t.x += __shfl_xor_sync(0xffffffffu, t.x, 8); t.x += __shfl_xor_sync(0xffffffffu, t.x, 16);
            t.y += __shfl_xor_sync(0xffffffffu, t.y, 8); t.y += __shfl_xor_sync(0xffffffffu, t.y, 16);
            t.z += __shfl_xor_sync(0xffffffffu, t.z, 8); t.z += __shfl_xor_sync(0xffffffffu, t.z, 16);
            t.w += __shfl_xor_sync(0xffffffffu, t.w, 8); t.w += __shfl_xor_sync(0xffffffffu, t.w, 16);
            if (grp == 0) *reinterpret_cast<float4*>(&s.acc[warp][g][4 * sub + 32 * e]) = t;
        }
        if (lane == 0) { s.m[warp][g] = M; s.l[warp][g] = L; }
    }
    consumer_bar_sync();
    for (int idx = tid; idx < G * HD; idx += kFusedConsumers * 32) {
        const int g = idx / HD, d = idx % HD;
        float M = -INFINITY;
#pragma unroll
        for (int w = 0; w < kFusedConsumers; ++w) M = fmaxf(M, s.m[w][g]);
        float L = 0.f, O = 0.f;
        if (M != -INFINITY) {
#pragma unroll
            for (int w = 0; w < kFusedConsumers; ++w) {
                const float e = expf(s.m[w][g] - M);
                L += s.l[w][g] * e;
                O += s.acc[w][g][d] * e;
            }
        }
        float* p = a.partial + ((size_t)(kvh * G + g) * a.nsplit + split) * kFusedPartialStride;
        p[d] = O;
        if (d == 0) { p[HD] = M; p[HD + 1] = L; }
    }
    // the split partials are merged by the consumers of the next phase (Consumer::load_attn), after the grid barrier
}

// ------------------------------------------------------------------------------------------------ the kernel
// PACKET_RESID = false: grid barriers after the attention, o_proj, gate/up and down.  PACKET_RESID = true: grid barriers after
// the attention and between gate/up and down (their exchanges are large or need an extra hop as packets: measured slower),
// tagged packets for the two residual-stream exchanges per layer -- the ones that cross GPUs under tensor parallelism.
// In both modes the qkv rows go to the attention as packets inside each kv-head group (qkv_slab): the attention CTA (g, split) needs
// only its group's q / k / v rows, so it waits for the group's nsplit CTAs instead of a grid barrier behind all of them.
template <int G, bool PACKET_RESID>
__global__ void __launch_bounds__(kFusedThreads, 1) decode_step_fused_kernel(FusedArgs a) {
    extern __shared__ __align__(1024) uint8_t fused_smem_raw[];
    uint8_t* ringbuf = fused_smem_raw;
    uint64_t* full = reinterpret_cast<uint64_t*>(fused_smem_raw + (size_t)kFusedStages * kFusedStageBytes);
    uint64_t* empty = full + kFusedStages;
    float* red = reinterpret_cast<float*>(empty + kFusedStages);
    uint32_t* gate = reinterpret_cast<uint32_t*>(red) + kFusedGateWord;   // the producer's run-ahead gate (Consumer::enter)
    float* xown = red + 32;                                     // [kFusedMaxOwnRows] (barrier mode only: PACKET_RESID keeps the whole stream in xres)
    float* cs = xown + (PACKET_RESID ? 0 : kFusedMaxOwnRows);   // [128] cos | sin of the step's rotary angles
    float* xs = cs + 128;                                       // [kFusedMaxK] activations / attention scratch
    uint16_t* spages = reinterpret_cast<uint16_t*>(xs + kFusedMaxK);   // [kFusedMaxPages] page table copy (physical page ids)
    float* xres = reinterpret_cast<float*>(spages + kFusedMaxPages);   // [kFusedMaxH] PACKET_RESID: the residual stream (not carved in barrier mode)
    AttnSmem<G>* as = reinterpret_cast<AttnSmem<G>*>(xs);
    static_assert(sizeof(AttnSmem<G>) <= kFusedMaxK * sizeof(float), "attention scratch must fit in the xs region");

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int i = 0; i < kFusedStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        *gate = kFusedAheadBytes;   // before the first phase the consumers are in an empty one
    }
    if ((a.dbg & 64) && tid == 0) { unsigned smid; asm volatile("mov.u32 %0, %%smid;" : "=r"(smid)); a.trace[8192 + blockIdx.x * 256 + 255] = smid; }
    const int t_new = a.st->pos;
    const int rope_delta = a.st->rope_delta;
    const uint32_t token = min(a.st->token, (uint32_t)(a.V - 1));   // a NaN logit row publishes 0x7fffffff: never index the embedding table with it
    const int ctx = t_new + 1;
    for (int i = tid; i < (ctx + kPage - 1) / kPage && i < kFusedMaxPages; i += kFusedThreads) spages[i] = (uint16_t)a.page_table[i];
    if (tid < 64) {   // RoPE angle of this step (same for every layer): cos/sin once per kernel
        const float ang = (float)(t_new + rope_delta) * a.inv_freq[tid];
        cs[tid] = cosf(ang);
        cs[64 + tid] = sinf(ang);
    }
    __syncthreads();
    Ring ring{ringbuf, full, empty};

    if (warp == kFusedConsumers) {
        // =================================================== PRODUCER (one elected lane)
        if (lane == 0) {
            Producer p;
            p.ring = ring;
            p.ns = (unsigned)a.stages;
            p.use_hint = (a.dbg & 16) == 0;      // dbg bit4 switches the L2 evict-first hint off (A/B runs)
            p.hint_kv = (a.dbg & 32) == 0;       // bit5: same switch for the KV half-page copies
            p.policy = l2_evict_first_policy();
            p.pages = spages;
            p.gate = gate;
#ifdef AHA_STAGE_TRACE
            if ((a.dbg & 128) && (int)blockIdx.x == ((a.dbg >> 16) & 0xff)) p.st_trace = a.trace + 8192;
#endif
            int pe = 0;
            AHA_STAMP(a, 1, pe);
            if (a.dbg & 512) return;   // sync-only experiment: no weight stream
            FusedLayer nxt = a.layers[0];
            for (int l = 0; l < a.L; ++l) {
                const FusedLayer Ly = nxt;
                if (l + 1 < a.L) nxt = a.layers[l + 1];   // pointer table one layer ahead: off the issue path
                p.rows(Ly.qkv, a.qkv_dim, a.H, qkv_slab(a.nh, a.nkv, a.hd, a.nsplit)); AHA_STAMP(a, 1, pe);
                p.attn(a, l, ctx); AHA_STAMP(a, 1, pe);
                p.rows(Ly.o, a.H, a.nh * a.hd, cta_slab(a.H, 1));
                AHA_STAMP(a, 1, pe);
                p.rows(Ly.gu, 2 * a.I, a.H, cta_slab(2 * a.I, 2)); AHA_STAMP(a, 1, pe);
                p.rows(Ly.down, a.H, a.I, cta_slab(a.H, 1));
                AHA_STAMP(a, 1, pe);
            }
            p.rows(a.lm_head + (size_t)a.v0 * a.H, a.V_l, a.H, cta_slab(a.V_l, 1)); AHA_STAMP(a, 1, pe);
        }
        return;
    }
    // ======================================================= CONSUMERS
    Consumer c;
    c.ring = ring; c.ns = (unsigned)a.stages; c.xs = xs; c.red = red; c.xown = xown; c.warp = warp; c.lane = lane;
#ifdef AHA_STAGE_TRACE
    if ((a.dbg & 128) && (int)blockIdx.x == ((a.dbg >> 16) & 0xff)) c.st_trace = a.trace + 8192;
#endif
    c.xres = xres; c.ll_abort = a.ll_abort;
    c.skip_loads = (a.dbg & 256) != 0;
    c.sync_only = (a.dbg & 512) != 0;
    unsigned long long* sy = nullptr;
#ifdef AHA_STAGE_TRACE
    if ((a.dbg & 1024) && (int)blockIdx.x == ((a.dbg >> 16) & 0xff)) { sy = a.trace + 8192 + 32768; c.sy_trace = sy; }
#endif
    unsigned seq = 0;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    const __half* emb_row = a.embed + (size_t)token * a.H;
    int own_r0, own_r1;
    cta_rows(a.H, 1, own_r0, own_r1);
    if (!PACKET_RESID && tid < own_r1 - own_r0) xown[tid] = __half2float(emb_row[own_r0 + tid]);   // the rows of the residual stream this CTA owns start as the embedding row
    int ce = 0;
#define CSTAMP() do { if (tid == 0) AHA_STAMP(a, 0, ce); } while (0)
    CSTAMP();
    FusedLayer nxtc = a.layers[0];
    for (int l = 0; l < a.L; ++l) {
        const FusedLayer Ly = nxtc;
        if (l + 1 < a.L) nxtc = a.layers[l + 1];
        const bool first = (l == 0);
        if constexpr (PACKET_RESID) {
            const uint32_t tag = a.ll_tag + (uint32_t)l;
            // P1: x = residual + down partial sums of layer l - 1 (packets, all ranks); qkv leaves as packets to the kv group
            if (first) c.load_x(a.H, nullptr, emb_row, Ly.ln1, a.eps, true);
            else if (a.tp_world == 1) c.template load_ll<false>(a.H, a.ll_xp_local[1], a.tp_world, (size_t)a.H, tag - 1u, Ly.ln1, a.eps, a.ll_flag_xp_local[1], (int)gridDim.x); else c.template load_ll<true>(a.H, a.ll_xp_local[1], a.tp_world, (size_t)a.H, tag - 1u, Ly.ln1, a.eps, a.ll_flag_xp_local[1], (int)gridDim.x);
            CSTAMP();
            c.template gemv<FE_QKV, true>(a, a.qkv_dim, a.H, Ly.qkv_b, nullptr, best, bi, tag); CSTAMP();
            CSTAMP();
            // P2: attention (split partials as plain floats)
            CSTAMP();
            fused_attention<G>(a, c, *as, cs, spages, l, Ly, t_new, tag); CSTAMP();
            grid_barrier(&a.sync[0], seq, a.dbg, a.trace, sy); CSTAMP();
            // P3: merge the splits, o_proj partial sums -> packets to every rank (no barrier: P4 polls them)
            c.load_attn(a); CSTAMP();
            c.template gemv<FE_RESID, true>(a, a.H, a.nh * a.hd, Ly.o_b, nullptr, best, bi, tag, 0); CSTAMP();
            CSTAMP();
            // P4: x = residual + o_proj partial sums (packets, all ranks); h = silu(gate) * up on rmsnorm(x)
            if (a.tp_world == 1) c.template load_ll<false>(a.H, a.ll_xp_local[0], a.tp_world, (size_t)a.H, tag, Ly.ln2, a.eps, a.ll_flag_xp_local[0], (int)gridDim.x); else c.template load_ll<true>(a.H, a.ll_xp_local[0], a.tp_world, (size_t)a.H, tag, Ly.ln2, a.eps, a.ll_flag_xp_local[0], (int)gridDim.x);
            CSTAMP();
            c.template gemv<FE_SWIGLU>(a, 2 * a.I, a.H, nullptr, a.h1, best, bi); CSTAMP();
            grid_barrier(&a.sync[0], seq, a.dbg, a.trace, sy); CSTAMP();
            // P5: down partial sums -> packets
            c.load_x(a.I, a.h1, nullptr, nullptr, 0.f); CSTAMP();
            c.template gemv<FE_RESID, true>(a, a.H, a.I, nullptr, nullptr, best, bi, tag, 1); CSTAMP();
            CSTAMP();
        } else {
        const uint32_t tag = a.ll_tag + (uint32_t)l;
        // P1: qkv = Wqkv . rmsnorm(x)      (layer 0 reads the embedding row directly: Embedding::forward); the rows leave as
        // packets that only the CTAs of their kv group wait for (qkv_slab): no grid barrier before the attention
        c.load_x(a.H, a.x, first ? emb_row : nullptr, Ly.ln1, a.eps);
        CSTAMP();
        c.template gemv<FE_QKV, true>(a, a.qkv_dim, a.H, Ly.qkv_b, nullptr, best, bi, tag); CSTAMP();
        CSTAMP();
        // P2: attention over the paged cache (+ q/k norm, RoPE, KV append)
        CSTAMP();
        fused_attention<G>(a, c, *as, cs, spages, l, Ly, t_new, tag); CSTAMP();
        grid_barrier(&a.sync[0], seq, a.dbg, a.trace, sy); CSTAMP();
        // P3: x = resid + Wo . attn
        c.load_attn(a); CSTAMP();
        c.template gemv<FE_RESID>(a, a.H, a.nh * a.hd, Ly.o_b, a.x, best, bi); CSTAMP();
        grid_barrier(&a.sync[0], seq, a.dbg, a.trace, sy); CSTAMP();
        // P4: h = silu(gate) * up, gate/up rows interleaved, input rmsnorm(x)
        c.load_x(a.H, a.x, nullptr, Ly.ln2, a.eps);
        CSTAMP();
        c.template gemv<FE_SWIGLU>(a, 2 * a.I, a.H, nullptr, a.h1, best, bi); CSTAMP();
        grid_barrier(&a.sync[0], seq, a.dbg, a.trace, sy); CSTAMP();
        // P5: x = x + Wdown . h
        c.load_x(a.I, a.h1, nullptr, nullptr, 0.f); CSTAMP();
        c.template gemv<FE_RESID>(a, a.H, a.I, nullptr, a.x, best, bi); CSTAMP();
        grid_barrier(&a.sync[0], seq, a.dbg, a.trace, sy); CSTAMP();
        }
    }
    // final: logits = lm_head . rmsnorm(x) over this rank's vocabulary shard, per-CTA argmax candidate
    if constexpr (PACKET_RESID) if (a.tp_world == 1) c.template load_ll<false>(a.H, a.ll_xp_local[1], a.tp_world, (size_t)a.H, a.ll_tag + (uint32_t)a.L - 1u, a.final_norm, a.eps, a.ll_flag_xp_local[1], (int)gridDim.x); else c.template load_ll<true>(a.H, a.ll_xp_local[1], a.tp_world, (size_t)a.H, a.ll_tag + (uint32_t)a.L - 1u, a.final_norm, a.eps, a.ll_flag_xp_local[1], (int)gridDim.x);
    else c.load_x(a.H, a.x, nullptr, a.final_norm, a.eps);
    best = -INFINITY; bi = 0x7fffffff;
    c.template gemv<FE_LOGITS>(a, a.V_l, a.H, nullptr, a.logits + a.v0, best, bi, 0, 0, a.v0); CSTAMP();
    // CTA-level argmax (first maximal index), then the last CTA to arrive reduces across CTAs
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (lane == 0) { red[warp] = best; reinterpret_cast<int*>(red)[16 + warp] = bi; }
    consumer_bar_sync();
    if (tid == 0) {
        for (int w = 1; w < kFusedConsumers; ++w) {
            const float ov = red[w];
            const int oi = reinterpret_cast<int*>(red)[16 + w];
            if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
        }
        a.pmax[blockIdx.x] = best;
        a.pidx[blockIdx.x] = bi;
        const unsigned ticket = atom_acq_rel_add(&a.sync[1], 1u);
        reinterpret_cast<int*>(red)[31] = (ticket == gridDim.x - 1) ? 1 : 0;
    }
    consumer_bar_sync();
    if (warp == 0 && reinterpret_cast<int*>(red)[31]) {   // last CTA to arrive: warp 0 reduces the per-CTA candidates
        float gb = -INFINITY;
        int gi = 0x7fffffff;
        for (unsigned i = lane; i < gridDim.x; i += 32) {
            const float v = __ldcg(a.pmax + i);
            const int id = __ldcg(a.pidx + i);
            if (v > gb || (v == gb && id < gi)) { gb = v; gi = id; }
        }
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, gb, o);
            const int oi = __shfl_xor_sync(0xffffffffu, gi, o);
            if (ov > gb || (ov == gb && oi < gi)) { gb = ov; gi = oi; }
        }
        if (PACKET_RESID && a.tp_world > 1) {
            // vocabulary shards: every rank publishes its (value, index) candidate to every rank and picks the same winner
            // (largest value, lowest index on ties)
            const uint32_t ftag = a.ll_tag + (uint32_t)a.L;
            if (lane < a.tp_world) {
                ll_store<true>(a.ll_peers->cand[lane] + a.tp_rank * 2, gb, ftag);
                ll_store<true>(a.ll_peers->cand[lane] + a.tp_rank * 2 + 1, __int_as_float(gi), ftag);
            }
            float cb = -INFINITY;
            int ci = 0x7fffffff;
            if (lane < a.tp_world) {
                cb = ll_wait1<true>(a.ll_cand_local + lane * 2, ftag, a.ll_abort);
                ci = __float_as_int(ll_wait1<true>(a.ll_cand_local + lane * 2 + 1, ftag, a.ll_abort));
            }
            for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, cb, o);
                const int oi = __shfl_xor_sync(0xffffffffu, ci, o);
                if (ov > cb || (ov == cb && oi < ci)) { cb = ov; ci = oi; }
            }
            gb = cb; gi = ci;
        }
        if (gi < 0 || gi >= a.V) gi = 0;   // all-NaN logits: publish a valid id (the reference would pick some index too)
        if (lane == 0) {
            *a.argmax_out = (uint32_t)gi;
            DecodeState* st = a.st;
            st->token = (uint32_t)gi;
            st->pos = t_new + 1;
            if (st->n_hist < a.hist_cap) a.history[st->n_hist] = (uint32_t)gi;
            st->n_hist += 1;
        }
    }
}

template <int G>
inline size_t fused_smem_bytes(bool packet_resid) {
    return (packet_resid ? (size_t)kFusedMaxH * sizeof(float) : (size_t)kFusedMaxOwnRows * sizeof(float)) + (size_t)kFusedStages * kFusedStageBytes + 2 * kFusedStages * sizeof(uint64_t) + (32 + 128) * sizeof(float) + (size_t)kFusedMaxK * sizeof(float) +
           (size_t)kFusedMaxPages * sizeof(uint16_t) + 64;
}

}  // namespace aha
