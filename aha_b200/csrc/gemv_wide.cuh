// gemv_wide.cuh -- decode projections for a WIDE batch on the tensor cores: Y[b][N] = epi(W[N,K] . X[b][K]), 1 <= nb <= 64.
//
// gemv_batch.cuh runs one fp32 FMA chain per (row, sequence) on the CUDA cores, so every extra sequence adds FMAs per weight byte and 8
// sequences are already bound by the activations, not by the weight stream (DESIGN.md section 4.4).  Here the weights are the wgmma A
// operand and the sequences the B operand, with the split-fp16 scheme of gemm_tc.cuh: W is exact fp16, X is pre-split into X = hi + lo
// (fp16 each, by rmsnorm_split_kernel or split_f32_to_f16x2_kernel: BatchDecoder::wide_prep) and W.hi + W.lo accumulate in fp32.
//
// Structure (one 128-row W tile x one K range per CTA, 288 threads, two CTAs per SM):
//   warp 8          : TMA producer -- per k-block the W tile (128 rows x 64 halfs) and the X hi / X lo tiles (64 sequences x 64 halfs,
//                     L2-resident) into a 3-stage mbarrier ring, as in gemm_tc.cuh;
//   warpgroups 0, 1 : 64 W rows each, 8 wgmma.m64n64k16 per k-block (4 k-steps x {hi, lo}).
// The B tile is ALWAYS 64 sequences wide (rows nb..63 of X are zero or stale and their columns are never stored): one MMA shape for every
// nb, so column b's sums do not depend on nb, on the other columns or on b itself.  The step is bound by the weight stream, so the unused
// columns cost tensor-core time that is idle anyway.
//
// Split-K: a projection with few 128-row tiles (o_proj, down: N = H) would leave most of the 132 SMs idle, so its K range is cut into
// `splits` parts that depend only on (N, K) and the SM count (wide_plan), never on nb.  Every CTA writes its fp32 partial tile to a
// workspace; the last CTA of a row tile (an atomic counter, reset by that CTA) adds the partials in split order 0, 1, ... and runs the
// epilogue.  No float atomics: the sums are the same whichever CTA finishes last.
//
// LoRA tail (TAIL = true, lora.cuh): after its base k-blocks the last split streams the k-blocks of the device list a.tail -- a B_pool tile
// (128 rows x 64 columns) and the t hi / lo tiles of the same 64 columns in place of W and X -- into the same ring and accumulator.  The
// tail rides in that one split whatever the list holds, so a row's partial sums keep their split order.
#pragma once
#include "gemm_tc.cuh"
#include "gemv.cuh"   // GemvEpi
#include "lora.cuh"   // LoraTail

namespace aha {

constexpr int kWideSeqs = 64;                     // sequences per B tile = the widest batch
constexpr int kWideBM = 128;                      // W rows per CTA (two consumer warpgroups)
constexpr int kWideThreads = 288;                 // 2 consumer warpgroups + 1 producer warp
constexpr int kWideStages = 3;
constexpr int kWideWBytes = kWideBM * kTcBK * 2;  // 16 KB
constexpr int kWideXBytes = kWideSeqs * kTcBK * 2;// 8 KB per half
constexpr int kWideStageBytes = kWideWBytes + 2 * kWideXBytes;
constexpr int kWidePartFloats = kWideBM * kWideSeqs;   // one CTA's partial tile
constexpr int kWideMinKb = 2;                     // k-blocks per split at least: the partial tile (32 KB) is never more than the weights behind it

inline size_t gemv_wide_smem_bytes() { return (size_t)kWideStages * kWideStageBytes + 2 * kWideStages * sizeof(uint64_t) + 1024; }

struct WidePlan { int tiles, splits, kper; };
// Split-K plan of an [N, K] projection: enough CTAs for two per SM where K allows it.  Depends on (N, K, SM count) only.
inline WidePlan wide_plan(int N, int K, int num_sms) {
    WidePlan p;
    p.tiles = ceil_div(N, kWideBM);
    const int nkb = K / kTcBK, target = 2 * num_sms;
    int s = 1;
    if (p.tiles < target) s = std::max(1, std::min(ceil_div(target, p.tiles), nkb / kWideMinKb));
    p.kper = ceil_div(nkb, s);
    p.splits = ceil_div(nkb, p.kper);
    return p;
}
inline bool gemv_wide_supported(int N, int K) { return N >= 64 && K >= 64 && N % 64 == 0 && K % 64 == 0; }

struct WideArgs {
    const float* bias;              // [N] or nullptr
    const float* resid; int ldr;    // [nb][N] (GEPI_RESID; may alias out)
    float* out; int ldo;            // [nb][N] (or [nb][N/2] for GEPI_SWIGLU)
    int N, K, nb;
    int splits, kper;               // wide_plan
    float* ws;                      // [tiles * splits][kWidePartFloats] when splits > 1
    int* counters;                  // [tiles], zero between launches
    const int* tail = nullptr;      // TAIL: device [count, k-block indices] of the LoRA pool (lora.cuh)
};

template <int EPI, bool TAIL>
__global__ void __launch_bounds__(kWideThreads, 2) gemv_wide_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_hi,
                                                                    const __grid_constant__ CUtensorMap tm_lo, const __grid_constant__ CUtensorMap tm_b,
                                                                    const __grid_constant__ CUtensorMap tm_thi, const __grid_constant__ CUtensorMap tm_tlo,
                                                                    WideArgs a) {
    extern __shared__ __align__(1024) uint8_t wide_smem_raw[];
    uint8_t* tiles = wide_smem_raw + ((1024u - (smem_u32(wide_smem_raw) & 1023u)) & 1023u);   // [stages][W | X hi | X lo]
    uint64_t* full = reinterpret_cast<uint64_t*>(tiles + (size_t)kWideStages * kWideStageBytes);
    uint64_t* empty = full + kWideStages;
    __shared__ int s_last;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tile = blockIdx.x, split = blockIdx.y, n0 = tile * kWideBM;
    const int kb0 = split * a.kper, nk = min(a.K / kTcBK, kb0 + a.kper) - kb0;
    const int nt = TAIL && split == a.splits - 1 ? a.tail[0] : 0;

    if (tid == 0) {
        for (int i = 0; i < kWideStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            for (int i = 0; i < nk + nt; ++i) {
                const int s = i % kWideStages;
                mbar_wait(&empty[s], ((i / kWideStages) & 1) ^ 1);
                uint8_t* st = tiles + (size_t)s * kWideStageBytes;
                mbar_expect_tx(&full[s], kWideStageBytes);
                if (!TAIL || i < nk) {
                    const int k = (kb0 + i) * kTcBK;
                    tma_load_2d(st, &tm_w, k, n0, &full[s]);
                    tma_load_2d(st + kWideWBytes, &tm_hi, k, 0, &full[s]);
                    tma_load_2d(st + kWideWBytes + kWideXBytes, &tm_lo, k, 0, &full[s]);
                } else {
                    const int k = a.tail[1 + i - nk] * kTcBK;
                    tma_load_2d(st, &tm_b, k, n0, &full[s]);
                    tma_load_2d(st + kWideWBytes, &tm_thi, k, 0, &full[s]);
                    tma_load_2d(st + kWideWBytes + kWideXBytes, &tm_tlo, k, 0, &full[s]);
                }
            }
        }
        return;
    }
    const int wg = warp >> 2;
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    for (int i = 0; i < nk + nt; ++i) {
        const int s = i % kWideStages;
        mbar_wait(&full[s], (i / kWideStages) & 1);
        const uint32_t st = smem_u32(tiles + (size_t)s * kWideStageBytes);
        const uint64_t d_w = wgmma_desc_sw128(st + wg * 64 * 128);
        const uint64_t d_hi = wgmma_desc_sw128(st + kWideWBytes), d_lo = wgmma_desc_sw128(st + kWideWBytes + kWideXBytes);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < kTcBK / 16; ++ks) {
            const uint64_t adv = (uint64_t)((ks * 16 * 2) >> 4);
            wgmma_ss_n64(acc, d_w + adv, d_hi + adv);
            wgmma_ss_n64(acc, d_w + adv, d_lo + adv);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (i > 0 && lane == 0) mbar_arrive(&empty[(i - 1) % kWideStages]);
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);

    // acc[4j + 2h + c] = D[row (lane / 4) + 8h of this warp's 16][sequence 8j + 2 (lane % 4) + c]; columns 8j >= nb are never read
    if (a.splits > 1) {
        float4* mine = reinterpret_cast<float4*>(a.ws) + ((size_t)(tile * a.splits + split) * 8) * 256;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (8 * j < a.nb) mine[j * 256 + tid] = make_float4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]);
        __threadfence();
        asm volatile("bar.sync 1, 256;" ::: "memory");   // the 8 consumer warps (the producer warp has left)
        if (tid == 0) s_last = atomicAdd(&a.counters[tile], 1) == a.splits - 1;
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (!s_last) return;
        __threadfence();
        const float4* base = reinterpret_cast<const float4*>(a.ws) + (size_t)tile * a.splits * 8 * 256;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (8 * j >= a.nb) continue;
            float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int s = 0; s < a.splits; ++s) {   // split order, whichever CTA is last
                const float4 p = s == split ? make_float4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]) : __ldcg(base + ((size_t)s * 8 + j) * 256 + tid);
                r.x += p.x; r.y += p.y; r.z += p.z; r.w += p.w;
            }
            acc[4 * j] = r.x; acc[4 * j + 1] = r.y; acc[4 * j + 2] = r.z; acc[4 * j + 3] = r.w;
        }
        if (tid == 0) a.counters[tile] = 0;   // ready for the next launch (stream order)
    }

    const int row0 = n0 + wg * 64 + (warp & 3) * 16 + (lane >> 2), col0 = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (8 * j >= a.nb) break;   // uniform across the CTA
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int n = row0 + 8 * h;
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const int b = 8 * j + col0 + c;
                float v = acc[4 * j + 2 * h + c];
                if (EPI == GEPI_SWIGLU) {   // rows (2i, 2i + 1) = (gate_i, up_i) sit in lanes l and l ^ 4
                    const float up = __shfl_xor_sync(0xffffffffu, v, 4);
                    if (((lane >> 2) & 1) == 0 && n < a.N && b < a.nb) {
                        const float g = v + (a.bias ? a.bias[n] : 0.f), u = up + (a.bias ? a.bias[n + 1] : 0.f);
                        a.out[(size_t)b * a.ldo + (n >> 1)] = silu_f(g) * u;
                    }
                } else if (n < a.N && b < a.nb) {
                    if (a.bias) v += a.bias[n];
                    if (EPI == GEPI_RESID) v += a.resid[(size_t)b * a.ldr + n];
                    a.out[(size_t)b * a.ldo + n] = v;
                }
            }
        }
    }
}

inline void gemv_wide_init() {
    const int smem = (int)gemv_wide_smem_bytes();
    AHA_CUDA_CHECK(cudaFuncSetAttribute(gemv_wide_kernel<GEPI_STORE, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    AHA_CUDA_CHECK(cudaFuncSetAttribute(gemv_wide_kernel<GEPI_RESID, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    AHA_CUDA_CHECK(cudaFuncSetAttribute(gemv_wide_kernel<GEPI_SWIGLU, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    AHA_CUDA_CHECK(cudaFuncSetAttribute(gemv_wide_kernel<GEPI_STORE, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    AHA_CUDA_CHECK(cudaFuncSetAttribute(gemv_wide_kernel<GEPI_RESID, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    AHA_CUDA_CHECK(cudaFuncSetAttribute(gemv_wide_kernel<GEPI_SWIGLU, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
}

// X hi / lo: [64][K] fp16 (rows >= nb zero or stale), tm_w: W [N, K] with 128-row boxes (make_tmap_f16 / LinearW::tmap).
// ws / counters: sized by wide_ws_floats / the tile count of the widest projection.
// tail (optional, Rp > 0): t hi / lo [64][Rp], B_pool [N][Rp] and the device list of k-blocks to stream (lora.cuh).
inline void gemv_wide(cudaStream_t st, int epi, const CUtensorMap& tm_w, const __half* x_hi, const __half* x_lo, WideArgs a, int num_sms,
                      const LoraTail* tail = nullptr) {
    AHA_REQUIRE(a.nb >= 1 && a.nb <= kWideSeqs, "gemv_wide: 1..64 sequences");
    AHA_REQUIRE(gemv_wide_supported(a.N, a.K), "gemv_wide: N and K must be multiples of 64");
    const WidePlan p = wide_plan(a.N, a.K, num_sms);
    a.splits = p.splits; a.kper = p.kper;
    AHA_REQUIRE(p.splits == 1 || (a.ws && a.counters), "gemv_wide: split-K needs a workspace");
    const CUtensorMap tm_hi = make_tmap_f16_rows(x_hi, kWideSeqs, (uint64_t)a.K, kWideSeqs);
    const CUtensorMap tm_lo = make_tmap_f16_rows(x_lo, kWideSeqs, (uint64_t)a.K, kWideSeqs);
    const dim3 grid(p.tiles, p.splits);
    const size_t smem = gemv_wide_smem_bytes();
    if (tail && tail->Rp > 0) {
        AHA_REQUIRE(tail->Rp % kTcBK == 0 && tail->list, "gemv_wide: the LoRA tail needs a pool of whole k-blocks and a k-block list");
        const CUtensorMap tm_b = make_tmap_f16(tail->B, (uint64_t)a.N, (uint64_t)tail->Rp);
        const CUtensorMap tm_thi = make_tmap_f16_rows(tail->t_hi, kWideSeqs, (uint64_t)tail->Rp, kWideSeqs);
        const CUtensorMap tm_tlo = make_tmap_f16_rows(tail->t_lo, kWideSeqs, (uint64_t)tail->Rp, kWideSeqs);
        a.tail = tail->list;
        switch (epi) {
            case GEPI_STORE: gemv_wide_kernel<GEPI_STORE, true><<<grid, kWideThreads, smem, st>>>(tm_w, tm_hi, tm_lo, tm_b, tm_thi, tm_tlo, a); break;
            case GEPI_RESID: gemv_wide_kernel<GEPI_RESID, true><<<grid, kWideThreads, smem, st>>>(tm_w, tm_hi, tm_lo, tm_b, tm_thi, tm_tlo, a); break;
            case GEPI_SWIGLU: gemv_wide_kernel<GEPI_SWIGLU, true><<<grid, kWideThreads, smem, st>>>(tm_w, tm_hi, tm_lo, tm_b, tm_thi, tm_tlo, a); break;
            default: AHA_REQUIRE(false, "gemv_wide: bad epilogue");
        }
        AHA_CUDA_CHECK(cudaGetLastError());
        return;
    }
    switch (epi) {   // (the tail maps are not read: the base W / X maps fill their places)
        case GEPI_STORE: gemv_wide_kernel<GEPI_STORE, false><<<grid, kWideThreads, smem, st>>>(tm_w, tm_hi, tm_lo, tm_w, tm_hi, tm_lo, a); break;
        case GEPI_RESID: gemv_wide_kernel<GEPI_RESID, false><<<grid, kWideThreads, smem, st>>>(tm_w, tm_hi, tm_lo, tm_w, tm_hi, tm_lo, a); break;
        case GEPI_SWIGLU: gemv_wide_kernel<GEPI_SWIGLU, false><<<grid, kWideThreads, smem, st>>>(tm_w, tm_hi, tm_lo, tm_w, tm_hi, tm_lo, a); break;
        default: AHA_REQUIRE(false, "gemv_wide: bad epilogue");
    }
    AHA_CUDA_CHECK(cudaGetLastError());
}
// workspace floats / counters one [N, K] projection needs (0 floats when it does not split)
inline size_t wide_ws_floats(int N, int K, int num_sms) {
    const WidePlan p = wide_plan(N, K, num_sms);
    return p.splits > 1 ? (size_t)p.tiles * p.splits * kWidePartFloats : 0;
}

}  // namespace aha
