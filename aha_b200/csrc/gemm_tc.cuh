// gemm_tc.cuh -- Hopper tensor-core GEMM (wgmma + TMA) for prefill / ViT / audio Linear layers on sm_90a:
//     C[M,N] = A[M,K] (fp32 activations) x W[N,K]^T (fp16 weights)  with fp32-grade accuracy.
//
// The tensor cores take fp16 operands, but the parity budget (1e-3 on logits) does not survive rounding
// activations to fp16 (DESIGN.md section 2).  So A is split once into A = hi + lo (both fp16, |lo| <= 2^-11 |hi|) and
// every weight tile is multiplied by both halves into the SAME fp32 accumulator: the weight products are
// exact (fp16 x fp16 -> fp32) and the dropped remainder of A is ~2^-22 relative.  Twice the MMA work, still
// tensor-pipe bound instead of CUDA-core bound.
//
// Structure (one 128 x BN output tile per CTA, BN = 128 or 256, 288 threads):
//   warp 8     : TMA producer -- cp.async.bulk.tensor.2d (SWIZZLE_128B) of A_hi, A_lo (128 rows x 64 halfs) and the W k-block
//                (BN rows x 64 halfs) into a shared-memory ring, completion on `full` mbarriers;
//   warpgroups 0, 1: consumers -- 64 rows each: per k-block 8 wgmma.m64nBNk16 (4 k-steps x {hi, lo}) into the fp32 accumulator
//                in registers; a slot is released on its `empty` mbarrier once the wgmmas that read it have retired, then
//                the fused bias / residual / activation / SwiGLU epilogue stores straight from the accumulator fragment.
// LoRA tail (TAIL = true, lora.cuh): after the base k-blocks the producer streams the k-blocks of the device list g.tail -- t hi / lo
// (128 rows x 64 columns) and B_pool (BN rows x 64 columns) in place of A and W -- into the same ring and accumulator.
// Replaces candle Linear::forward at the reference call sites src/models/common/modules.rs:81-87,
// 538-577 and qwen3vl/model.rs:96-103,168-184,232-278 (prefill shapes); validated against gemm_simt.cuh.
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "decode_fused.cuh"  // mbarrier helpers
#include "gemm_simt.cuh"
#include "lora.cuh"
#include "wgmma.cuh"

namespace aha {

constexpr int kTcBM = 128, kTcBK = 64;
constexpr int kTcTileBytes = kTcBM * kTcBK * 2;             // 16 KB: one A half (hi or lo) of a k-block
constexpr int kTcThreads = 288;                             // 2 consumer warpgroups + 1 producer warp
template <int BN> __host__ __device__ constexpr int tc_stages() { return BN == 128 ? 4 : 3; }   // 4 x 48 KB / 3 x 64 KB of the 227 KB an H100 block may use
template <int BN> __host__ __device__ constexpr int tc_stage_bytes() { return 2 * kTcTileBytes + BN * kTcBK * 2; }

// ------------------------------------------------------------------------------------------------ host: tensor maps
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                        const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                        CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline PFN_tmapEncodeTiled tmap_encode_fn() {
    static PFN_tmapEncodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        AHA_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
        AHA_REQUIRE(q == cudaDriverEntryPointSuccess && p, "cuTensorMapEncodeTiled is not available in this driver");
        fn = reinterpret_cast<PFN_tmapEncodeTiled>(p);
    }
    return fn;
}
// fp16 row-major [rows, K] matrix, box = 128 rows x 64 halfs (128 bytes), 128-byte swizzle, OOB rows read as zero
inline CUtensorMap make_tmap_f16(const void* ptr, uint64_t rows, uint64_t K) {
    CUtensorMap m;
    const cuuint64_t gdim[2] = {K, rows};
    const cuuint64_t gstride[1] = {K * 2};
    const cuuint32_t box[2] = {(cuuint32_t)kTcBK, (cuuint32_t)kTcBM};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = tmap_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    AHA_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
    return m;
}

// ------------------------------------------------------------------------------------------------ device helpers
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* tm, int c0, int c1, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(dst)),
                 "l"(tm), "r"(c0), "r"(c1), "r"(smem_u32(bar))
                 : "memory");
}

// ------------------------------------------------------------------------------------------------ A = hi + lo split
__global__ void split_f32_to_f16x2_kernel(const float* __restrict__ a, int lda, __half* __restrict__ hi, __half* __restrict__ lo, int M, int K) {
    const size_t i4 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;   // index of a float4 inside [M, K]
    const size_t per_row = K / 4;
    if (i4 >= (size_t)M * per_row) return;
    const size_t r = i4 / per_row, c = (i4 % per_row) * 4;
    const float4 v = *reinterpret_cast<const float4*>(a + r * lda + c);
    const float x[4] = {v.x, v.y, v.z, v.w};
    __half h[4], l[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        h[e] = __float2half_rn(x[e]);
        l[e] = __float2half_rn(x[e] - __half2float(h[e]));
    }
    *reinterpret_cast<uint2*>(hi + r * K + c) = make_uint2(*reinterpret_cast<uint32_t*>(&h[0]), *reinterpret_cast<uint32_t*>(&h[2]));
    *reinterpret_cast<uint2*>(lo + r * K + c) = make_uint2(*reinterpret_cast<uint32_t*>(&l[0]), *reinterpret_cast<uint32_t*>(&l[2]));
}

// ------------------------------------------------------------------------------------------------ the GEMM kernel
struct GemmTcArgs {
    const float* bias;
    const float* resid; int ldr;
    float* C; int ldc;
    int M, N, K;
    int act;
    __half* out_hi = nullptr;   // when set, the result (after bias / activation / SwiGLU) is written as fp16 hi + lo halves [M, ldo] for the
    __half* out_lo = nullptr;   // next GEMM instead of fp32 C (EPI_STORE / EPI_ACT / EPI_SWIGLU)
    int ldo = 0;
    const int* tail = nullptr;  // TAIL: device [count, k-block indices] of the LoRA pool
};

// one thread's two adjacent accumulator columns (n, n + 1) of output row `row` (n even): bias / residual / activation / SwiGLU, then
// fp32 stores -- or, when g.out_hi is set, the fp16 hi + lo halves the next GEMM reads
template <int EPI>
__device__ __forceinline__ void tc_epilogue_pair(const GemmTcArgs& g, float v0, float v1, int row, int n) {
    if (row >= g.M || n >= g.N) return;
    if (g.bias) { v0 += g.bias[n]; v1 += g.bias[n + 1]; }
    if (EPI == EPI_SWIGLU) {   // W rows are interleaved (gate, up): the pair is one gate / up couple -> output column n / 2
        const float r = silu_f(v0) * v1;
        if (g.out_hi) {
            const size_t o = (size_t)row * g.ldo + n / 2;
            const __half h = __float2half_rn(r);
            g.out_hi[o] = h;
            g.out_lo[o] = __float2half_rn(r - __half2float(h));
        } else {
            g.C[(size_t)row * g.ldc + n / 2] = r;
        }
        return;
    }
    if (EPI == EPI_ACT) { v0 = apply_act(g.act, v0); v1 = apply_act(g.act, v1); }
    if (EPI == EPI_RESID) {
        const float2 r2 = *reinterpret_cast<const float2*>(g.resid + (size_t)row * g.ldr + n);
        v0 += r2.x; v1 += r2.y;
    }
    if (EPI != EPI_RESID && g.out_hi) {
        const size_t o = (size_t)row * g.ldo + n;
        const __half2 h = __floats2half2_rn(v0, v1);
        *reinterpret_cast<__half2*>(g.out_hi + o) = h;
        *reinterpret_cast<__half2*>(g.out_lo + o) = __floats2half2_rn(v0 - __low2float(h), v1 - __high2float(h));
        return;
    }
    *reinterpret_cast<float2*>(g.C + (size_t)row * g.ldc + n) = make_float2(v0, v1);
}

template <int BN>
__device__ __forceinline__ void tc_mma(float (&acc)[BN / 2], uint64_t da, uint64_t db) {
    if constexpr (BN == 128) wgmma_ss_n128(acc, da, db);
    else wgmma_ss_n256(acc, da, db);
}

// ------------------------------------------------------------------------------------------------ the shared mainloop
// The ring is walked by a position `it` that counts k-blocks over the CTA's whole life: slot it % S, phase it / S.  gemm_tc_kernel walks
// one tile (it = kb); score_head_kernel (score_head.cuh) walks several W tiles of the same A rows back to back through the same ring.
//
// TMA producer: k-block kb of A rows [m0, m0 + 128) and W rows [n0, n0 + BN) into the slot of ring position `it`
template <int BN>
__device__ __forceinline__ void tc_produce(uint8_t* tiles, uint64_t* full, uint64_t* empty, const CUtensorMap* tm_hi, const CUtensorMap* tm_lo,
                                           const CUtensorMap* tm_w, int it, int kb, int m0, int n0) {
    constexpr int S = tc_stages<BN>(), SB = tc_stage_bytes<BN>();
    const int s = it % S;
    mbar_wait(&empty[s], ((it / S) & 1) ^ 1);
    uint8_t* st = tiles + (size_t)s * SB;
    mbar_expect_tx(&full[s], SB);
    tma_load_2d(st, tm_hi, kb * kTcBK, m0, &full[s]);
    tma_load_2d(st + kTcTileBytes, tm_lo, kb * kTcBK, m0, &full[s]);
    tma_load_2d(st + 2 * kTcTileBytes, tm_w, kb * kTcBK, n0, &full[s]);
}
// consumer warpgroup wg (rows [64 wg, 64 wg + 64) of the tile): acc = the tile's products over nkb k-blocks taken from ring positions
// it0 .. it0 + nkb - 1, every k-block as 4 k-steps x {hi, lo}.  Every slot but the last one is released on its `empty` barrier; the caller
// releases that one (or ends) once the accumulator has been read.
template <int BN>
__device__ __forceinline__ void tc_mainloop(float (&acc)[BN / 2], uint8_t* tiles, uint64_t* full, uint64_t* empty, int it0, int nkb, int wg, int lane) {
    constexpr int S = tc_stages<BN>(), SB = tc_stage_bytes<BN>();
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < nkb; ++kb) {
        const int it = it0 + kb, s = it % S;
        mbar_wait(&full[s], (it / S) & 1);
        const uint32_t st = smem_u32(tiles + (size_t)s * SB);
        const uint64_t d_hi = wgmma_desc_sw128(st + wg * 64 * 128), d_lo = wgmma_desc_sw128(st + kTcTileBytes + wg * 64 * 128);
        const uint64_t d_w = wgmma_desc_sw128(st + 2 * kTcTileBytes);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < kTcBK / 16; ++ks) {
            const uint64_t adv = (uint64_t)((ks * 16 * 2) >> 4);   // 32 bytes per K = 16 step inside the 128-byte swizzle atom
            tc_mma<BN>(acc, d_hi + adv, d_w + adv);
            tc_mma<BN>(acc, d_lo + adv, d_w + adv);
        }
        wgmma_commit();
        wgmma_wait<1>();                                      // the group of k-block kb - 1 has retired: its slot is free
        if (kb > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % S]);
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
}

// ------------------------------------------------------------------------------------------------ the GEMM kernel
template <int EPI, int BN, bool TAIL>
__global__ void __launch_bounds__(kTcThreads, 1) gemm_tc_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo,
                                                               const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_thi,
                                                               const __grid_constant__ CUtensorMap tm_tlo, const __grid_constant__ CUtensorMap tm_b,
                                                               GemmTcArgs g) {
    constexpr int S = tc_stages<BN>(), SB = tc_stage_bytes<BN>();
    extern __shared__ __align__(1024) uint8_t tc_smem_raw[];
    // SWIZZLE_128B tiles need 1024-byte alignment in the shared window: align by hand (1 KB of slack is allocated)
    uint8_t* tiles = tc_smem_raw + ((1024u - (smem_u32(tc_smem_raw) & 1023u)) & 1023u);   // [stages][A_hi | A_lo | W]
    uint64_t* full = reinterpret_cast<uint64_t*>(tiles + (size_t)S * SB);
    uint64_t* empty = full + S;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m0 = blockIdx.y * kTcBM, n0 = blockIdx.x * BN;
    const int nkb = g.K / kTcBK, nt = TAIL ? g.tail[0] : 0;

    if (tid == 0) {
        for (int i = 0; i < S; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }   // 8 consumer warps release a slot
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        // ======================= TMA producer
        if (lane == 0) {
            for (int kb = 0; kb < nkb; ++kb) tc_produce<BN>(tiles, full, empty, &tm_hi, &tm_lo, &tm_w, kb, kb, m0, n0);
            for (int i = 0; i < nt; ++i) tc_produce<BN>(tiles, full, empty, &tm_thi, &tm_tlo, &tm_b, nkb + i, g.tail[1 + i], m0, n0);
        }
        return;
    }
    // ======================= consumer warpgroup wg: rows [64 wg, 64 wg + 64) of the tile
    const int wg = warp >> 2;
    float acc[BN / 2];
    tc_mainloop<BN>(acc, tiles, full, empty, 0, nkb + nt, wg, lane);
    const int row = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2), col = n0 + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        tc_epilogue_pair<EPI>(g, acc[4 * j], acc[4 * j + 1], row, col + 8 * j);
        tc_epilogue_pair<EPI>(g, acc[4 * j + 2], acc[4 * j + 3], row + 8, col + 8 * j);
    }
}
template <int BN>
inline size_t gemm_tc_smem_bytes() { return (size_t)tc_stages<BN>() * tc_stage_bytes<BN>() + 2 * tc_stages<BN>() * sizeof(uint64_t) + 1024; }

inline bool gemm_tc_supported(int M, int N, int K) { return K % kTcBK == 0 && N % 32 == 0 && M >= 1; }

// The > 48 KB dynamic shared memory opt-in is a per-device function attribute: aha_b200_create calls this after
// cudaSetDevice for every handle (a process-wide once-flag would leave a second device without it).
template <int BN, bool TAIL>
inline void gemm_tc_init_bn() {
    const int smem = (int)gemm_tc_smem_bytes<BN>();
    AHA_CUDA_CHECK(cudaFuncSetAttribute(gemm_tc_kernel<EPI_STORE, BN, TAIL>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    AHA_CUDA_CHECK(cudaFuncSetAttribute(gemm_tc_kernel<EPI_RESID, BN, TAIL>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    AHA_CUDA_CHECK(cudaFuncSetAttribute(gemm_tc_kernel<EPI_ACT, BN, TAIL>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    AHA_CUDA_CHECK(cudaFuncSetAttribute(gemm_tc_kernel<EPI_SWIGLU, BN, TAIL>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
}
inline void gemm_tc_init() {
    gemm_tc_init_bn<128, false>();
    gemm_tc_init_bn<256, false>();
    gemm_tc_init_bn<128, true>();
    gemm_tc_init_bn<256, true>();
}

// W map with `box_rows`-row boxes (the 128 x 256 tile loads 256 W rows per k-block)
inline CUtensorMap make_tmap_f16_rows(const void* ptr, uint64_t rows, uint64_t K, uint32_t box_rows) {
    CUtensorMap m;
    const cuuint64_t gdim[2] = {K, rows};
    const cuuint64_t gstride[1] = {K * 2};
    const cuuint32_t box[2] = {(cuuint32_t)kTcBK, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = tmap_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    AHA_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
    return m;
}

// A already split: hi/lo fp16 [M, K] row-major.  tm_w describes W [N, K] with BN-row boxes (make_tmap_f16 for 128,
// make_tmap_f16_rows(w, N, K, 256) for 256).  tail (optional, Rp > 0): t hi / lo [M][Rp], B_pool [N][Rp] and the device list of k-blocks.
template <int BN>
inline void gemm_tc_launch(cudaStream_t st, int epi, const __half* a_hi, const __half* a_lo, const CUtensorMap& tm_w, const GemmTcArgs& g0,
                           const LoraTail* tail = nullptr) {
    GemmTcArgs g = g0;
    const CUtensorMap tm_hi = make_tmap_f16(a_hi, (uint64_t)g.M, (uint64_t)g.K);
    const CUtensorMap tm_lo = make_tmap_f16(a_lo, (uint64_t)g.M, (uint64_t)g.K);
    const size_t smem = gemm_tc_smem_bytes<BN>();
    dim3 grid(ceil_div(g.N, BN), ceil_div(g.M, kTcBM));
    if (tail && tail->Rp > 0) {
        AHA_REQUIRE(tail->Rp % kTcBK == 0 && tail->list, "gemm_tc: the LoRA tail needs a pool of whole k-blocks and a k-block list");
        const CUtensorMap tm_thi = make_tmap_f16(tail->t_hi, (uint64_t)g.M, (uint64_t)tail->Rp);
        const CUtensorMap tm_tlo = make_tmap_f16(tail->t_lo, (uint64_t)g.M, (uint64_t)tail->Rp);
        const CUtensorMap tm_b = make_tmap_f16_rows(tail->B, (uint64_t)g.N, (uint64_t)tail->Rp, BN);
        g.tail = tail->list;
        switch (epi) {
#define AHA_TC_TAIL_CASE(E)                                                                                                        \
    case E: gemm_tc_kernel<E, BN, true><<<grid, kTcThreads, smem, st>>>(tm_hi, tm_lo, tm_w, tm_thi, tm_tlo, tm_b, g); break;
            AHA_TC_TAIL_CASE(EPI_STORE)
            AHA_TC_TAIL_CASE(EPI_RESID)
            AHA_TC_TAIL_CASE(EPI_ACT)
            AHA_TC_TAIL_CASE(EPI_SWIGLU)
            default: AHA_REQUIRE(false, "gemm_tc: bad epilogue");
        }
#undef AHA_TC_TAIL_CASE
        AHA_CUDA_CHECK(cudaGetLastError());
        return;
    }
#define AHA_TC_CASE(E)                                                                                                             \
    case E: gemm_tc_kernel<E, BN, false><<<grid, kTcThreads, smem, st>>>(tm_hi, tm_lo, tm_w, tm_hi, tm_lo, tm_w, g); break;
    switch (epi) {
        AHA_TC_CASE(EPI_STORE)
        AHA_TC_CASE(EPI_RESID)
        AHA_TC_CASE(EPI_ACT)
        AHA_TC_CASE(EPI_SWIGLU)
        default: AHA_REQUIRE(false, "gemm_tc: bad epilogue");
    }
#undef AHA_TC_CASE
    AHA_CUDA_CHECK(cudaGetLastError());
}

}  // namespace aha
