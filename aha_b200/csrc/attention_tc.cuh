// attention_tc.cuh -- flash attention on the Hopper tensor cores (wgmma + TMA) for head_dim 64 (the ViT segments of
// Qwen3-VL: 8160 tokens x 16 heads per layer for a 1080p image, and the audio encoder) and 128 (LLM prefill, causal, GQA).
//
// Same contract as flash_attn_kernel / flash_attn_mma_kernel: softmax(Q K^T * scale) V per head, never materialising
// S x S (reference: Qwen3VLVisionAttention::forward, src/models/qwen3vl/model.rs:232-278;
// eager_attention_forward, src/models/common/modules.rs:757-813; NaiveAttention, modules.rs:201-242).
// Accuracy: like every tensor-core path here, operands are split x = hi + lo (fp16 each) and each product is formed as
// hi*hi + hi*lo + lo*hi into the same fp32 accumulator.
//
// One CTA = 128 queries of one head, KV tiles of 64 tokens, 288 threads:
//   warp 8 (one elected lane): TMA loads -- Q once, then K and V^T tiles into a two-stage ring (full / empty mbarriers), so
//     tile t + 1 streams in while tile t is computed;
//   warpgroups 0, 1: 64 query rows each.  S[64 x 64] = Q K^T by wgmma from shared memory (3 products per k-step), the online
//     softmax in fp32 on the accumulator fragment (a row lives in 4 lanes: two shuffles per reduction), then P = hi + lo is
//     repacked in registers as the A operand of PV[64 x HD] += P V (wgmma with A from registers, B = the V^T tile), so P never
//     touches shared memory.  The two warpgroups overlap each other's softmax and MMAs.
// V is staged transposed ([head][d][token], written by the split pass) so that every shared-memory operand is K-major with
// the one descriptor form gemm_tc.cuh uses.
#pragma once
#include "attention_mma.cuh"
#include "gemm_tc.cuh"

namespace aha {

constexpr int kFaBQ = 128, kFaBKV = 64, kFaThreads = 288;
constexpr int kFaWork = 5;   // ints per work item of the varlen kernel

// fp16 row-major [rows, cols] matrix, box = box_rows x 64 halfs (128 bytes), 128-byte swizzle, OOB reads as zero
inline CUtensorMap make_tmap_f16_box(const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
    CUtensorMap m;
    const cuuint64_t gdim[2] = {cols, rows};
    const cuuint64_t gstride[1] = {cols * 2};
    const cuuint32_t box[2] = {64u, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = tmap_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    AHA_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
    return m;
}

// ---- split pass: q, k -> packed fp16 hi | lo [head][token][64]; v -> TRANSPOSED hi | lo [head][64][skv_pad] (zero padded) ----
struct SplitTcArgs {
    FlashArgs f;
    __half *q_hi, *q_lo, *k_hi, *k_lo, *vt_hi, *vt_lo;
    int nheads, nkv, skv_pad;
};
// blockIdx.y: 0 = q, 1 = k (one row per block, like split_qkv_kernel); 2 = v: 64-token tile per block, transposed through shared memory
template <int HD>
__global__ void split_qkv_tc_kernel(SplitTcArgs s) {
    const int which = blockIdx.y;
    if (which < 2) {
        const int S = which == 0 ? s.f.Sq : s.f.Skv, H = which == 0 ? s.nheads : s.nkv;
        // HD / 4 threads x float4 per row, 512 / HD rows per pass of the 128 threads
        constexpr int TPR = HD / 4, RPP = 128 / TPR;
        for (size_t row = (size_t)blockIdx.x * RPP + threadIdx.x / TPR; row < (size_t)S * H; row += (size_t)gridDim.x * RPP) {
            const int head = (int)(row / S), tok = (int)(row % S);
            const float* src = which == 0 ? s.f.q + (size_t)(s.f.q0 + tok) * s.f.q_tok_stride + (size_t)head * s.f.q_head_stride
                                          : s.f.kv.k + s.f.kv.off(s.f.kv0 + tok, head);
            __half* hi = (which == 0 ? s.q_hi : s.k_hi) + row * HD;
            __half* lo = (which == 0 ? s.q_lo : s.k_lo) + row * HD;
            {
                const int c4 = (threadIdx.x % TPR) * 4;
                const float4 v = *reinterpret_cast<const float4*>(src + c4);
                uint32_t h0, l0, h1, l1;
                split2(v.x, v.y, h0, l0);
                split2(v.z, v.w, h1, l1);
                *reinterpret_cast<uint2*>(hi + c4) = make_uint2(h0, h1);
                *reinterpret_cast<uint2*>(lo + c4) = make_uint2(l0, l1);
            }
        }
        return;
    }
    __shared__ float tile[64][HD + 1];
    const int tiles_per_head = s.skv_pad / 64;
    for (int job = blockIdx.x; job < s.nkv * tiles_per_head; job += gridDim.x) {
        const int head = job / tiles_per_head, t0 = (job % tiles_per_head) * 64;
        __syncthreads();
        for (int idx = threadIdx.x; idx < 64 * HD; idx += blockDim.x) {
            const int r = idx / HD, c = idx % HD;
            tile[r][c] = (t0 + r < s.f.Skv) ? s.f.kv.v[s.f.kv.off(s.f.kv0 + t0 + r, head) + c] : 0.f;
        }
        __syncthreads();
        for (int idx = threadIdx.x; idx < HD * 64; idx += blockDim.x) {
            const int d = idx / 64, r = idx % 64;
            const float x = tile[r][d];
            const __half h = __float2half_rn(x);
            const size_t o = ((size_t)head * HD + d) * s.skv_pad + t0 + r;
            s.vt_hi[o] = h;
            s.vt_lo[o] = __float2half_rn(x - __half2float(h));
        }
    }
}

struct FlashTcArgs {
    float* out; size_t o_tok_stride, o_head_stride;
    __half *out_hi, *out_lo;   // when set: the output goes out as fp16 hi + lo halves (operand format of the next GEMM) instead of fp32
    int Sq, Skv, q0, groups;
    float scaling;
    const int* work = nullptr;   // VARLEN: [gridDim.x][kFaWork] = (q_start, q_len, kv_start, kv_len, qt0), one 128-query tile of one segment per item
};

__device__ __forceinline__ float ex2_approx(float x) {   // 2^x on the MUFU, flush-to-zero (inputs here are <= 0; -inf -> 0)
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}


template <int HD>
__device__ __forceinline__ void fa_mma_pv(float (&o)[HD / 2], const uint32_t (&a)[4], uint64_t db) {
    if constexpr (HD == 64) wgmma_rs_n64(o, a, db);
    else wgmma_rs_n128(o, a, db);
}

// VARLEN: independent segments packed back to back (Sq: the pack's query rows, Skv: its gathered key rows).  blockIdx.x picks a work item;
// inside it the queries are rows [q_start, q_start + q_len) and the keys rows [kv_start, kv_start + kv_len), so Sq = q_len, Skv = kv_len and
// the causal diagonal shifts by kv_len - q_len (a segment whose first kv_len - q_len keys are a cached prefix), while the KV tile grid and the
// masks stay relative to the segment.  So each query row goes through the same operations in the same order as when its segment runs alone:
// keys of the next segment that enter the last tile are masked (kj >= kv_len or kj > qi + shift) and their V rows are multiplied by P = 0.
// kv_start must be a multiple of 16 tokens (flash_attn_tc_varlen).
template <int HD, bool CAUSAL, bool VARLEN = false>
__global__ void __launch_bounds__(kFaThreads, 1) flash_attn_tc_kernel(const __grid_constant__ CUtensorMap tm_qh, const __grid_constant__ CUtensorMap tm_ql,
                                                                     const __grid_constant__ CUtensorMap tm_kh, const __grid_constant__ CUtensorMap tm_kl,
                                                                     const __grid_constant__ CUtensorMap tm_vh, const __grid_constant__ CUtensorMap tm_vl, FlashTcArgs a) {
    constexpr int BQ = kFaBQ, BKV = kFaBKV, KB = HD / 64;   // KB: 64-half k-blocks per head row (one TMA box each)
    constexpr int kQBytes = BQ * HD * 2, kKBytes = BKV * HD * 2, kVBytes = HD * BKV * 2;   // head_dim 64: 16, 8, 8 KB
    constexpr int kQBlk = BQ * 128, kKBlk = BKV * 128;       // bytes of one k-block of the Q / K tile
    constexpr int kStage = 2 * kKBytes + 2 * kVBytes;        // Kh | Kl | Vh | Vl
    extern __shared__ __align__(1024) uint8_t fa_tc_smem_raw[];
    uint8_t* base = fa_tc_smem_raw + ((1024u - (smem_u32(fa_tc_smem_raw) & 1023u)) & 1023u);
    uint8_t* Qh = base;
    uint8_t* Ql = Qh + kQBytes;
    uint8_t* ring = Ql + kQBytes;                            // [2][kStage]
    uint64_t* bars = reinterpret_cast<uint64_t*>(ring + 2 * kStage);
    uint64_t *bar_q = bars, *full = bars + 1, *empty = bars + 3;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int head = blockIdx.y, kvh = head / a.groups;
    int q_start = 0, kv_start = 0, Sq = a.Sq, Skv = a.Skv, qt0 = blockIdx.x * BQ;
    if constexpr (VARLEN) {
        const int* w = a.work + kFaWork * blockIdx.x;
        q_start = __ldg(w); Sq = __ldg(w + 1); kv_start = __ldg(w + 2); Skv = __ldg(w + 3); qt0 = __ldg(w + 4);
    }
    const int causal_shift = Skv - Sq;
    int kv_end = Skv;
    if (CAUSAL) kv_end = min(Skv, qt0 + BQ + causal_shift);
    const int ntiles = (kv_end + BKV - 1) / BKV;

    if (tid == 0) {
        mbar_init(bar_q, 1);
        for (int i = 0; i < 2; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }   // 8 consumer warps release a stage
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        // ======================= producer lane: Q once, then the K / V^T tiles through the two-stage ring
        if (lane == 0) {
            const int qrow = head * a.Sq + q_start + qt0, krow = kvh * a.Skv + kv_start, vrow = kvh * HD;
            mbar_expect_tx(bar_q, 2 * kQBytes);
#pragma unroll
            for (int kb = 0; kb < KB; ++kb) {
                tma_load_2d(Qh + kb * kQBlk, &tm_qh, kb * 64, qrow, bar_q);
                tma_load_2d(Ql + kb * kQBlk, &tm_ql, kb * 64, qrow, bar_q);
            }
            for (int t = 0; t < ntiles; ++t) {
                const int s = t & 1;
                mbar_wait(&empty[s], ((t >> 1) & 1) ^ 1);
                uint8_t* st = ring + s * kStage;
                mbar_expect_tx(&full[s], kStage);
#pragma unroll
                for (int kb = 0; kb < KB; ++kb) {
                    tma_load_2d(st + kb * kKBlk, &tm_kh, kb * 64, krow + t * BKV, &full[s]);
                    tma_load_2d(st + kKBytes + kb * kKBlk, &tm_kl, kb * 64, krow + t * BKV, &full[s]);
                }
                tma_load_2d(st + 2 * kKBytes, &tm_vh, kv_start + t * BKV, vrow, &full[s]);
                tma_load_2d(st + 2 * kKBytes + kVBytes, &tm_vl, kv_start + t * BKV, vrow, &full[s]);
            }
        }
        return;
    }

    // ======================= consumer warpgroup wg: query rows qt0 + 64 wg + [0, 64); this thread holds rows r0 and r0 + 8
    const int wg = warp >> 2;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int c0 = 2 * (lane & 3);
    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // m in the log2 domain: exp(x) = 2^(x * log2 e); l: this thread's partial row sums
    const float scale_log2 = a.scaling * 1.4426950408889634f;
    const uint32_t qh = smem_u32(Qh) + wg * 64 * 128, ql = smem_u32(Ql) + wg * 64 * 128;
    mbar_wait(bar_q, 0);
    for (int t = 0; t < ntiles; ++t) {
        const int s = t & 1, kt0 = t * BKV;
        mbar_wait(&full[s], (t >> 1) & 1);
        const uint32_t kh = smem_u32(ring + s * kStage), kl = kh + kKBytes, vh = kh + 2 * kKBytes, vl = vh + kVBytes;
        float sc[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) sc[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < HD / 16; ++ks) {   // k-block ks / 4 of the tiles, 32 bytes per K = 16 step inside its 128-byte swizzle atom
            const uint32_t qa = (ks >> 2) * kQBlk + (ks & 3) * 32, ka = (ks >> 2) * kKBlk + (ks & 3) * 32;
            wgmma_ss_n64(sc, wgmma_desc_sw128(qh + qa), wgmma_desc_sw128(kh + ka));
            wgmma_ss_n64(sc, wgmma_desc_sw128(qh + qa), wgmma_desc_sw128(kl + ka));
            wgmma_ss_n64(sc, wgmma_desc_sw128(ql + qa), wgmma_desc_sw128(kh + ka));
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(sc);
        // masking only on the tiles that can need it (the last one / the causal diagonal); the max on raw scores (scale > 0 commutes
        // with max); scale and max subtraction in ONE fma feeding ex2.approx
        const bool mask_tile = (kt0 + BKV > Skv) || (CAUSAL && kt0 + BKV - 1 > qt0 + wg * 64 + causal_shift);
        float alpha[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int qi = qt0 + r0 + 8 * r;
            float rmax = -INFINITY;
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    float& x = sc[4 * j + 2 * r + c];
                    const int kj = kt0 + 8 * j + c0 + c;
                    if (mask_tile && (kj >= Skv || (CAUSAL && kj > qi + causal_shift))) x = -INFINITY;
                    rmax = fmaxf(rmax, x);
                }
            rmax = fmaxf(rmax, __shfl_xor_sync(0xffffffffu, rmax, 1));
            rmax = fmaxf(rmax, __shfl_xor_sync(0xffffffffu, rmax, 2));
            const float mn = fmaxf(m[r], rmax * scale_log2);
            const float mu = (mn == -INFINITY) ? 0.f : mn;
            alpha[r] = ex2_approx(m[r] - mu);
            float rs = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    float& x = sc[4 * j + 2 * r + c];
                    x = ex2_approx(fmaf(x, scale_log2, -mu));
                    rs += x;
                }
            l[r] = l[r] * alpha[r] + rs;
            m[r] = mn;
        }
#pragma unroll
        for (int j = 0; j < HD / 8; ++j) {
            o[4 * j] *= alpha[0]; o[4 * j + 1] *= alpha[0];
            o[4 * j + 2] *= alpha[1]; o[4 * j + 3] *= alpha[1];
        }
        // P -> fp16 hi | lo A fragments: k-chunk kk (kv columns 16 kk .. 16 kk + 15) is accumulator registers 8 kk .. 8 kk + 7
        uint32_t ph[4][4], pl[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
            for (int q = 0; q < 4; ++q) split2(sc[8 * kk + 2 * q], sc[8 * kk + 2 * q + 1], ph[kk][q], pl[kk][q]);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const uint32_t adv = kk * 32;
            fa_mma_pv<HD>(o, ph[kk], wgmma_desc_sw128(vh + adv));
            fa_mma_pv<HD>(o, ph[kk], wgmma_desc_sw128(vl + adv));
            fa_mma_pv<HD>(o, pl[kk], wgmma_desc_sw128(vh + adv));
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);   // this warp's reads of the stage have retired
    }
    if constexpr (VARLEN) {   // read again rather than held through the KV loop (keeps the register count of the plain kernel)
        const int* w = a.work + kFaWork * blockIdx.x;
        asm volatile("ld.global.nc.s32 %0, [%1];" : "=r"(q_start) : "l"(w));
        asm volatile("ld.global.nc.s32 %0, [%1];" : "=r"(Sq) : "l"(w + 1));
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
        const int qi = qt0 + r0 + 8 * r;
        if (qi >= Sq) continue;
        const float inv = 1.0f / l[r];
        const size_t off = (size_t)(a.q0 + q_start + qi) * a.o_tok_stride + (size_t)head * a.o_head_stride + c0;
#pragma unroll
        for (int j = 0; j < HD / 8; ++j) {
            const float x = o[4 * j + 2 * r] * inv, y = o[4 * j + 2 * r + 1] * inv;
            if (a.out_hi) {
                uint32_t h, lo;
                split2(x, y, h, lo);
                *reinterpret_cast<uint32_t*>(a.out_hi + off + 8 * j) = h;
                *reinterpret_cast<uint32_t*>(a.out_lo + off + 8 * j) = lo;
            } else {
                *reinterpret_cast<float2*>(a.out + off + 8 * j) = make_float2(x, y);
            }
        }
    }
}

template <int HD>
inline size_t flash_tc_smem_bytes() { return (size_t)(2 * kFaBQ * HD * 2 + 2 * (2 * kFaBKV * HD * 2 + 2 * HD * kFaBKV * 2)) + 5 * sizeof(uint64_t) + 1024; }
inline int flash_tc_skv_pad(int Skv) { return ceil_div(Skv, 64) * 64; }
// workspace halfs: q hi|lo + k hi|lo ([head][token][HD]) + v^T hi|lo ([head][HD][skv_pad])
template <int HD>
inline size_t flash_tc_ws_halfs(const FlashArgs& a, int nheads) {
    const int nkv = nheads / a.groups;
    return 2 * ((size_t)nheads * a.Sq + (size_t)nkv * a.Skv + (size_t)nkv * flash_tc_skv_pad(a.Skv)) * HD;
}
inline void flash_attn_tc_init() {
    AHA_CUDA_CHECK(cudaFuncSetAttribute(flash_attn_tc_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)flash_tc_smem_bytes<64>()));
    AHA_CUDA_CHECK(cudaFuncSetAttribute(flash_attn_tc_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)flash_tc_smem_bytes<64>()));
    AHA_CUDA_CHECK(cudaFuncSetAttribute(flash_attn_tc_kernel<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)flash_tc_smem_bytes<128>()));
    AHA_CUDA_CHECK(cudaFuncSetAttribute(flash_attn_tc_kernel<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)flash_tc_smem_bytes<128>()));
    AHA_CUDA_CHECK(cudaFuncSetAttribute(flash_attn_tc_kernel<128, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)flash_tc_smem_bytes<128>()));
}
// The split pass over all of `a`, then the tensor maps and kernel arguments of the attention launch.
struct FlashTcLaunch {
    CUtensorMap tqh, tql, tkh, tkl, tvh, tvl;
    FlashTcArgs m;
};
template <int HD>
inline FlashTcLaunch flash_tc_prepare(cudaStream_t st, const FlashArgs& a, int nheads, __half* ws, int num_sms) {
    const int nkv = nheads / a.groups, pad = flash_tc_skv_pad(a.Skv);
    SplitTcArgs sp;
    sp.f = a; sp.nheads = nheads; sp.nkv = nkv; sp.skv_pad = pad;
    const size_t nq = (size_t)nheads * a.Sq * HD, nk = (size_t)nkv * a.Skv * HD, nv = (size_t)nkv * HD * pad;
    sp.q_hi = ws; sp.q_lo = ws + nq; sp.k_hi = ws + 2 * nq; sp.k_lo = sp.k_hi + nk; sp.vt_hi = sp.k_lo + nk; sp.vt_lo = sp.vt_hi + nv;
    const unsigned blocks = (unsigned)std::min<size_t>(std::max<size_t>(ceil_div((int)std::max((size_t)nheads * a.Sq, (size_t)nkv * a.Skv), 512 / HD), (size_t)nkv * (pad / 64)), (size_t)num_sms * 32);
    split_qkv_tc_kernel<HD><<<dim3(blocks, 3), 128, 0, st>>>(sp);
    FlashTcLaunch L;
    L.tqh = make_tmap_f16_box(sp.q_hi, (uint64_t)nheads * a.Sq, HD, kFaBQ); L.tql = make_tmap_f16_box(sp.q_lo, (uint64_t)nheads * a.Sq, HD, kFaBQ);
    L.tkh = make_tmap_f16_box(sp.k_hi, (uint64_t)nkv * a.Skv, HD, kFaBKV); L.tkl = make_tmap_f16_box(sp.k_lo, (uint64_t)nkv * a.Skv, HD, kFaBKV);
    L.tvh = make_tmap_f16_box(sp.vt_hi, (uint64_t)nkv * HD, (uint64_t)pad, HD); L.tvl = make_tmap_f16_box(sp.vt_lo, (uint64_t)nkv * HD, (uint64_t)pad, HD);
    FlashTcArgs& m = L.m;
    m.out = a.out; m.o_tok_stride = a.o_tok_stride; m.o_head_stride = a.o_head_stride; m.out_hi = a.out_hi; m.out_lo = a.out_lo;
    m.Sq = a.Sq; m.Skv = a.Skv; m.q0 = a.q0; m.groups = a.groups; m.scaling = a.scaling;
    return L;
}
// head_dim 64 (ViT, audio encoder: 96 KB of shared memory) and 128 (LLM prefill, causal, GQA, paged KV: 192 KB).  `ws`: at least flash_tc_ws_halfs<HD>() halfs.
template <int HD>
inline void flash_attn_tc(cudaStream_t st, const FlashArgs& a, int nheads, bool causal, __half* ws, int num_sms) {
    if (a.Sq == 0) return;
    const FlashTcLaunch L = flash_tc_prepare<HD>(st, a, nheads, ws, num_sms);
    dim3 grid(ceil_div(a.Sq, kFaBQ), nheads);
    const size_t smem = flash_tc_smem_bytes<HD>();
    if (causal) flash_attn_tc_kernel<HD, true><<<grid, kFaThreads, smem, st>>>(L.tqh, L.tql, L.tkh, L.tkl, L.tvh, L.tvl, L.m);
    else flash_attn_tc_kernel<HD, false><<<grid, kFaThreads, smem, st>>>(L.tqh, L.tql, L.tkh, L.tkl, L.tvh, L.tvl, L.m);
    AHA_CUDA_CHECK(cudaGetLastError());
}
// Causal attention over independent segments packed back to back (head_dim 128; packed embeddings, packed admission).  `a` covers the
// whole pack (Sq query rows, Skv key rows; q0 = kv0 = 0): the split pass runs once over it, then one launch of (n_work, nheads) CTAs.  work:
// device [n_work][kFaWork] = (q_start, q_len, kv_start, kv_len, qt0), one item per 128-query tile of every segment; a segment without a
// cached prefix has q_start = kv_start and q_len = kv_len.  `ws`: at least flash_tc_ws_halfs<128>(a) halfs.  kv_start is the innermost TMA
// coordinate of the V^T tiles, so it must keep them on a 16-byte boundary: callers lay segments out on multiples of 16 tokens.
inline void flash_attn_tc_varlen(cudaStream_t st, const FlashArgs& a, int nheads, const int* work, int n_work, __half* ws, int num_sms) {
    if (n_work == 0) return;
    AHA_REQUIRE(a.Sq <= a.Skv && a.q0 == 0 && a.kv0 == 0, "flash_attn_tc_varlen: the pack's key rows start at 0 and hold at least its query rows");
    FlashTcLaunch L = flash_tc_prepare<128>(st, a, nheads, ws, num_sms);
    L.m.work = work;
    flash_attn_tc_kernel<128, true, true><<<dim3(n_work, nheads), kFaThreads, flash_tc_smem_bytes<128>(), st>>>(L.tqh, L.tql, L.tkh, L.tkl, L.tvh, L.tvl, L.m);
    AHA_CUDA_CHECK(cudaGetLastError());
}

}  // namespace aha
