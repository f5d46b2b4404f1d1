// score_head.cuh -- the lm_head over many rows with a log-softmax epilogue (aha_b200_score / aha_b200_score_batch): stage 1 of logprobs.cuh
// computed straight from the tensor-core accumulator, so that no [rows, V] logits block is ever written.
//
//   score_head_kernel, grid (P = lp_parts(V), ceil(M / 128)), 384 threads (kShThreads): CTA (p, y) multiplies the 128 rows [128 y, 128 y + 128) of
//   A = rmsnorm(x) (fp16 hi + lo, the split-activation format of gemm_tc.cuh) by the lm_head rows of vocabulary slice p, [2048 p, 2048 p + 2048),
//   as up to 8 sub-tiles of 256 columns.  The TMA producer walks the sub-tiles' k-blocks through one 3-stage ring without a break, and the
//   consumers run the k-block loop of gemm_tc_kernel<., 256> (tc_mainloop), so every logit is bit-identical to gemm_tc's EPI_STORE output.
//   After each sub-tile a row's quad of lanes (4 lanes x 64 columns) folds its logits into
//     m_p = the running maximum, s_p = sum exp(x - m_p) (each lane rescales its own partial sum when m_p grows),
//     the top n by (logit desc, id asc): a sorted list per row in shared memory; each lane marks its entries that beat the list's n-th
//     entry, then the quad's four lanes take turns inserting their marked entries (sh_select),
//   and the lane holding the row's target column writes that raw logit to tlogit[row].  At the end the quad adds its four sums (xor tree)
//   and writes (m_p, s_p, list) in logprob_partial_rows_kernel's layout; score_final_rows_kernel (logprobs.cuh) is stage 2.
//
// Columns >= V (TMA zero-fills the lm_head rows beyond V) are -inf, sub-tiles without a column < V are skipped, and rows >= M are zero-filled
// and never written.  No atomics, no cross-row reduction: a row's record depends on its own hidden state only, not on M, on its place in
// the tile or on the rows beside it.  n = 0 is its own instantiation without lists or selection.
#pragma once
#include "gemm_tc.cuh"
#include "logprobs.cuh"

namespace aha {

constexpr int kShBN = 256;                   // W rows per sub-tile: gemm_tc_kernel's 128 x 256 tile
constexpr int kShSub = kLpSlice / kShBN;     // sub-tiles per vocabulary slice
// 2 consumer warpgroups + 1 producer warpgroup (one TMA warp, three idle).  A full third warpgroup lets setmaxnreg move registers: the
// block launches at 168 a thread (384 x 168 of the SM's 65536; with 288 threads the cap is also 168, because three warps then share an SM
// sub-partition's 16384), the producers drop to 40 and the consumers rise to 232, enough for the 128-register accumulator, the row state
// and the selection without spilling.
constexpr int kShThreads = 384;

struct ScoreHeadArgs {
    int M, V, K;
    int n;                   // top count (1 .. kLpMaxTop in the TOP instantiation)
    const uint32_t* tgt;     // [M] target id of every row (< V)
    float* part;             // [M][P][kLpPartFloats]  (m_p, s_p, candidate logits)
    int* part_id;            // [M][P][kLpMaxTop]      candidate ids
    float* tlogit;           // [M] raw logit of the target
};

// one sub-tile folded into the running maximum m, this lane's sum s and the target logit of row `row`: H = 0 / 1 picks the accumulator
// entries of the thread's first / second row (columns >= V already -inf); c0 = the column of its entries j = 0
template <int H>
__device__ __forceinline__ void sh_stats(const float (&acc)[kShBN / 2], const ScoreHeadArgs& a, int c0, int q, int row, uint32_t tg, float& m, float& s) {
    // entry k of the row's 64 logits of this sub-tile: column c0 + 8 (k / 2) + k % 2
    auto x = [&](int k) { return acc[4 * (k >> 1) + 2 * H + (k & 1)]; };
    float tmax = -INFINITY;
#pragma unroll
    for (int k = 0; k < kShBN / 4; ++k) tmax = fmaxf(tmax, x(k));
    tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 1));
    tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 2));
    const float mn = fmaxf(m, tmax);
    float sum = s * expf(m - mn);   // the first sub-tile: 0 * exp(-inf) = 0
#pragma unroll
    for (int k = 0; k < kShBN / 4; ++k) sum += expf(x(k) - mn);   // masked columns add exp(-inf) = 0
    s = sum;
    m = mn;
    if (tg - (uint32_t)(c0 - 2 * q) < (uint32_t)kShBN) {
#pragma unroll
        for (int k = 0; k < kShBN / 4; ++k)
            if ((uint32_t)(c0 + 8 * (k >> 1) + (k & 1)) == tg) a.tlogit[row] = x(k);
    }
}

// (v, c) into the sorted list lv / li of n entries when it beats the n-th one; tv / ti: that bar, updated
__device__ __forceinline__ void sh_insert(float* lv, int* li, int n, float v, int c, float& tv, int& ti) {
    if (!(v > -INFINITY && lp_before(v, c, tv, ti))) return;   // (-inf: a column >= V)
    int i = n - 1;
    for (; i > 0 && lp_before(v, c, lv[i - 1], li[i - 1]); --i) { lv[i] = lv[i - 1]; li[i] = li[i - 1]; }
    lv[i] = v; li[i] = c;
    tv = lv[n - 1];
    ti = li[n - 1];
}

// one sub-tile into the sorted lists of the thread's two rows (lv0 / li0, lv1 / li1 in shared memory).  Every lane first checks whether
// any of its entries beats its row's bar (the list's n-th entry); then the quad's four lanes pass over their entries one lane after the
// other, inserting each entry that beats the bar as it rises.  Any insertion order gives the top n under the total (logit desc, id asc)
// order.  A lane runs its pass once, both rows entry by entry, so each accumulator entry dies as soon as it has been visited: the lane waits
// for the lanes before it with q __syncwarp()s and releases the lanes after it with 4 - q.  Apart from the accumulator the state is the
// two bars and one flag.
__device__ __forceinline__ void sh_select(const float (&acc)[kShBN / 2], int n, int c0, int q, float* lv0, int* li0, float* lv1, int* li1) {
    float tv0 = lv0[n - 1], tv1 = lv1[n - 1];
    int ti0 = li0[n - 1], ti1 = li1[n - 1];
    bool any = false;
#pragma unroll
    for (int k = 0; k < kShBN / 4; ++k) {
        const int c = c0 + 8 * (k >> 1) + (k & 1);
        any |= lp_before(acc[4 * (k >> 1) + (k & 1)], c, tv0, ti0) | lp_before(acc[4 * (k >> 1) + 2 + (k & 1)], c, tv1, ti1);
    }
    for (int l = 0; l < q; ++l) __syncwarp();
    if (any) {
        tv0 = lv0[n - 1]; ti0 = li0[n - 1];   // the lanes before this one may have raised the bars
        tv1 = lv1[n - 1]; ti1 = li1[n - 1];
#pragma unroll
        for (int k = 0; k < kShBN / 4; ++k) {
            const int c = c0 + 8 * (k >> 1) + (k & 1);
            sh_insert(lv0, li0, n, acc[4 * (k >> 1) + (k & 1)], c, tv0, ti0);
            sh_insert(lv1, li1, n, acc[4 * (k >> 1) + 2 + (k & 1)], c, tv1, ti1);
        }
    }
    for (int l = q; l < 4; ++l) __syncwarp();
}

template <bool TOP>
__global__ void __launch_bounds__(kShThreads, 1) score_head_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo,
                                                                  const __grid_constant__ CUtensorMap tm_w, ScoreHeadArgs a) {
    constexpr int S = tc_stages<kShBN>(), SB = tc_stage_bytes<kShBN>();
    extern __shared__ __align__(1024) uint8_t sh_smem_raw[];
    uint8_t* tiles = sh_smem_raw + ((1024u - (smem_u32(sh_smem_raw) & 1023u)) & 1023u);   // [stages][A_hi | A_lo | W]
    uint64_t* full = reinterpret_cast<uint64_t*>(tiles + (size_t)S * SB);
    uint64_t* empty = full + S;
    float* cv = reinterpret_cast<float*>(empty + S);             // TOP: [128][kLpMaxTop] every row's sorted candidate logits
    int* ci = reinterpret_cast<int*>(cv + kTcBM * kLpMaxTop);    //      and their ids

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int p = blockIdx.x, m0 = blockIdx.y * kTcBM, v0 = p * kLpSlice;
    const int nkb = a.K / kTcBK;
    const int nsub = min(kShSub, (a.V - v0 + kShBN - 1) / kShBN);   // sub-tiles that hold a column < V

    if (tid == 0) {
        for (int i = 0; i < S; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }   // 8 consumer warps release a slot
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp >= 8) {
        // ======================= TMA producer warpgroup: warp 8 issues the k-blocks of every sub-tile in order, one ring position each
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 8 && lane == 0)
            for (int t = 0, it = 0; t < nsub; ++t)
                for (int kb = 0; kb < nkb; ++kb, ++it) tc_produce<kShBN>(tiles, full, empty, &tm_hi, &tm_lo, &tm_w, it, kb, m0, v0 + t * kShBN);
        return;
    }
    // ======================= consumers: this thread holds columns 2 q + 8 j + {0, 1} of local rows rl and rl + 8
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = warp >> 2, q = lane & 3;
    const int rl = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    float m[2] = {-INFINITY, -INFINITY}, s[2] = {0.f, 0.f};
    uint32_t tg[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) tg[h] = m0 + rl + 8 * h < a.M ? a.tgt[m0 + rl + 8 * h] : 0xffffffffu;
    if (TOP) {
        if (q == 0)
            for (int h = 0; h < 2; ++h)
                for (int k = 0; k < kLpMaxTop; ++k) { cv[(rl + 8 * h) * kLpMaxTop + k] = -INFINITY; ci[(rl + 8 * h) * kLpMaxTop + k] = kLpNone; }
        __syncwarp();
    }
    float acc[kShBN / 2];
    for (int t = 0; t < nsub; ++t) {
        const int n0 = v0 + t * kShBN;
        tc_mainloop<kShBN>(acc, tiles, full, empty, t * nkb, nkb, wg, lane);
        if (lane == 0) mbar_arrive(&empty[(t * nkb + nkb - 1) % S]);   // the accumulator is in registers: the sub-tile's last slot is free
        if (n0 + kShBN > a.V) {   // the sub-tile that crosses V: its columns beyond V (zero-filled W rows) are no entries
#pragma unroll
            for (int j = 0; j < kShBN / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    if (n0 + 2 * q + 8 * j + e >= a.V) { acc[4 * j + e] = -INFINITY; acc[4 * j + 2 + e] = -INFINITY; }
        }
        sh_stats<0>(acc, a, n0 + 2 * q, q, m0 + rl, tg[0], m[0], s[0]);
        sh_stats<1>(acc, a, n0 + 2 * q, q, m0 + rl + 8, tg[1], m[1], s[1]);
        if (TOP) sh_select(acc, a.n, n0 + 2 * q, q, cv + rl * kLpMaxTop, ci + rl * kLpMaxTop, cv + (rl + 8) * kLpMaxTop, ci + (rl + 8) * kLpMaxTop);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float sum = s[h];
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        const int row = m0 + rl + 8 * h;
        if (row >= a.M) continue;
        float* out = a.part + ((size_t)row * gridDim.x + p) * kLpPartFloats;
        if (q == 0) { out[0] = m[h]; out[1] = sum; }
        if (TOP) {
            int* out_id = a.part_id + ((size_t)row * gridDim.x + p) * kLpMaxTop;
            for (int k = q; k < a.n; k += 4) { out[2 + k] = cv[(rl + 8 * h) * kLpMaxTop + k]; out_id[k] = ci[(rl + 8 * h) * kLpMaxTop + k]; }
        }
    }
}

inline size_t score_head_smem_bytes(bool top) {
    return gemm_tc_smem_bytes<kShBN>() + (top ? (size_t)kTcBM * kLpMaxTop * (sizeof(float) + sizeof(int)) : 0);
}
// the > 48 KB dynamic shared memory opt-in (per device, like gemm_tc_init)
inline void score_head_init() {
    AHA_CUDA_CHECK(cudaFuncSetAttribute(score_head_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)score_head_smem_bytes(false)));
    AHA_CUDA_CHECK(cudaFuncSetAttribute(score_head_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)score_head_smem_bytes(true)));
}
inline bool score_head_supported(int K) { return K % kTcBK == 0; }

// stage 1 over M rows already normalised and split (hi / lo [M, K]); tm_w: lm_head [V, K] with 256-row boxes (make_tmap_f16_rows)
inline void score_head_launch(cudaStream_t st, const __half* a_hi, const __half* a_lo, const CUtensorMap& tm_w, const ScoreHeadArgs& a) {
    const CUtensorMap tm_hi = make_tmap_f16(a_hi, (uint64_t)a.M, (uint64_t)a.K);
    const CUtensorMap tm_lo = make_tmap_f16(a_lo, (uint64_t)a.M, (uint64_t)a.K);
    const dim3 grid(lp_parts(a.V), ceil_div(a.M, kTcBM));
    if (a.n > 0) score_head_kernel<true><<<grid, kShThreads, score_head_smem_bytes(true), st>>>(tm_hi, tm_lo, tm_w, a);
    else score_head_kernel<false><<<grid, kShThreads, score_head_smem_bytes(false), st>>>(tm_hi, tm_lo, tm_w, a);
    AHA_CUDA_CHECK(cudaGetLastError());
}

}  // namespace aha
