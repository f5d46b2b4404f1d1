// logprobs.cuh -- token log-probabilities and top alternatives on the device (new design: the reference builds every response with
// `logprobs: None`).  For the token t a step produced from its fp32 logits row x:
//     logprob(t) = x[t] - (M + log sum_j exp(x[j] - M)),  M = max_j x[j]
// i.e. the model's own distribution, taken BEFORE repeat penalty, temperature, top-k and top-p, so that greedy and sampled requests
// report comparable numbers.  top_logprobs: the n (0 <= n <= 20) largest entries ordered by raw logit descending, ties by ascending id
// (the order ArgMax breaks ties in, so a greedy token without penalty is top_ids[0] with the identical logprob).
//
// Two stages over `rows` logits rows (row j belongs to slot act[j]; act == nullptr: one row, slot 0):
//   1. logprob_partial_rows_kernel, grid (P, rows): CTA p covers vocabulary entries [p * kLpSlice, (p + 1) * kLpSlice) and writes its
//      max m_p, s_p = sum exp(x - m_p) (every thread adds its entries in index order, then a fixed shuffle tree, then the warp totals in
//      order) and its top n candidates sorted by (logit desc, id asc).  P = ceil(V / kLpSlice) depends on V only.
//   2. logprob_final_rows_kernel, one CTA per row: M = max m_p, S = sum_p s_p exp(m_p - M) in p order, a P-way merge of the sorted
//      lists, and one aha_logprobs record written in the host layout.  The token is the row's final one (tok[slot]: the sampler's draw
//      for sampled rows, the ArgMax otherwise); its index is DecodeState::n_hist - 1 after a decode step, 0 for a first token.
// Every launch argument is the same at every step, so the pair sits inside a captured step graph.  No atomics: a record depends only
// on its logits row, and the single-request path and both batch widths share these kernels.
#pragma once
#include <climits>
#include <cstddef>

#include "../../include/aha_b200.h"
#include "kernels_common.cuh"

namespace aha {

constexpr int kLpMaxTop = AHA_MAX_TOP_LOGPROBS;
constexpr int kLpSlice = 2048;                          // vocabulary entries per stage-1 CTA
constexpr int kLpThreads = 256;                         // stage 1
constexpr int kLpPerThread = kLpSlice / kLpThreads;     // entries per stage-1 thread (kept in registers)
constexpr int kLpMaxParts = 128;                        // stage 2: one list head per thread -> V <= 128 * 2048
constexpr int kLpPartFloats = 2 + kLpMaxTop;            // m_p, s_p, the candidates' logits
constexpr int kLpNone = INT_MAX;                        // id of an empty candidate (a slice with fewer than n entries)
inline int lp_parts(int V) { return (V + kLpSlice - 1) / kLpSlice; }

// the record is written on the device straight in the layout the host reads
static_assert(sizeof(aha_logprobs) == 184, "aha_logprobs layout");
static_assert(offsetof(aha_logprobs, token) == 0 && offsetof(aha_logprobs, index) == 4 && offsetof(aha_logprobs, logprob) == 8 &&
              offsetof(aha_logprobs, n_top) == 12 && offsetof(aha_logprobs, top_ids) == 16 && offsetof(aha_logprobs, top_logprobs) == 96 &&
              offsetof(aha_logprobs, valid) == 176, "aha_logprobs layout");

__device__ __forceinline__ bool lp_before(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

// (value desc, id asc) maximum over the CTA; every thread gets the winner
template <int NT>
__device__ __forceinline__ void lp_block_best(float& v, int& i, float* rv, int* ri) {
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (lp_before(ov, oi, v, i)) { v = ov; i = oi; }
    }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) { rv[w] = v; ri[w] = i; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < NT / 32; ++k) if (lp_before(rv[k], ri[k], rv[0], ri[0])) { rv[0] = rv[k]; ri[0] = ri[k]; }
    }
    __syncthreads();
    v = rv[0]; i = ri[0];
    __syncthreads();
}

// on[slot]: 0 = the slot's request asked for no record, else 1 + its top count
__global__ void __launch_bounds__(kLpThreads) logprob_partial_rows_kernel(const float* __restrict__ logits, int ld, int V, const int* __restrict__ act,
                                                                          const int* __restrict__ on, float* __restrict__ part, int* __restrict__ part_id) {
    __shared__ float rv[kLpThreads / 32];
    __shared__ int ri[kLpThreads / 32];
    const int row = blockIdx.y, p = blockIdx.x, tid = threadIdx.x;
    const int slot = act ? act[row] : 0;
    const int n = on[slot] - 1;
    if (n < 0) return;
    const float* x = logits + (size_t)row * ld;
    const int i0 = p * kLpSlice + tid;
    float v[kLpPerThread];
    float mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < kLpPerThread; ++k) {
        const int i = i0 + k * kLpThreads;
        v[k] = i < V ? x[i] : -INFINITY;
        mx = fmaxf(mx, v[k]);
    }
    int dummy = 0;
    lp_block_best<kLpThreads>(mx, dummy, rv, ri);
    float s = 0.f;
    if (mx != -INFINITY) {
#pragma unroll
        for (int k = 0; k < kLpPerThread; ++k) if (i0 + k * kLpThreads < V) s += expf(v[k] - mx);
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((tid & 31) == 0) rv[tid >> 5] = s;
    __syncthreads();
    float* out = part + ((size_t)row * gridDim.x + p) * kLpPartFloats;
    int* out_id = part_id + ((size_t)row * gridDim.x + p) * kLpMaxTop;
    if (tid == 0) {
        float t = 0.f;
        for (int w = 0; w < kLpThreads / 32; ++w) t += rv[w];
        out[0] = mx; out[1] = t;
    }
    __syncthreads();
    // top n of the slice: n rounds of a CTA-wide (logit desc, id asc) maximum over the entries not taken yet
    unsigned taken = 0u;
    for (int r = 0; r < n; ++r) {
        float bv = -INFINITY;
        int bi = kLpNone;
#pragma unroll
        for (int k = 0; k < kLpPerThread; ++k) {
            const int i = i0 + k * kLpThreads;
            if (i < V && !((taken >> k) & 1u) && lp_before(v[k], i, bv, bi)) { bv = v[k]; bi = i; }
        }
        lp_block_best<kLpThreads>(bv, bi, rv, ri);
        if (bi != kLpNone && (bi - p * kLpSlice) % kLpThreads == tid) taken |= 1u << ((bi - p * kLpSlice) / kLpThreads);
        if (tid == 0) { out[2 + r] = bv; out_id[r] = bi; }
    }
}

// stage 2 of one row, run by a CTA of kLpMaxParts threads: the row's P slice results pr / pi (n candidates each) -> record `rec` for token t
// at `index`; xt: the row's logit of t (nullptr: t is outside the vocabulary, logprob -inf)
__device__ __forceinline__ void lp_final_record(const float* __restrict__ pr, const int* __restrict__ pi, int P, int n, uint32_t t, const float* xt,
                                                int index, aha_logprobs* __restrict__ rec) {
    __shared__ float rv[kLpMaxParts / 32];
    __shared__ int ri[kLpMaxParts / 32];
    __shared__ float s_lse;
    const int tid = threadIdx.x;
    if (tid == 0) {
        float M = -INFINITY;
        for (int p = 0; p < P; ++p) M = fmaxf(M, pr[(size_t)p * kLpPartFloats]);
        float S = 0.f;
        for (int p = 0; p < P; ++p) {
            const float sp = pr[(size_t)p * kLpPartFloats + 1];
            if (sp > 0.f) S += sp * expf(pr[(size_t)p * kLpPartFloats] - M);
        }
        const float lse = M + logf(S);
        s_lse = lse;
        rec->token = t;
        rec->index = (uint32_t)index;
        rec->logprob = xt ? *xt - lse : -INFINITY;
        rec->n_top = (uint32_t)n;
        rec->valid = 1u;
        rec->reserved = 0u;
    }
    __syncthreads();
    const float lse = s_lse;
    // P-way merge of the sorted candidate lists: thread p holds the head of list p
    int head = 0;
    for (int r = 0; r < n; ++r) {
        float bv = -INFINITY;
        int bi = kLpNone;
        if (tid < P && head < n) { bv = pr[(size_t)tid * kLpPartFloats + 2 + head]; bi = pi[(size_t)tid * kLpMaxTop + head]; }
        lp_block_best<kLpMaxParts>(bv, bi, rv, ri);
        if (tid < P && head < n && pi[(size_t)tid * kLpMaxTop + head] == bi) ++head;
        if (tid == 0) { rec->top_ids[r] = bi == kLpNone ? 0u : (uint32_t)bi; rec->top_logprobs[r] = bv - lse; }
    }
    for (int r = n + tid; r < kLpMaxTop; r += kLpMaxParts) { rec->top_ids[r] = 0u; rec->top_logprobs[r] = 0.f; }
}

__global__ void __launch_bounds__(kLpMaxParts) logprob_final_rows_kernel(const float* __restrict__ logits, int ld, int V, int P, const int* __restrict__ act,
                                                                         const int* __restrict__ on, const float* __restrict__ part,
                                                                         const int* __restrict__ part_id, const uint32_t* __restrict__ tok,
                                                                         const DecodeState* __restrict__ st, int first, aha_logprobs* __restrict__ out,
                                                                         int by_index, int out_cap) {
    const int row = blockIdx.x;
    const int slot = act ? act[row] : 0;
    const int n = on[slot] - 1;
    if (n < 0) return;
    const int index = first ? 0 : st[slot].n_hist - 1;
    if (by_index && (index < 0 || index >= out_cap)) return;
    const uint32_t t = tok[slot];
    lp_final_record(part + (size_t)row * P * kLpPartFloats, part_id + (size_t)row * P * kLpMaxTop, P, n, t,
                    t < (uint32_t)V ? logits + (size_t)row * ld + t : nullptr, index, out + (by_index ? index : slot));
}

// stage 2 of scored rows (score_head.cuh): row r's record for token tgt[r] at index[r] goes to out[r].  Its logit is tlogit[r] (written by
// score_head_kernel) or, when tlogit is nullptr, logits[r * ld + tgt[r]] (a logits block from gemm_tc).  tgt[r] < V.
__global__ void __launch_bounds__(kLpMaxParts) score_final_rows_kernel(const float* __restrict__ part, const int* __restrict__ part_id, int P, int n,
                                                                       const uint32_t* __restrict__ tgt, const float* __restrict__ tlogit,
                                                                       const float* __restrict__ logits, int ld, const uint32_t* __restrict__ index,
                                                                       aha_logprobs* __restrict__ out) {
    const int row = blockIdx.x;
    const uint32_t t = tgt[row];
    lp_final_record(part + (size_t)row * P * kLpPartFloats, part_id + (size_t)row * P * kLpMaxTop, P, n, t,
                    tlogit ? tlogit + row : logits + (size_t)row * ld + t, (int)index[row], out + row);
}

// the two stages over `rows` logits rows (ld floats apart); part / part_id: [rows][lp_parts(V)] candidate lists
inline void logprobs_rows(cudaStream_t stream, const float* logits, int ld, int V, int rows, const int* act, const int* on, float* part, int* part_id,
                          const uint32_t* tok, const DecodeState* st, int first, aha_logprobs* out, int by_index, int out_cap) {
    const int P = lp_parts(V);
    logprob_partial_rows_kernel<<<dim3(P, rows), kLpThreads, 0, stream>>>(logits, ld, V, act, on, part, part_id);
    logprob_final_rows_kernel<<<rows, kLpMaxParts, 0, stream>>>(logits, ld, V, P, act, on, part, part_id, tok, st, first, out, by_index, out_cap);
}

}  // namespace aha
