// sampling.cuh -- the sampler of the decode loop on the device: repeat penalty, temperature softmax, top-k / top-p /
// multinomial draw from a ChaCha12 stream, so that non-greedy requests never move the 608 KB logits row to the host.
//
// Replaces (reference): sample_and_push (src/models/common/generate.rs:70-86), get_logit_processor and
// use_repeat_penalty (src/models/common/sample.rs:7-60) and, behind them, candle-transformers' LogitsProcessor /
// apply_repeat_penalty and rand's StdRng / WeightedIndex.  The arithmetic is restated line by line in oracle/sample.py,
// including the two places where it deliberately fixes an order the crates leave to their implementation (blocked fp32
// sums over the vocabulary; top-k candidates sorted by descending probability, ties by ascending id).
//
// One CTA of 1024 threads per token (the vocabulary row, 0.6 MB, sits in L2); every sum over the vocabulary is formed over
// 256-element chunks left to right (thread c owns chunk c) and then over the chunk totals left to right (thread 0), i.e.
// it is deterministic and identical to the oracle's `blocked_sum`.
#pragma once
#include <cstdint>

#include "../../include/aha_b200.h"
#include "common.cuh"
#include "kernels_common.cuh"

namespace aha {

constexpr int kSampleThreads = 1024;
constexpr int kSampleChunk = 256;
constexpr int kSampleMaxTopK = 1024;
constexpr int kSampleMaxRows = 64;          // rows of one sample_rows_kernel launch: the widest batch session
constexpr const char* kSampleWeightsError =
    "sampler: the token weights are all zero or not finite (rand::distr::weighted::WeightedIndex::new fails in the reference)";

enum SampleMode { SAMPLE_ARGMAX = 0, SAMPLE_ALL = 1, SAMPLE_TOPP = 2, SAMPLE_TOPK = 3, SAMPLE_TOPK_TOPP = 4 };

struct SampleArgs {
    const float* logits;     // [V] raw logits of the step
    float* work;             // [V] scratch (penalised logits -> probabilities)
    int V;
    int mode;
    float inv_temp;          // (float)(1.0 / temperature)
    float top_p;
    int top_k;
    float penalty;           // 1.0 = off
    int last_n;              // repeat_last_n (0 = off)
    uint32_t key[8];         // ChaCha key = seed_from_u64(seed)
    DecodeState* st;         // token / n_hist / n_draws live here so that steps chain on the device
    uint32_t* history;       // [hist_cap] tokens generated so far in this request (the repeat-penalty context)
    int hist_cap;
    uint32_t* token_out;
    int overwrite;           // 1: the step kernel already pushed its argmax token (history[n_hist - 1], st->token): replace it
    int* error;              // set to 1 when the weights are all zero / not finite (WeightedIndex::new fails in the reference)
    // token automaton of a constrained request (aha_b200_fsm_create; null: unconstrained): state s allows the ascending tokens
    // fsm_tok[fsm_off[s] .. fsm_off[s + 1]), and fsm_next[j] is the state after fsm_tok[j].  The current state is st->fsm_state.
    const uint64_t* fsm_off;
    const uint32_t* fsm_tok;
    const uint32_t* fsm_next;
    // logit rules (aha_b200_rules_create): bias_vals[j] is added to the logit of bias_ids[j] (distinct ids); with a count row `cnt` ([V],
    // zero between draws; null: no penalties), every token generated before this draw loses frequency per occurrence and presence once
    const uint32_t* bias_ids;
    const float* bias_vals;
    int n_bias;
    float presence;
    float frequency;
    int* cnt;
};

// ---- StdRng: ChaCha12 block `counter` of the stream keyed by `key`, word `w` (rand_chacha: 64-bit counter in words 12-13, stream 0)
__device__ __forceinline__ uint32_t rotl32(uint32_t x, int n) { return (x << n) | (x >> (32 - n)); }
__device__ inline uint32_t chacha12_word(const uint32_t* key, unsigned long long counter, int w) {
    uint32_t s[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, key[0], key[1], key[2], key[3], key[4], key[5], key[6], key[7],
                      (uint32_t)counter, (uint32_t)(counter >> 32), 0u, 0u};
    uint32_t x[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) x[i] = s[i];
#define AHA_QR(a, b, c, d)                                                                   \
    x[a] += x[b]; x[d] = rotl32(x[d] ^ x[a], 16); x[c] += x[d]; x[b] = rotl32(x[b] ^ x[c], 12); \
    x[a] += x[b]; x[d] = rotl32(x[d] ^ x[a], 8);  x[c] += x[d]; x[b] = rotl32(x[b] ^ x[c], 7);
#pragma unroll 1
    for (int r = 0; r < 6; ++r) {
        AHA_QR(0, 4, 8, 12) AHA_QR(1, 5, 9, 13) AHA_QR(2, 6, 10, 14) AHA_QR(3, 7, 11, 15)
        AHA_QR(0, 5, 10, 15) AHA_QR(1, 6, 11, 12) AHA_QR(2, 7, 8, 13) AHA_QR(3, 4, 9, 14)
    }
#undef AHA_QR
    uint32_t out = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) if (i == w) out = x[i] + s[i];
    return out;
}
// Uniform<f32>: 23 random mantissa bits with exponent 0, minus one
__device__ __forceinline__ float uniform01_from_word(uint32_t w) { return __uint_as_float((w >> 9) | 0x3f800000u) - 1.0f; }

struct SampleSmem {
    float csum[kSampleThreads];      // chunk totals
    float cpre[kSampleThreads];      // exclusive prefix of the chunk totals
    int ccnt[kSampleThreads];        // chunk tie counts -> exclusive prefix
    float cand_p[kSampleMaxTopK];
    int cand_i[kSampleMaxTopK];
    unsigned hist[256];
    float redf[32];
    int redi[32];
    float bc_f[4];
    int bc_i[4];
};

// Blocked sum of f(i) over i < V: thread c adds its chunk left to right, thread 0 adds the chunk totals left to right.
// Leaves the chunk totals in s.csum and their exclusive prefix in s.cpre; returns the total to every thread.
template <typename F>
__device__ float blocked_sum_dev(SampleSmem& s, int V, F f) {
    const int nch = (V + kSampleChunk - 1) / kSampleChunk;
    const int c = threadIdx.x;
    if (c < nch) {
        float t = 0.f;
        const int i0 = c * kSampleChunk, i1 = min(V, i0 + kSampleChunk);
        for (int i = i0; i < i1; ++i) t += f(i);
        s.csum[c] = t;
    }
    __syncthreads();
    if (c == 0) {
        float run = 0.f;
        for (int j = 0; j < nch; ++j) { s.cpre[j] = run; run += s.csum[j]; }
        s.bc_f[0] = run;
    }
    __syncthreads();
    const float tot = s.bc_f[0];
    __syncthreads();
    return tot;
}

// WeightedIndex over w(i) with the blocked cumulative sums of the oracle's `blocked_pick`; every thread gets the index.
template <typename F>
__device__ int blocked_pick_dev(SampleSmem& s, int V, F w, float draw01, int* error) {
    const float total = blocked_sum_dev(s, V, w);
    const int nch = (V + kSampleChunk - 1) / kSampleChunk;
    if (!(total > 0.f) || !isfinite(total)) {
        if (threadIdx.x == 0) *error = 1;
        return 0;
    }
    const float u = draw01 * total;
    // chunks whose last cumulative value is <= u lie entirely before the pick (the cumulative sequence is monotone)
    int before = 0;
    if ((int)threadIdx.x < nch && s.cpre[threadIdx.x] + s.csum[threadIdx.x] <= u) before = 1;
    before = __syncthreads_count(before);
    if (threadIdx.x == 0) {
        int idx = V - 1;
        if (before < nch) {
            const int i0 = before * kSampleChunk, i1 = min(V, i0 + kSampleChunk);
            const float pre = s.cpre[before];
            float run = 0.f;
            idx = i1 - 1;
            for (int i = i0; i < i1; ++i) {
                run += w(i);
                if (!(pre + run <= u)) { idx = i; break; }
            }
        }
        s.bc_i[0] = idx;
    }
    __syncthreads();
    const int r = s.bc_i[0];
    __syncthreads();
    return r;
}

// The sampler of one token, run by a CTA of kSampleThreads threads: sample_kernel (one request) and sample_rows_kernel (a wide batch step)
// share it, so a request draws the same token whichever of the two runs it.
__device__ __forceinline__ void sample_dev(const SampleArgs& a, SampleSmem& s) {
    const int tid = threadIdx.x, V = a.V;
    float* p = a.work;
    const int n_hist = a.st->n_hist;
    const int n_ctx = a.overwrite ? n_hist - 1 : n_hist;     // tokens generated before this one
    const unsigned draw = a.st->n_draws;
    const bool fsm = a.fsm_off != nullptr;
    if (!fsm) {
        for (int i = tid; i < V; i += kSampleThreads) p[i] = a.logits[i];
    } else {
        // masked logits: -inf, then the allowed entries scattered from the state's row (O(V + allowed), no per-state bitmap)
        const uint32_t fs = a.st->fsm_state;
        const uint64_t f0 = a.fsm_off[fs], f1 = a.fsm_off[fs + 1];
        for (int i = tid; i < V; i += kSampleThreads) p[i] = -INFINITY;
        __syncthreads();
        for (uint64_t j = f0 + tid; j < f1; j += kSampleThreads) { const uint32_t t = a.fsm_tok[j]; p[t] = a.logits[t]; }
    }
    __syncthreads();
    // ---- logit bias: one fp32 add per listed token (a masked entry stays -inf: the values are finite)
    if (a.n_bias > 0) {
        for (int j = tid; j < a.n_bias; j += kSampleThreads) { const uint32_t t = a.bias_ids[j]; p[t] = __fadd_rn(p[t], a.bias_vals[j]); }
        __syncthreads();
    }
    // occurrence counts of the generated tokens, scattered now and consumed after the repeat penalty (frequency / presence)
    const bool counts = a.cnt != nullptr && n_ctx > 0;
    if (counts)
        for (int t = tid; t < n_ctx; t += kSampleThreads) { const uint32_t tok = a.history[t]; if (tok < (uint32_t)V) atomicAdd(&a.cnt[tok], 1); }
    // ---- penalised logits (use_repeat_penalty: every distinct token of the last `last_n` generated ones, once; a masked entry stays -inf)
    if (!(a.penalty == 1.0f || a.last_n == 0) && n_ctx > 0) {
        const int start = max(0, n_ctx - a.last_n);
        for (int t = start + tid; t < n_ctx; t += kSampleThreads) {
            const uint32_t tok = a.history[t];
            bool first = true;
            for (int u = start; u < t; ++u) if (a.history[u] == tok) { first = false; break; }
            if (first && tok < (uint32_t)V) {
                const float x = p[tok];
                if (!(fsm && x == -INFINITY)) p[tok] = x >= 0.f ? x / a.penalty : x * a.penalty;
            }
        }
        __syncthreads();
    }
    // ---- frequency and presence: the first position to take a token's count applies y - c * frequency - presence once (product and
    // differences rounded separately, as the oracle states them), and the exchange leaves the count row zero for the next draw
    if (counts) {
        __syncthreads();
        for (int t = tid; t < n_ctx; t += kSampleThreads) {
            const uint32_t tok = a.history[t];
            if (tok >= (uint32_t)V) continue;
            const int c = atomicExch(&a.cnt[tok], 0);
            if (c > 0) p[tok] = __fsub_rn(__fsub_rn(p[tok], __fmul_rn((float)c, a.frequency)), a.presence);
        }
        __syncthreads();
    }
    int token = 0;
    if (a.mode == SAMPLE_ARGMAX) {
        float best = -INFINITY;
        int bi = 0x7fffffff;
        for (int i = tid; i < V; i += kSampleThreads) { const float v = p[i]; if (v > best || (v == best && i < bi)) { best = v; bi = i; } }
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
        }
        if ((tid & 31) == 0) { s.redf[tid >> 5] = best; s.redi[tid >> 5] = bi; }
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < kSampleThreads / 32; ++w) if (s.redf[w] > best || (s.redf[w] == best && s.redi[w] < bi)) { best = s.redf[w]; bi = s.redi[w]; }
            s.bc_i[1] = (bi < 0 || bi >= V) ? 0 : bi;
            if (fsm && !(best > -INFINITY)) *a.error = 1;      // no allowed token has a finite logit
        }
        __syncthreads();
        token = s.bc_i[1];
    } else {
        // ---- prs = softmax(logits * (1 / temperature)), blocked denominator
        float mx = -INFINITY;
        for (int i = tid; i < V; i += kSampleThreads) { const float x = p[i] * a.inv_temp; p[i] = x; mx = fmaxf(mx, x); }
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if ((tid & 31) == 0) s.redf[tid >> 5] = mx;
        __syncthreads();
        if (tid == 0) { float m = s.redf[0]; for (int w = 1; w < kSampleThreads / 32; ++w) m = fmaxf(m, s.redf[w]); s.bc_f[1] = m; }
        __syncthreads();
        mx = s.bc_f[1];
        for (int i = tid; i < V; i += kSampleThreads) p[i] = expf(p[i] - mx);
        __syncthreads();
        const float denom = blocked_sum_dev(s, V, [&](int i) { return p[i]; });
        for (int i = tid; i < V; i += kSampleThreads) p[i] = p[i] / denom;
        __syncthreads();
        const float u01 = uniform01_from_word(chacha12_word(a.key, draw >> 4, (int)(draw & 15u)));
        const uint32_t* key = reinterpret_cast<const uint32_t*>(p);      // p >= 0: the bit pattern orders like the value
        // candle's own shortcuts to the plain multinomial: TopP with p outside (0, 1) (the TopP arm of LogitsProcessor::sample_f) and
        // TopK with k >= V (sample_topk).  TopKThenTopP with k >= V has none: sample_topk_topp runs sample_topp, which with p = 1 still
        // drops the smallest entries once the fp32 sum of the kept ones reaches 1 (and keeps every entry when p > 1).
        const bool plain = a.mode == SAMPLE_ALL || (a.mode == SAMPLE_TOPP && (a.top_p <= 0.f || a.top_p >= 1.f)) ||
                           (a.mode == SAMPLE_TOPK && a.top_k >= V);
        const bool nucleus = !plain && (a.mode == SAMPLE_TOPP || (a.mode == SAMPLE_TOPK_TOPP && a.top_k >= V));
        if (plain) {
            token = blocked_pick_dev(s, V, [&](int i) { return p[i]; }, u01, a.error);
        } else if (nucleus) {
            // sample_topp: T = smallest key with A(T) = blocked_sum(p[key > T]) < top_p (31 halvings of the key range)
            uint32_t lo = 0u, hi = 0x7f800000u;
            while (lo < hi) {
                const uint32_t mid = lo + ((hi - lo) >> 1);
                const float A = blocked_sum_dev(s, V, [&](int i) { return key[i] > mid ? p[i] : 0.f; });
                if (A < a.top_p) hi = mid; else lo = mid + 1u;
            }
            const uint32_t T = lo;
            const float A = blocked_sum_dev(s, V, [&](int i) { return key[i] > T ? p[i] : 0.f; });
            // ties at T are kept in id order while A + j * value < top_p: j = number of ties with a smaller id
            const int nch = (V + kSampleChunk - 1) / kSampleChunk;
            if (tid < nch) {
                int cnt = 0;
                const int i0 = tid * kSampleChunk, i1 = min(V, i0 + kSampleChunk);
                for (int i = i0; i < i1; ++i) cnt += key[i] == T;
                s.ccnt[tid] = cnt;
            }
            __syncthreads();
            if (tid == 0) { int run = 0; for (int j = 0; j < nch; ++j) { const int c = s.ccnt[j]; s.ccnt[j] = run; run += c; } }
            __syncthreads();
            const float tv = __uint_as_float(T);
            if (tid < nch) {   // zero the rejected entries in place: the chunk owner walks its ties in id order
                int j = s.ccnt[tid];
                const int i0 = tid * kSampleChunk, i1 = min(V, i0 + kSampleChunk);
                for (int i = i0; i < i1; ++i) {
                    const uint32_t k = key[i];
                    if (k < T) p[i] = 0.f;
                    // product and sum rounded separately, as the oracle states them (a contracted FMA rounds once and can decide a tie differently)
                    else if (k == T) { if (!(__fadd_rn(A, __fmul_rn((float)j, tv)) < a.top_p)) p[i] = 0.f; ++j; }
                }
            }
            __syncthreads();
            token = blocked_pick_dev(s, V, [&](int i) { return p[i]; }, u01, a.error);
        } else {
            // ---- top-k: radix select of the k-th largest key (4 passes of 8 bits, integer histograms)
            const int k = a.top_k;
            uint32_t prefix = 0u, pmask = 0u;
            int remaining = k;      // rank (1-based, from the top) still to locate inside the current prefix bucket
            for (int shift = 24; shift >= 0; shift -= 8) {
                for (int b = tid; b < 256; b += kSampleThreads) s.hist[b] = 0u;
                __syncthreads();
                for (int i = tid; i < V; i += kSampleThreads) {
                    const uint32_t kk = key[i];
                    if ((kk & pmask) == prefix) atomicAdd(&s.hist[(kk >> shift) & 255u], 1u);
                }
                __syncthreads();
                if (tid == 0) {
                    int run = 0, b = 255;
                    for (; b > 0; --b) { if (run + (int)s.hist[b] >= remaining) break; run += (int)s.hist[b]; }
                    s.bc_i[2] = b; s.bc_i[3] = remaining - run;
                }
                __syncthreads();
                prefix |= (uint32_t)s.bc_i[2] << shift; pmask |= 255u << shift; remaining = s.bc_i[3];
                __syncthreads();
            }
            const uint32_t Kk = prefix;          // the k-th largest key; `remaining` of the entries equal to it belong to the top k (lowest ids)
            const int nch = (V + kSampleChunk - 1) / kSampleChunk;
            if (tid < nch) {
                int cnt = 0;
                const int i0 = tid * kSampleChunk, i1 = min(V, i0 + kSampleChunk);
                for (int i = i0; i < i1; ++i) cnt += key[i] == Kk;
                s.ccnt[tid] = cnt;
            }
            if (tid == 0) s.bc_i[0] = 0;
            __syncthreads();
            if (tid == 0) { int run = 0; for (int j = 0; j < nch; ++j) { const int c = s.ccnt[j]; s.ccnt[j] = run; run += c; } }
            __syncthreads();
            if (tid < nch) {
                int j = s.ccnt[tid];
                const int i0 = tid * kSampleChunk, i1 = min(V, i0 + kSampleChunk);
                for (int i = i0; i < i1; ++i) {
                    const uint32_t kk = key[i];
                    const bool take = kk > Kk || (kk == Kk && j++ < remaining);
                    if (take) { const int pos = atomicAdd(&s.bc_i[0], 1); if (pos < kSampleMaxTopK) { s.cand_p[pos] = p[i]; s.cand_i[pos] = i; } }
                }
            }
            __syncthreads();
            // sort the k candidates by (probability descending, id ascending): bitonic network over the padded power of two
            int n2 = 1;
            while (n2 < k) n2 <<= 1;
            for (int i = k + tid; i < n2; i += kSampleThreads) { s.cand_p[i] = -1.f; s.cand_i[i] = 0x7fffffff; }
            __syncthreads();
            for (int size = 2; size <= n2; size <<= 1) {
                for (int stride = size >> 1; stride > 0; stride >>= 1) {
                    for (int i = tid; i < n2; i += kSampleThreads) {
                        const int j = i ^ stride;
                        if (j > i) {
                            const bool up = (i & size) == 0;       // ascending position = earlier in the final order
                            const float pi = s.cand_p[i], pj = s.cand_p[j];
                            const int ii = s.cand_i[i], ij = s.cand_i[j];
                            const bool i_after_j = pi < pj || (pi == pj && ii > ij);
                            if (i_after_j == up) { s.cand_p[i] = pj; s.cand_p[j] = pi; s.cand_i[i] = ij; s.cand_i[j] = ii; }
                        }
                    }
                    __syncthreads();
                }
            }
            if (tid == 0) {
                float total = 0.f;
                for (int j = 0; j < k; ++j) total += s.cand_p[j];          // sum_p, left to right
                if (a.mode == SAMPLE_TOPK_TOPP && !(a.top_p <= 0.f || a.top_p >= total)) {
                    float cum = 0.f;   // sample_topp on the candidate list
                    for (int j = 0; j < k; ++j) { if (cum >= a.top_p) s.cand_p[j] = 0.f; else cum += s.cand_p[j]; }
                    total = 0.f;
                    for (int j = 0; j < k; ++j) total += s.cand_p[j];
                }
                int idx = k - 1;
                if (!(total > 0.f) || !isfinite(total)) { *a.error = 1; idx = 0; }
                else {
                    const float u = u01 * total;
                    float run = 0.f;
                    for (int j = 0; j < k; ++j) { run += s.cand_p[j]; if (!(run <= u)) { idx = j; break; } }
                }
                s.bc_i[1] = s.cand_i[idx];
            }
            __syncthreads();
            token = s.bc_i[1];
        }
    }
    if (tid == 0) {
        if (token < 0 || token >= V) token = 0;
        *a.token_out = (uint32_t)token;
        DecodeState* st = a.st;
        if (a.mode != SAMPLE_ARGMAX) st->n_draws = draw + 1u;
        if (a.overwrite) {
            st->token = (uint32_t)token;
            if (n_hist >= 1 && n_hist - 1 < a.hist_cap) a.history[n_hist - 1] = (uint32_t)token;
        }
        if (fsm) {   // advance: the token's entry in the state's sorted row; a token the state does not allow is an error, never a transition
            const uint32_t fs = st->fsm_state;
            const uint64_t f1 = a.fsm_off[fs + 1];
            uint64_t lo = a.fsm_off[fs], hi = f1;
            while (lo < hi) { const uint64_t mid = lo + ((hi - lo) >> 1); if (a.fsm_tok[mid] < (uint32_t)token) lo = mid + 1; else hi = mid; }
            if (lo < f1 && a.fsm_tok[lo] == (uint32_t)token) st->fsm_state = a.fsm_next[lo];
            else *a.error = 1;
        }
    }
}

__global__ void __launch_bounds__(kSampleThreads) sample_kernel(SampleArgs a) {
    __shared__ SampleSmem s;
    sample_dev(a, s);
}

// Row-indexed sampler of a wide batch step: CTA j samples logits row j for the slot act[j] with that slot's SampleArgs (args[slot]); a
// row whose request does not sample (on[slot] == 0) returns at once.  Which slots run is read from device memory, so one launch serves
// every composition of the same width.
__global__ void __launch_bounds__(kSampleThreads) sample_rows_kernel(const SampleArgs* __restrict__ args, const int* __restrict__ on,
                                                                     const int* __restrict__ act, const float* logits, int ld, int overwrite) {
    __shared__ SampleSmem s;
    const int slot = act[blockIdx.x];
    if (!on[slot]) return;
    SampleArgs a = args[slot];
    a.logits = logits + (size_t)blockIdx.x * ld;
    a.overwrite = overwrite;
    sample_dev(a, s);
}

// ----------------------------------------------------------------------------------------------------------------------- host side
// A request's sampler.  inactive = plain ArgMax, which the step kernels compute themselves.  `args` holds the parameters only; the buffers
// (logits, work, state, history, token, error flag) are filled where the sampler is bound to a row (TextModel::bind_sampler).
struct Sampler {
    bool active = false;
    SampleArgs args{};
    uint32_t fsm_start = 0;      // the automaton's start state: a first token is drawn from it
    uint32_t fsm_id = 0;         // the automaton's id on the handle (0: unconstrained)
    uint32_t rules_id = 0;       // the logit-rules object's id on the handle (0: none)
    bool counts = false;         // frequency or presence penalty: the row it is bound to needs a count row
};

// a token automaton in device memory (aha_b200_fsm_create)
struct TokenFsmDev {
    const uint64_t* off = nullptr;
    const uint32_t* tok = nullptr;
    const uint32_t* next = nullptr;
    uint32_t start = 0;
};

// the logit rules of a request with the bias list in device memory (aha_b200_rules_create)
struct LogitRulesDev {
    const uint32_t* ids = nullptr;
    const float* vals = nullptr;
    int n_bias = 0;
    float presence = 0.f;
    float frequency = 0.f;
};

// get_logit_processor (sample.rs:7-38): the Sampling a request's parameters select, checked against what the device sampler supports
// A constrained request (fsm != null) or one with logit rules always samples on the device, greedy included: ArgMax over its
// allowed tokens and transformed logits.
inline Sampler make_sampler(const aha_gen_params& p, int V, const TokenFsmDev* fsm = nullptr, const LogitRulesDev* rules = nullptr) {
    const bool has_t = !(p.temperature < 1e-7f);
    const bool has_k = p.top_k > 0, has_p = p.top_p > 0.f;
    const int mode = !has_t ? SAMPLE_ARGMAX : !has_k ? (has_p ? SAMPLE_TOPP : SAMPLE_ALL) : (has_p ? SAMPLE_TOPK_TOPP : SAMPLE_TOPK);
    const bool pen = !(p.repeat_penalty == 1.0f || p.repeat_last_n == 0);
    Sampler s;
    s.active = mode != SAMPLE_ARGMAX || pen || fsm != nullptr || rules != nullptr;
    if (!s.active) return s;
    AHA_REQUIRE(V <= kSampleThreads * kSampleChunk, "vocabulary too large for the device sampler");
    AHA_REQUIRE(!(mode == SAMPLE_TOPK || mode == SAMPLE_TOPK_TOPP) || p.top_k >= 1, "top_k must be >= 1");
    AHA_REQUIRE(!(mode == SAMPLE_TOPK || mode == SAMPLE_TOPK_TOPP) || p.top_k >= V || p.top_k <= kSampleMaxTopK,
                "top_k > 1024 is not supported by the device sampler");
    SampleArgs& a = s.args;
    a.V = V; a.mode = mode;
    a.inv_temp = mode == SAMPLE_ARGMAX ? 1.0f : (float)(1.0 / (double)p.temperature);
    a.top_p = p.top_p; a.top_k = p.top_k; a.penalty = p.repeat_penalty; a.last_n = p.repeat_last_n;
    if (fsm) { a.fsm_off = fsm->off; a.fsm_tok = fsm->tok; a.fsm_next = fsm->next; s.fsm_start = fsm->start; }
    if (rules) {
        a.bias_ids = rules->ids; a.bias_vals = rules->vals; a.n_bias = rules->n_bias;
        a.presence = rules->presence; a.frequency = rules->frequency;
        // both zero: y - fl(c * 0) - 0 = y, so the counting pass is skipped and no count row is needed
        s.counts = rules->presence != 0.f || rules->frequency != 0.f;
    }
    // rand_core::SeedableRng::seed_from_u64: eight PCG32 outputs fill the 32-byte ChaCha seed
    uint64_t stt = p.seed;
    for (int i = 0; i < 8; ++i) {
        stt = stt * 6364136223846793005ull + 11634580027462260723ull;
        const uint32_t xs = (uint32_t)(((stt >> 18) ^ stt) >> 27);
        const uint32_t rot = (uint32_t)(stt >> 59);
        a.key[i] = (xs >> rot) | (xs << ((32u - rot) & 31u));
    }
    return s;
}

}  // namespace aha
