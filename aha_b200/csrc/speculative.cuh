// speculative.cuh -- speculative decoding: verify passes of R = max_draft + 1 rows per request through one weight stream, for one request
// (aha_b200_generate_speculative) or for the speculative requests of a wide batch session beside its plain ones (aha_b200_batch_step_spec)
// (new design; the reference decodes one token per forward_step, src/models/common/generate.rs:115-159, and ignores the `prediction` field
// of its request schema, src/params/chat.rs:102-105).
//
// A pass runs R rows of each speculative request:
//     row 0       the last emitted token, at position pos (DecodeState::pos of the request)
//     row r >= 1  draft r, at position pos + r
// and emits the longest run the request's own sampler reproduces.  A launch holds np plain rows first (one per plain session slot; np = 0
// for a single request), then every speculative request's R rows.  Its launches (captured into a CUDA graph per launch shape) are
//     [draft]    spec_draft_kernel        one CTA per request: drafts of this pass -> the request's history behind the emitted tokens, one
//                                         DecodeState per verify row
//     [embed]    embed_rows_kernel        plain row j <- its slot's token; verify row r <- its token
// then per layer
//     [qkv]      wide projection          over all rows (gemv_wide.cuh: a row's bits do not depend on the other rows)
//     [attn]     decode_attn_batch_kernel over the plain rows, as in a plain step
//     [K/V]      spec_qk_rows_kernel      verify rows: q/k RMSNorm, RoPE at pos + r + rope_delta, K/V stored through the row's own request's
//                                         page table for every row BEFORE any row attends
//     [attn]     spec_verify_attn_kernel + spec_verify_merge_kernel over the verify rows
//     [o_proj], [gate/up + SwiGLU], [down]   wide projections over all rows
// then one lm_head and ArgMax stage 1 over all rows; the plain rows' ArgMax stage 2, sampler and records advance their slots (a plain step);
// the verify rows' do not advance anything, and
//     [accept]   spec_accept_kernel       one CTA per request: compares samples with drafts, emits the run, applies EOS / max_tokens,
//                                         advances the request.
// Which slots and requests a launch holds -- the row -> request map, each request's first row, R, control block and page table -- is read
// from device memory, so a graph serves every composition of the same (plain rows, requests, verify rows, records) shape.
//
// Exactness.  Row r is sampled with the request's sampler at draw index n_draws + r and with the repeat-penalty context "history
// followed by drafts 1..r" (the drafts sit in the history buffer right behind the emitted tokens, and row r's DecodeState says
// n_hist = emitted + r).  If the first j drafts equal the samples of the rows before them, rows 0..j computed exactly what j + 1
// sequential steps of the same kernels compute, so the pass emits their j + 1 samples and consumes j + 1 draws.  Every row is computed
// independently of its index, of R and of the other rows of the launch (column-invariant projections, the row-invariant attention below,
// row-indexed head kernels), so a request's ids and log-probability records do not depend on the drafts, max_draft, graphs or its
// neighbours: a wrong draft costs time, never the answer.  K/V of rejected positions are stale; the next pass's rows overwrite them before
// any row reads them, and no row reads past its own position.
//
// Draft rule (spec_draft_kernel; restated in tests/spec_ref.py).  e[0..E) = the emitted tokens.  For n = min(ngram, E) down to 1, and
// for each source in order -- first the caller's prediction p[0..P), then, with prompt lookup, the text "prompt followed by e[0..E)" --
// take the largest i with src[i .. i+n) == e[E-n .. E) and i + n < |src| (at least one token follows).  The first (n, source) that has
// one gives the drafts src[i+n .. min(i+n+max_draft, |src|)).  No match: no drafts.  Rows behind the drafts are padded with token 0 and
// their samples are ignored.
#pragma once
#include <array>

#include "attention.cuh"
#include "batch_decode.cuh"
#include "kernels_common.cuh"
#include "logprobs.cuh"
#include "sampling.cuh"

namespace aha {

constexpr int kSpecMaxRows = AHA_SPEC_MAX_ROWS;   // max_draft + 1
constexpr int kSpecChunk = 2 * kPage;       // KV positions per verify-attention chunk: a fixed multiple of the page, never ctx / splits
constexpr int kSpecDefaultNgram = 3;
constexpr int kSpecMaxNgram = 8;
constexpr int kSpecDraftThreads = 256;
constexpr int kSpecAttnThreads = 256;

// device-side control block of a speculative request: set by the host when the request starts, advanced by the accept kernel
struct SpecCtl {
    const uint32_t* pred; int n_pred;        // the caller's prediction (may be empty)
    const uint32_t* prompt; int n_prompt;    // prompt lookup: the prompt (n_prompt = 0 without lookup)
    const uint32_t* stop; int n_stop;        // the handle's stop ids
    int max_tokens;                          // sample_len: tokens the request may emit, the first included
    int ngram;
    uint32_t draw_step;                      // draws per token: 1 when the sampler draws, 0 for ArgMax
    int lp;                                  // records asked: the accept kernel copies the accepted rows' records
    int done;                                // EOS or max_tokens reached: later passes change nothing
    int n_draft;                             // drafts of the current pass
    uint32_t passes, drafted, accepted;
    DecodeState* req;                        // the request's state: token = last emitted, pos = its position, n_hist = E emitted tokens
    uint32_t* hist;                          // its history (the emitted tokens, then this pass's drafts)
    // the records of the tokens a pass emits: token k of the pass (output index E + k) goes to lp_out[E + k] when lp_by_index, else to
    // lp_out[k]; the last one also to *lp_last when it is set
    aha_logprobs* lp_out; int lp_by_index;
    aha_logprobs* lp_last;
};

// a speculative request of a launch: its control block, its page table and its verify rows [row0, row0 + R); ctx = the position of its
// last row + 1, written by spec_draft_kernel so that the attention finds everything it needs in one load
struct SpecReq {
    SpecCtl* ctl;
    const int* table;
    int row0, R;
    int ctx;
};

// ---------------------------------------------------------------------------------------------------------------------------- draft
__device__ __forceinline__ uint32_t spec_src_at(const SpecCtl& c, const uint32_t* hist, int src, int i) {
    if (src == 0) return c.pred[i];
    return i < c.n_prompt ? c.prompt[i] : hist[i - c.n_prompt];
}

// One CTA per request (reqs[blockIdx.x]); rows: the launch's verify-row states, the request's at [row0, row0 + R).
__global__ void __launch_bounds__(kSpecDraftThreads) spec_draft_kernel(SpecReq* __restrict__ reqs, DecodeState* __restrict__ rows) {
    __shared__ int red[kSpecDraftThreads / 32];
    __shared__ int s_src, s_start, s_nd;
    const SpecReq q = reqs[blockIdx.x];
    SpecCtl* ctl = q.ctl;
    const SpecCtl c = *ctl;
    const DecodeState st = *c.req;
    uint32_t* hist = c.hist;
    const int R = q.R;
    rows += q.row0;
    const int E = st.n_hist, tid = threadIdx.x;
    if (tid == 0) { s_src = 0; s_start = 0; s_nd = 0; }
    __syncthreads();
    if (!c.done) {
        bool found = false;
        for (int n = min(c.ngram, E); n >= 1 && !found; --n) {
            for (int src = 0; src < 2 && !found; ++src) {
                const int L = src == 0 ? c.n_pred : (c.n_prompt > 0 ? c.n_prompt + E : 0);
                int best = -1;
                for (int i = tid; i + n < L; i += kSpecDraftThreads) {
                    bool eq = true;
                    for (int k = 0; k < n && eq; ++k) eq = spec_src_at(c, hist, src, i + k) == hist[E - n + k];
                    if (eq) best = i;    // i grows along the thread's stride: the last match is its largest
                }
                for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
                if ((tid & 31) == 0) red[tid >> 5] = best;
                __syncthreads();
                if (tid == 0) {
                    int b = -1;
                    for (int w = 0; w < kSpecDraftThreads / 32; ++w) b = max(b, red[w]);
                    if (b >= 0) { s_src = src; s_start = b + n; s_nd = min(R - 1, L - (b + n)); }
                }
                __syncthreads();
                found = s_nd > 0;
                __syncthreads();
            }
        }
    }
    const int nd = s_nd, src = s_src, start = s_start;
    for (int r = tid; r < R; r += kSpecDraftThreads) {
        uint32_t tok = st.token;
        if (r > 0) {
            tok = r - 1 < nd ? spec_src_at(c, hist, src, start + r - 1) : 0u;
            hist[E + r - 1] = tok;
        }
        DecodeState s = st;
        s.token = tok;
        s.pos = st.pos + r;
        s.n_hist = E + r;
        s.n_draws = st.n_draws + (uint32_t)r * c.draw_step;
        rows[r] = s;
    }
    if (tid == 0) { ctl->n_draft = nd; reqs[blockIdx.x].ctx = st.pos + R; }
}

// --------------------------------------------------------------------------------------------------------------- row K/V append
struct SpecRowArgs {
    float* qkv; int ld;                      // [rows][ld] raw projections of the verify rows; q is normalised and rotated in place
    const float* qw; const float* kw; float eps;
    const float* inv_freq;
    const DecodeState* rows;                 // row r's position and rope_delta
    const int* const* row_table;             // row r's request's page table, which it writes through
    float* kbase; float* vbase;              // layer bases into the pool (writable)
    KVSrc kv;                                // layer bases; the row's request's table replaces page_table
    int nh, nkv;
};

// grid (ceil((nh + 2 nkv) / 8), rows), 256 threads: warp = one head slot of one row (q heads, k heads, v heads), the arithmetic of
// decode_attn_body's prologue
template <int HD>
__global__ void __launch_bounds__(256) spec_qk_rows_kernel(SpecRowArgs a) {
    static_assert(HD == 128, "speculative decoding is specialised for head_dim 128");
    const int lane = threadIdx.x & 31, slot = blockIdx.x * 8 + (threadIdx.x >> 5), r = blockIdx.y;
    if (slot >= a.nh + 2 * a.nkv) return;
    KVSrc kv = a.kv;
    kv.page_table = a.row_table[r];
    float* row = a.qkv + (size_t)r * a.ld;
    const DecodeState st = a.rows[r];
    const int pos = st.pos;
    const float4 x = *reinterpret_cast<const float4*>(row + (size_t)slot * HD + lane * 4);
    if (slot >= a.nh + a.nkv) {
        const size_t off = kv.off(pos, slot - a.nh - a.nkv) + lane * 4;
        *reinterpret_cast<float4*>(a.vbase + off) = make_float4(kv_store_round(x.x), kv_store_round(x.y), kv_store_round(x.z), kv_store_round(x.w));
        return;
    }
    const bool is_q = slot < a.nh;
    const float rpos = (float)(pos + st.rope_delta);
    float ss = x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
    ss = warp_sum(ss);
    const float inv = 1.0f / sqrtf(ss / (float)HD + a.eps);
    const float4 w = *reinterpret_cast<const float4*>((is_q ? a.qw : a.kw) + lane * 4);
    float n[4] = {x.x * inv * w.x, x.y * inv * w.y, x.z * inv * w.z, x.w * inv * w.w};
    float o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float partner = __shfl_xor_sync(0xffffffffu, n[e], 16);  // element d +- 64
        const int d = lane * 4 + e;
        const int j = d & (HD / 2 - 1);
        const float ang = rpos * a.inv_freq[j];
        const float rot = (d < HD / 2) ? -partner : partner;
        o[e] = n[e] * cosf(ang) + rot * sinf(ang);
    }
    if (is_q) {
        *reinterpret_cast<float4*>(row + (size_t)slot * HD + lane * 4) = make_float4(o[0], o[1], o[2], o[3]);
    } else {
        const size_t off = kv.off(pos, slot - a.nh) + lane * 4;
        *reinterpret_cast<float4*>(a.kbase + off) = make_float4(kv_store_round(o[0]), kv_store_round(o[1]), kv_store_round(o[2]), kv_store_round(o[3]));
    }
}

// ------------------------------------------------------------------------------------------------------------ verify attention
// Multi-query split-KV attention of each request's R rows over its own page table.  CTA (x, kvh, q) serves request q: it takes the chunks
// c = x, x + gridDim.x, ... of kSpecChunk positions [c * kSpecChunk, (c + 1) * kSpecChunk) of that request, stages the chunk's K and V in
// shared memory once and serves every (row, q head) pair of the request's KV group from it, so a KV page is read once per pass, not once
// per row.  Row r attends to positions 0 .. pos_r (= its own position: causal inside the draft).
//
// Invariant: row r's output depends only on its own position and its q -- not on its index, R, its request's index or the other
// requests of the launch.
//   * Chunk boundaries are fixed multiples of the page, not a function of the context length, of R or of the grid.
//   * Inside a chunk a warp walks the row's positions lo .. min(hi, pos_r + 1) - 1 in order, one online-softmax update each; positions
//     past pos_r are never visited, so they leave m / l / acc bit-unchanged (there is no masked update, hence no -inf - -inf).
//     Which warp or CTA serves a row does not matter: every warp runs the same sequence of operations.
//   * spec_verify_merge_kernel merges the row's chunks 0 .. pos_r / kSpecChunk in index order.
struct SpecAttnArgs {
    const float* q; int ldq;                 // verify row r, head h: q + r * ldq + h * HD (normalised and rotated)
    KVSrc kv;                                // layer bases; request q's table replaces page_table
    const SpecReq* reqs;                     // [gridDim.z] the requests of the launch
    const DecodeState* rows;                 // verify-row positions
    float* partial;                          // [rows][nh][max_chunks][spec_part_stride(HD)]: acc (unnormalised), m, l
    int max_chunks;
    float* out; int ldo;                     // verify row r, head h: out + r * ldo + h * HD
    int nh, nkv;
    float scaling;
};

// a chunk partial: acc[HD], m, l, padded to 16 bytes so that acc is stored as float4
__host__ __device__ constexpr int spec_part_stride(int hd) { return hd + 4; }

template <int HD>
inline size_t spec_attn_smem_bytes() { return (size_t)2 * kSpecChunk * HD * sizeof(float); }

template <int HD>
__global__ void __launch_bounds__(kSpecAttnThreads) spec_verify_attn_kernel(SpecAttnArgs a) {
    static_assert(HD == 128, "speculative decoding is specialised for head_dim 128");
    constexpr int NW = kSpecAttnThreads / 32;
    extern __shared__ __align__(16) float spec_smem[];
    float* Ks = spec_smem;
    float* Vs = Ks + kSpecChunk * HD;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, kvh = blockIdx.y;
    const SpecReq rq = a.reqs[blockIdx.z];
    KVSrc kv = a.kv;
    kv.page_table = rq.table;
    const DecodeState* rows = a.rows + rq.row0;
    const int G = a.nh / a.nkv, Q = rq.R * G;
    const int ctx = rq.ctx;
    const int nchunks = (ctx + kSpecChunk - 1) / kSpecChunk;
    for (int c = blockIdx.x; c < nchunks; c += gridDim.x) {
        const int lo = c * kSpecChunk, hi = min(ctx, lo + kSpecChunk);
        __syncthreads();   // the previous chunk is consumed
        for (int idx = tid; idx < (hi - lo) * (HD / 4); idx += kSpecAttnThreads) {
            const int t = idx / (HD / 4), c4 = idx % (HD / 4);
            const size_t off = kv.off(lo + t, kvh) + c4 * 4;
            *reinterpret_cast<float4*>(Ks + t * HD + c4 * 4) = *reinterpret_cast<const float4*>(kv.k + off);
            *reinterpret_cast<float4*>(Vs + t * HD + c4 * 4) = *reinterpret_cast<const float4*>(kv.v + off);
        }
        __syncthreads();
        for (int qi = warp; qi < Q; qi += NW) {
            const int r = qi / G, h = kvh * G + (qi - r * G);
            const int pr = rows[r].pos;
            if (pr < lo) continue;                       // the chunk lies after the row's position: the merge stops before it
            const int end = min(hi, pr + 1) - lo;
            const int gr = rq.row0 + r;                  // the row among the launch's verify rows
            const float4 q = *reinterpret_cast<const float4*>(a.q + (size_t)gr * a.ldq + (size_t)h * HD + lane * 4);
            float m = -INFINITY, l = 0.f;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int t0 = 0; t0 < end; t0 += 4) {
                float s[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {   // four independent dot products in flight; the updates below stay in position order
                    const int t = min(t0 + i, end - 1);
                    const float4 k = *reinterpret_cast<const float4*>(Ks + t * HD + lane * 4);
                    s[i] = q.x * k.x + q.y * k.y + q.z * k.z + q.w * k.w;
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) s[i] += __shfl_xor_sync(0xffffffffu, s[i], o);
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    if (t0 + i >= end) break;
                    const float sc = s[i] * a.scaling;
                    const float4 v = *reinterpret_cast<const float4*>(Vs + (t0 + i) * HD + lane * 4);
                    const float mnew = fmaxf(m, sc);
                    const float alpha = expf(m - mnew);      // m = -inf on the first position only: alpha = 0
                    const float p = expf(sc - mnew);
                    l = l * alpha + p;
                    acc.x = acc.x * alpha + p * v.x;
                    acc.y = acc.y * alpha + p * v.y;
                    acc.z = acc.z * alpha + p * v.z;
                    acc.w = acc.w * alpha + p * v.w;
                    m = mnew;
                }
            }
            float* p = a.partial + (((size_t)gr * a.nh + h) * a.max_chunks + c) * spec_part_stride(HD);
            *reinterpret_cast<float4*>(p + lane * 4) = acc;
            if (lane == 0) { p[HD] = m; p[HD + 1] = l; }
        }
    }
}

// grid (nh, rows), HD threads: verify row r, head h merges its chunks 0 .. pos_r / kSpecChunk in index order (every one holds >= 1 position)
template <int HD>
__global__ void __launch_bounds__(HD) spec_verify_merge_kernel(SpecAttnArgs a) {
    const int h = blockIdx.x, r = blockIdx.y, d = threadIdx.x;
    const int nc = a.rows[r].pos / kSpecChunk + 1;
    const float* pb = a.partial + ((size_t)r * a.nh + h) * a.max_chunks * spec_part_stride(HD);
    float M = -INFINITY;
    for (int c = 0; c < nc; ++c) M = fmaxf(M, pb[(size_t)c * spec_part_stride(HD) + HD]);
    float L = 0.f, O = 0.f;
    for (int c = 0; c < nc; ++c) {
        const float e = expf(pb[(size_t)c * spec_part_stride(HD) + HD] - M);
        L += pb[(size_t)c * spec_part_stride(HD) + HD + 1] * e;
        O += pb[(size_t)c * spec_part_stride(HD) + d] * e;
    }
    a.out[(size_t)r * a.ldo + (size_t)h * HD + d] = O / L;
}

// ---------------------------------------------------------------------------------------------------------------------------- accept
// One CTA per request (reqs[blockIdx.x]).  row_tok[row0 + r]: the final token of its row r (the sample, or the ArgMax of a greedy request);
// hist[E + r - 1]: draft r.  Emits rows 0 .. j (j = leading drafts equal to the sample of the row before them), cut after an EOS token or at
// max_tokens, copies their records (index set to the token's place in the output) and advances the request.
__global__ void __launch_bounds__(128) spec_accept_kernel(const SpecReq* __restrict__ reqs, const uint32_t* __restrict__ row_tok,
                                                         const aha_logprobs* __restrict__ row_lp) {
    __shared__ int s_n, s_E;
    const int tid = threadIdx.x;
    const SpecReq q = reqs[blockIdx.x];
    SpecCtl* ctl = q.ctl;
    if (ctl->done) return;
    row_tok += q.row0;
    row_lp += q.row0;
    if (tid == 0) {
        SpecCtl& c = *ctl;
        DecodeState& st = *c.req;
        uint32_t* hist = c.hist;
        const int E = st.n_hist, nd = c.n_draft;
        int j = 0;
        while (j < nd && hist[E + j] == row_tok[j]) ++j;
        int n = 0;
        bool done = false;
        for (int k = 0; k <= j && !done; ++k) {
            const uint32_t t = row_tok[k];
            hist[E + k] = t;
            ++n;
            if (E + n >= c.max_tokens) done = true;
            for (int s = 0; s < c.n_stop; ++s) if (c.stop[s] == t) done = true;   // an EOS token is pushed, then the request ends
        }
        st.token = row_tok[n - 1];
        st.pos += n;
        st.n_hist = E + n;
        st.n_draws += (uint32_t)n * c.draw_step;
        c.passes += 1u;
        c.drafted += (uint32_t)nd;
        c.accepted += (uint32_t)min(j, n);
        c.done = done ? 1 : 0;
        s_n = c.lp ? n : 0;
        s_E = E;
    }
    __syncthreads();
    constexpr int W = (int)(sizeof(aha_logprobs) / sizeof(uint32_t));
    const SpecCtl& c = *ctl;
    aha_logprobs* out = c.lp_by_index ? c.lp_out + s_E : c.lp_out;
    for (int idx = tid; idx < s_n * W; idx += blockDim.x) {
        const int k = idx / W, w = idx % W;
        uint32_t v = reinterpret_cast<const uint32_t*>(row_lp + k)[w];
        if (w == (int)(offsetof(aha_logprobs, index) / sizeof(uint32_t))) v = (uint32_t)(s_E + k);
        reinterpret_cast<uint32_t*>(out + k)[w] = v;
        if (k == s_n - 1 && c.lp_last) reinterpret_cast<uint32_t*>(c.lp_last)[w] = v;
    }
}

// ----------------------------------------------------------------------------------------------------------------------- host side
// The verify passes on the wide decoder's activation buffers (BatchDecoder::init_wide: xb / qkvb / attnb / hb / logitsb, rows np .. np + ns - 1
// after the plain rows) with per-row arrays of their own: verify-row states, samplers, tokens, sampler scratch, count rows and records.  The
// plain rows of a session step keep their slots' arrays.  Control blocks: one per session slot (a single request uses block 0; the
// single-request entry refuses an open session).
struct SpecDecoder {
    TextModel* T = nullptr;
    BatchDecoder* B = nullptr;
    SpecCtl* d_ctl = nullptr;                          // [kWideSeqs]
    SpecReq* d_reqs = nullptr;                         // [kWideSeqs] the requests of the current composition
    const int** d_row_table = nullptr;                 // [kWideSeqs] verify row -> its request's page table, in the current composition
    int* d_ident = nullptr;                            // [kWideSeqs] r -> r: the verify rows' "active list"
    DecodeState* d_vst = nullptr;                      // [kWideSeqs] verify-row states (spec_draft_kernel)
    uint32_t* d_vtok = nullptr;                        // [kWideSeqs] verify-row final tokens
    SampleArgs* d_vsamp = nullptr;                     // [kWideSeqs] the sampler of each verify row's request, bound to the row
    int* d_vsamp_on = nullptr;                         // [kWideSeqs]
    int* d_vlp_on = nullptr;                           // [kWideSeqs] 1 + top count of the row's request, or 0
    aha_logprobs* d_vlp_rec = nullptr;                 // [kWideSeqs] verify-row records
    aha_logprobs* d_slot_lp = nullptr;                 // [kWideSeqs][kSpecMaxRows] records of the tokens a session slot's last pass emitted
    float* d_vwork = nullptr;                          // [kWideSeqs][V] sampler scratch
    int* d_vcnt = nullptr;                             // [kWideSeqs][V] count rows, allocated when a request first asks
    float* partial = nullptr; int max_chunks = 0, partial_rows = 0;
    uint32_t* d_buf[kWideSeqs] = {}; size_t buf_cap[kWideSeqs] = {};   // per control block: prediction | prompt | stop ids
    GraphCache<int> graphs;                            // single requests: keyed by R
    GraphCache<std::array<int, 4>> steps;              // session steps: keyed by (plain rows, requests, verify rows, records)
    std::vector<int> built_plain, built_spec;          // the composition the device copies were built for
    uint64_t built_epoch = ~0ull;

    void destroy() {
        graphs.clear();
        steps.clear();
        for (int i = 0; i < kWideSeqs; ++i) if (d_buf[i]) { cudaFree(d_buf[i]); d_buf[i] = nullptr; buf_cap[i] = 0; }
        if (partial) { cudaFree(partial); partial = nullptr; partial_rows = 0; }
    }
    // `rows`: verify rows the passes may hold (kSpecMaxRows for a single request, kWideSeqs in a session)
    void init(TextModel& t, BatchDecoder& b, int rows) {
        T = &t; B = &b;
        B->init_wide(t);
        B->ensure_lp();
        if (!T->d_lp) T->set_logprobs(0);     // the single request's record buffer (the accept kernel's target) exists before any capture
        Ctx& c = *t.ctx;
        if (!d_ctl) {
            const int n = kWideSeqs;
            d_ctl = c.alloc<SpecCtl>(n);
            d_reqs = c.alloc<SpecReq>(n);
            d_row_table = c.alloc<const int*>(n);
            d_ident = c.alloc<int>(n);
            d_vst = c.alloc<DecodeState>(n);
            d_vtok = c.alloc<uint32_t>(n);
            d_vsamp = c.alloc<SampleArgs>(n);
            d_vsamp_on = c.alloc<int>(n);
            d_vlp_on = c.alloc<int>(n);
            d_vlp_rec = c.alloc<aha_logprobs>(n);
            d_slot_lp = c.alloc<aha_logprobs>((size_t)n * kSpecMaxRows);
            d_vwork = c.alloc<float>((size_t)n * t.cfg.V);
            std::vector<int> ident(n);
            for (int i = 0; i < n; ++i) ident[i] = i;
            AHA_CUDA_CHECK(cudaMemcpy(d_ident, ident.data(), n * sizeof(int), cudaMemcpyHostToDevice));
            AHA_CUDA_CHECK(cudaMemset(d_ctl, 0, n * sizeof(SpecCtl)));
            max_chunks = ceil_div(t.max_ctx, kSpecChunk);
            AHA_CUDA_CHECK(cudaFuncSetAttribute(spec_verify_attn_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)spec_attn_smem_bytes<128>()));
        }
        if (rows > partial_rows) {   // the graphs hold the old buffer: they are captured again
            if (partial) { AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream)); AHA_CUDA_CHECK(cudaFree(partial)); partial = nullptr; }
            graphs.clear();
            steps.clear();
            AHA_CUDA_CHECK(cudaMalloc(&partial, (size_t)rows * t.nh_l * max_chunks * spec_part_stride(t.cfg.hd) * sizeof(float)));
            partial_rows = rows;
        }
    }
    int* counts(const Sampler& s, int r) {
        if (!s.counts) return nullptr;
        if (!d_vcnt) d_vcnt = T->alloc_counts(kWideSeqs);
        return d_vcnt + (size_t)r * T->cfg.V;
    }
    // control block i of a request: its draft sources in block i's buffer, its state / history / page table and where its records go
    void set_ctl(int i, const Sampler& samp, const std::vector<uint32_t>& pred, const uint32_t* prompt, size_t n_prompt,
                 const std::vector<uint32_t>& stop, int max_tokens, int ngram, int lp_on, DecodeState* req, uint32_t* hist,
                 aha_logprobs* lp_out, int lp_by_index, aha_logprobs* lp_last) {
        Ctx& c = *T->ctx;
        const size_t need = pred.size() + n_prompt + stop.size();
        if (need > buf_cap[i]) {
            if (d_buf[i]) { AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream)); AHA_CUDA_CHECK(cudaFree(d_buf[i])); d_buf[i] = nullptr; buf_cap[i] = 0; }
            AHA_CUDA_CHECK(cudaMalloc(&d_buf[i], need * sizeof(uint32_t)));
            buf_cap[i] = need;
        }
        std::vector<uint32_t> h(pred);
        h.insert(h.end(), prompt, prompt + n_prompt);
        h.insert(h.end(), stop.begin(), stop.end());
        SpecCtl s{};
        uint32_t* buf = d_buf[i];
        s.pred = buf; s.n_pred = (int)pred.size();
        s.prompt = buf + pred.size(); s.n_prompt = (int)n_prompt;
        s.stop = buf + pred.size() + n_prompt; s.n_stop = (int)stop.size();
        s.max_tokens = max_tokens; s.ngram = ngram;
        s.draw_step = samp.active && samp.args.mode != SAMPLE_ARGMAX ? 1u : 0u;
        s.lp = lp_on > 0 ? 1 : 0;
        s.req = req; s.hist = hist;
        s.lp_out = lp_out; s.lp_by_index = lp_by_index; s.lp_last = lp_last;
        if (!h.empty()) AHA_CUDA_CHECK(cudaMemcpyAsync(buf, h.data(), h.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_ctl + i, &s, sizeof(s), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));   // host temporaries
    }
    // the device copy of a composition: requests (slot = control block, page table, R) in order, their rows after each other, every
    // verify row bound to its request's sampler (the request's history, the row's own state / token / scratch / count row) and record flag,
    // which of[q] holds (R in of[q]->req)
    void build(const std::vector<int>& ctl_of, const std::vector<const int*>& table_of, const std::vector<const BatchSlot*>& of,
               const std::vector<uint32_t*>& hist_of) {
        Ctx& c = *T->ctx;
        std::vector<SpecReq> reqs;
        std::vector<const int*> row_table;
        std::vector<int> on(kWideSeqs, 0), lp(kWideSeqs, 0);
        std::vector<SampleArgs> samp(kWideSeqs);
        int row = 0;
        for (size_t q = 0; q < ctl_of.size(); ++q) {
            const BatchSlot& s = *of[q];
            reqs.push_back(SpecReq{d_ctl + ctl_of[q], table_of[q], row, s.req.R, 0});
            for (int r = 0; r < s.req.R; ++r, ++row) {
                row_table.push_back(table_of[q]);
                on[row] = s.sampler.active ? 1 : 0;
                lp[row] = s.lp;
                // the request's history holds the emitted tokens followed by the drafts, so row r's counts (frequency / presence, each row
                // its own count row) cover the context a sequential decode would see at that draw
                if (s.sampler.active) samp[row] = T->bind_sampler(s.sampler, d_vst + row, hist_of[q], d_vtok + row, d_vwork + (size_t)row * T->cfg.V, counts(s.sampler, row));
            }
        }
        AHA_REQUIRE(row <= kWideSeqs, "speculative step: more than 64 verify rows");
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_reqs, reqs.data(), reqs.size() * sizeof(SpecReq), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_row_table, row_table.data(), row_table.size() * sizeof(const int*), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_vsamp_on, on.data(), on.size() * sizeof(int), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_vsamp, samp.data(), samp.size() * sizeof(SampleArgs), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_vlp_on, lp.data(), lp.size() * sizeof(int), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));   // host temporaries
    }

    // ---- one request (aha_b200_generate_speculative): control block 0 on the model's own state, history, page table and record buffer
    void prepare(int R, const Sampler& samp, const std::vector<uint32_t>& pred, const uint32_t* prompt, size_t n_prompt,
                 const std::vector<uint32_t>& stop, int max_tokens, int ngram, int lp_on) {
        set_ctl(0, samp, pred, prompt, n_prompt, stop, max_tokens, ngram, lp_on, T->d_state, T->d_history, T->d_lp, 1, nullptr);
        BatchSlot s; s.req.R = R; s.sampler = samp; s.lp = lp_on;
        build({0}, {T->table.d}, {&s}, {T->d_history});
        built_epoch = ~0ull;                  // a later session builds its own composition
        B->zero_rows_from(R);
    }
    void pass(int R) {
        if (!T->use_graph) { launches(0, 1, R, true); return; }
        graphs.run(*T->ctx, R, [&] { launches(0, 1, R, true); });   // (the record kernels always run: one graph per R)
    }

    // ---- a session step: the plain slots `plain` (rows 0 .. np-1, the decoder's active list) and the speculative slots `spec`
    void step(const std::vector<int>& plain, const std::vector<int>& spec) {
        if (B->epoch != built_epoch || plain != built_plain || spec != built_spec) {
            B->build_attn_table(plain);
            std::vector<const int*> tab;
            std::vector<const BatchSlot*> of;
            std::vector<uint32_t*> hist;
            for (int s : spec) { tab.push_back(B->slots[s].table.d); of.push_back(&B->slots[s]); hist.push_back(B->d_hist + (size_t)s * T->hist_cap); }
            build(spec, tab, of, hist);
            built_plain = plain; built_spec = spec; built_epoch = B->epoch;
        }
        const int np = (int)plain.size(), nq = (int)spec.size();
        int ns = 0;
        bool lp = false;
        for (int s : plain) lp = lp || B->slots[s].lp > 0;
        for (int s : spec) { ns += B->slots[s].req.R; lp = lp || B->slots[s].lp > 0; }
        B->zero_rows_from(np + ns);
        if (!B->use_graph) { launches(np, nq, ns, lp); return; }
        steps.run(*T->ctx, {np, nq, ns, lp ? 1 : 0}, [&] { launches(np, nq, ns, lp); });
    }

    static int attn_ctas(int max_chunks, int nkv, int num_sms) { return std::max(1, std::min(max_chunks, ceil_div(2 * num_sms, nkv))); }
    // np plain rows, then the ns verify rows of nq requests; lp: the record kernels run
    void launches(int np, int nq, int ns, bool lp) {
        Ctx& c = *T->ctx;
        cudaStream_t st = c.stream;
        const TextCfg& cf = T->cfg;
        const int H = cf.H, nb = np + ns;
        float* qkv_v = B->qkvb + (size_t)np * T->qkv_dim;
        float* attn_v = B->attnb + (size_t)np * T->nh_l * cf.hd;
        spec_draft_kernel<<<nq, kSpecDraftThreads, 0, st>>>(d_reqs, d_vst);
        c.cnt.kernels++;
        if (np) { embed_rows_kernel<<<np, 256, 0, st>>>(B->d_act, B->d_states, T->embed, B->xb, H, cf.V); c.cnt.kernels++; }
        embed_rows_kernel<<<ns, 256, 0, st>>>(d_ident, d_vst, T->embed, B->xb + (size_t)np * H, H, cf.V);
        c.cnt.kernels++;
        for (int l = 0; l < cf.L; ++l) {
            TextLayer& Ly = T->layers[l];
            B->proj(GEPI_STORE, Ly.qkv, B->xb, H, Ly.ln1, nullptr, 0, B->qkvb, T->qkv_dim, nb);
            if (np) B->attn(l, np);
            const KVSrc kv = T->kv_src(l, T->table);
            SpecRowArgs ra{};
            ra.qkv = qkv_v; ra.ld = T->qkv_dim; ra.qw = Ly.qn; ra.kw = Ly.kn; ra.eps = cf.eps; ra.inv_freq = T->inv_freq; ra.rows = d_vst;
            ra.row_table = d_row_table;
            ra.kbase = const_cast<float*>(kv.k); ra.vbase = const_cast<float*>(kv.v); ra.kv = kv; ra.nh = T->nh_l; ra.nkv = T->nkv_l;
            spec_qk_rows_kernel<128><<<dim3(ceil_div(T->nh_l + 2 * T->nkv_l, 8), ns), 256, 0, st>>>(ra);
            SpecAttnArgs aa{};
            aa.q = qkv_v; aa.ldq = T->qkv_dim;
            aa.kv = kv; aa.reqs = d_reqs; aa.rows = d_vst;
            aa.partial = partial; aa.max_chunks = max_chunks;
            aa.out = attn_v; aa.ldo = T->nh_l * cf.hd;
            aa.nh = T->nh_l; aa.nkv = T->nkv_l;
            aa.scaling = (float)(1.0 / std::sqrt((double)cf.hd));
            spec_verify_attn_kernel<128><<<dim3(attn_ctas(max_chunks, T->nkv_l * nq, c.num_sms), T->nkv_l, nq), kSpecAttnThreads, spec_attn_smem_bytes<128>(), st>>>(aa);
            spec_verify_merge_kernel<128><<<dim3(T->nh_l, ns), 128, 0, st>>>(aa);
            c.cnt.kernels += 3;
            B->proj(GEPI_RESID, Ly.o, B->attnb, T->nh_l * cf.hd, nullptr, B->xb, H, B->xb, H, nb);
            B->proj(GEPI_SWIGLU, Ly.gu, B->xb, H, Ly.ln2, nullptr, 0, B->hb, T->I_l, nb);
            B->proj(GEPI_RESID, Ly.down, B->hb, T->I_l, nullptr, B->xb, H, B->xb, H, nb);
        }
        B->lm_head(nb);
        // plain rows: a decode step's ArgMax / sampler / records; verify rows: the same kernels without advancing any state
        if (np) B->head_rows_at(0, np, B->d_act, B->d_tok, B->d_states, B->d_hist, B->d_samp, B->d_samp_on, B->d_lp_on, B->d_lp_rec, false, lp);
        B->head_rows_at(np, ns, d_ident, d_vtok, d_vst, T->d_history, d_vsamp, d_vsamp_on, d_vlp_on, d_vlp_rec, true, lp);
        spec_accept_kernel<<<nq, 128, 0, st>>>(d_reqs, d_vtok, d_vlp_rec);
        c.cnt.kernels++;
        AHA_CUDA_CHECK(cudaGetLastError());
    }
};

}  // namespace aha
