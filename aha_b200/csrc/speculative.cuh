// speculative.cuh -- speculative decoding of ONE request: verify passes of R = max_draft + 1 rows through one weight stream
// (new design; the reference decodes one token per forward_step, src/models/common/generate.rs:115-159, and ignores the
// `prediction` field of its request schema, src/params/chat.rs:102-105).
//
// A pass runs R rows of the same request:
//     row 0       the last emitted token, at position pos (DecodeState::pos of the request)
//     row r >= 1  draft r, at position pos + r
// and emits the longest run the request's own sampler reproduces.  Its launches (captured once per R into a CUDA graph) are
//     [draft]    spec_draft_kernel        drafts of this pass -> the request's history behind the emitted tokens, one DecodeState per row
//     [embed]    embed_rows_kernel        row r <- its token
// then per layer
//     [qkv]      wide projection          (gemv_wide.cuh: a row's bits do not depend on the other rows)
//     [K/V]      spec_qk_rows_kernel      q/k RMSNorm, RoPE at pos + r + rope_delta, K/V stored for every row BEFORE any row attends
//     [attn]     spec_verify_attn_kernel + spec_verify_merge_kernel
//     [o_proj], [gate/up + SwiGLU], [down]   wide projections
// then the head of BatchDecoder (lm_head, row ArgMax, sample_rows_kernel, logprobs_rows) and
//     [accept]   spec_accept_kernel       compares samples with drafts, emits the run, applies EOS / max_tokens, advances the request.
//
// Exactness.  Row r is sampled with the request's sampler at draw index n_draws + r and with the repeat-penalty context "history
// followed by drafts 1..r" (the drafts sit in the history buffer right behind the emitted tokens, and row r's DecodeState says
// n_hist = emitted + r).  If the first j drafts equal the samples of the rows before them, rows 0..j computed exactly what j + 1
// sequential steps of the same kernels compute, so the pass emits their j + 1 samples and consumes j + 1 draws.  Every row is computed
// independently of its index and of R (column-invariant projections, the row-invariant attention below, row-indexed head kernels), so a
// request's ids and log-probability records do not depend on the drafts, max_draft or graphs: a wrong draft costs time, never the answer.
// K/V of rejected positions are stale; the next pass's rows overwrite them before any row reads them, and no row reads past its own position.
//
// Draft rule (spec_draft_kernel; restated in tests/spec_ref.py).  e[0..E) = the emitted tokens.  For n = min(ngram, E) down to 1, and
// for each source in order -- first the caller's prediction p[0..P), then, with prompt lookup, the text "prompt followed by e[0..E)" --
// take the largest i with src[i .. i+n) == e[E-n .. E) and i + n < |src| (at least one token follows).  The first (n, source) that has
// one gives the drafts src[i+n .. min(i+n+max_draft, |src|)).  No match: no drafts.  Rows behind the drafts are padded with token 0 and
// their samples are ignored.
#pragma once
#include "attention.cuh"
#include "batch_decode.cuh"
#include "kernels_common.cuh"
#include "logprobs.cuh"
#include "sampling.cuh"

namespace aha {

constexpr int kSpecMaxRows = 16;            // max_draft + 1
constexpr int kSpecChunk = 2 * kPage;       // KV positions per verify-attention chunk: a fixed multiple of the page, never ctx / splits
constexpr int kSpecDefaultNgram = 3;
constexpr int kSpecMaxNgram = 8;
constexpr int kSpecDraftThreads = 256;
constexpr int kSpecAttnThreads = 256;

// device-side control block of a speculative request: set by the host before the first pass, advanced by the accept kernel
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
};

// ---------------------------------------------------------------------------------------------------------------------------- draft
__device__ __forceinline__ uint32_t spec_src_at(const SpecCtl& c, const uint32_t* hist, int src, int i) {
    if (src == 0) return c.pred[i];
    return i < c.n_prompt ? c.prompt[i] : hist[i - c.n_prompt];
}

// One CTA.  req: the request's state (token = last emitted, pos = its position, n_hist = E emitted tokens); rows: [R] per-row states.
__global__ void __launch_bounds__(kSpecDraftThreads) spec_draft_kernel(SpecCtl* __restrict__ ctl, const DecodeState* __restrict__ req,
                                                                       uint32_t* __restrict__ hist, DecodeState* __restrict__ rows, int R) {
    __shared__ int red[kSpecDraftThreads / 32];
    __shared__ int s_src, s_start, s_nd;
    const SpecCtl c = *ctl;
    const DecodeState st = *req;
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
                    for (int q = 0; q < n && eq; ++q) eq = spec_src_at(c, hist, src, i + q) == hist[E - n + q];
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
    if (tid == 0) ctl->n_draft = nd;
}

// --------------------------------------------------------------------------------------------------------------- row K/V append
struct SpecRowArgs {
    float* qkv; int ld;                      // [R][ld] raw projections; q is normalised and rotated in place
    const float* qw; const float* kw; float eps;
    const float* inv_freq;
    const DecodeState* rows;                 // row r's position and rope_delta
    float* kbase; float* vbase;              // layer bases into the pool (writable)
    KVSrc kv;
    int nh, nkv;
};

// grid (ceil((nh + 2 nkv) / 8), R), 256 threads: warp = one head slot of one row (q heads, k heads, v heads), the arithmetic of
// decode_attn_body's prologue
template <int HD>
__global__ void __launch_bounds__(256) spec_qk_rows_kernel(SpecRowArgs a) {
    static_assert(HD == 128, "speculative decoding is specialised for head_dim 128");
    const int lane = threadIdx.x & 31, slot = blockIdx.x * 8 + (threadIdx.x >> 5), r = blockIdx.y;
    if (slot >= a.nh + 2 * a.nkv) return;
    float* row = a.qkv + (size_t)r * a.ld;
    const DecodeState st = a.rows[r];
    const int pos = st.pos;
    const float4 x = *reinterpret_cast<const float4*>(row + (size_t)slot * HD + lane * 4);
    if (slot >= a.nh + a.nkv) {
        const size_t off = a.kv.off(pos, slot - a.nh - a.nkv) + lane * 4;
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
        const size_t off = a.kv.off(pos, slot - a.nh) + lane * 4;
        *reinterpret_cast<float4*>(a.kbase + off) = make_float4(kv_store_round(o[0]), kv_store_round(o[1]), kv_store_round(o[2]), kv_store_round(o[3]));
    }
}

// ------------------------------------------------------------------------------------------------------------ verify attention
// Multi-query split-KV attention of the R rows over the request's page table.  CTA (x, kvh) takes the chunks c = x, x + gridDim.x, ...
// of kSpecChunk positions [c * kSpecChunk, (c + 1) * kSpecChunk), stages the chunk's K and V in shared memory once and serves every
// (row, q head) pair of the KV group from it, so a KV page is read once per pass, not once per row.  Row r attends to positions
// 0 .. pos_r (= its own position: causal inside the draft).
//
// Invariant: row r's output depends only on its own position and its q.
//   * Chunk boundaries are fixed multiples of the page, not a function of the context length or of R.
//   * Inside a chunk a warp walks the row's positions lo .. min(hi, pos_r + 1) - 1 in order, one online-softmax update each; positions
//     past pos_r are never visited, so they leave m / l / acc bit-unchanged (there is no masked update, hence no -inf - -inf).
//     Which warp serves a row does not matter: every warp runs the same sequence of operations.
//   * spec_verify_merge_kernel merges the row's chunks 0 .. pos_r / kSpecChunk in index order.
struct SpecAttnArgs {
    const float* q; int ldq;                 // row r, head h: q + r * ldq + h * HD (normalised and rotated)
    KVSrc kv;
    const DecodeState* rows;                 // [R] positions
    float* partial;                          // [R][nh][max_chunks][spec_part_stride(HD)]: acc (unnormalised), m, l
    int max_chunks;
    float* out; int ldo;                     // row r, head h: out + r * ldo + h * HD
    int R, nh, nkv;
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
    const int G = a.nh / a.nkv, Q = a.R * G;
    const int ctx = a.rows[a.R - 1].pos + 1;
    const int nchunks = (ctx + kSpecChunk - 1) / kSpecChunk;
    for (int c = blockIdx.x; c < nchunks; c += gridDim.x) {
        const int lo = c * kSpecChunk, hi = min(ctx, lo + kSpecChunk);
        __syncthreads();   // the previous chunk is consumed
        for (int idx = tid; idx < (hi - lo) * (HD / 4); idx += kSpecAttnThreads) {
            const int t = idx / (HD / 4), c4 = idx % (HD / 4);
            const size_t off = a.kv.off(lo + t, kvh) + c4 * 4;
            *reinterpret_cast<float4*>(Ks + t * HD + c4 * 4) = *reinterpret_cast<const float4*>(a.kv.k + off);
            *reinterpret_cast<float4*>(Vs + t * HD + c4 * 4) = *reinterpret_cast<const float4*>(a.kv.v + off);
        }
        __syncthreads();
        for (int qi = warp; qi < Q; qi += NW) {
            const int r = qi / G, h = kvh * G + (qi - r * G);
            const int pr = a.rows[r].pos;
            if (pr < lo) continue;                       // the chunk lies after the row's position: the merge stops before it
            const int end = min(hi, pr + 1) - lo;
            const float4 q = *reinterpret_cast<const float4*>(a.q + (size_t)r * a.ldq + (size_t)h * HD + lane * 4);
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
            float* p = a.partial + (((size_t)r * a.nh + h) * a.max_chunks + c) * spec_part_stride(HD);
            *reinterpret_cast<float4*>(p + lane * 4) = acc;
            if (lane == 0) { p[HD] = m; p[HD + 1] = l; }
        }
    }
}

// grid (nh, R), HD threads: row r, head h merges its chunks 0 .. pos_r / kSpecChunk in index order (every one holds >= 1 position)
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
// One CTA.  row_tok[r]: the final token of row r (the sample, or the ArgMax of a greedy request); hist[E + r - 1]: draft r.
// Emits rows 0 .. j (j = leading drafts equal to the sample of the row before them), cut after an EOS token or at max_tokens, copies
// their records (index set to the token's place in the output) and advances the request.
__global__ void __launch_bounds__(128) spec_accept_kernel(SpecCtl* __restrict__ ctl, DecodeState* __restrict__ req, uint32_t* __restrict__ hist,
                                                         const uint32_t* __restrict__ row_tok, const aha_logprobs* __restrict__ row_lp,
                                                         aha_logprobs* __restrict__ lp_out) {
    __shared__ int s_n, s_E;
    const int tid = threadIdx.x;
    if (ctl->done) return;
    if (tid == 0) {
        SpecCtl& c = *ctl;
        DecodeState& st = *req;
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
    for (int idx = tid; idx < s_n * W; idx += blockDim.x) {
        const int k = idx / W, w = idx % W;
        uint32_t v = reinterpret_cast<const uint32_t*>(row_lp + k)[w];
        if (w == (int)(offsetof(aha_logprobs, index) / sizeof(uint32_t))) v = (uint32_t)(s_E + k);
        reinterpret_cast<uint32_t*>(lp_out + s_E + k)[w] = v;
    }
}

// ----------------------------------------------------------------------------------------------------------------------- host side
// The passes of a speculative request on the wide decoder's buffers (BatchDecoder::init_wide): rows 0 .. R-1 of xb / qkvb / attnb / hb /
// logitsb and of its per-slot DecodeState / SampleArgs / token / record arrays.  Safe because the single-request entries refuse an open
// batch session.  One pass graph per R.
struct SpecDecoder {
    TextModel* T = nullptr;
    BatchDecoder* B = nullptr;
    SpecCtl* d_ctl = nullptr;
    float* partial = nullptr; int max_chunks = 0;
    uint32_t* d_buf = nullptr; size_t buf_cap = 0;     // prediction | prompt | stop ids of the current request
    GraphCache<int> graphs;                            // keyed by R
    void destroy() {
        graphs.clear();
        if (d_buf) { cudaFree(d_buf); d_buf = nullptr; buf_cap = 0; }
    }
    void init(TextModel& t, BatchDecoder& b) {
        T = &t; B = &b;
        B->init_wide(t);
        B->ensure_lp();
        if (!T->d_lp) T->set_logprobs(0);     // the request's record buffer (the accept kernel's target) exists before any capture
        if (d_ctl) return;
        Ctx& c = *t.ctx;
        d_ctl = c.alloc<SpecCtl>(1);
        max_chunks = ceil_div(t.max_ctx, kSpecChunk);
        partial = c.alloc<float>((size_t)kSpecMaxRows * t.nh_l * max_chunks * spec_part_stride(t.cfg.hd));
        AHA_CUDA_CHECK(cudaFuncSetAttribute(spec_verify_attn_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)spec_attn_smem_bytes<128>()));
    }
    // the request's control block, rows 0..R-1 of the decoder's active list / samplers / record flags (lp_on = 1 + top count, or 0)
    void prepare(int R, const Sampler& samp, const std::vector<uint32_t>& pred, const uint32_t* prompt, size_t n_prompt,
                 const std::vector<uint32_t>& stop, int max_tokens, int ngram, int lp_on) {
        Ctx& c = *T->ctx;
        const size_t need = pred.size() + n_prompt + stop.size();
        if (need > buf_cap) {
            if (d_buf) { AHA_CUDA_CHECK(cudaFree(d_buf)); d_buf = nullptr; buf_cap = 0; }
            AHA_CUDA_CHECK(cudaMalloc(&d_buf, need * sizeof(uint32_t)));
            buf_cap = need;
        }
        std::vector<uint32_t> h(pred);
        h.insert(h.end(), prompt, prompt + n_prompt);
        h.insert(h.end(), stop.begin(), stop.end());
        SpecCtl s{};
        s.pred = d_buf; s.n_pred = (int)pred.size();
        s.prompt = d_buf + pred.size(); s.n_prompt = (int)n_prompt;
        s.stop = d_buf + pred.size() + n_prompt; s.n_stop = (int)stop.size();
        s.max_tokens = max_tokens; s.ngram = ngram;
        s.draw_step = samp.active && samp.args.mode != SAMPLE_ARGMAX ? 1u : 0u;
        s.lp = lp_on > 0 ? 1 : 0;
        std::vector<int> act(kSpecMaxRows), on(kSpecMaxRows, samp.active ? 1 : 0), lp(kSpecMaxRows, lp_on);
        std::vector<SampleArgs> rows(kSpecMaxRows);
        for (int r = 0; r < kSpecMaxRows; ++r) {
            act[r] = r;
            // the request's sampler on every row; the shared history holds the emitted tokens followed by the drafts, so row r's counts
            // (frequency / presence, each row its own count row) cover the context a sequential decode would see at that draw
            if (samp.active) rows[r] = T->bind_sampler(samp, B->d_states + r, T->d_history, B->d_tok + r, B->workb + (size_t)r * T->cfg.V, B->counts(samp, r));
        }
        if (!h.empty()) AHA_CUDA_CHECK(cudaMemcpyAsync(d_buf, h.data(), h.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_ctl, &s, sizeof(s), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(B->d_act, act.data(), act.size() * sizeof(int), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(B->d_samp_on, on.data(), on.size() * sizeof(int), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(B->d_samp, rows.data(), rows.size() * sizeof(SampleArgs), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(B->d_lp_on, lp.data(), lp.size() * sizeof(int), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));   // host temporaries
        B->composition_changed();             // a later session rebuilds its own device copies
        B->zero_rows_from(R);
        B->lp_any = true;                     // the record kernels always run (rows that ask for none return at once): one graph per R
    }
    SpecAttnArgs attn_args(int l, int R) const {
        SpecAttnArgs a{};
        a.q = B->qkvb; a.ldq = T->qkv_dim;
        a.kv = T->kv_src(l, T->table);
        a.rows = B->d_states;
        a.partial = partial; a.max_chunks = max_chunks;
        a.out = B->attnb; a.ldo = T->nh_l * T->cfg.hd;
        a.R = R; a.nh = T->nh_l; a.nkv = T->nkv_l;
        a.scaling = (float)(1.0 / std::sqrt((double)T->cfg.hd));
        return a;
    }
    static int attn_ctas(int max_chunks, int nkv, int num_sms) { return std::max(1, std::min(max_chunks, ceil_div(2 * num_sms, nkv))); }
    void launches(int R) {
        Ctx& c = *T->ctx;
        cudaStream_t st = c.stream;
        const TextCfg& cf = T->cfg;
        const int H = cf.H;
        spec_draft_kernel<<<1, kSpecDraftThreads, 0, st>>>(d_ctl, T->d_state, T->d_history, B->d_states, R);
        embed_rows_kernel<<<R, 256, 0, st>>>(B->d_act, B->d_states, T->embed, B->xb, H, cf.V);
        c.cnt.kernels += 2;
        for (int l = 0; l < cf.L; ++l) {
            TextLayer& Ly = T->layers[l];
            B->proj(GEPI_STORE, Ly.qkv, B->xb, H, Ly.ln1, nullptr, 0, B->qkvb, T->qkv_dim, R);
            const KVSrc kv = T->kv_src(l, T->table);
            SpecRowArgs ra{};
            ra.qkv = B->qkvb; ra.ld = T->qkv_dim; ra.qw = Ly.qn; ra.kw = Ly.kn; ra.eps = cf.eps; ra.inv_freq = T->inv_freq; ra.rows = B->d_states;
            ra.kbase = const_cast<float*>(kv.k); ra.vbase = const_cast<float*>(kv.v); ra.kv = kv; ra.nh = T->nh_l; ra.nkv = T->nkv_l;
            spec_qk_rows_kernel<128><<<dim3(ceil_div(T->nh_l + 2 * T->nkv_l, 8), R), 256, 0, st>>>(ra);
            const SpecAttnArgs aa = attn_args(l, R);
            spec_verify_attn_kernel<128><<<dim3(attn_ctas(max_chunks, T->nkv_l, c.num_sms), T->nkv_l), kSpecAttnThreads, spec_attn_smem_bytes<128>(), st>>>(aa);
            spec_verify_merge_kernel<128><<<dim3(T->nh_l, R), 128, 0, st>>>(aa);
            c.cnt.kernels += 3;
            B->proj(GEPI_RESID, Ly.o, B->attnb, T->nh_l * cf.hd, nullptr, B->xb, H, B->xb, H, R);
            B->proj(GEPI_SWIGLU, Ly.gu, B->xb, H, Ly.ln2, nullptr, 0, B->hb, T->I_l, R);
            B->proj(GEPI_RESID, Ly.down, B->hb, T->I_l, nullptr, B->xb, H, B->xb, H, R);
        }
        B->head(R, true);   // lm_head, row ArgMax and samplers without advancing any state, records of the rows
        spec_accept_kernel<<<1, 128, 0, st>>>(d_ctl, T->d_state, T->d_history, B->d_tok, B->d_lp_rec, T->d_lp);
        c.cnt.kernels++;
        AHA_CUDA_CHECK(cudaGetLastError());
    }
    void pass(int R) {
        if (!T->use_graph) { launches(R); return; }
        graphs.run(*T->ctx, R, [&] { launches(R); });
    }
};

}  // namespace aha
