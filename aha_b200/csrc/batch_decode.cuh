// batch_decode.cuh -- several sequences decoded in lockstep on one handle (SURVEY 8f rank 4, second half).
//
// The reference holds one request at a time behind a lock (src/server/api.rs:117) and every decode step
// streams all weights for ONE token.  Here several sequences share a step: each slot owns a PageTable over the common paged KV pool
// (text_model.cuh; the TextModel's PagePool maps its pages when it is admitted, its prefill writes through that table, and the pool takes the
// pages back when it is released), its own DecodeState (token, position, rope_delta, sampler draw index), history and sampler parameters; a step is
//     [embedding]      embed_rows_kernel        row j <- the last token of slot act[j]
// then per layer
//     [rmsnorm + qkv]  projection               all sequences, every weight row read once
//     [attention]      decode_attn_batch_kernel grid.z = sequence: q/k norm, RoPE, KV append, split-KV attention, merge
//     [o_proj + res]   projection
//     [rmsnorm + gate/up + SwiGLU], [down + res]
// then the head: final norm + lm_head for all rows, the two-stage ArgMax that advances every row's DecodeState, and the sampler of every row
// whose request samples, then, while a running request asks for them, the log-probability records (logprobs.cuh).  Everything that depends on
// WHICH slots run is read from device memory -- the active list d_act (row j -> slot), the attention table d_attn, the per-slot sampler
// arguments d_samp and log-probability flags d_lp_on -- so one CUDA graph per (running count, any request asks) serves every composition.
// Finished sequences leave the step (the activation rows are rebuilt from the token embeddings every step, so compaction is free).
// Packed admission (aha_b200_batch_add_many) borrows xb / logitsb between two steps for the first tokens of several requests at once (head_rows).
//
// The two widths differ only in how a projection is computed:
//   * narrow (init, aha_b200_batch_open / generate_batch): up to 8 sequences on gemv_batch.cuh's CUDA-core GEMV.  It accumulates every
//     (row, sequence) in gemv_kernel's order and the attention / ArgMax / sampler bodies are the single-sequence ones, so each sequence produces
//     exactly the tokens it would produce alone (tests/test_batch_gpu.py compares every sequence with its own single-request run);
//   * wide (init_wide, aha_b200_batch_open_wide): up to 64 sequences on gemv_wide.cuh's tensor-core kernel, each fed by a prep kernel that
//     normalises and / or splits the nb fp32 rows into the fp16 hi / lo rows the kernel's TMA reads.  A sequence's sums do not depend on its
//     row or on the other rows (one MMA width, split-K fixed by the shape), so its ids do not depend on its slot, its neighbours or the step it
//     joined at; they are not those of the single-sequence gemv_kernel, whose sums run in another order.
#pragma once
#include "gemv_batch.cuh"
#include "gemv_wide.cuh"
#include "kv_fork.cuh"
#include "kv_swap.cuh"
#include "text_model.cuh"

namespace aha {

// The host state of the request a batch-session slot runs (api.cu's session layer keeps it; a speculative step reads R)
struct SlotRequest {
    bool used = false;                   // the slot runs a request
    size_t budget = 0, produced = 0;     // its max_tokens and the tokens it has delivered
    size_t hit = 0;                      // prompt tokens it took from the prefix cache
    bool spec = false;                   // a speculative request, stepped in verify passes of R rows
    int R = 1;
    aha_spec_stats spec_stats{};         // its counters
    bool lp_valid = false;               // the slot's record row holds the record of the last token its request delivered
    int last_n = 0;                      // tokens its last speculative pass delivered (0: its last token came from admission or a plain step)
    uint32_t lora = 0;                   // the LoRA adapter it runs (aha_b200_batch_add_lora; 0: the base model)
    // a finished request: the slot is free, and its record, last_n and spec counters stay readable until the slot is taken again
    void release() { used = false; hit = 0; spec = false; lora = 0; }
    // a cancelled or suspended request, or a failed admission: as release, but the slot shows no record
    void clear() { release(); lp_valid = false; last_n = 0; }
};

struct BatchSlot {                       // one sequence of the batch
    PageTable table;                     // its pages, which it holds from its prefill until it is released; device copy: row of BatchDecoder::d_tables
    bool samp_active = false;
    SampleArgs samp{};                   // sampler of the request with the pointers of this slot
    int lp = 0;                          // 0: the request asked for no log-probabilities, else 1 + its top count
    uint32_t fsm_id = 0;                 // the token automaton the request is constrained by (0: none); it cannot be destroyed while the slot runs
    uint32_t rules_id = 0;               // the request's logit-rules object (0: none); it cannot be destroyed while the slot runs
    Sampler sampler;                     // the request's sampler as bound (a suspended request takes it along and is bound again at resume)
    SlotRequest req;
};

struct BatchDecoder {
    TextModel* T = nullptr;
    int cap = 0;                         // slots allocated
    float *xb = nullptr, *qkvb = nullptr, *attnb = nullptr, *hb = nullptr, *logitsb = nullptr, *partialb = nullptr;
    int* countersb = nullptr;
    float* pmaxb = nullptr; int* pidxb = nullptr; int n_pcand = 0;
    DecodeState* d_states = nullptr;     // [cap]
    uint32_t* d_hist = nullptr;          // [cap][hist_cap]
    uint32_t* d_tok = nullptr;           // [cap] token of the last step per slot
    int* d_tables = nullptr;             // [cap][num_pages]
    DecodeAttnArgs* d_attn = nullptr;    // [L][cap] attention arguments of the current active list
    int* d_act = nullptr;                // [cap] row -> slot
    SampleArgs* d_samp = nullptr;        // [cap] per-slot sampler arguments
    int* d_samp_on = nullptr;            // [cap]
    float* workb = nullptr;              // [cap][V] sampler scratch, one row per slot (the rows sample concurrently)
    int* cntb = nullptr;                 // [cap][V] count rows of frequency / presence penalties, allocated when a request of the handle first asks
    // log-probabilities (logprobs.cuh), allocated when a request of the session first asks: per slot the on flag and the record of its
    // latest token; the candidate lists of every row
    int* d_lp_on = nullptr;              // [cap] BatchSlot::lp
    aha_logprobs* d_lp_rec = nullptr;    // [cap]
    float* lp_part = nullptr; int* lp_part_id = nullptr;
    bool lp_any = false;                 // a request of the current composition asks: the head computes records
    std::vector<BatchSlot> slots;
    std::vector<int> table_for;          // active list the device copy of the composition was built for
    // set when a session opens (AHA_BATCH_GEMV, AHA_BATCH_GRAPH): the narrow step's projections -- 0 = batched GEMV with the weights in
    // registers, 1 = exact SIMT GEMM (validation twin), 2 = batched GEMV with the cp.async weight ring -- and eager launches instead of graphs
    int gemv = 2;
    bool use_graph = true;
    // one CUDA graph per (running count, any request asks for log-probabilities, any runs a LoRA adapter) (~170 launches per step become
    // one); they outlive composition changes
    GraphCache<std::pair<int, int>> graphs;
    // LoRA (lora.cuh), wide sessions only: per slot the index of its request's adapter (-1: none), the tail lists of the adapters the
    // composition runs and the t rows of the step; allocated from T->lora's memory, so they are re-made whenever its pools are rebuilt
    bool lora_any = false;               // a request of the current composition runs an adapter
    uint64_t lora_version = 0;           // the pools (LoraSet::version) the buffers and the adapter graphs were made for
    int* d_slot_lora = nullptr;          // [cap]
    int* d_lora_list = nullptr;          // [4][LoraSet::list_stride()]
    __half *lt_hi = nullptr, *lt_lo = nullptr;   // [64][LoraSet::Rmax]
    // the set of running requests or a slot's sampler changed: the device copy of the composition is rebuilt before the next step
    void composition_changed() { table_for.clear(); ++epoch; }
    uint64_t epoch = 0;                  // counts composition changes (a speculative step rebuilds its own device copies on a new one)
    // no sequence holds a slot any more (a session opens or closes)
    void reset() {
        for (auto& sl : slots) { sl.table.mapped = 0; sl.lp = 0; sl.req = SlotRequest{}; }
        table_for.clear();
        lp_any = false;
        lora_any = false;
        graphs.clear();
    }

    // ---- wide mode
    struct WideAct { __half* hi = nullptr; __half* lo = nullptr; int K = 0; };   // [64][K] operand rows of one K
    bool wide = false;
    WideAct act_h, act_q, act_i;         // K = H (qkv, gate_up, lm_head), K = heads x head_dim (o_proj), K = I (down)
    int rows_live = 0;                   // operand rows that may be non-zero (rows >= the running count are zeroed when it falls)
    float* wide_ws = nullptr; int* wide_cnt = nullptr;

    // a wide decoder of kWideSeqs slots: the kernel's B tile is 64 sequences wide whatever the session width, so the buffers are too
    void init_wide(TextModel& t) {
        init(t, kWideSeqs);
        if (wide) return;
        Ctx& c = *t.ctx;
        const TextCfg& cf = t.cfg;
        auto mk = [&](int K) {
            WideAct a; a.K = K;
            a.hi = c.alloc<__half>((size_t)kWideSeqs * K); a.lo = c.alloc<__half>((size_t)kWideSeqs * K);
            AHA_CUDA_CHECK(cudaMemset(a.hi, 0, (size_t)kWideSeqs * K * sizeof(__half)));
            AHA_CUDA_CHECK(cudaMemset(a.lo, 0, (size_t)kWideSeqs * K * sizeof(__half)));
            return a;
        };
        act_h = mk(cf.H); act_q = mk(t.nh_l * cf.hd); act_i = mk(t.I_l);
        size_t ws = 0; int tiles = 0;
        auto need = [&](int N, int K) { ws = std::max(ws, wide_ws_floats(N, K, c.num_sms)); tiles = std::max(tiles, wide_plan(N, K, c.num_sms).tiles); };
        need(t.qkv_dim, cf.H); need(cf.H, t.nh_l * cf.hd); need(2 * t.I_l, cf.H); need(cf.H, t.I_l); need(cf.V, cf.H);
        if (ws) wide_ws = c.alloc<float>(ws);
        wide_cnt = c.alloc<int>(tiles);
        AHA_CUDA_CHECK(cudaMemset(wide_cnt, 0, (size_t)tiles * sizeof(int)));
        rows_live = 0;
        wide = true;
    }
    // every projection of the model tiles the wide kernel (N and K multiples of 64)
    static bool wide_shapes_ok(const TextModel& t) {
        const TextCfg& cf = t.cfg;
        return gemv_wide_supported(t.qkv_dim, cf.H) && gemv_wide_supported(cf.H, t.nh_l * cf.hd) && gemv_wide_supported(2 * t.I_l, cf.H) &&
               gemv_wide_supported(cf.H, t.I_l) && gemv_wide_supported(cf.V, cf.H);
    }

    void init(TextModel& t, int n) {
        T = &t;
        if (n <= cap) return;
        AHA_REQUIRE(cap == 0, "batch decoder already sized");   // one size per handle: kGemvBatchMax
        Ctx& c = *t.ctx;
        cap = n;
        const TextCfg& cf = t.cfg;
        xb = c.alloc<float>((size_t)n * cf.H); qkvb = c.alloc<float>((size_t)n * t.qkv_dim); attnb = c.alloc<float>((size_t)n * t.nh_l * cf.hd);
        hb = c.alloc<float>((size_t)n * t.I_l); logitsb = c.alloc<float>((size_t)n * cf.V);
        partialb = c.alloc<float>((size_t)n * t.nh_l * kDecodeSplits * (cf.hd + 2));
        countersb = c.alloc<int>((size_t)n * t.nkv_l);
        AHA_CUDA_CHECK(cudaMemset(countersb, 0, (size_t)n * t.nkv_l * sizeof(int)));
        n_pcand = 64;
        pmaxb = c.alloc<float>((size_t)n * n_pcand); pidxb = c.alloc<int>((size_t)n * n_pcand);
        d_states = c.alloc<DecodeState>(n);
        d_hist = c.alloc<uint32_t>((size_t)n * t.hist_cap);
        d_tok = c.alloc<uint32_t>(n);
        d_tables = c.alloc<int>((size_t)n * t.num_pages);
        d_attn = c.alloc<DecodeAttnArgs>((size_t)cf.L * n);
        d_act = c.alloc<int>(n);
        d_samp = c.alloc<SampleArgs>(n);
        d_samp_on = c.alloc<int>(n);
        workb = c.alloc<float>((size_t)n * cf.V);
        slots.resize(n);
        for (int i = 0; i < n; ++i) { slots[i].table.h.assign(t.num_pages, 0); slots[i].table.d = d_tables + (size_t)i * t.num_pages; }
    }

    // after the first token of slot i: its decode state starts from that token (history[0]) at position seq_len, with the draw index and
    // automaton state the first token left
    void adopt(int i, uint32_t first_token, int seq_len, int rope_delta, uint32_t n_draws, uint32_t fsm_state) {
        Ctx& c = *T->ctx;
        DecodeState st{first_token, seq_len, rope_delta, 1, n_draws, fsm_state, {0, 0}};
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_states + i, &st, sizeof(st), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_hist + (size_t)i * T->hist_cap, &first_token, sizeof(uint32_t), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));   // stack temporaries
    }
    // the K/V of positions [0, n_tokens) of slot src copied into slots dst, whose tables already map those pages (kv_fork.cuh)
    void fork(int src, const std::vector<int>& dst, int n_tokens) {
        kv_fork(*T->ctx, T->kv_pool, T->layer_stride, T->page_stride, T->cfg.L, d_tables, T->num_pages, src, dst.data(), (int)dst.size(),
                ceil_div(n_tokens, kPage));
    }
    void ensure_lp() {
        if (d_lp_rec) return;
        Ctx& c = *T->ctx;
        const int P = lp_parts(T->cfg.V);
        d_lp_on = c.alloc<int>(cap);
        d_lp_rec = c.alloc<aha_logprobs>(cap);
        lp_part = c.alloc<float>((size_t)cap * P * kLpPartFloats);
        lp_part_id = c.alloc<int>((size_t)cap * P * kLpMaxTop);
        AHA_CUDA_CHECK(cudaMemset(d_lp_on, 0, (size_t)cap * sizeof(int)));
    }
    // the request's sampler becomes slot i's, with the slot's own state, history, token and scratch row
    void bind_sampler(int i, const Sampler& s) {
        BatchSlot& sl = slots[i];
        sl.samp_active = s.active;
        sl.sampler = s;
        sl.fsm_id = s.fsm_id;
        sl.rules_id = s.rules_id;
        if (s.active) sl.samp = T->bind_sampler(s, d_states + i, d_hist + (size_t)i * T->hist_cap, d_tok + i, workb + (size_t)i * T->cfg.V, counts(s, i));
    }
    // slot i's count row when the request has frequency or presence penalties (else null)
    int* counts(const Sampler& s, int i) {
        if (!s.counts) return nullptr;
        if (!cntb) cntb = T->alloc_counts(cap);
        return cntb + (size_t)i * T->cfg.V;
    }

    // the device copy of the composition `act`: attention table, active list and every slot's sampler arguments
    void build_attn_table(const std::vector<int>& act) {
        const TextCfg& cf = T->cfg;
        const int nb = (int)act.size();
        std::vector<DecodeAttnArgs> h((size_t)cf.L * cap);
        const float scaling = (float)(1.0 / std::sqrt((double)cf.hd));
        for (int l = 0; l < cf.L; ++l) {
            TextLayer& Ly = T->layers[l];
            for (int j = 0; j < nb; ++j) {
                DecodeAttnArgs d{};
                const int slot = act[j];
                const KVSrc kv = T->kv_src(l, slots[slot].table);
                d.qkv = qkvb + (size_t)j * T->qkv_dim; d.qw = Ly.qn; d.kw = Ly.kn; d.eps = cf.eps; d.inv_freq = T->inv_freq; d.st = d_states + slot;
                d.kbase = const_cast<float*>(kv.k); d.vbase = const_cast<float*>(kv.v);
                d.kv = kv;
                d.partial = partialb + (size_t)j * T->nh_l * kDecodeSplits * (cf.hd + 2);
                d.counters = countersb + (size_t)j * T->nkv_l;
                d.out = attnb + (size_t)j * T->nh_l * cf.hd;
                d.nh = T->nh_l; d.nkv = T->nkv_l; d.nsplit = kDecodeSplits; d.scaling = scaling;
                h[(size_t)l * cap + j] = d;
            }
        }
        std::vector<SampleArgs> samp((size_t)cap);
        std::vector<int> on((size_t)cap, 0);
        for (int i = 0; i < cap; ++i) { on[i] = slots[i].samp_active ? 1 : 0; if (on[i]) samp[i] = slots[i].samp; }
        std::vector<int> lp_on((size_t)cap, 0);
        lp_any = false;
        for (int i = 0; i < cap; ++i) lp_on[i] = slots[i].lp;
        for (int s : act) lp_any = lp_any || slots[s].lp > 0;
        Ctx& c = *T->ctx;
        lora_table(act);
        if (d_lp_on) AHA_CUDA_CHECK(cudaMemcpyAsync(d_lp_on, lp_on.data(), lp_on.size() * sizeof(int), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_attn, h.data(), h.size() * sizeof(DecodeAttnArgs), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_act, act.data(), act.size() * sizeof(int), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_samp, samp.data(), samp.size() * sizeof(SampleArgs), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_samp_on, on.data(), on.size() * sizeof(int), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
        table_for = act;
    }

    template <int G>
    void launch_attn(int l, int nb) {
        decode_attn_batch_kernel<128, G><<<dim3(kDecodeSplits, T->nkv_l, nb), 256, 0, T->ctx->stream>>>(d_attn + (size_t)l * cap);
    }

    // the attention of rows 0..nb-1 (the active list's first nb slots) in layer l
    void attn(int l, int nb) {
        switch (T->nh_l / T->nkv_l) {
            case 1: launch_attn<1>(l, nb); break;
            case 2: launch_attn<2>(l, nb); break;
            case 4: launch_attn<4>(l, nb); break;
            default: launch_attn<6>(l, nb); break;
        }
        T->ctx->cnt.kernels++;
    }

    // rows 0..nb-1: out = epi(W . x), x RMSNorm-ed with norm_w first when given; (l, g): the layer and LoRA group of a projection adapters
    // may target (g < 0: none)
    void proj(int epi, const LinearW& W, const float* x, int ldx, const float* norm_w, const float* resid, int ldr, float* out, int ldo, int nb,
              int l = -1, int g = -1) {
        Ctx& c = *T->ctx;
        if (wide) {
            const WideAct& in = W.K == act_h.K ? act_h : (W.K == act_i.K ? act_i : act_q);   // (any [64][K] operand of the right K will do)
            wide_prep(x, ldx, norm_w, in, nb);
            LoraTail tail;
            if (lora_any && g >= 0 && T->lora.Rp[g] > 0) {   // the rows' shrink outputs from the operand the projection reads, then the tail
                const LoraSet& Lr = T->lora;
                lora_shrink(c.stream, nb, in.hi, in.lo, nullptr, in.K, in.K, Lr.A[g][l], Lr.Rp[g], Lr.d_tab, g, d_slot_lora, d_act, lt_hi, lt_lo, nullptr);
                c.cnt.kernels++;
                tail.t_hi = lt_hi; tail.t_lo = lt_lo; tail.B = Lr.B[g][l]; tail.Rp = Lr.Rp[g];
                tail.list = d_lora_list + (size_t)g * Lr.list_stride();
            }
            wide_proj(epi, W, in, resid, ldr, out, ldo, nb, &tail);
            return;
        }
        if (gemv == 1) {   // validation twin: the exact fp32 SIMT GEMM over the nb rows (normalised beforehand when a prologue is asked for)
            const float* a = x; int lda = ldx;
            if (norm_w) {
                rmsnorm_kernel<<<nb, 256, 0, c.stream>>>(x, norm_w, T->cfg.eps, T->xn, W.K); c.cnt.kernels++;   // xn: [max_prefill >= 8][H] scratch of the prefill
                a = T->xn; lda = W.K;
            }
            GemmArgs g{};
            g.A = a; g.lda = lda; g.W = W.w; g.bias = W.b; g.resid = resid; g.ldr = ldr; g.C = out; g.ldc = ldo; g.M = nb; g.N = W.N; g.K = W.K; g.act = ACT_NONE;
            gemm_simt(c.stream, epi == GEPI_STORE ? EPI_STORE : (epi == GEPI_RESID ? EPI_RESID : EPI_SWIGLU), g);
            c.cnt.kernels++;
            return;
        }
        GemvBatchArgs a{};
        a.W = W.w; a.x = x; a.ldx = ldx; a.norm_w = norm_w; a.eps = T->cfg.eps; a.bias = W.b; a.resid = resid; a.ldr = ldr; a.out = out; a.ldo = ldo;
        a.N = W.N; a.K = W.K; a.nb = nb;
        gemv_batch(c.stream, norm_w ? PRO_RMSNORM : PRO_NONE, epi, a, gemv == 2);
        c.cnt.kernels++;
    }

    // The adapters of the composition `act` (wide sessions): the slots' adapter indices and the tail lists to the device.  New pools
    // (an adapter was created or destroyed) drop the buffers and the step graphs that read the old ones.
    void lora_table(const std::vector<int>& act) {
        LoraSet& Lr = T->lora;
        if (lora_version != Lr.version) {
            lora_version = Lr.version;
            d_slot_lora = d_lora_list = nullptr; lt_hi = lt_lo = nullptr;
            std::vector<GraphCache<std::pair<int, int>>::Entry> keep;
            for (auto& e : graphs.entries) {
                if (e.key.second & 2) { if (e.exec) cudaGraphExecDestroy(e.exec); }
                else keep.push_back(e);
            }
            graphs.entries.swap(keep);
        }
        std::vector<int> ad((size_t)cap, -1), used;
        lora_any = false;
        for (int s : act) {
            if (!slots[s].req.lora) continue;
            ad[s] = Lr.index_of(slots[s].req.lora);
            AHA_REQUIRE(ad[s] >= 0, "batch step: slot " + std::to_string(s) + " runs an adapter that is not loaded");
            used.push_back(ad[s]);
            lora_any = true;
        }
        if (!lora_any) return;
        AHA_REQUIRE(wide, "LoRA adapters run in wide sessions only");
        Ctx& c = *T->ctx;
        if (!d_slot_lora) {
            d_slot_lora = Lr.dalloc<int>((size_t)cap);
            d_lora_list = Lr.dalloc<int>((size_t)kLoraGroups * Lr.list_stride());
            lt_hi = Lr.dalloc<__half>((size_t)kWideSeqs * Lr.Rmax);
            lt_lo = Lr.dalloc<__half>((size_t)kWideSeqs * Lr.Rmax);
            AHA_CUDA_CHECK(cudaMemsetAsync(lt_hi, 0, (size_t)kWideSeqs * Lr.Rmax * sizeof(__half), c.stream));
            AHA_CUDA_CHECK(cudaMemsetAsync(lt_lo, 0, (size_t)kWideSeqs * Lr.Rmax * sizeof(__half), c.stream));
        }
        const std::vector<int> lists = Lr.lists(used);
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_slot_lora, ad.data(), ad.size() * sizeof(int), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_lora_list, lists.data(), lists.size() * sizeof(int), cudaMemcpyHostToDevice, c.stream));
        AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));   // host vectors
    }

    // one decode step of the sequences in `act` (slot indices, at most cap); leaves every slot's next token in d_tok[slot] and its DecodeState advanced
    void step(const std::vector<int>& act) {
        Ctx& c = *T->ctx;
        AHA_REQUIRE(!act.empty() && (int)act.size() <= cap, "batch step: bad active list");
        if (T->lora.version != lora_version) table_for.clear();
        if (act != table_for) build_attn_table(act);
        const int nb = (int)act.size();
        if (wide) zero_rows_from(nb);
        if (!use_graph) { launches(nb); return; }
        graphs.run(c, {nb, (lp_any ? 1 : 0) | (lora_any ? 2 : 0)}, [&] { launches(nb); });
    }
    void launches(int nb) {
        Ctx& c = *T->ctx;
        const TextCfg& cf = T->cfg;
        const int H = cf.H;
        embed_rows_kernel<<<nb, 256, 0, c.stream>>>(d_act, d_states, T->embed, xb, H, cf.V);
        c.cnt.kernels++;
        for (int l = 0; l < cf.L; ++l) {
            TextLayer& Ly = T->layers[l];
            proj(GEPI_STORE, Ly.qkv, xb, H, Ly.ln1, nullptr, 0, qkvb, T->qkv_dim, nb, l, LORA_QKV);
            attn(l, nb);
            proj(GEPI_RESID, Ly.o, attnb, T->nh_l * cf.hd, nullptr, xb, H, xb, H, nb, l, LORA_O);
            proj(GEPI_SWIGLU, Ly.gu, xb, H, Ly.ln2, nullptr, 0, hb, T->I_l, nb, l, LORA_GU);
            proj(GEPI_RESID, Ly.down, hb, T->I_l, nullptr, xb, H, xb, H, nb, l, LORA_DOWN);
        }
        head(nb, false);
    }
    // Final norm + lm_head over rows 0 .. nb-1 of xb, then for row j the two-stage ArgMax of slot d_act[j] and, when its request samples, its
    // sampler, then, when a request of the composition asks, the log-probability records of the rows whose request asks (into d_lp_rec[slot]).
    // A decode step (first = false) advances the slot's DecodeState and the sampled token replaces the ArgMax one the step pushed
    // (the single-sequence loop does the same).  A request's first token (first = true, packed admission) is drawn the way forward_any draws
    // it: no advance, no overwrite, against the slot's state as the caller set it (empty history, draw index 0); only n_draws moves.
    void head(int nb, bool first) {
        lm_head(nb);
        head_rows_at(0, nb, d_act, d_tok, d_states, d_hist, d_samp, d_samp_on, d_lp_on, d_lp_rec, first, lp_any);
    }
    // final norm + lm_head and ArgMax stage 1 over rows 0 .. nb-1
    void lm_head(int nb) {
        Ctx& c = *T->ctx;
        const TextCfg& cf = T->cfg;
        LinearW lm; lm.w = T->lm_head; lm.b = nullptr; lm.N = cf.V; lm.K = cf.H;
        proj(GEPI_STORE, lm, xb, cf.H, T->norm, nullptr, 0, logitsb, cf.V, nb);
        argmax_partial_rows_kernel<<<dim3(n_pcand, nb), 256, 0, c.stream>>>(logitsb, cf.V, cf.V, pmaxb, pidxb);
        c.cnt.kernels++;
    }
    // ArgMax stage 2, sampler and (lp) records of rows r0 .. r0 + n - 1, row r0 + j standing for entry act[j] of the per-row arrays given
    // (tok, st, hist, samp, samp_on, lp_on, rec: a slot's, or a speculative verify row's)
    void head_rows_at(int r0, int n, const int* act, uint32_t* tok, DecodeState* st, uint32_t* hist, const SampleArgs* samp, const int* samp_on,
                      const int* lp_on, aha_logprobs* rec, bool first, bool lp) {
        Ctx& c = *T->ctx;
        cudaStream_t s = c.stream;
        const int V = T->cfg.V;
        const float* logits = logitsb + (size_t)r0 * V;
        argmax_final_rows_kernel<<<n, 32, 0, s>>>(pmaxb + (size_t)r0 * n_pcand, pidxb + (size_t)r0 * n_pcand, n_pcand, act, tok, st, hist, T->hist_cap, first ? 0 : 1);
        sample_rows_kernel<<<n, kSampleThreads, 0, s>>>(samp, samp_on, act, logits, V, first ? 0 : 1);
        c.cnt.kernels += 2;
        if (lp) {
            const size_t P = (size_t)lp_parts(V);
            logprobs_rows(s, logits, V, V, n, act, lp_on, lp_part + (size_t)r0 * P * kLpPartFloats, lp_part_id + (size_t)r0 * P * kLpMaxTop, tok, st,
                          first ? 1 : 0, rec, 0, cap);
            c.cnt.kernels += 2;
        }
        AHA_CUDA_CHECK(cudaGetLastError());
    }
    // the first tokens of the slots in `act`, whose last prompt rows packed admission gathered into xb and whose samplers were just bound
    void head_rows(const std::vector<int>& act, bool first) {
        build_attn_table(act);
        const int nb = (int)act.size();
        if (wide) zero_rows_from(nb);
        head(nb, first);
    }

    // ---- the wide projection
    // operand rows nb..63 left by a wider step are zeroed: their columns are never stored, but a zero B column keeps the stated invariant
    void zero_rows_from(int nb) {
        if (nb < rows_live) {
            cudaStream_t st = T->ctx->stream;
            for (const WideAct* a : {&act_h, &act_q, &act_i}) {
                const size_t off = (size_t)nb * a->K, n = (size_t)(rows_live - nb) * a->K * sizeof(__half);
                AHA_CUDA_CHECK(cudaMemsetAsync(a->hi + off, 0, n, st));
                AHA_CUDA_CHECK(cudaMemsetAsync(a->lo + off, 0, n, st));
            }
        }
        rows_live = nb;
    }
    // prep: rows 0..nb-1 of x (ldx floats apart) -> the hi / lo operand rows of `in`, RMSNorm-ed with norm_w when given
    void wide_prep(const float* x, int ldx, const float* norm_w, const WideAct& in, int nb) {
        Ctx& c = *T->ctx;
        if (norm_w) {
            AHA_REQUIRE(ldx == in.K, "wide prep: normalised rows must be packed");
            rmsnorm_split_kernel<<<nb, 256, 0, c.stream>>>(x, norm_w, T->cfg.eps, in.hi, in.lo, in.K);
        } else {
            const size_t n4 = (size_t)nb * in.K / 4;
            split_f32_to_f16x2_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, c.stream>>>(x, ldx, in.hi, in.lo, nb, in.K);
        }
        c.cnt.kernels++;
    }
    void wide_proj(int epi, const LinearW& W, const WideAct& in, const float* resid, int ldr, float* out, int ldo, int nb, const LoraTail* tail = nullptr) {
        Ctx& c = *T->ctx;
        WideArgs a{};
        a.bias = W.b; a.resid = resid; a.ldr = ldr; a.out = out; a.ldo = ldo; a.N = W.N; a.K = W.K; a.nb = nb;
        a.ws = wide_ws; a.counters = wide_cnt;
        AHA_REQUIRE(W.K == in.K, "wide projection: operand width mismatch");
        const CUtensorMap tm = W.has_tmap ? W.tmap : make_tmap_f16(W.w, (uint64_t)W.N, (uint64_t)W.K);
        gemv_wide(c.stream, epi, tm, in.hi, in.lo, a, c.num_sms, tail);
        c.cnt.kernels++;
    }
};

}  // namespace aha
