// api.cu -- extern "C" entry points of libaha_b200.so (see include/aha_b200.h for the contract and the
// reference items each entry replaces).  Host side = the C++ mirror of aha's model structs:
// Qwen3Model (src/models/qwen3/model.rs:94-214), Qwen3VLModel (qwen3vl/model.rs:837-1324),
// Qwen3ASRModel (qwen3_asr/model.rs:308-425) and generate_generic (common/generate.rs:115-159).
#include <array>
#include <cassert>
#include <chrono>
#include <cstdio>
#include <functional>
#include <limits>
#include <map>
#include <mutex>
#include <set>
#include <unordered_map>
#include <system_error>
#include <thread>
#include <type_traits>

#include "audio_model.cuh"
#include "preprocess.cuh"
#include "score_head.cuh"
#include "text_model.cuh"
#include "batch_decode.cuh"
#include "speculative.cuh"
#include "vision_model.cuh"

using namespace aha;

namespace {
std::mutex g_err_mu;
std::string g_create_error;
// the error of a call without a handle, read by aha_b200_last_error(NULL)
void set_create_error(const char* what) {
    std::lock_guard<std::mutex> lk(g_err_mu);
    g_create_error = what;
}
template <typename F>
int guarded_host(F&& f) {   // host-only entries (no handle)
    try { f(); return 0; }
    catch (const std::exception& e) { set_create_error(e.what()); return 1; }
}
}  // namespace

// A batch session's prefix cache (aha_b200_batch_prefix_cache): full 32-token pages of admitted prompts, keyed by their token ids and their
// parent page, so that a later request whose prompt starts with the same pages maps them into its table instead of prefilling them.  Every
// block holds one reference on its page (PagePool::refs); the blocks form a tree from the prompts' first pages.  A key's hash only narrows
// the search: a match is confirmed on the 32 ids.  A prompt's first page hangs below the root of the LoRA adapter its request ran
// (root(0) = -1 for the base model), so a request only finds pages written under its own adapter.
struct PrefixIndex {
    static int root(uint32_t lora) { return -1 - (int)lora; }
    struct Block {
        uint32_t ids[kPage];
        int parent = -1;     // page of the block before it in the prompt (< 0: the prompt's first page, below root(its adapter))
        int children = 0;    // cached blocks whose parent this is
        uint64_t used = 0;   // LRU clock of the last admission that hit or inserted it
    };
    size_t max_pages = 0;                          // 0: off
    std::unordered_map<int, Block> blocks;         // by page
    std::unordered_multimap<uint64_t, int> by_key; // hash(parent, ids) -> page
    uint64_t clock = 0, hit_tokens = 0, lookups = 0, evicted = 0;
    bool on() const { return max_pages > 0; }
    static uint64_t key(int parent, const uint32_t* ids) {
        uint64_t h = 0x9e3779b97f4a7c15ull ^ (uint64_t)(uint32_t)parent;
        for (int i = 0; i < kPage; ++i) { h = (h ^ ids[i]) * 0xff51afd7ed558ccdull; h ^= h >> 29; }
        return h;
    }
    // the page caching ids[0, kPage) after `parent`, or -1
    int find(int parent, const uint32_t* ids) const {
        auto r = by_key.equal_range(key(parent, ids));
        for (auto it = r.first; it != r.second; ++it) {
            const Block& b = blocks.at(it->second);
            if (b.parent == parent && std::equal(ids, ids + kPage, b.ids)) return it->second;
        }
        return -1;
    }
    // the pages of the longest cached chain of full pages that starts ids[0, n) under adapter `lora`
    std::vector<int> chain(const uint32_t* ids, size_t n, uint32_t lora) const {
        std::vector<int> pages;
        int parent = root(lora);
        for (size_t t = 0; t + kPage <= n; t += kPage) {
            const int p = find(parent, ids + t);
            if (p < 0) break;
            pages.push_back(p);
            parent = p;
        }
        return pages;
    }
    // pages the index alone holds, outside `keep`: every one can be evicted, leaves first (a page a table holds keeps its ancestors held too)
    size_t evictable(const PagePool& pool, const std::set<int>& keep) const {
        size_t k = 0;
        for (const auto& e : blocks) k += pool.refs[e.first] == 1 && !keep.count(e.first);
        return k;
    }
    // drop the least recently used leaf only the index holds, outside `keep`; false when there is none
    bool evict_one(PagePool& pool, const std::set<int>& keep) {
        int victim = -1;
        uint64_t best = 0;
        for (const auto& e : blocks)
            if (pool.refs[e.first] == 1 && e.second.children == 0 && !keep.count(e.first) && (victim < 0 || e.second.used < best)) {
                victim = e.first;
                best = e.second.used;
            }
        if (victim < 0) return false;
        erase(pool, victim);
        ++evicted;
        return true;
    }
    void erase(PagePool& pool, int page) {
        const Block& b = blocks.at(page);
        auto r = by_key.equal_range(key(b.parent, b.ids));
        for (auto it = r.first; it != r.second; ++it) if (it->second == page) { by_key.erase(it); break; }
        if (b.parent >= 0) blocks.at(b.parent).children -= 1;
        blocks.erase(page);
        pool.unref(page);
    }
    // every block cached under adapter `lora` (aha_b200_lora_destroy): one pass finds each block's root and depth (memoised along the
    // chain), then the adapter's blocks are erased deepest first, so every block is a leaf when it goes
    void drop(PagePool& pool, uint32_t lora) {
        std::unordered_map<int, std::pair<int, int>> at;   // page -> (root, depth)
        std::vector<int> chain;
        for (const auto& e : blocks) {
            int q = e.first;
            chain.clear();
            while (q >= 0 && !at.count(q)) { chain.push_back(q); q = blocks.at(q).parent; }
            std::pair<int, int> rd = q >= 0 ? at.at(q) : std::make_pair(q, -1);
            for (auto it = chain.rbegin(); it != chain.rend(); ++it) { rd.second += 1; at[*it] = rd; }
        }
        std::vector<std::pair<int, int>> mine;   // (depth, page)
        for (const auto& e : at) if (e.second.first == root(lora)) mine.emplace_back(e.second.second, e.first);
        std::sort(mine.rbegin(), mine.rend());
        for (const auto& d : mine) erase(pool, d.second);
    }
    // The full pages of an admitted prompt that the table `t` holds (its first hit / kPage of them are the cached chain it hit), in prompt
    // order.  Inserting beyond max_pages evicts LRU leaves first; the chain stops at the first page that cannot be inserted.
    void insert(PagePool& pool, const uint32_t* ids, size_t n, const PageTable& t, uint32_t lora) {
        ++clock;
        int parent = root(lora);
        for (size_t b = 0; (b + 1) * kPage <= n; ++b) {
            const int page = t.h[b];
            const int have = find(parent, ids + b * kPage);
            if (have >= 0) {   // the chain this request hit, or the same ids inserted earlier in this call from another request's pages
                blocks.at(have).used = clock;
                if (have != page) return;
                parent = page;
                continue;
            }
            while (blocks.size() >= max_pages) if (!evict_one(pool, {})) return;
            Block& nb = blocks[page];
            std::copy(ids + b * kPage, ids + (b + 1) * kPage, nb.ids);
            nb.parent = parent;
            nb.used = clock;
            if (parent >= 0) blocks.at(parent).children += 1;
            by_key.emplace(key(parent, nb.ids), page);
            pool.ref(page);
            parent = page;
        }
    }
    // max_tokens 0: every block lets go of its page
    void clear(PagePool& pool) {
        for (const auto& e : blocks) pool.unref(e.first);
        blocks.clear();
        by_key.clear();
    }
};

struct aha_model {
    enum Kind { QWEN3, QWEN3VL, QWEN3_ASR } kind = QWEN3;
    Ctx ctx;
    TextModel text;
    VisionModel vision;
    AudioModel audio;
    std::vector<uint32_t> stop_ids;
    std::string last_error;
    // Qwen3-VL state / config
    int image_token_id = -1, video_token_id = -1, vision_start_token_id = -1;
    bool have_rope_delta = false;  // rope_deltas: Option<Tensor>, qwen3vl/model.rs:842
    int rope_delta = 0;
    int audio_token_id = -1;
    int* d_scatter_idx = nullptr;
    int max_scatter = 0;
    int* d_pack_work = nullptr;   // packed prefills (embed_batch, batch_add_many): varlen attention work list ([max_prefill][kFaWork]), the rows
    int* d_pack_rows = nullptr;   // taken from the pack ([max_prefill]) and the pack's page table ([num_pages]); allocated on first use
    int* d_pack_table = nullptr;
    int* d_pack_read = nullptr;   // the read table of a pack with cached prefixes ([num_pages]); allocated when a batch_add_many first hits
    double last_vision_secs = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    // pinned staging for the host<->device scalars of a step / the tokens of a burst
    uint32_t* h_pin = nullptr;
    aha_logprobs* h_lp_pin = nullptr;        // [32] the records of a burst (generate_logprobs), allocated the first time a request asks
    static constexpr int kStreamBurst = 8;   // streaming: steps the device may run ahead of the token being delivered
    cudaEvent_t ev_tok[kStreamBurst] = {};
    // KV reuse across requests (SURVEY 8f rank 4; new design: the reference clears the cache after every request, common/generate.rs:147,
    // and serialises requests behind one lock, server/api.rs:117).  A request that carries AHA_GEN_REUSE_PREFIX leaves its K/V in the paged
    // cache; the next such request prefills only what follows the longest common prefix.
    std::vector<uint32_t> cached_ids;   // tokens whose K/V occupy positions 0 .. n-1 of the paged cache
    uint64_t cached_mm_fp = 0;          // fingerprint of the multimodal tensors those tokens were embedded with (0 = none)
    size_t last_prefix_hit = 0;         // tokens the last generate call did not have to prefill
    BatchDecoder batch;                 // several sequences decoded in lockstep (aha_b200_generate_batch); buffers allocated on first use
    BatchDecoder wide_batch;            // the tensor-core decoder of wide sessions (aha_b200_batch_open_wide); buffers allocated on first use
    // Continuous batching (aha_b200_batch_open / _add / _step / _close): requests join and leave a running batch between steps.  Each slot's
    // request state is the decoder's BatchSlot, its host bookkeeping BatchSlot::req.
    struct BatchSession {
        bool open = false;
        bool wide = false;              // opened by batch_open_wide: wide_batch runs it
        int width = kGemvBatchMax;      // slots of the session
        PrefixIndex prefix;             // aha_b200_batch_prefix_cache; dropped with the session
    } session;
    BatchDecoder& sess() { return session.wide ? wide_batch : batch; }   // the decoder of the open session (batch when none is open)
    SpecDecoder spec;                   // speculative requests (generate_speculative, batch_add_speculative) on wide_batch's buffers
    // scoring (aha_b200_score / _score_batch): the buffers of one head launch over up to max_prefill rows and the lm_head's tensor map,
    // set up by the first scoring call
    struct ScoreBufs {
        int* rows = nullptr;            // [M] rows of TextModel::x to score
        uint32_t* tgt = nullptr;        // [M] the token each row is scored at
        uint32_t* index = nullptr;      // [M] the records' index fields
        float* tlogit = nullptr;        // [M] the targets' raw logits (score_head_kernel)
        float* part = nullptr;          // [M][P][kLpPartFloats] slice results
        int* part_id = nullptr;         // [M][P][kLpMaxTop]
        int* on = nullptr;              // [1] 1 + the top count (the twin's logprob_partial_rows_kernel)
        aha_logprobs* rec = nullptr;    // [M]
    } score;
    CUtensorMap score_tm_w{};
    bool score_ready = false;
    // token automata of constrained requests (aha_b200_fsm_create): id -> one device allocation holding offsets | tokens | next
    struct Fsm {
        void* mem = nullptr;
        TokenFsmDev dev;
    };
    std::map<uint32_t, Fsm> fsms;
    uint32_t next_fsm_id = 1;
    // logit-rules objects (aha_b200_rules_create): id -> the penalties, one device allocation holding bias ids | values, and the automaton
    // the object names (0: none)
    struct Rules {
        void* mem = nullptr;
        LogitRulesDev dev;
        uint32_t fsm = 0;
    };
    std::map<uint32_t, Rules> rules;
    uint32_t next_rules_id = 1;
    uint32_t next_lora_id = 1;          // LoRA adapters (aha_b200_lora_create) live in text.lora
    // Swap preemption (aha_b200_batch_swap_space / _suspend / _resume): a pinned host arena of host pages, each holding one KV page of every
    // layer ([layer][page_stride] fp32), kept across sessions until it is resized or the handle is destroyed, and its free list -- a pool of
    // its own, apart from the device PagePool.  The counters run for the handle's lifetime.
    struct SwapArena {
        float* host = nullptr;          // cudaHostAlloc-ed
        size_t pages = 0;
        std::vector<int> free;          // free host pages
        uint64_t pages_out = 0, pages_in = 0;
        double suspend_secs = 0, resume_secs = 0;
    } swap;
    // a suspended request of the open session (aha_b200_batch_suspend): everything its slot held, its K/V in the arena
    struct Suspended {
        std::vector<int> host_pages;    // logical page p -> host page
        int mapped = 0;                 // pages its table held
        DecodeState st{};
        std::vector<uint32_t> hist;     // history [0, st.n_hist)
        Sampler sampler;                // BatchSlot::sampler, ::lp and ::req
        int lp = 0;
        SlotRequest req;
    };
    std::map<uint32_t, Suspended> suspended;   // by id (>= 1)
    uint32_t next_suspend_id = 1;
    size_t swap_page_bytes() const { return (size_t)text.cfg.L * text.page_stride * sizeof(float); }
};

namespace {

void bind(aha_model* m) { AHA_CUDA_CHECK(cudaSetDevice(m->ctx.device)); }

template <typename F>
int guarded(aha_model* m, F&& f) {
    try {
        if (!m) throw std::runtime_error("null model handle");
        bind(m);
        f();
        return 0;
    } catch (const std::exception& e) {
        if (m) m->last_error = e.what();
        else set_create_error(e.what());
        // leave the stream usable: drop a dangling capture, clear sticky launch errors
        if (m && m->ctx.stream) {
            cudaStreamCaptureStatus cs;
            if (cudaStreamIsCapturing(m->ctx.stream, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone) {
                cudaGraph_t g = nullptr; cudaStreamEndCapture(m->ctx.stream, &g); if (g) cudaGraphDestroy(g);
            }
        }
        cudaGetLastError();
        return 1;
    }
}

const aha_tensor_desc* mm_entry(const aha_mm* mm, size_t i) {
    if (!mm || i >= mm->n) return nullptr;
    const aha_tensor_desc* d = &mm->data_vec[i];
    return d->data ? d : nullptr;
}

std::vector<float> desc_to_f32(const aha_tensor_desc& d) {
    const size_t n = WeightTable::numel(d);
    std::vector<float> v(n);
    if (d.dtype == AHA_F32) std::memcpy(v.data(), d.data, n * sizeof(float));
    else for (size_t i = 0; i < n; ++i) v[i] = WeightTable::at(d, i);
    return v;
}
std::vector<int64_t> desc_to_i64(const aha_tensor_desc& d) {
    const size_t n = WeightTable::numel(d);
    std::vector<int64_t> v(n);
    for (size_t i = 0; i < n; ++i) {
        switch (d.dtype) {
            case AHA_U32: v[i] = reinterpret_cast<const uint32_t*>(d.data)[i]; break;
            case AHA_I64: v[i] = reinterpret_cast<const int64_t*>(d.data)[i]; break;
            case AHA_U8: v[i] = reinterpret_cast<const uint8_t*>(d.data)[i]; break;
            default: throw std::runtime_error("integer tensor expected");
        }
    }
    return v;
}

// Qwen3VLModel::get_rope_index, image branch (src/models/qwen3vl/model.rs:901-1071,1072-1090):
// text runs get equal t/h/w ids; an image of merged grid (t,h',w') gets t_idx = base, h_idx = base+0..h'-1,
// w_idx = base+0..w'-1; the next run starts at max+1; rope_delta = max+1-S.  pos3 is [3][S].
// video_grid: video_grid_thw with every (t, h, w) row already expanded to t rows of (1, h, w) (model.rs:907-925): each frame group has
// its own <|vision_start|><|video_pad|>... run in the prompt (timestamps sit between them).
void get_rope_index(const uint32_t* ids, int S, const std::vector<std::array<int, 3>>& grid, const std::vector<std::array<int, 3>>& video_grid, int merge,
                    int image_tok, int video_tok, int vstart_tok, std::vector<int>& pos3, int& delta) {
    pos3.assign((size_t)3 * S, 0);
    if (grid.empty() && video_grid.empty()) {
        for (int r = 0; r < 3; ++r) for (int i = 0; i < S; ++i) pos3[(size_t)r * S + i] = i;
        delta = 0;
        return;
    }
    int out = 0;            // tokens emitted so far
    int last_max = -1;      // max of the last pushed chunk
    bool any = false;
    int text_start = 0, text_end = 0;
    size_t image_index = 0, video_index = 0;
    std::array<int, 3> thw{0, 0, 0};
    bool have_thw = false;
    auto push_text = [&](int len) {
        const int start = any ? last_max + 1 : 0;
        for (int i = 0; i < len; ++i) for (int r = 0; r < 3; ++r) pos3[(size_t)r * S + out + i] = start + i;
        if (len > 0) last_max = start + len - 1;
        // an empty chunk has no max in the reference either; it only matters that `any` flips
        any = true;
        out += len;
        return start + len;
    };
    for (int j0 = 0; j0 < S; ++j0) {
        if ((int)ids[j0] != vstart_tok) continue;
        const int j = j0 + 1;
        if (j >= S) throw std::runtime_error("vision_start token at the end of the prompt");
        if ((int)ids[j] == image_tok) {
            if (image_index >= grid.size()) throw std::runtime_error("more image placeholders than image_grid_thw rows");
            thw = grid[image_index++];
            have_thw = true;
            text_end = j;
        }
        if ((int)ids[j] == video_tok && video_tok >= 0) {
            if (video_index >= video_grid.size()) throw std::runtime_error("more video placeholder runs than video_grid_thw frames");
            thw = video_grid[video_index++];
            have_thw = true;
            text_end = j;
        }
        if (!have_thw) throw std::runtime_error("vision_start not followed by an image or video token");
        const int gt = thw[0], gh = thw[1] / merge, gw = thw[2] / merge;
        const int text_len = text_end - text_start;
        if (out + text_len + gt * gh * gw > S) throw std::runtime_error("image placeholders exceed the prompt length");
        const int base = push_text(text_len);
        for (int t = 0; t < gt; ++t)
            for (int h = 0; h < gh; ++h)
                for (int w = 0; w < gw; ++w) {
                    const int i = out + (t * gh + h) * gw + w;
                    pos3[i] = base + t; pos3[(size_t)S + i] = base + h; pos3[(size_t)2 * S + i] = base + w;
                }
        last_max = base + std::max(gt, std::max(gh, gw)) - 1;
        out += gt * gh * gw;
        text_start = text_end + gt * gh * gw;
    }
    if (text_start < S) push_text(S - text_start);
    if (out != S) throw std::runtime_error("get_rope_index: placeholder layout does not cover the prompt");
    int mx = 0;
    for (int v : pos3) mx = std::max(mx, v);
    delta = mx + 1 - S;
}

void upload_ids(aha_model* m, const uint32_t* ids, size_t S) {
    TextModel& T = m->text;
    AHA_REQUIRE(S >= 1, "empty input_ids");
    AHA_REQUIRE((int)S <= T.max_prefill, "prompt of " + std::to_string(S) + " tokens exceeds max_prefill " + std::to_string(T.max_prefill));
    for (size_t i = 0; i < S; ++i) AHA_REQUIRE(ids[i] < (uint32_t)T.cfg.V, "token id out of range");
    AHA_CUDA_CHECK(cudaMemcpyAsync(T.d_ids, ids, S * sizeof(uint32_t), cudaMemcpyHostToDevice, m->ctx.stream));
}
void upload_pos(aha_model* m, const std::vector<int>& pos3) {
    AHA_CUDA_CHECK(cudaMemcpyAsync(m->text.d_pos3, pos3.data(), pos3.size() * sizeof(int), cudaMemcpyHostToDevice, m->ctx.stream));
    AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));  // pos3 may be a temporary
}
void upload_scatter_idx(aha_model* m, const std::vector<int>& idx) {
    AHA_REQUIRE((int)idx.size() <= m->max_scatter, "too many placeholder tokens");
    AHA_CUDA_CHECK(cudaMemcpyAsync(m->d_scatter_idx, idx.data(), idx.size() * sizeof(int), cudaMemcpyHostToDevice, m->ctx.stream));
    AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
}

void fetch_outputs(aha_model* m, float* logits_out, uint32_t* argmax_out) {
    TextModel& T = m->text;
    if (logits_out) AHA_CUDA_CHECK(cudaMemcpyAsync(logits_out, T.logits, (size_t)T.cfg.V * sizeof(float), cudaMemcpyDeviceToHost, m->ctx.stream));
    if (argmax_out) AHA_CUDA_CHECK(cudaMemcpyAsync(m->h_pin, T.d_argmax, sizeof(uint32_t), cudaMemcpyDeviceToHost, m->ctx.stream));
    AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
    T.check_ll_abort();
    if (argmax_out) *argmax_out = m->h_pin[0];
}


// ---- KV reuse across requests: which prefix of the new prompt is already in the cache --------------------------------------------
// Longest prefix of `ids` whose K/V can be taken from a cache holding `cached`: the common prefix, cut to n - 1 (the last prompt token is
// always run: its logits are the request's first output).  Placeholder tokens (<|image_pad|>, <|video_pad|>, <|audio_pad|>) stand for rows
// of the multimodal tensors, so they only count when those tensors are the same (`same_mm`), and every placeholder of BOTH sequences must
// lie inside the common prefix -- the suffix is then plain text whose M-RoPE positions are index + rope_delta (qwen3vl/model.rs:1250-1264).
size_t prefix_match(const uint32_t* cached, size_t n_cached, const uint32_t* ids, size_t n, const uint32_t* mm_tokens, size_t n_mm_tokens, bool same_mm) {
    if (n == 0 || n_cached == 0 || !same_mm) return 0;
    size_t lcp = 0;
    while (lcp < n && lcp < n_cached && cached[lcp] == ids[lcp]) ++lcp;
    auto is_mm = [&](uint32_t t) { for (size_t i = 0; i < n_mm_tokens; ++i) if (mm_tokens[i] == t) return true; return false; };
    for (size_t i = lcp; i < n; ++i) if (is_mm(ids[i])) return 0;
    for (size_t i = lcp; i < n_cached; ++i) if (is_mm(cached[i])) return 0;
    return std::min(lcp, n - 1);
}

// 64-bit fingerprint of a host buffer: four independent multiply-xorshift lanes over 8-byte words, folded with the length.  Buffers
// beyond 1 MiB are cut into 1 MiB blocks hashed by up to 8 threads and folded in block order (the value does not depend on the thread
// count).  Not cryptographic: it guards a cache, not a boundary.
uint64_t fingerprint_block(const unsigned char* p, size_t n, uint64_t seed) {
    uint64_t h[4] = {seed ^ 0x9e3779b97f4a7c15ull, seed ^ 0xbf58476d1ce4e5b9ull, seed ^ 0x94d049bb133111ebull, seed ^ 0x2545f4914f6cdd1dull};
    const uint64_t k = 0xff51afd7ed558ccdull;
    size_t i = 0;
    for (; i + 32 <= n; i += 32) {
        uint64_t w[4];
        std::memcpy(w, p + i, 32);
        for (int l = 0; l < 4; ++l) { h[l] = (h[l] ^ w[l]) * k; h[l] ^= h[l] >> 29; }
    }
    uint64_t tail[4] = {0, 0, 0, 0};
    if (n > i) std::memcpy(tail, p + i, n - i);
    for (int l = 0; l < 4; ++l) { h[l] = (h[l] ^ tail[l]) * k; h[l] ^= h[l] >> 29; }
    uint64_t r = (uint64_t)n * 0xc4ceb9fe1a85ec53ull;
    for (int l = 0; l < 4; ++l) { r = (r ^ h[l]) * k; r ^= r >> 32; }
    return r;
}
uint64_t fingerprint_bytes(const void* data, size_t n, uint64_t seed) {
    const unsigned char* p = static_cast<const unsigned char*>(data);
    constexpr size_t kBlock = (size_t)1 << 20;
    if (n <= kBlock) return fingerprint_block(p, n, seed);
    const size_t nb = (n + kBlock - 1) / kBlock;
    std::vector<uint64_t> hb(nb);
    const unsigned nt = (unsigned)std::min<size_t>(std::min<size_t>(8, std::max(1u, std::thread::hardware_concurrency())), nb);
    auto work = [&](unsigned t) { for (size_t b = t; b < nb; b += nt) hb[b] = fingerprint_block(p + b * kBlock, std::min(kBlock, n - b * kBlock), seed + b); };
    std::vector<std::thread> th;
    unsigned started = 1;   // lane 0 is this thread
    try {
        for (unsigned t = 1; t < nt; ++t) { th.emplace_back(work, t); ++started; }
    } catch (const std::system_error&) {}   // no more threads to be had: the lanes that did not start are hashed here (same blocks, same value)
    work(0);
    for (unsigned t = started; t < nt; ++t) work(t);
    for (auto& x : th) x.join();
    return fingerprint_block(reinterpret_cast<const unsigned char*>(hb.data()), nb * sizeof(uint64_t), seed ^ (uint64_t)n);
}
// fingerprint of a request's MultiModalData (0 when it carries no tensor): dtype, shape and bytes of every present entry
uint64_t mm_fingerprint(const aha_mm* mm) {
    uint64_t fp = 0;
    for (size_t i = 0; mm && i < mm->n; ++i) {
        const aha_tensor_desc* d = mm_entry(mm, i);
        if (!d) continue;
        size_t esz = 4;
        switch (d->dtype) { case AHA_F16: case AHA_BF16: esz = 2; break; case AHA_I64: esz = 8; break; case AHA_U8: esz = 1; break; default: break; }
        uint64_t meta[11] = {(uint64_t)i + 1, (uint64_t)d->dtype, (uint64_t)d->rank};
        for (int r = 0; r < d->rank && r < 8; ++r) meta[3 + r] = (uint64_t)d->shape[r];
        fp = fingerprint_bytes(meta, sizeof(meta), fp);
        fp = fingerprint_bytes(d->data, WeightTable::numel(*d) * esz, fp);
        if (fp == 0) fp = 1;
    }
    return fp;
}
std::vector<uint32_t> mm_token_ids(const aha_model* m) {
    std::vector<uint32_t> t;
    for (int v : {m->image_token_id, m->video_token_id, m->audio_token_id}) if (v >= 0) t.push_back((uint32_t)v);
    return t;
}
void require_no_session(aha_model* m) {
    AHA_REQUIRE(!m->session.open, "a batch session is open on this handle: call aha_b200_batch_close first");
}
// the tensors a multimodal request must carry, present or empty (a qwen3 handle ignores them)
void require_mm_arity(const aha_model* m, const aha_mm* mm) {
    if (m->kind == aha_model::QWEN3VL) AHA_REQUIRE(mm && mm->n == 5, "Qwen3VL process data error, must have pixel_values, image_grid_thw, pixel_values_video, video_grid_thw, cache_position");
    if (m->kind == aha_model::QWEN3_ASR) AHA_REQUIRE(mm && mm->n == 1, "Qwen3 asr process data error, must have input_features");
}
// `for _ in 1..sample_len` (generate.rs): max_tokens 0 and 1 both yield exactly one token
size_t token_budget(const aha_gen_params& p) { return std::max<size_t>(p.max_tokens, 1); }
// the M-RoPE offset of the decode positions (rope_deltas; 0 for the models without one)
int decode_rope_delta(const aha_model* m) { return m->kind == aha_model::QWEN3VL ? m->rope_delta : 0; }
// device memory of one call, freed when the call returns or throws
struct Scratch {
    std::vector<void*> ptrs;
    Scratch() = default;
    Scratch(const Scratch&) = delete;
    Scratch& operator=(const Scratch&) = delete;
    ~Scratch() { for (void* p : ptrs) cudaFree(p); }
    template <typename T>
    T* alloc(size_t n) {
        void* p = nullptr;
        AHA_CUDA_CHECK(cudaMalloc(&p, n * sizeof(T)));
        ptrs.push_back(p);
        return static_cast<T*>(p);
    }
};
// device time (ms) of launch(0) .. launch(n - 1) between ev0 and ev1 on the model's stream; warm-ups are the caller's
template <typename F>
float timed_ms(aha_model* m, size_t n, F&& launch) {
    cudaStream_t st = m->ctx.stream;
    AHA_CUDA_CHECK(cudaEventRecord(m->ev0, st));
    for (size_t i = 0; i < n; ++i) launch(i);
    AHA_CUDA_CHECK(cudaEventRecord(m->ev1, st));
    AHA_CUDA_CHECK(cudaStreamSynchronize(st));
    float ms = 0.f;
    AHA_CUDA_CHECK(cudaEventElapsedTime(&ms, m->ev0, m->ev1));
    return ms;
}
using clk = std::chrono::steady_clock;
double seconds(clk::duration d) { return std::chrono::duration<double>(d).count(); }
void add_usage(aha_usage* u, size_t prompt_tokens, size_t completion_tokens, double prompt_secs, double completion_secs, double vision_secs) {
    if (!u) return;
    u->prompt_tokens += (uint32_t)prompt_tokens;
    u->completion_tokens += (uint32_t)completion_tokens;
    u->prompt_secs += prompt_secs;
    u->completion_secs += completion_secs;
    u->vision_secs += vision_secs;
}
bool env_flag(const char* name, bool dflt) { const char* v = std::getenv(name); return v ? std::atoi(v) != 0 : dflt; }
int env_int(const char* name, int dflt) { const char* v = std::getenv(name); return v ? std::atoi(v) : dflt; }
// AHA_GEN_LOGPROBS / AHA_GEN_TOP_LOGPROBS(n) of a request: -1 = no records, else the top count n (bits 8 and up of flags, unmasked)
int logprob_request(const aha_gen_params& p, const TextModel& T, const std::string& who) {
    const uint32_t n = p.flags >> 8;
    if (!(p.flags & AHA_GEN_LOGPROBS)) {
        AHA_REQUIRE(n == 0, who + "AHA_GEN_TOP_LOGPROBS(" + std::to_string(n) + ") needs AHA_GEN_LOGPROBS");
        return -1;
    }
    AHA_REQUIRE(n <= AHA_MAX_TOP_LOGPROBS, who + "AHA_GEN_TOP_LOGPROBS(" + std::to_string(n) + "): at most " + std::to_string(AHA_MAX_TOP_LOGPROBS) + " alternatives");
    AHA_REQUIRE(n <= (uint32_t)T.cfg.V, who + "AHA_GEN_TOP_LOGPROBS(" + std::to_string(n) + ") exceeds the vocabulary of " + std::to_string(T.cfg.V));
    AHA_REQUIRE(T.tp_world == 1, who + "log-probabilities are single-GPU (under tensor parallelism the decode step holds only a vocabulary shard)");
    AHA_REQUIRE(T.cfg.V <= kLpMaxParts * kLpSlice, who + "vocabulary too large for the log-probability kernels");
    return (int)n;
}
// the entries that return no records refuse a request for them
void refuse_logprobs(const aha_gen_params& p, const std::string& who, const std::string& instead) {
    AHA_REQUIRE((p.flags & AHA_GEN_LOGPROBS) == 0 && (p.flags >> 8) == 0, who + " returns no log-probabilities: use " + instead);
}
// Everything aha_token_fsm promises, checked on the host before an automaton reaches the device: the kernels index with these values
// unchecked (sampling.cuh), and a state without a token would leave a request nothing to draw.
void fsm_validate(const aha_token_fsm* f, size_t vocab) {
    AHA_REQUIRE(f, "token automaton: fsm is NULL");
    AHA_REQUIRE(f->n_states >= 1, "token automaton: n_states must be at least 1");
    AHA_REQUIRE(f->offsets, "token automaton: offsets is NULL");
    const uint64_t n_trans = f->offsets[f->n_states];
    AHA_REQUIRE(n_trans == 0 || (f->tokens && f->next), "token automaton: tokens and next are required");
    AHA_REQUIRE(f->start < f->n_states, "token automaton: start " + std::to_string(f->start) + " is not below n_states " + std::to_string(f->n_states));
    AHA_REQUIRE(f->offsets[0] == 0, "token automaton: offsets[0] must be 0");
    for (uint32_t st = 0; st < f->n_states; ++st) {
        const uint64_t a = f->offsets[st], b = f->offsets[st + 1];
        AHA_REQUIRE(a <= b && b <= n_trans, "token automaton: offsets must be non-decreasing up to offsets[n_states] (state " + std::to_string(st) + ")");
        AHA_REQUIRE(b > a, "token automaton: state " + std::to_string(st) + " allows no token");
        for (uint64_t j = a; j < b; ++j) {
            AHA_REQUIRE(f->tokens[j] < vocab, "token automaton: state " + std::to_string(st) + " allows token " + std::to_string(f->tokens[j]) +
                                                  ", outside the vocabulary of " + std::to_string(vocab));
            AHA_REQUIRE(j == a || f->tokens[j] > f->tokens[j - 1], "token automaton: the tokens of state " + std::to_string(st) +
                                                                       " are not strictly ascending");
            AHA_REQUIRE(f->next[j] < f->n_states, "token automaton: next[" + std::to_string(j) + "] = " + std::to_string(f->next[j]) +
                                                      " is not below n_states " + std::to_string(f->n_states));
        }
    }
}
// bytes of an automaton's device copy: offsets [n_states + 1] (u64), then tokens and next [transitions] (u32)
size_t fsm_bytes(const aha_token_fsm& f) { return (size_t)(f.n_states + 1) * sizeof(uint64_t) + (size_t)f.offsets[f.n_states] * 2 * sizeof(uint32_t); }
// a validated automaton copied into `mem` (fsm_bytes(f) bytes of device memory)
TokenFsmDev fsm_upload(const aha_token_fsm& f, void* mem) {
    const size_t n_off = (size_t)f.n_states + 1, n = (size_t)f.offsets[f.n_states];
    TokenFsmDev d;
    char* p = static_cast<char*>(mem);
    d.off = reinterpret_cast<const uint64_t*>(p);
    d.tok = reinterpret_cast<const uint32_t*>(p + n_off * sizeof(uint64_t));
    d.next = d.tok + n;
    d.start = f.start;
    AHA_CUDA_CHECK(cudaMemcpy(p, f.offsets, n_off * sizeof(uint64_t), cudaMemcpyHostToDevice));
    if (n) {
        AHA_CUDA_CHECK(cudaMemcpy(const_cast<uint32_t*>(d.tok), f.tokens, n * sizeof(uint32_t), cudaMemcpyHostToDevice));
        AHA_CUDA_CHECK(cudaMemcpy(const_cast<uint32_t*>(d.next), f.next, n * sizeof(uint32_t), cudaMemcpyHostToDevice));
    }
    return d;
}
// Everything aha_logit_rules promises, checked on the host: the kernel scatters the bias by id unchecked and relies on distinct ids (one
// thread per entry), and the ranges are OpenAI's.
void rules_validate(const aha_logit_rules* r, size_t vocab) {
    AHA_REQUIRE(r, "logit rules: rules is NULL");
    auto in = [](float x, float lim) { return std::isfinite(x) && x >= -lim && x <= lim; };
    AHA_REQUIRE(in(r->presence_penalty, 2.f), "logit rules: presence_penalty " + std::to_string(r->presence_penalty) + " is not a finite value in [-2, 2]");
    AHA_REQUIRE(in(r->frequency_penalty, 2.f), "logit rules: frequency_penalty " + std::to_string(r->frequency_penalty) + " is not a finite value in [-2, 2]");
    AHA_REQUIRE(r->reserved[0] == 0 && r->reserved[1] == 0 && r->reserved[2] == 0, "logit rules: reserved must be 0");
    AHA_REQUIRE(r->n_bias <= vocab, "logit rules: n_bias " + std::to_string(r->n_bias) + " exceeds the vocabulary of " + std::to_string(vocab));
    if (r->n_bias == 0) return;
    AHA_REQUIRE(r->bias_ids && r->bias_values, "logit rules: bias_ids and bias_values are required when n_bias > 0");
    std::vector<char> seen(vocab, 0);
    for (size_t j = 0; j < r->n_bias; ++j) {
        const uint32_t t = r->bias_ids[j];
        AHA_REQUIRE(t < vocab, "logit rules: bias id " + std::to_string(t) + " is outside the vocabulary of " + std::to_string(vocab));
        AHA_REQUIRE(!seen[t], "logit rules: bias id " + std::to_string(t) + " is listed twice");
        seen[t] = 1;
        AHA_REQUIRE(in(r->bias_values[j], 100.f), "logit rules: the bias of token " + std::to_string(t) + " (" + std::to_string(r->bias_values[j]) +
                                                       ") is not a finite value in [-100, 100]");
    }
}
// a validated rules object's bias list copied into `mem` (n_bias ids, then n_bias values)
LogitRulesDev rules_upload(const aha_logit_rules& r, void* mem) {
    LogitRulesDev d;
    d.n_bias = (int)r.n_bias; d.presence = r.presence_penalty; d.frequency = r.frequency_penalty;
    if (r.n_bias == 0) return d;
    uint32_t* ids = static_cast<uint32_t*>(mem);
    float* vals = reinterpret_cast<float*>(ids + r.n_bias);
    AHA_CUDA_CHECK(cudaMemcpy(ids, r.bias_ids, r.n_bias * sizeof(uint32_t), cudaMemcpyHostToDevice));
    AHA_CUDA_CHECK(cudaMemcpy(vals, r.bias_values, r.n_bias * sizeof(float), cudaMemcpyHostToDevice));
    d.ids = ids; d.vals = vals;
    return d;
}
// What a request's AHA_GEN_CONSTRAINED / AHA_GEN_LOGIT_RULES resolve to on the handle: its automaton (directly, or the one its rules name)
// and its rules, each with its id (0 and null: none).  Refused where neither runs.
struct RequestRules {
    const TokenFsmDev* fsm = nullptr;
    uint32_t fsm_id = 0;
    const LogitRulesDev* rules = nullptr;
    uint32_t rules_id = 0;
};
RequestRules request_rules(const aha_model* m, const aha_gen_params& p, const std::string& who) {
    RequestRules q;
    const bool con = (p.flags & AHA_GEN_CONSTRAINED) != 0, lr = (p.flags & AHA_GEN_LOGIT_RULES) != 0;
    if (!con && !lr) return q;
    AHA_REQUIRE(!(con && lr), who + "AHA_GEN_CONSTRAINED and AHA_GEN_LOGIT_RULES exclude each other (params.reserved holds one id): name the "
                                    "automaton in the logit-rules object (aha_logit_rules.fsm) instead");
    uint32_t fsm_id = p.reserved;
    if (lr) {
        AHA_REQUIRE(m->text.tp_world == 1, who + "logit rules are single-GPU (under tensor parallelism the decode step holds only a vocabulary shard)");
        const auto it = m->rules.find(p.reserved);
        AHA_REQUIRE(it != m->rules.end(), who + "AHA_GEN_LOGIT_RULES: no logit-rules object has id " + std::to_string(p.reserved) + " on this handle");
        q.rules = &it->second.dev;
        q.rules_id = p.reserved;
        fsm_id = it->second.fsm;
        if (fsm_id == 0) return q;
    }
    AHA_REQUIRE(m->text.tp_world == 1, who + "constrained decoding is single-GPU (under tensor parallelism the decode step holds only a vocabulary shard)");
    const auto it = m->fsms.find(fsm_id);
    AHA_REQUIRE(it != m->fsms.end(), who + "AHA_GEN_CONSTRAINED: no token automaton has id " + std::to_string(fsm_id) + " on this handle");
    q.fsm = &it->second.dev;
    q.fsm_id = fsm_id;
    return q;
}
// the request's sampler (make_sampler), constrained by its automaton and transformed by its logit rules when it asks
Sampler request_sampler(const aha_model* m, const aha_gen_params& p, const std::string& who) {
    const RequestRules q = request_rules(m, p, who);
    Sampler s = make_sampler(p, m->text.cfg.V, q.fsm, q.rules);
    s.fsm_id = q.fsm_id;
    s.rules_id = q.rules_id;
    return s;
}

// AHA_BATCH_GEMV's default (BatchDecoder::gemv).  The two batched GEMVs are bit-identical on every tested shape and neither wins everywhere: on
// one H100 80GB HBM3 at 400 W (profiles/run_batch.py, ms per step at 1 / 8 requests) v2 takes 2.25 / 4.68-4.76 against v1's 2.22 / 4.17 on the
// VL2 text stack, and 1.30 / 2.71 against 1.33 / 2.63-2.64 on the Qwen3-0.6B shape.
constexpr int kBatchGemvDefault = 2;

// model.clear_cache(): pages, rope_deltas, and what the prefix cache remembered
void drop_cache(aha_model* m) {
    m->text.pages.reset();
    m->text.table.mapped = 0;
    m->have_rope_delta = false;  // qwen3vl/model.rs:1279-1282
    m->rope_delta = 0;
    m->cached_ids.clear();
    m->cached_mm_fp = 0;
}
// model.clear_cache() (generate.rs:147) when a single request ends -- also on the error path, so that a failed request never leaves
// rope_delta / pages behind -- unless the request keeps its K/V for the next one (REUSE_PREFIX)
struct RequestReset {
    aha_model* m;
    bool keep = false;
    ~RequestReset() { if (!keep) drop_cache(m); m->text.clear_sampler(); }
};
// ends the batch session, if one is open, and leaves the handle as clear_cache() does
void session_close(aha_model* m) {
    for (auto& e : m->suspended) m->swap.free.insert(m->swap.free.end(), e.second.host_pages.begin(), e.second.host_pages.end());
    m->suspended.clear();   // suspended requests belong to the session
    for (BatchDecoder* B : {&m->batch, &m->wide_batch}) B->reset();
    m->spec.steps.clear();
    m->spec.built_epoch = ~0ull;
    m->session = aha_model::BatchSession{};
    drop_cache(m);
    m->text.clear_sampler();
}

void alloc_pack_buffers(aha_model* m) {
    if (m->d_pack_work) return;
    const TextModel& T = m->text;
    m->d_pack_work = m->ctx.alloc<int>((size_t)kFaWork * T.max_prefill);
    m->d_pack_rows = m->ctx.alloc<int>((size_t)T.max_prefill);
    m->d_pack_table = m->ctx.alloc<int>((size_t)T.num_pages);
}

// One packed prefill (embed_batch, batch_add_many): inputs [first, last) laid out in input order, input j starting at token start[j - first].
// The first input starts at 0, every later one on the next multiple of the caller's alignment.  The gap behind an input is filled with token 0
// and joins that input's segment: its rows come after every real row, so the causal mask keeps them out of the input's own rows.  The last
// input of a pack is not padded.
struct Pack {
    size_t first = 0, last = 0;
    size_t S = 0;                    // tokens in the pack
    size_t KV = 0;                   // key rows of the pack: S plus the cached prefixes of its inputs
    std::vector<size_t> start;
    std::vector<size_t> kv_start;    // where each input's keys (its prefix, then its own rows) start among the KV rows
    std::vector<uint32_t> ids;       // [S]
    std::vector<int> pos3;           // [3][S]: positions restart at the input's prefix length (0 without one) in every segment
    PrefillSegments sg;              // (start, length) of every segment; the work list's device copy is set by upload_pack
    std::vector<int> work;           // [n_work][kFaWork] work list of flash_attn_tc_varlen
    std::vector<int> rows;           // the last row of every input
};
// The pack that begins at input `first`: as many inputs as fit `cap` tokens, each starting on a multiple of `align`.  pre (optional): the
// cached prefix of every input, a multiple of `align` tokens that the pack does not run but its attention reads; then the pack's key rows
// (every input's prefix and segment, laid end to end) must also fit `kv_cap`.
Pack plan_pack(const std::vector<const uint32_t*>& ids, const std::vector<size_t>& lens, size_t first, size_t align, size_t cap,
               const std::vector<size_t>& pre = {}, size_t kv_cap = 0) {
    Pack p;
    p.first = p.last = first;
    auto pre_of = [&](size_t j) { return pre.empty() ? (size_t)0 : pre[j]; };
    while (p.last < lens.size()) {
        const size_t s0 = p.last == first ? 0 : (p.S + align - 1) / align * align;
        const size_t kv0 = p.last == first ? 0 : p.kv_start.back() + pre_of(p.last - 1) + (s0 - p.start.back());
        if (s0 + lens[p.last] > cap) break;
        if (!pre.empty() && kv0 + pre[p.last] + lens[p.last] > kv_cap) break;
        p.start.push_back(s0);
        p.kv_start.push_back(kv0);
        p.S = s0 + lens[p.last];
        p.KV = kv0 + pre_of(p.last) + lens[p.last];
        ++p.last;
    }
    AHA_REQUIRE(p.last > first, "packed prefill: an input of " + std::to_string(lens[first]) + " tokens exceeds the pack capacity of " + std::to_string(cap));
    const size_t S = p.S;
    p.ids.assign(S, 0);
    p.pos3.resize((size_t)3 * S);
    for (size_t j = p.first; j < p.last; ++j) {
        const int s0 = (int)p.start[j - first], len = (int)lens[j], pj = (int)pre_of(j), kv0 = (int)p.kv_start[j - first];
        const int seg = (j + 1 < p.last ? (int)p.start[j + 1 - first] : (int)S) - s0;   // the input and the filler behind it
        std::memcpy(p.ids.data() + s0, ids[j], (size_t)len * sizeof(uint32_t));
        for (int k = 0; k < 3; ++k) for (int i = 0; i < seg; ++i) p.pos3[(size_t)k * S + s0 + i] = pj + i;
        p.sg.segs.emplace_back(s0, seg);
        if (!pre.empty()) p.sg.kv.emplace_back(kv0, pj + seg);
        for (int q = 0; q < seg; q += kFaBQ) p.work.insert(p.work.end(), {s0, seg, kv0, pj + seg, q});
        p.rows.push_back(s0 + len - 1);
    }
    return p;
}
// the pack's ids, positions, work list and last rows to the device (synchronises: the host vectors are free after it)
void upload_pack(aha_model* m, Pack& p) {
    cudaStream_t st = m->ctx.stream;
    p.sg.d_work = m->d_pack_work;
    p.sg.n_work = (int)(p.work.size() / kFaWork);
    AHA_CUDA_CHECK(cudaMemcpyAsync(m->text.d_ids, p.ids.data(), p.S * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    AHA_CUDA_CHECK(cudaMemcpyAsync(m->d_pack_work, p.work.data(), p.work.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    AHA_CUDA_CHECK(cudaMemcpyAsync(m->d_pack_rows, p.rows.data(), p.rows.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    upload_pos(m, p.pos3);
}

// The multi-token forward (prefill) of the sequence of table `pt`.  Mirrors Qwen3Model::forward / Qwen3VLModel::forward / Qwen3ASRThinker::forward.
void forward_prefill(aha_model* m, PageTable& pt, const uint32_t* ids, size_t S, size_t offset, const aha_mm* mm, bool initial) {
    TextModel& T = m->text;
    Ctx& c = m->ctx;
    upload_ids(m, ids, S);
    std::vector<int> pos3((size_t)3 * S);
    std::vector<const float*> deepstack;
    int n_visual = 0;
    bool embeds_ready = false;
    m->last_vision_secs = 0;
    if (m->kind == aha_model::QWEN3VL) {
        const aha_tensor_desc* pv = initial ? mm_entry(mm, 0) : nullptr;
        const aha_tensor_desc* thw = initial ? mm_entry(mm, 1) : nullptr;
        const aha_tensor_desc* pvv = initial ? mm_entry(mm, 2) : nullptr;
        const aha_tensor_desc* vthw = initial ? mm_entry(mm, 3) : nullptr;
        if (!(pv && thw)) { pv = nullptr; thw = nullptr; }       // `if let Some(pixel_values) && let Some(image_grid_thw)` (model.rs:1150-1151)
        if (!(pvv && vthw)) { pvv = nullptr; vthw = nullptr; }   // the same for the video pair (model.rs:1169-1170)
        std::vector<std::array<int, 3>> grid, vgrid, vgrid_frames;
        auto read_grid = [&](const aha_tensor_desc& d, std::vector<std::array<int, 3>>& out, const char* what) {
            auto g = desc_to_i64(d);
            AHA_REQUIRE(g.size() % 3 == 0 && !g.empty(), std::string(what) + " must be (n, 3)");
            int N = 0;
            for (size_t i = 0; i < g.size(); i += 3) { out.push_back({(int)g[i], (int)g[i + 1], (int)g[i + 2]}); N += (int)(g[i] * g[i + 1] * g[i + 2]); }
            return N;
        };
        if (pv || pvv) {
            VisionModel& V = m->vision;
            const int N_img = pv ? read_grid(*thw, grid, "image_grid_thw") : 0;
            const int N_vid = pvv ? read_grid(*vthw, vgrid, "video_grid_thw") : 0;
            for (auto& g : vgrid) for (int t = 0; t < g[0]; ++t) vgrid_frames.push_back({1, g[1], g[2]});
            const int N = N_img + N_vid, m2 = V.cfg.merge * V.cfg.merge;
            if (pv) AHA_REQUIRE(pv->rank == 2 && pv->shape[0] == N_img && pv->shape[1] == V.patch_dim, "pixel_values shape does not match image_grid_thw");
            if (pvv) AHA_REQUIRE(pvv->rank == 2 && pvv->shape[0] == N_vid && pvv->shape[1] == V.patch_dim, "pixel_values_video shape does not match video_grid_thw");
            AHA_REQUIRE(N <= V.max_patches, "image needs " + std::to_string(N) + " patches, max_patches is " + std::to_string(V.max_patches));
            // placeholder positions + count checks (model.rs:1158-1164, 1176-1183: the video branch raises the same text); the scatter list is
            // the image positions followed by the video positions, matching the row order of the tower's output below
            std::vector<int> idx, vidx;
            for (size_t i = 0; i < S; ++i) {
                if (pv && (int)ids[i] == m->image_token_id) idx.push_back((int)i);
                if (pvv && (int)ids[i] == m->video_token_id) vidx.push_back((int)i);
            }
            if (pv && (int)idx.size() != N_img / m2)
                throw std::runtime_error("n_image_token num: " + std::to_string(idx.size()) + " not equal to image_embed len: " + std::to_string(N_img / m2));
            if (pvv && (int)vidx.size() != N_vid / m2)
                throw std::runtime_error("n_image_token num: " + std::to_string(vidx.size()) + " not equal to image_embed len: " + std::to_string(N_vid / m2));
            idx.insert(idx.end(), vidx.begin(), vidx.end());
            const int n_embed = N / m2;
            // pixel rows -> HBM (images, then video frames), one pass of the tower over both: every grid entry is independent through all
            // blocks and mergers, so this equals the reference's two get_vision_features calls
            auto put = [&](const aha_tensor_desc& d, size_t row0, size_t rows) {
                float* dst = V.pix + row0 * V.patch_dim;
                if (d.dtype == AHA_F32) AHA_CUDA_CHECK(cudaMemcpyAsync(dst, d.data, rows * V.patch_dim * sizeof(float), cudaMemcpyHostToDevice, c.stream));
                else { auto f = desc_to_f32(d); AHA_CUDA_CHECK(cudaMemcpyAsync(dst, f.data(), f.size() * sizeof(float), cudaMemcpyHostToDevice, c.stream)); AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream)); }
            };
            if (pv) put(*pv, 0, (size_t)N_img);
            if (pvv) put(*pvv, (size_t)N_img, (size_t)N_vid);
            std::vector<std::array<int, 3>> all = grid;
            all.insert(all.end(), vgrid.begin(), vgrid.end());
            AHA_CUDA_CHECK(cudaEventRecord(m->ev0, c.stream));
            V.forward(N, all);
            AHA_CUDA_CHECK(cudaEventRecord(m->ev1, c.stream));
            upload_scatter_idx(m, idx);
            embed_gather_kernel<<<(unsigned)S, 256, 0, c.stream>>>(T.d_ids, T.embed, T.x, (int)S, T.cfg.H, T.cfg.V); c.cnt.kernels++;
            scatter_rows_kernel<<<n_embed, 256, 0, c.stream>>>(m->d_scatter_idx, V.image_embeds, T.x, T.cfg.H, 0); c.cnt.kernels++;
            embeds_ready = true;
            n_visual = n_embed;   // deepstack: x[idx[r]] += ds[r] over the same list = the joint embedding of model.rs:1189-1225
            for (float* p : V.ds_out) deepstack.push_back(p);
        }
        // positions: first call -> get_rope_index, later -> arange + offset + rope_deltas (model.rs:1226-1264)
        if (!m->have_rope_delta || (initial && offset == 0)) {   // cache_position[0] == 0 recomputes get_rope_index even when rope_deltas is set (model.rs:1228)
            int delta = 0;
            get_rope_index(ids, (int)S, grid, vgrid_frames, m->vision.cfg.merge, m->image_token_id, m->video_token_id, m->vision_start_token_id, pos3, delta);
            m->rope_delta = delta; m->have_rope_delta = true;
        } else {
            for (int r = 0; r < 3; ++r) for (size_t i = 0; i < S; ++i) pos3[(size_t)r * S + i] = (int)(i + offset) + m->rope_delta;
        }
    } else if (m->kind == aha_model::QWEN3_ASR) {
        const aha_tensor_desc* feat = initial ? mm_entry(mm, 0) : nullptr;
        if (feat) {
            AHA_REQUIRE(feat->rank == 2 && feat->shape[0] == m->audio.cfg.mel, "input_features must be (num_mel_bins, frames)");
            const int Tm = (int)feat->shape[1];
            AHA_REQUIRE(Tm <= m->audio.max_frames, "input_features longer than max_frames");
            auto f = desc_to_f32(*feat);
            AHA_CUDA_CHECK(cudaMemcpyAsync(m->audio.d_mel, f.data(), f.size() * sizeof(float), cudaMemcpyHostToDevice, c.stream));
            AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
            AHA_CUDA_CHECK(cudaEventRecord(m->ev0, c.stream));
            const int n_tok = m->audio.forward(m->audio.d_mel, Tm);
            AHA_CUDA_CHECK(cudaEventRecord(m->ev1, c.stream));
            std::vector<int> idx;
            for (size_t i = 0; i < S; ++i) if ((int)ids[i] == m->audio_token_id) idx.push_back((int)i);
            if ((int)idx.size() != n_tok)  // qwen3_asr/model.rs:348-354
                throw std::runtime_error("n_audio_tokens num: " + std::to_string(idx.size()) + " not equal to audio_feature len: " + std::to_string(n_tok));
            upload_scatter_idx(m, idx);
            embed_gather_kernel<<<(unsigned)S, 256, 0, c.stream>>>(T.d_ids, T.embed, T.x, (int)S, T.cfg.H, T.cfg.V); c.cnt.kernels++;
            scatter_rows_kernel<<<n_tok, 256, 0, c.stream>>>(m->d_scatter_idx, m->audio.audio_embeds, T.x, T.cfg.H, 0); c.cnt.kernels++;
            embeds_ready = true;
        }
        for (int r = 0; r < 3; ++r) for (size_t i = 0; i < S; ++i) pos3[(size_t)r * S + i] = (int)(i + offset);
    } else {
        for (int r = 0; r < 3; ++r) for (size_t i = 0; i < S; ++i) pos3[(size_t)r * S + i] = (int)(i + offset);
    }
    upload_pos(m, pos3);
    T.prefill(pt, (int)S, (int)offset, embeds_ready, m->d_scatter_idx, n_visual, deepstack);
}

// A prompt longer than the activation workspace (max_prefill) runs as consecutive chunks against the growing cache: the first chunk is
// the reference's call (multimodal rows are scattered there), the others are continuations.  Same K/V, same logits for the last token.
// after_chunk(done, n) runs after the chunk of tokens [done, done + n), while its rows are still in TextModel::x.
void prefill_chunked(aha_model* m, PageTable& pt, const uint32_t* ids, size_t S, size_t offset, const aha_mm* mm, bool initial, bool has_mm, bool extend,
                     const std::function<void(size_t, size_t)>& after_chunk = nullptr) {
    const size_t chunk = (size_t)m->text.max_prefill;
    size_t done = 0;
    while (done < S) {
        const size_t n = std::min(chunk, S - done);
        const bool first = done == 0;
        if (first && !extend) {
            if (n < S && has_mm) {   // every placeholder row must be embedded by the call that carries the tensors
                const auto mmt = mm_token_ids(m);
                for (size_t i = n; i < S; ++i) for (uint32_t t : mmt) AHA_REQUIRE(ids[i] != t, "prompt exceeds max_prefill before its last multimodal placeholder");
            }
            // (Qwen3-VL: get_rope_index over the first chunk yields the whole prompt's rope_delta, because only text follows the last placeholder)
            forward_prefill(m, pt, ids, n, offset, mm, initial);
        } else forward_prefill(m, pt, ids + done, n, offset + done, nullptr, false);
        if (after_chunk) after_chunk(done, n);
        done += n;
    }
}

// `extend`: prefill continuation (new design) -- S >= 1 further tokens against a cache that already holds `offset` tokens; the causal mask is
// the (S, offset + S) one the reference never builds (its (S, S) mask makes a multi-token call with a non-empty cache fail, qwen3/model.rs:164-175).
// `pt`: the sequence's page table.  The decode step runs on the model's own table only, so a single token on any other table (a batch slot's
// first prefill) is prefilled.
void forward_any(aha_model* m, PageTable& pt, const uint32_t* ids, size_t S, size_t offset, const aha_mm* mm, bool initial, float* logits_out,
                 uint32_t* argmax_out, bool extend = false) {
    TextModel& T = m->text;
    AHA_REQUIRE(ids != nullptr && S >= 1, "input_ids must hold at least one token");
    AHA_REQUIRE(offset + S <= (size_t)T.max_ctx, "context exceeds max_ctx");
    const bool has_mm = initial && mm && ((m->kind == aha_model::QWEN3VL && (mm_entry(mm, 0) || mm_entry(mm, 2))) || (m->kind == aha_model::QWEN3_ASR && mm_entry(mm, 0)));
    if (initial) require_mm_arity(m, mm);
    if (S == 1 && !has_mm && !extend && &pt == &T.table && (m->kind != aha_model::QWEN3VL || m->have_rope_delta)) {
        // decode step: single token against the cache
        AHA_REQUIRE(ids[0] < (uint32_t)T.cfg.V, "token id out of range");
        T.pages.map(T.table, (int)offset + 1);
        T.set_state(ids[0], (int)offset, decode_rope_delta(m), 0);
        T.decode_step(logits_out != nullptr);
    } else {
        // The reference builds an (S,S) causal mask with offset 0 for every multi-token call
        // (qwen3/model.rs:164-175); with a non-empty cache its broadcast_add against (S, off+S) scores fails.
        if (!extend) AHA_REQUIRE(offset == 0, "seq_len > 1 with seqlen_offset > 0 is not supported (the reference's mask shape rejects it too)");
        else AHA_REQUIRE(offset <= (size_t)pt.mapped * kPage, "forward_extend: seqlen_offset is beyond the tokens in the cache");
        prefill_chunked(m, pt, ids, S, offset, mm, initial, has_mm, extend);
        T.finish_argmax(0);
        T.sample(0);   // device sampler of generate(): penalty / temperature / top-k / top-p on the prefill logits (no-op for plain ArgMax)
    }
    fetch_outputs(m, logits_out, argmax_out);
    if (m->kind != aha_model::QWEN3 && has_mm) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, m->ev0, m->ev1) == cudaSuccess) m->last_vision_secs = ms * 1e-3;
    }
}

// A request's first token (forward_initial + sample_and_push): its sampler is set on the model against an empty history at draw index
// draws0, the prompt is prefilled on `pt` -- from `hit` on, as a continuation, when the cache already holds ids[0, hit) -- and the token is
// drawn from the last row's logits.
uint32_t first_token(aha_model* m, PageTable& pt, const uint32_t* ids, size_t seq_len, size_t hit, const aha_mm* mm, const Sampler& samp,
                     uint32_t draws0) {
    TextModel& T = m->text;
    T.set_sampler(samp);
    T.set_state(0, 0, 0, 0, draws0, samp.fsm_start);    // empty history: the first token sees no repeat-penalty context
    uint32_t tok = 0;
    if (hit > 0) forward_any(m, pt, ids + hit, seq_len - hit, hit, nullptr, false, nullptr, &tok, true);   // only the tokens the cache does not hold yet
    else forward_any(m, pt, ids, seq_len, 0, mm, true, nullptr, &tok);
    T.check_sample_error();
    return tok;
}

// The handoff to decode after first_token: every page positions [0, ctx) can touch is mapped on `pt` (the step kernels only read the
// table), and the decode state starts from `tok` at position seq_len, with history[0] = tok and the draw index the first token left.  The
// state is the model's own, or batch slot `slot`'s; the automaton state the first token left travels with it.
void handoff(aha_model* m, PageTable& pt, size_t ctx, uint32_t tok, size_t seq_len, int slot = -1) {
    TextModel& T = m->text;
    T.pages.map(pt, (int)ctx);
    DecodeState cur;
    AHA_CUDA_CHECK(cudaMemcpy(&cur, T.d_state, sizeof(cur), cudaMemcpyDeviceToHost));
    if (slot >= 0) {
        m->sess().adopt(slot, tok, (int)seq_len, decode_rope_delta(m), cur.n_draws, cur.fsm_state);
        return;
    }
    T.set_state(tok, (int)seq_len, decode_rope_delta(m), 1, cur.n_draws, cur.fsm_state);
    AHA_CUDA_CHECK(cudaMemcpy(T.d_history, &tok, sizeof(uint32_t), cudaMemcpyHostToDevice));
}

// a request that asks for records (lp_n >= 0 alternatives each); a burst's records are staged in pinned memory
void request_logprobs(aha_model* m, int lp_n) {
    if (lp_n < 0) return;
    m->text.set_logprobs(lp_n);
    if (!m->h_lp_pin) AHA_CUDA_CHECK(cudaMallocHost(&m->h_lp_pin, 32 * sizeof(aha_logprobs)));
}

}  // namespace

extern "C" {

int aha_b200_abi_version(void) { return AHA_B200_ABI_VERSION; }

int aha_b200_create(const char* kind, const char* config_json, const aha_tensor_desc* weights, size_t n_weights, const uint32_t* eos_ids,
                    size_t n_eos, const aha_options* opts, aha_model** out) {
    if (!out) return 1;
    *out = nullptr;
    aha_model* m = nullptr;
    try {
        AHA_REQUIRE(kind && config_json && weights, "kind, config_json and weights are required");
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
            throw std::runtime_error("no CUDA device visible: libaha_b200 has no CPU fallback");
        aha_options o{};
        if (opts) o = *opts;
        o.use_graph = opts ? opts->use_graph : 1;
        AHA_REQUIRE(o.device >= 0 && o.device < ndev, "invalid device ordinal");
        cudaDeviceProp prop;
        AHA_CUDA_CHECK(cudaGetDeviceProperties(&prop, o.device));
        AHA_REQUIRE(prop.major == 9 && prop.minor == 0, std::string("device '") + prop.name + "' is not sm_90 (this library is built for sm_90a only)");
        m = new aha_model();
        m->ctx.device = o.device;
        m->ctx.num_sms = prop.multiProcessorCount;
        AHA_REQUIRE(o.gemm_impl >= 0 && o.gemm_impl <= 3, "gemm_impl must be 0 (auto), 1 (SIMT), 2 or 3 (wgmma 128 x 128 / 128 x 256 tiles)");
        m->ctx.gemm_impl = o.gemm_impl;
        { const char* e = getenv("AHA_GEMM_WIDE"); if (e) m->ctx.gemm_wide = atoi(e) != 0; }
        { const char* e = getenv("AHA_PRESPLIT"); if (e) m->ctx.presplit = atoi(e) != 0; }
        m->ctx.attn_impl = o.reserved[0];   // 0 = wgmma flash attention, 1 = fp32 SIMT twin, 2 = mma.sync kernel everywhere
        AHA_CUDA_CHECK(cudaSetDevice(o.device));
        AHA_CUDA_CHECK(cudaStreamCreateWithFlags(&m->ctx.stream, cudaStreamNonBlocking));
        AHA_CUDA_CHECK(cudaEventCreate(&m->ev0));
        AHA_CUDA_CHECK(cudaEventCreate(&m->ev1));
        AHA_CUDA_CHECK(cudaMallocHost(&m->h_pin, 64 * sizeof(uint32_t)));
        for (auto& e : m->ev_tok) AHA_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        gemv_init();
        gemm_tc_init();
        score_head_init();
        gemv_wide_init();
        flash_attn_tc_init();
        const std::string k = kind;
        const std::string cfg_text = config_json;
        Json root = JsonParser(cfg_text).parse();
        WeightTable wt(weights, n_weights);
        const int tp_rank = o.tp_world > 1 ? o.tp_rank : 0, tp_world = o.tp_world > 1 ? o.tp_world : 1;
        const int max_ctx = o.max_ctx > 0 ? o.max_ctx : 8192;
        const int max_prefill = o.max_prefill > 0 ? o.max_prefill : max_ctx;
        TextCfg tc;
        if (k == "qwen3") {
            m->kind = aha_model::QWEN3;
            tc = TextCfg::from_json(root);
            const std::string prefix = wt.has("model.embed_tokens.weight") ? "model." : "";  // qwen3/model.rs:105-109
            m->text.load(m->ctx, tc, wt, prefix, "lm_head.weight", tp_rank, tp_world);
        } else if (k == "qwen3vl") {
            m->kind = aha_model::QWEN3VL;
            tc = TextCfg::from_json(root.at("text_config"));
            tc.tie = root.boolean_or("tie_word_embeddings", false);  // lm_head tying follows the TOP-LEVEL flag (model.rs:853-861)
            AHA_REQUIRE(tc.mrope, "text_config.rope_scaling.mrope_section is required for Qwen3-VL");
            m->image_token_id = root.integer("image_token_id"); m->video_token_id = root.integer_or("video_token_id", -1);
            m->vision_start_token_id = root.integer("vision_start_token_id");
            m->text.load(m->ctx, tc, wt, "model.language_model.", "lm_head.weight", tp_rank, tp_world);
            m->vision.load(m->ctx, VisionCfg::from_json(root.at("vision_config")), wt, "model.visual.", o.max_patches > 0 ? o.max_patches : 16384);
            AHA_REQUIRE(m->vision.cfg.out_hidden == tc.H, "vision out_hidden_size must equal the text hidden_size");
        } else if (k == "qwen3_asr") {
            m->kind = aha_model::QWEN3_ASR;
            const Json& tk = root.at("thinker_config");
            tc = TextCfg::from_json(tk.at("text_config"));
            tc.mrope_asr = true;  // apply_interleaved_mrope_asr index rule (rope.rs:478-500); rows are identical so it is numerically a no-op
            m->audio_token_id = tk.integer("audio_token_id");
            m->text.load(m->ctx, tc, wt, "thinker.model.", "thinker.lm_head.weight", tp_rank, tp_world);
            m->audio.load(m->ctx, AudioCfg::from_json(tk.at("audio_config")), wt, "thinker.audio_tower.", o.max_frames > 0 ? o.max_frames : 3000);
            AHA_REQUIRE(m->audio.cfg.out_dim == tc.H, "audio output_dim must equal the text hidden_size");
        } else {
            throw std::runtime_error("unknown model kind '" + k + "' (expected qwen3 | qwen3vl | qwen3_asr)");
        }
        m->text.alloc_runtime(max_ctx, max_prefill, o.use_graph != 0, o.decode_impl);
        m->text.init_tp(o.tp_comm);
        if (m->kind == aha_model::QWEN3VL) m->vision.set_tp(m->text.tp_rank, m->text.tp_world, m->text.comm);   // images sharded over the ranks
        m->max_scatter = max_prefill;
        m->d_scatter_idx = m->ctx.alloc<int>(max_prefill);
        for (size_t i = 0; i < n_eos; ++i) m->stop_ids.push_back(eos_ids[i]);
        AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
        AHA_CUDA_CHECK(cudaDeviceSynchronize());
        *out = m;
        return 0;
    } catch (const std::exception& e) {
        set_create_error(e.what());
        cudaGetLastError();
        if (m) aha_b200_destroy(m);
        return 1;
    }
}

int aha_b200_forward_initial(aha_model* m, const uint32_t* ids, size_t seq_len, size_t seqlen_offset, const aha_mm* mm, float* logits_out,
                             uint32_t* argmax_out) {
    return guarded(m, [&] { require_no_session(m); m->cached_ids.clear(); forward_any(m, m->text.table, ids, seq_len, seqlen_offset, mm, true, logits_out, argmax_out); });
}

int aha_b200_forward_step(aha_model* m, const uint32_t* ids, size_t seq_len, size_t seqlen_offset, float* logits_out, uint32_t* argmax_out) {
    return guarded(m, [&] { require_no_session(m); m->cached_ids.clear(); forward_any(m, m->text.table, ids, seq_len, seqlen_offset, nullptr, false, logits_out, argmax_out); });
}

int aha_b200_forward_extend(aha_model* m, const uint32_t* ids, size_t seq_len, size_t seqlen_offset, float* logits_out, uint32_t* argmax_out) {
    return guarded(m, [&] { require_no_session(m); m->cached_ids.clear(); forward_any(m, m->text.table, ids, seq_len, seqlen_offset, nullptr, false, logits_out, argmax_out, true); });
}

size_t aha_b200_last_prefix_hit(aha_model* m) { return m ? m->last_prefix_hit : 0; }

size_t aha_b200_prefix_match(const uint32_t* cached, size_t n_cached, const uint32_t* ids, size_t n, const uint32_t* mm_token_ids, size_t n_mm_tokens,
                             int same_mm) {
    if ((!cached && n_cached) || (!ids && n) || (!mm_token_ids && n_mm_tokens)) return 0;
    return prefix_match(cached, n_cached, ids, n, mm_token_ids, n_mm_tokens, same_mm != 0);
}

uint64_t aha_b200_mm_fingerprint(const aha_mm* mm) { return mm_fingerprint(mm); }

int aha_b200_clear_cache(aha_model* m) {
    return guarded(m, [&] {
        AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
        if (m->session.open) session_close(m);   // clear_cache ends a batch session too: every sequence's K/V is gone
        else drop_cache(m);
    });
}

size_t aha_b200_stop_token_ids(aha_model* m, uint32_t* out, size_t cap) {
    if (!m) return 0;
    for (size_t i = 0; i < m->stop_ids.size() && i < cap && out; ++i) out[i] = m->stop_ids[i];
    return m->stop_ids.size();
}

namespace {

struct GenSink {   // receives every generated token in order (with its record when the request asked); returns true to stop the request (client went away)
    std::function<bool(uint32_t token, size_t index, const aha_logprobs* lp)> push;
};

// generate_generic / generate_stream_generic (common/generate.rs:115-159, 231-368) with the loop on the device:
// forward_initial + sample, then decode steps chained through DecodeState (token, position, history, RNG draw index all
// live in HBM); the host only looks at the tokens, a burst behind the device.  `stream`: tokens are handed to the sink one
// by one as their step completes (per-step event) while the device keeps running ahead inside the burst.
// lp_n >= 0: every token's log-probability record (lp_n alternatives) is computed after its step and travels with it.
void generate_impl(aha_model* m, const uint32_t* ids, size_t seq_len, const aha_mm* mm, const aha_gen_params& params, const GenSink& sink, bool stream,
                   aha_usage* usage, size_t* n_generated, int lp_n = -1) {
    TextModel& T = m->text;
    require_no_session(m);
    request_rules(m, params, "");
    const bool lp = lp_n >= 0;
    request_logprobs(m, lp_n);
    const size_t sample_len = token_budget(params);
    AHA_REQUIRE(seq_len + sample_len <= (size_t)T.max_ctx,
                "prompt + max_tokens exceeds max_ctx (the handle's KV capacity, aha_options.max_ctx; the reference's cache is unbounded)");
    const auto t0 = clk::now();   // prompt_secs covers everything up to the first token, the prefix lookup (fingerprint of the tensors) included
    const bool eos_on_first = (params.flags & AHA_GEN_EOS_ON_FIRST) != 0;
    // KV reuse (AHA_GEN_REUSE_PREFIX): how much of this prompt the cache already holds.  Every path that is not a hit starts from
    // model.clear_cache(), exactly where the reference starts every request.
    const bool reuse = (params.flags & AHA_GEN_REUSE_PREFIX) != 0;
    size_t hit = 0;
    uint64_t mm_fp = 0;
    if (reuse) {
        mm_fp = mm_fingerprint(mm);
        const auto mmt = mm_token_ids(m);
        hit = prefix_match(m->cached_ids.data(), m->cached_ids.size(), ids, seq_len, mmt.data(), mmt.size(), mm_fp == m->cached_mm_fp);
    }
    if (hit == 0) drop_cache(m);
    m->cached_ids.clear();   // the cache is being written: nothing is reusable until this request has completed
    m->last_prefix_hit = hit;
    std::vector<uint32_t> produced;   // what the request generated (the K/V of all but the last token end up in the cache)
    RequestReset reset{m};
    uint32_t draws0 = 0;
    if ((params.flags & AHA_GEN_CONTINUE_RNG) != 0) {   // one LogitsProcessor across the chunks of a request: keep its stream position
        DecodeState cur;
        AHA_CUDA_CHECK(cudaMemcpy(&cur, T.d_state, sizeof(cur), cudaMemcpyDeviceToHost));
        draws0 = cur.n_draws;
    }
    auto is_eos = [&](uint32_t t) { for (uint32_t e : m->stop_ids) if (e == t) return true; return false; };
    const uint32_t tok = first_token(m, T.table, ids, seq_len, hit, mm, request_sampler(m, params, ""), draws0);
    if (lp) {   // the first token's record, from the prefill logits
        T.logprobs(true, T.d_lp, true);
        AHA_CUDA_CHECK(cudaMemcpyAsync(m->h_lp_pin, T.d_lp, sizeof(aha_logprobs), cudaMemcpyDeviceToHost, m->ctx.stream));
        AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
    }
    const auto t1 = clk::now();
    const double vision_secs = m->last_vision_secs;
    size_t done = 1;
    produced.push_back(tok);
    bool stop = sink.push(tok, 0, lp ? m->h_lp_pin : nullptr) || (eos_on_first && is_eos(tok));   // generate_generic never EOS-checks the first token; the ASR loop does
    if (sample_len > 1 && !stop) {
        handoff(m, T.table, seq_len + sample_len, tok, seq_len);
        const size_t burst_max = stream ? (size_t)aha_model::kStreamBurst : 32;
        while (done < sample_len && !stop) {
            const size_t n = std::min<size_t>(burst_max, sample_len - done);
            for (size_t i = 0; i < n; ++i) {
                T.decode_step(lp);
                if (lp) T.logprobs(false, T.d_lp, true);
                if (stream) {
                    AHA_CUDA_CHECK(cudaMemcpyAsync(m->h_pin + i, T.d_history + done + i, sizeof(uint32_t), cudaMemcpyDeviceToHost, m->ctx.stream));
                    if (lp) AHA_CUDA_CHECK(cudaMemcpyAsync(m->h_lp_pin + i, T.d_lp + done + i, sizeof(aha_logprobs), cudaMemcpyDeviceToHost, m->ctx.stream));
                    AHA_CUDA_CHECK(cudaEventRecord(m->ev_tok[i], m->ctx.stream));
                }
            }
            if (!stream) {
                AHA_CUDA_CHECK(cudaMemcpyAsync(m->h_pin, T.d_history + done, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, m->ctx.stream));
                if (lp) AHA_CUDA_CHECK(cudaMemcpyAsync(m->h_lp_pin, T.d_lp + done, n * sizeof(aha_logprobs), cudaMemcpyDeviceToHost, m->ctx.stream));
                AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
            }
            for (size_t i = 0; i < n && !stop; ++i) {
                if (stream) AHA_CUDA_CHECK(cudaEventSynchronize(m->ev_tok[i]));
                const uint32_t t = m->h_pin[i];
                ++done;
                produced.push_back(t);
                stop = sink.push(t, done - 1, lp ? m->h_lp_pin + i : nullptr) || is_eos(t);   // an EOS token is pushed before the break (generate.rs:139-141)
            }
            AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
            T.check_ll_abort();
            T.check_sample_error();
        }
    }
    const auto t2 = clk::now();
    if (reuse) {
        // the cache now holds the prompt and every generated token that was fed back (all but the last one): step j wrote the K/V of token j-1.
        // Steps the device ran past an EOS inside a burst wrote positions beyond that; they are simply overwritten by the next request.
        m->cached_ids.assign(ids, ids + seq_len);
        m->cached_ids.insert(m->cached_ids.end(), produced.begin(), produced.end() - 1);
        m->cached_mm_fp = mm_fp;
        reset.keep = true;
    }
    if (n_generated) *n_generated = done;
    add_usage(usage, seq_len, done, seconds(t1 - t0), seconds(t2 - t1), vision_secs);
}

// generate_impl's request in verify passes (speculative.cuh): the same prefill, first token, Reset guard and Usage split; then passes of
// R = max_draft + 1 rows in bursts, the emitted tokens (and records) read from the request's history after each burst.
// The checks every speculative request passes before any device work (generate_speculative, batch_add_speculative) -> its ngram
int spec_request_check(aha_model* m, const aha_gen_params& params, const aha_spec_params& sp, const std::string& who) {
    TextModel& T = m->text;
    AHA_REQUIRE(T.tp_world == 1, who + "speculative decoding is single-GPU");
    AHA_REQUIRE(m->kind != aha_model::QWEN3_ASR, who + "Qwen3-ASR handles decode through asr_generate");
    AHA_REQUIRE(BatchDecoder::wide_shapes_ok(T) && T.cfg.hd == 128,
                who + "every projection's rows and columns must be multiples of 64 and head_dim 128 (hidden " + std::to_string(T.cfg.H) +
                    ", intermediate " + std::to_string(T.I_l) + ", qkv rows " + std::to_string(T.qkv_dim) + ", vocabulary " + std::to_string(T.cfg.V) + ")");
    AHA_REQUIRE(sp.max_draft >= 1 && sp.max_draft <= (uint32_t)(kSpecMaxRows - 1), who + "max_draft must be 1 to " + std::to_string(kSpecMaxRows - 1));
    const int ngram = sp.ngram == 0 ? kSpecDefaultNgram : (int)sp.ngram;
    AHA_REQUIRE(ngram >= 1 && ngram <= kSpecMaxNgram, who + "ngram must be 0 (default " + std::to_string(kSpecDefaultNgram) + ") to " + std::to_string(kSpecMaxNgram));
    AHA_REQUIRE((sp.flags & ~AHA_SPEC_PROMPT_LOOKUP) == 0, who + "unknown spec flags");
    AHA_REQUIRE(sp.prediction || sp.n_prediction == 0, who + "prediction is NULL but n_prediction is not 0");
    for (size_t i = 0; i < sp.n_prediction; ++i) AHA_REQUIRE(sp.prediction[i] < (uint32_t)T.cfg.V, who + "prediction token id out of range");
    AHA_REQUIRE((params.flags & (AHA_GEN_REUSE_PREFIX | AHA_GEN_CONTINUE_RNG | AHA_GEN_EOS_ON_FIRST)) == 0,
                who + "REUSE_PREFIX, CONTINUE_RNG and EOS_ON_FIRST are not supported with speculative decoding");
    AHA_REQUIRE((params.flags & AHA_GEN_CONSTRAINED) == 0,
                who + "AHA_GEN_CONSTRAINED is not supported with speculative decoding (a verify row's mask would depend on the drafts before it)");
    AHA_REQUIRE(request_rules(m, params, who).fsm == nullptr,
                who + "logit rules that name a token automaton are not supported with speculative decoding (a verify row's mask would depend on "
                      "the drafts before it)");
    return ngram;
}

void generate_speculative_impl(aha_model* m, const uint32_t* ids, size_t seq_len, const aha_mm* mm, const aha_gen_params& params,
                               const aha_spec_params& sp, uint32_t* out_tokens, aha_logprobs* out_lp, size_t cap, size_t* n_out, aha_usage* usage,
                               aha_spec_stats* stats) {
    TextModel& T = m->text;
    const std::string who = "generate_speculative: ";
    require_no_session(m);
    const int ngram = spec_request_check(m, params, sp, who);
    const int lp_n = logprob_request(params, T, who);
    AHA_REQUIRE(lp_n < 0 || out_lp, who + "AHA_GEN_LOGPROBS needs out_logprobs");
    const size_t sample_len = token_budget(params);
    AHA_REQUIRE(cap >= sample_len, who + "out_tokens capacity is smaller than max_tokens");
    const size_t need = seq_len + sample_len + sp.max_draft;
    AHA_REQUIRE(need <= (size_t)T.max_ctx, who + "prompt + max_tokens + max_draft = " + std::to_string(need) + " tokens exceeds max_ctx " + std::to_string(T.max_ctx));
    const int R = (int)sp.max_draft + 1;
    SpecDecoder& S = m->spec;
    S.init(T, m->wide_batch, kSpecMaxRows);
    request_logprobs(m, lp_n);
    const auto t0 = clk::now();
    drop_cache(m);
    m->last_prefix_hit = 0;
    RequestReset reset{m};
    const Sampler samp = request_sampler(m, params, who);
    const uint32_t tok = first_token(m, T.table, ids, seq_len, 0, mm, samp, 0);
    if (lp_n >= 0) T.logprobs(true, T.d_lp, true);   // record 0, from the prefill logits
    const auto t1 = clk::now();
    const double vision_secs = m->last_vision_secs;
    SpecCtl ctl{};
    size_t E = 1;
    if (sample_len > 1) {
        handoff(m, T.table, need, tok, seq_len);
        const std::vector<uint32_t> pred(sp.prediction, sp.prediction + sp.n_prediction);
        const bool lookup = (sp.flags & AHA_SPEC_PROMPT_LOOKUP) != 0;
        S.prepare(R, samp, pred, ids, lookup ? seq_len : 0, m->stop_ids, (int)sample_len, ngram, lp_n >= 0 ? lp_n + 1 : 0);
        DecodeState cur;
        while (true) {
            // a pass emits 1 .. R tokens: never launch more passes than the remaining budget could need at R tokens each
            const size_t burst = std::min<size_t>(8, std::max<size_t>(1, (sample_len - E + R - 1) / R));
            for (size_t i = 0; i < burst; ++i) S.pass(R);
            AHA_CUDA_CHECK(cudaMemcpyAsync(&ctl, S.d_ctl, sizeof(ctl), cudaMemcpyDeviceToHost, m->ctx.stream));
            AHA_CUDA_CHECK(cudaMemcpyAsync(&cur, T.d_state, sizeof(cur), cudaMemcpyDeviceToHost, m->ctx.stream));
            AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
            T.check_sample_error();
            E = (size_t)cur.n_hist;
            if (ctl.done) break;
        }
    }
    AHA_CUDA_CHECK(cudaMemcpy(out_tokens, T.d_history, E * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    out_tokens[0] = tok;
    if (lp_n >= 0) AHA_CUDA_CHECK(cudaMemcpy(out_lp, T.d_lp, E * sizeof(aha_logprobs), cudaMemcpyDeviceToHost));
    const auto t2 = clk::now();
    *n_out = E;
    if (stats) { *stats = aha_spec_stats{}; stats->passes = ctl.passes; stats->drafted = ctl.drafted; stats->accepted = ctl.accepted; }
    add_usage(usage, seq_len, E, seconds(t1 - t0), seconds(t2 - t1), vision_secs);
}

}  // namespace

namespace {
// One request into slot `slot` of the batch decoder: the reference's forward_initial + sample_and_push on the slot's own page table (the
// single-request code, so tower / M-RoPE / deepstack / sampler-on-prefill are shared), then its decode state, history and sampler move into the
// slot.  hit > 0: the table already starts with the prefix cache's pages of ids[0, hit) and only the rest is prefilled, as a continuation (a
// text-only prompt, so on Qwen3-VL its positions are the plain ones, rope_delta 0).  If this throws, the slot's table holds whatever pages it
// took and the caller releases them with the slot.
uint32_t batch_prefill_slot(aha_model* m, int slot, const aha_batch_request& r, size_t sample_len, int lp_n, size_t hit = 0) {
    TextModel& T = m->text;
    BatchDecoder& B = m->sess();
    PageTable& pt = B.slots[slot].table;
    m->have_rope_delta = hit > 0; m->rope_delta = 0;
    const Sampler samp = request_sampler(m, r.params, "");
    const uint32_t tok = first_token(m, pt, r.ids, r.seq_len, hit, r.mm, samp, 0);
    if (lp_n >= 0) {   // the first token's record goes straight into the slot's record row
        T.set_logprobs(lp_n);
        B.ensure_lp();
        T.logprobs(true, B.d_lp_rec + slot, false);
    }
    B.slots[slot].lp = lp_n + 1;
    B.bind_sampler(slot, samp);
    handoff(m, pt, r.seq_len + sample_len, tok, r.seq_len, slot);
    return tok;
}

// The hit rule of every admission path: the longest cached chain of full pages that starts the prompt, capped at seq_len - 1 tokens and,
// unless every GEMM runs on the SIMT kernel, at seq_len - kPage, so that the rows still prefilled run on the wgmma GEMM as the cold prefill of
// the same rows does (gemm_on_tc: M < 32 takes SIMT).  The pages it returns hold ids[0, kPage * size()).  Multimodal requests never hit.
std::vector<int> prefix_hit(const aha_model* m, const uint32_t* ids, size_t seq_len, bool has_mm, uint32_t lora) {
    const PrefixIndex& X = m->session.prefix;
    if (!X.on() || has_mm) return {};
    const size_t cap = m->ctx.gemm_impl == 1 ? seq_len - 1 : (seq_len >= (size_t)kPage ? seq_len - kPage : 0);
    return X.chain(ids, cap / kPage * kPage, lora);
}
// Admission's page check: `pages` fresh pages must fit the free list plus the pages only the prefix cache holds, less those this call hits
// (`keep`).  Once the call has passed every check, prefix_make_room evicts LRU leaves only as far as the call needs.
void prefix_check_room(const aha_model* m, size_t pages, const std::set<int>& keep, const std::string& what) {
    const TextModel& T = m->text;
    const PrefixIndex& X = m->session.prefix;
    const size_t avail = T.pages.free_count() + (X.on() ? X.evictable(T.pages, keep) : 0);
    AHA_REQUIRE(pages <= avail, what + std::to_string(pages * kPage) + " tokens of KV capacity, " + std::to_string(avail * kPage) +
                                    " are free (max_ctx " + std::to_string(T.max_ctx) + ")");
}
void prefix_make_room(aha_model* m, size_t pages, const std::set<int>& keep) {
    while (m->text.pages.free_count() < pages) AHA_REQUIRE(m->session.prefix.evict_one(m->text.pages, keep), "prefix cache: no page left to evict");
}
// the shared pages first in the (empty) table of each admitted request that hit; the debug assert states why no step ever writes them:
// decode writes positions >= seq_len, and the hit ends at or before seq_len - 1
void prefix_share(aha_model* m, int slot, const std::vector<int>& pages, size_t seq_len) {
    assert(pages.size() * kPage < seq_len);
    if (!pages.empty()) m->text.pages.share(m->sess().slots[slot].table, pages);
    (void)seq_len;
}
// after a successful admission: the request's full prompt pages enter the index, and the statistics count its lookup
void prefix_admitted(aha_model* m, int slot, const uint32_t* ids, size_t seq_len, size_t hit, uint32_t lora) {
    PrefixIndex& X = m->session.prefix;
    if (!X.on()) return;
    X.lookups += 1;
    X.hit_tokens += hit;
    X.insert(m->text.pages, ids, seq_len, m->sess().slots[slot].table, lora);
}

// ---- continuous batching: the same slots and the same step, with requests joining and leaving between steps -------------------------
// (new design; the reference's server holds ONE request behind a write lock, server/api.rs:117.)  A finished request's pages go back to the
// free list at once, so a waiting request can take its place while the others keep decoding.
aha_model::BatchSession& open_session(aha_model* m) {
    AHA_REQUIRE(m->session.open, "no batch session is open (aha_b200_batch_open)");
    return m->session;
}
SlotRequest& slot_req(aha_model* m, int slot) { return m->sess().slots[slot].req; }
// a finished request leaves its slot (SlotRequest::release)
void session_release(aha_model* m, int slot) {
    BatchSlot& sl = m->sess().slots[slot];
    m->text.pages.release(sl.table);
    sl.samp_active = false;
    sl.lp = 0;
    sl.req.release();
    m->sess().composition_changed();
}
// a cancelled or suspended request, or one whose admission failed, leaves its slot (SlotRequest::clear)
void session_clear(aha_model* m, int slot) {
    session_release(m, slot);
    slot_req(m, slot).clear();
}
// verify rows of the running requests: R for a speculative request, 1 for a plain one
int session_rows(aha_model* m) {
    int rows = 0;
    for (int i = 0; i < m->session.width; ++i) {
        const SlotRequest& r = slot_req(m, i);
        if (r.used) rows += r.spec ? r.R : 1;
    }
    return rows;
}
bool session_has_spec(aha_model* m) {
    for (int i = 0; i < m->session.width; ++i) if (slot_req(m, i).used && slot_req(m, i).spec) return true;
    return false;
}
// The n lowest free slots for an admission or a resume, after the slot checks: enough free slots (batch_add_n counts choices), and room for
// `rows` more step rows.  Beside speculative requests a step's rows must fit the wide kernel's 64-row B tile; without them the rows are the
// running slots, which the session width already bounds.
std::vector<int> free_slots(aha_model* m, size_t n, int rows, const std::string& who, bool choices = false) {
    const std::string width = std::to_string(m->session.width);
    std::vector<int> slot;
    for (int i = 0; i < m->session.width; ++i) if (!slot_req(m, i).used) slot.push_back(i);
    AHA_REQUIRE(choices || !slot.empty(), who + "all " + width + " slots are decoding (step until one finishes)");
    AHA_REQUIRE(n <= slot.size(), who + std::to_string(n) + (choices ? " choices" : " requests") + ", but only " + std::to_string(slot.size()) +
                                      " of the " + width + " slots are free (step until requests finish)");
    slot.resize(n);
    const int now = session_rows(m);
    AHA_REQUIRE(now + rows <= kWideSeqs, who + "the step rows of the running requests (" + std::to_string(now) + ", a speculative request counts "
                                              "max_draft + 1) plus " + std::to_string(rows) + " exceed " + std::to_string(kWideSeqs));
    return slot;
}
void require_ctx(const aha_model* m, size_t ctx, const std::string& what) {
    AHA_REQUIRE(ctx <= (size_t)m->text.max_ctx, what + std::to_string(ctx) + " tokens exceeds max_ctx " + std::to_string(m->text.max_ctx));
}
// What admission needs of one request, from the checks every admission path runs on it before any device work
struct AdmitReq {
    const aha_batch_request* r;
    int lp_n;                       // logprob_request
    size_t budget;                  // token_budget
    size_t ctx;                     // the positions its pages hold: prompt + budget (+ max_draft)
    bool has_mm;                    // (a qwen3 handle ignores the tensors)
    std::vector<int> hit_pages;     // prefix_hit: the cached pages its table starts with
    uint32_t lora = 0;              // its LoRA adapter (0: the base model)
    size_t hit() const { return hit_pages.size() * kPage; }
    // fresh pages for n copies of it (the first one shares the hit pages)
    size_t pages(size_t n = 1) const { return n * ((ctx + kPage - 1) / kPage) - hit_pages.size(); }
};
// i: the request's index in a batch_add_many call, -1 for the call's only request; extra: positions beyond prompt + budget
AdmitReq admit_check(aha_model* m, const aha_batch_request& r, const std::string& who, int i, size_t extra = 0, uint32_t lora = 0) {
    const TextModel& T = m->text;
    const std::string at = i < 0 ? who : who + "request " + std::to_string(i) + ": ";
    AHA_REQUIRE(r.ids && r.seq_len >= 1, who + (i < 0 ? "the request" : "request " + std::to_string(i)) + " needs input_ids");
    AdmitReq a{&r};
    a.lp_n = logprob_request(r.params, T, at);
    for (size_t k = 0; k < r.seq_len; ++k) AHA_REQUIRE(r.ids[k] < (uint32_t)T.cfg.V, "token id out of range");
    AHA_REQUIRE((r.params.flags & (AHA_GEN_CONTINUE_RNG | AHA_GEN_REUSE_PREFIX)) == 0, who + "CONTINUE_RNG / REUSE_PREFIX are per-handle states of the single-request calls");
    request_rules(m, r.params, at);
    require_mm_arity(m, r.mm);
    a.budget = token_budget(r.params);
    a.ctx = r.seq_len + a.budget + extra;
    for (size_t k = 0; m->kind != aha_model::QWEN3 && k < r.mm->n; ++k) a.has_mm = a.has_mm || mm_entry(r.mm, k) != nullptr;
    a.lora = lora;
    a.hit_pages = prefix_hit(m, r.ids, r.seq_len, a.has_mm, lora);
    return a;
}
// One admission call: its slots (request k into slots[k]; every choice of batch_add_n is a[0]'s) and its checked requests.  Once it has
// taken the slots and until it commits, its destructor leaves the session as it was: every slot it took is cleared with its pages.
struct Admission {
    aha_model* m;
    std::vector<int> slots;
    std::vector<AdmitReq> a;
    bool taken = false, ok = false;
    ~Admission() {
        if (!taken || ok) return;
        for (int s : slots) session_clear(m, s);
        m->have_rope_delta = false; m->rope_delta = 0; m->text.clear_sampler();
    }
    std::set<int> keep() const {   // pages the requests hit: never evicted by this call
        std::set<int> k;
        for (const AdmitReq& q : a) k.insert(q.hit_pages.begin(), q.hit_pages.end());
        return k;
    }
    void check_room(size_t pages, const std::string& what) const { prefix_check_room(m, pages, keep(), what); }
    // after every check: evicts cached prefixes as far as `pages` fresh pages need, takes the slots and starts each request's table with
    // its hit pages
    void take(size_t pages) {
        prefix_make_room(m, pages, keep());
        taken = true;
        for (int s : slots) slot_req(m, s).used = true;
        for (size_t k = 0; k < a.size(); ++k) prefix_share(m, slots[k], a[k].hit_pages, a[k].r->seq_len);
    }
    // Slot k has its first token tok[k]: the requests' prompt pages enter the prefix index, each slot's record starts (a slot whose first
    // token is also its last is released), and the outputs of slot k are filled.
    void commit(const std::vector<uint32_t>& tok, const std::vector<double>& secs, const std::vector<double>& vision, int32_t* slots_out,
                uint32_t* first_tokens, int32_t* finished, aha_usage* usage) {
        ok = true;
        for (size_t k = 0; k < a.size(); ++k) if (!a[k].has_mm) prefix_admitted(m, slots[k], a[k].r->ids, a[k].r->seq_len, a[k].hit(), a[k].lora);
        m->text.clear_sampler();
        m->sess().composition_changed();
        for (size_t k = 0; k < slots.size(); ++k) {
            const AdmitReq& q = a[std::min(k, a.size() - 1)];
            SlotRequest& r = slot_req(m, slots[k]);
            r = SlotRequest{};
            r.used = true; r.budget = q.budget; r.produced = 1; r.hit = k < a.size() ? q.hit() : 0; r.lp_valid = q.lp_n >= 0; r.lora = q.lora;
            bool stop = q.budget == 1;
            if ((q.r->params.flags & AHA_GEN_EOS_ON_FIRST) != 0) for (uint32_t e : m->stop_ids) if (e == tok[k]) stop = true;
            if (stop) session_release(m, slots[k]);
            if (usage) {
                usage[k] = aha_usage{};
                add_usage(&usage[k], q.r->seq_len, 1, secs[k], 0.0, vision[k]);
            }
            slots_out[k] = slots[k]; first_tokens[k] = tok[k]; finished[k] = stop ? 1 : 0;
        }
    }
};
// the first tokens just drawn into the session decoder's d_tok and their decode states (draw counts, automaton states), read back once,
// then the sampler check
void read_first_tokens(aha_model* m, std::vector<uint32_t>& tok, std::vector<DecodeState>& st) {
    BatchDecoder& B = m->sess();
    Ctx& c = m->ctx;
    tok.resize((size_t)B.cap);
    st.resize((size_t)B.cap);
    AHA_CUDA_CHECK(cudaMemcpyAsync(tok.data(), B.d_tok, tok.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, c.stream));
    AHA_CUDA_CHECK(cudaMemcpyAsync(st.data(), B.d_states, st.size() * sizeof(DecodeState), cudaMemcpyDeviceToHost, c.stream));
    AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
    m->text.check_sample_error();
}
// width 0: the narrow session (8 slots, batched CUDA-core GEMV); 1..64: a wide session (gemv_wide.cuh)
void session_open(aha_model* m, int width) {
    TextModel& T = m->text;
    require_no_session(m);
    AHA_REQUIRE(T.tp_world == 1, "batch sessions are single-GPU");
    if (width == 0) AHA_REQUIRE(T.max_prefill >= kGemvBatchMax, "batch sessions need max_prefill >= 8");
    else {
        AHA_REQUIRE(width >= 1 && width <= kWideSeqs, "batch_open_wide: max_seqs must be 1 to 64");
        AHA_REQUIRE(BatchDecoder::wide_shapes_ok(T), "batch_open_wide: every projection's rows and columns must be multiples of 64 "
                                                     "(hidden " + std::to_string(T.cfg.H) + ", intermediate " + std::to_string(T.I_l) +
                                                     ", qkv rows " + std::to_string(T.qkv_dim) + ", vocabulary " + std::to_string(T.cfg.V) + ")");
    }
    drop_cache(m);
    BatchDecoder& B = width == 0 ? m->batch : m->wide_batch;
    if (width == 0) B.init(T, kGemvBatchMax);
    else B.init_wide(T);
    B.reset();
    B.gemv = env_int("AHA_BATCH_GEMV", kBatchGemvDefault);   // (the wide step always runs gemv_wide)
    B.use_graph = env_flag("AHA_BATCH_GRAPH", true);
    m->session = aha_model::BatchSession{};
    m->session.open = true;
    m->session.wide = width != 0;
    m->session.width = width == 0 ? kGemvBatchMax : width;
}
// ---- ending and swapping requests between steps (aha_b200_batch_cancel / _suspend / _resume / _discard).  Every check runs before anything
// is copied or written (suspend first reads the slot's DecodeState), so a refused call changes nothing.
void session_check_slot(aha_model* m, int32_t slot, const std::string& who) {
    open_session(m);
    AHA_REQUIRE(slot >= 0 && slot < m->session.width, who + "slot " + std::to_string(slot) + " is outside the session's " +
                                                          std::to_string(m->session.width) + " slots");
    AHA_REQUIRE(slot_req(m, slot).used, who + "slot " + std::to_string(slot) + " runs no request");
}
// the request in `slot` ends as if it had finished: its pages go back at once (the prefix index keeps its references) and the slot shows
// no record; a speculative slot keeps its counters until the slot is taken again
void session_cancel(aha_model* m, int32_t slot) {
    session_check_slot(m, slot, "batch_cancel: ");
    session_clear(m, slot);
}
aha_model::Suspended& suspended_of(aha_model* m, uint32_t id, const std::string& who) {
    open_session(m);
    const auto it = m->suspended.find(id);
    AHA_REQUIRE(it != m->suspended.end(), who + "no suspended request of this session has id " + std::to_string(id));
    return it->second;
}
// The request in `slot` to the swap arena: the K/V pages it has written (logical pages 0 .. ceil(pos / 32) - 1, pos from its device
// DecodeState), its DecodeState, its history and the host-side slot state; then the slot and every page reference it held are released as
// session_release does.  -> its id.
uint32_t session_suspend(aha_model* m, int32_t slot) {
    const std::string who = "batch_suspend: ";
    session_check_slot(m, slot, who);
    AHA_REQUIRE(!slot_req(m, slot).spec, who + "slot " + std::to_string(slot) + " runs a speculative request, which cannot be suspended "
                                               "(aha_b200_batch_cancel ends it)");
    aha_model::SwapArena& A = m->swap;
    AHA_REQUIRE(A.pages > 0, who + "the handle has no swap space (aha_b200_batch_swap_space)");
    AHA_REQUIRE(m->next_suspend_id != 0, who + "the handle has used every suspended-request id");
    TextModel& T = m->text;
    BatchDecoder& B = m->sess();
    BatchSlot& sl = B.slots[slot];
    Ctx& c = m->ctx;
    const auto t0 = clk::now();
    aha_model::Suspended r;
    AHA_CUDA_CHECK(cudaMemcpyAsync(&r.st, B.d_states + slot, sizeof(DecodeState), cudaMemcpyDeviceToHost, c.stream));
    AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
    const int pages = ceil_div(r.st.pos, kPage);
    AHA_REQUIRE(pages >= 1 && pages <= sl.table.mapped && r.st.n_hist >= 1 && r.st.n_hist <= T.hist_cap, who + "slot " + std::to_string(slot) +
                                                                                                           " holds an inconsistent decode state");
    AHA_REQUIRE((size_t)pages <= A.free.size(), who + "the request has written " + std::to_string(pages) + " KV pages, but only " +
                                                    std::to_string(A.free.size()) + " of the " + std::to_string(A.pages) + " host pages are free");
    r.host_pages.assign(A.free.end() - pages, A.free.end());
    r.hist.resize((size_t)r.st.n_hist);
    kv_swap(c, true, T.kv_pool, T.layer_stride, T.page_stride, T.cfg.L, sl.table.h.data(), r.host_pages.data(), A.host, pages);
    AHA_CUDA_CHECK(cudaMemcpyAsync(r.hist.data(), B.d_hist + (size_t)slot * T.hist_cap, r.hist.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, c.stream));
    AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
    A.free.resize(A.free.size() - pages);
    r.mapped = sl.table.mapped;
    r.sampler = sl.sampler;
    r.lp = sl.lp;
    r.req = sl.req;
    const uint32_t id = m->next_suspend_id++;
    m->suspended.emplace(id, std::move(r));
    session_clear(m, slot);
    A.pages_out += (uint64_t)pages;
    A.suspend_secs += seconds(clk::now() - t0);
    return id;
}
// A suspended request back into the lowest free slot: the same number of pages it held (cached prefix pages may be evicted for them, as at
// admission; its shared prefix pages come back as its own), its K/V, DecodeState, history and slot state restored, its sampler bound to the
// new slot.  No token is delivered: its next one comes from the next step.  -> the slot.
int32_t session_resume(aha_model* m, uint32_t id) {
    const std::string who = "batch_resume: ";
    aha_model::Suspended& r = suspended_of(m, id, who);
    AHA_REQUIRE(!(r.req.lora && session_has_spec(m)), who + "suspended request " + std::to_string(id) + " runs LoRA adapter " +
                                                          std::to_string(r.req.lora) + " and a speculative request is running: speculative "
                                                          "requests and adapters do not share a session");
    const int slot = free_slots(m, 1, 1, who)[0];
    prefix_check_room(m, (size_t)r.mapped, {}, who + "the request needs ");
    prefix_make_room(m, (size_t)r.mapped, {});
    TextModel& T = m->text;
    BatchDecoder& B = m->sess();
    BatchSlot& sl = B.slots[slot];
    aha_model::SwapArena& A = m->swap;
    Ctx& c = m->ctx;
    const auto t0 = clk::now();
    const int pages = (int)r.host_pages.size();
    T.pages.map(sl.table, std::min(r.mapped * kPage, T.max_ctx));
    sl.req = r.req;              // budget, produced and hit; a suspended request ran plain steps only, so its spec state is clear
    sl.req.lp_valid = false;     // the record of its last token was read before it was suspended
    kv_swap(c, false, T.kv_pool, T.layer_stride, T.page_stride, T.cfg.L, sl.table.h.data(), r.host_pages.data(), A.host, pages);
    AHA_CUDA_CHECK(cudaMemcpyAsync(B.d_states + slot, &r.st, sizeof(DecodeState), cudaMemcpyHostToDevice, c.stream));
    AHA_CUDA_CHECK(cudaMemcpyAsync(B.d_hist + (size_t)slot * T.hist_cap, r.hist.data(), r.hist.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, c.stream));
    if (r.lp > 0) B.ensure_lp();
    sl.lp = r.lp;
    B.bind_sampler(slot, r.sampler);
    AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
    B.composition_changed();
    A.free.insert(A.free.end(), r.host_pages.begin(), r.host_pages.end());
    A.pages_in += (uint64_t)pages;
    A.resume_secs += seconds(clk::now() - t0);
    m->suspended.erase(id);
    return slot;
}
void session_discard(aha_model* m, uint32_t id) {
    aha_model::Suspended& r = suspended_of(m, id, "batch_discard: ");
    m->swap.free.insert(m->swap.free.end(), r.host_pages.begin(), r.host_pages.end());
    m->suspended.erase(id);
}
// The arena resized to max_tokens / 32 host pages (0 frees it); refused while a request is suspended.  The new arena is allocated before
// the old one is freed, so a failed allocation leaves the old one in place.
void swap_space(aha_model* m, size_t max_tokens) {
    aha_model::SwapArena& A = m->swap;
    AHA_REQUIRE(m->suspended.empty(), "batch_swap_space: " + std::to_string(m->suspended.size()) + " requests are suspended (resume or "
                                      "discard them first)");
    const size_t pages = max_tokens / kPage;
    if (pages == A.pages) return;
    float* host = nullptr;
    if (pages) AHA_CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&host), pages * m->swap_page_bytes(), cudaHostAllocPortable));
    AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
    if (A.host) AHA_CUDA_CHECK(cudaFreeHost(A.host));
    A.host = host; A.pages = pages;
    A.free.clear();
    for (int p = 0; p < (int)pages; ++p) A.free.push_back(p);
}

// The LoRA adapters of the rows of the prefills run while it lives: ad[row] an adapter index (< 0: the base model).  Rows of the base model
// alone set nothing, so such prefills run exactly as without adapters.
struct LoraPrefill {
    LoraSet& L;
    LoraPrefill(aha_model* m, const std::vector<int>& ad) : L(m->text.lora) {
        if (std::any_of(ad.begin(), ad.end(), [](int a) { return a >= 0; })) L.prefill_begin(m->ctx.stream, ad);
    }
    ~LoraPrefill() { L.prefill_end(); }
};
bool session_has_lora(aha_model* m) {
    for (int i = 0; i < m->session.width; ++i) if (slot_req(m, i).used && slot_req(m, i).lora) return true;
    return false;
}

// n requests admitted in one call (aha_b200_batch_add_many).  Text-only requests that fit max_prefill are cut, in input order, into packed
// prefills (TextModel::prefill with PrefillSegments: each request attends only to itself and its positions restart at 0), so one pass over the
// weights serves them all; their last rows then go through the step's batched lm_head and each request's own ArgMax / sampler.  A request
// with multimodal tensors, or one longer than max_prefill, is prefilled alone by batch_prefill_slot.  pack = false prefills every request
// alone (aha_b200_batch_add, generate_batch).
//
// Every request of a pack starts on a multiple of kPage tokens, so the pack's page table is the slots' own page lists laid end to end: pack
// position p of the request starting at s0 is its page (p - s0) / kPage at the same offset, and the prefill writes every request's K/V straight
// into that request's own pages.  The gap behind a request is filled with token 0 and joins its segment; those K/V land in the request's last
// page at positions >= seq_len, which its decode steps overwrite before any step reads them.  A 32-token round-up never reaches a 64-token KV
// tile or a 128-token query tile that the request's own rows do not already touch, so each request runs the attention tiles it runs alone.
void session_add_many(aha_model* m, const aha_batch_request* reqs, size_t n, int32_t* slots_out, uint32_t* first_tokens, int32_t* finished,
                      aha_usage* usage, bool pack, const uint32_t* adapters = nullptr) {
    TextModel& T = m->text;
    BatchDecoder& B = m->sess();
    Ctx& c = m->ctx;
    const std::string who = adapters ? "batch_add_lora: " : (pack ? "batch_add_many: " : "batch_add: ");
    auto lora_of = [&](size_t i) { return adapters ? adapters[i] : 0u; };
    // ---- every check before any device work: a refused call leaves the session untouched
    open_session(m);
    AHA_REQUIRE(n >= 1, who + "no requests");
    Admission ad{m, free_slots(m, n, (int)n, who)};   // request i takes the i-th lowest free slot
    size_t pages = 0;
    for (size_t i = 0; i < n; ++i) {
        ad.a.push_back(admit_check(m, reqs[i], who, (int)i, 0, lora_of(i)));
        pages += ad.a[i].pages();
    }
    ad.check_room(pages, who + "the requests need ");
    for (const AdmitReq& q : ad.a) require_ctx(m, q.ctx, "context of ");   // (only reachable when max_ctx is not a multiple of the page)
    ad.take(pages);
    const auto t0 = clk::now();
    const std::vector<int>& slot = ad.slots;
    std::vector<uint32_t> tok(n);
    std::vector<double> secs(n), vision(n, 0.0);
    std::vector<bool> packed(n);
    // ---- packed requests: map every page each can touch (as batch_prefill_slot does after its prefill), then prefill them pack by pack
    // With prefix hits a request's pack segment is the part of its prompt the cache does not hold: ids[hit, seq_len) at positions hit ..
    std::vector<size_t> pk, pk_pre;
    std::vector<const uint32_t*> pk_ids;
    std::vector<size_t> pk_lens;
    bool any_hit = false;
    for (size_t i = 0; i < n; ++i) {
        const size_t hit = ad.a[i].hit();
        packed[i] = pack && !ad.a[i].has_mm && reqs[i].seq_len <= (size_t)T.max_prefill;
        if (!packed[i]) continue;
        pk.push_back(i); pk_ids.push_back(reqs[i].ids + hit); pk_lens.push_back(reqs[i].seq_len - hit); pk_pre.push_back(hit);
        any_hit = any_hit || hit > 0;
        T.pages.map(B.slots[slot[i]].table, (int)ad.a[i].ctx);
    }
    if (!any_hit) pk_pre.clear();
    if (!pk.empty()) {
        alloc_pack_buffers(m);
        if (any_hit && !m->d_pack_read) m->d_pack_read = c.alloc<int>((size_t)T.num_pages);
        const int H = T.cfg.H;
        const size_t cap = (size_t)std::min(T.max_prefill, T.max_ctx);
        for (size_t first = 0; first < pk.size();) {
            // (key rows: the split workspace of the attention holds max_ctx of them, as for a continuation prefill)
            Pack p = plan_pack(pk_ids, pk_lens, first, kPage, cap, pk_pre, (size_t)T.max_ctx);
            // The pack's table: the requests' own pages laid end to end, all mapped above, so the prefill takes no page from the pool and
            // writes only pages no other table holds.  With prefixes, the attention reads a second table: every request's pages from its
            // first, the shared ones included, laid end to end the same way (every segment but the last ends on a page boundary).
            PageTable pt, rd;
            for (size_t j = p.first; j < p.last; ++j) {
                const std::vector<int>& own = B.slots[slot[pk[j]]].table.h;
                const int pre = any_hit ? (int)pk_pre[j] / kPage : 0, seg = p.sg.segs[j - p.first].second;
                pt.h.insert(pt.h.end(), own.begin() + pre, own.begin() + pre + ceil_div(seg, kPage));
                if (any_hit) rd.h.insert(rd.h.end(), own.begin(), own.begin() + pre + ceil_div(seg, kPage));
            }
            pt.mapped = (int)pt.h.size();
            AHA_REQUIRE(ceil_div((int)p.S, kPage) <= pt.mapped, "batch_add_many: the pack's page table does not cover the pack");
            pt.h.resize(T.num_pages, 0);
            pt.d = m->d_pack_table;
            AHA_CUDA_CHECK(cudaMemcpyAsync(pt.d, pt.h.data(), (size_t)pt.mapped * sizeof(int), cudaMemcpyHostToDevice, c.stream));
            if (any_hit) {
                AHA_REQUIRE(ceil_div((int)p.KV, kPage) <= (int)rd.h.size() && rd.h.size() <= (size_t)T.num_pages, "batch_add_many: the pack's read table does not cover its keys");
                AHA_CUDA_CHECK(cudaMemcpyAsync(m->d_pack_read, rd.h.data(), rd.h.size() * sizeof(int), cudaMemcpyHostToDevice, c.stream));
                p.sg.d_read = m->d_pack_read;
                p.sg.kv_rows = (int)p.KV;
            }
            upload_pack(m, p);
            std::vector<int> row_lora(p.S, -1);   // every row of a segment, its filler included, runs its request's adapter
            for (size_t j = p.first; j < p.last; ++j) {
                const auto& sg = p.sg.segs[j - p.first];
                std::fill(row_lora.begin() + sg.first, row_lora.begin() + sg.first + sg.second, T.lora.index_of(lora_of(pk[j])));
            }
            {
                LoraPrefill lp(m, row_lora);
                T.prefill(pt, (int)p.S, 0, false, nullptr, 0, {}, p.sg);
            }
            gather_rows_kernel<<<(unsigned)(p.last - p.first), 256, 0, c.stream>>>(m->d_pack_rows, T.x, B.xb + p.first * H, H);
            c.cnt.kernels++;
            first = p.last;
        }
        // first tokens: batched lm_head over the gathered rows, then each request's ArgMax / sampler against an empty state (forward_any's draw)
        std::vector<int> act;
        std::vector<DecodeState> empty((size_t)B.cap, DecodeState{0, 0, 0, 0, 0, 0, {0, 0}});   // per slot: empty history, draw index 0
        for (size_t i : pk) {
            const Sampler samp = request_sampler(m, reqs[i].params, who);
            B.bind_sampler(slot[i], samp);
            empty[slot[i]].fsm_state = samp.fsm_start;
            B.slots[slot[i]].lp = ad.a[i].lp_n + 1;
            if (ad.a[i].lp_n >= 0) B.ensure_lp();
            act.push_back(slot[i]);
        }
        for (int s : act) AHA_CUDA_CHECK(cudaMemcpyAsync(B.d_states + s, &empty[s], sizeof(DecodeState), cudaMemcpyHostToDevice, c.stream));
        B.head_rows(act, true);
        std::vector<uint32_t> h_tok;
        std::vector<DecodeState> h_st;
        read_first_tokens(m, h_tok, h_st);
        const double t_first = seconds(clk::now() - t0);
        for (size_t i : pk) {   // (their pages were mapped before the prefill)
            B.adopt(slot[i], h_tok[slot[i]], (int)reqs[i].seq_len, 0, h_st[slot[i]].n_draws, h_st[slot[i]].fsm_state);
            tok[i] = h_tok[slot[i]];
            secs[i] = t_first;
        }
    }
    // ---- the others: one prefill each, on the slot's own table
    for (size_t i = 0; i < n; ++i) {
        if (packed[i]) continue;
        LoraPrefill lp(m, std::vector<int>(std::min((size_t)T.max_prefill, reqs[i].seq_len - ad.a[i].hit()), T.lora.index_of(lora_of(i))));
        tok[i] = batch_prefill_slot(m, slot[i], reqs[i], ad.a[i].budget, ad.a[i].lp_n, ad.a[i].hit());
        secs[i] = seconds(clk::now() - t0);
        vision[i] = m->last_vision_secs;
    }
    ad.commit(tok, secs, vision, slots_out, first_tokens, finished, usage);
}

// OpenAI `n` (aha_b200_batch_add_n): n choices of one request in the n lowest free slots.  The prompt is prefilled once, into choice 0's
// slot, by batch_prefill_slot (tower, M-RoPE, deepstack, chunks beyond max_prefill: whatever batch_add does); its pages are copied into the
// other choices' own pages by one kv_fork launch.  Every other choice then draws its first token from the prefill logits, still in
// TextModel::logits, with the single-row kernels forward_any draws with -- finish_argmax, the choice's sampler against an empty state at draw
// index 0, its record -- so each choice yields exactly what batch_add yields for the request with its seed.  Nothing between two draws
// writes logits, pmax or pidx (the sampler works in sample_work, the records in their own partials).  After the call every choice is an
// ordinary slot that owns its pages.
void session_add_n(aha_model* m, const aha_batch_request& req, size_t n, const uint64_t* seeds, int32_t* slots_out, uint32_t* first_tokens,
                   int32_t* finished, aha_usage* usage) {
    TextModel& T = m->text;
    BatchDecoder& B = m->sess();
    Ctx& c = m->ctx;
    const std::string who = "batch_add_n: ";
    // ---- every check before any device work: a refused call leaves the session untouched
    open_session(m);
    AHA_REQUIRE(n >= 1, who + "n must be at least 1");
    Admission ad{m, free_slots(m, n, (int)n, who, true)};
    ad.a.push_back(admit_check(m, req, who, -1));
    const AdmitReq& q = ad.a[0];   // choice 0's table starts with its hit pages
    require_ctx(m, q.ctx, "context of ");
    const size_t pages = q.pages(n);
    ad.check_room(pages, who + std::to_string(n) + " choices need ");
    std::vector<aha_batch_request> r(n, req);
    std::vector<Sampler> samp(n);
    for (size_t i = 0; i < n; ++i) {
        r[i].params.seed = seeds ? seeds[i] : req.params.seed + i;
        samp[i] = request_sampler(m, r[i].params, who);
    }
    ad.take(pages);
    const auto t0 = clk::now();
    const std::vector<int>& slot = ad.slots;
    std::vector<uint32_t> tok(n);
    tok[0] = batch_prefill_slot(m, slot[0], r[0], q.budget, q.lp_n, q.hit());
    if (n > 1) {
        const std::vector<int> dst(slot.begin() + 1, slot.end());
        for (int s : dst) T.pages.map(B.slots[s].table, (int)q.ctx);
        B.fork(slot[0], dst, (int)req.seq_len);
        const DecodeState empty{0, 0, 0, 0, 0, samp[0].fsm_start, {0, 0}};   // first_token's state: empty history, draw index 0, start state
        for (size_t i = 1; i < n; ++i) {
            const int s = slot[i];
            T.set_sampler(samp[i]);
            AHA_CUDA_CHECK(cudaMemcpyAsync(T.d_state, &empty, sizeof(empty), cudaMemcpyHostToDevice, c.stream));
            T.finish_argmax(0);
            T.sample(0);
            if (q.lp_n >= 0) T.logprobs(true, B.d_lp_rec + s, false);
            // the draw's token and draw count, collected in the slot's own rows and read back once below
            AHA_CUDA_CHECK(cudaMemcpyAsync(B.d_tok + s, T.d_argmax, sizeof(uint32_t), cudaMemcpyDeviceToDevice, c.stream));
            AHA_CUDA_CHECK(cudaMemcpyAsync(B.d_states + s, T.d_state, sizeof(DecodeState), cudaMemcpyDeviceToDevice, c.stream));
            B.slots[s].lp = q.lp_n + 1;
            B.bind_sampler(s, samp[i]);
        }
        std::vector<uint32_t> h_tok;
        std::vector<DecodeState> h_st;
        read_first_tokens(m, h_tok, h_st);
        for (size_t i = 1; i < n; ++i) {
            tok[i] = h_tok[slot[i]];
            B.adopt(slot[i], tok[i], (int)req.seq_len, decode_rope_delta(m), h_st[slot[i]].n_draws, h_st[slot[i]].fsm_state);
        }
    }
    const double secs = seconds(clk::now() - t0), vision = m->last_vision_secs;
    ad.commit(tok, std::vector<double>(n, secs), std::vector<double>(n, vision), slots_out, first_tokens, finished, usage);
}

// One speculative request into the lowest free slot of the open wide session (aha_b200_batch_add_speculative): admitted as batch_add admits it
// (prefilled alone on the slot's table, prefix-cache hit and insert included), with pages for max_draft more positions, and from then on
// stepped in verify passes of R = max_draft + 1 rows by session_step_core.  Its control block is the slot's; drafts come from the slot's
// copy of the prediction and prompt.
void session_add_spec(aha_model* m, const aha_batch_request& req, const aha_spec_params& sp, int32_t* slot_out, uint32_t* first_token,
                      int32_t* finished, aha_usage* usage) {
    TextModel& T = m->text;
    const std::string who = "batch_add_speculative: ";
    // ---- every check before any device work: a refused call leaves the session untouched
    open_session(m);
    AHA_REQUIRE(m->session.wide, who + "speculative requests need a wide session (aha_b200_batch_open_wide): a narrow session promises the ids of "
                                       "single-request runs, which verify passes cannot keep");
    const int ngram = spec_request_check(m, req.params, sp, who);
    AHA_REQUIRE(!session_has_lora(m), who + "a LoRA request is running: speculative requests and adapters do not share a session");
    const int R = (int)sp.max_draft + 1;
    Admission ad{m, free_slots(m, 1, R, who)};
    ad.a.push_back(admit_check(m, req, who, -1, sp.max_draft));   // (spec_request_check refused its flags and rules already)
    const AdmitReq& q = ad.a[0];
    require_ctx(m, q.ctx, who + "prompt + max_tokens + max_draft = ");
    ad.check_room(q.pages(), who + "the request needs ");
    const Sampler samp = request_sampler(m, req.params, who);
    SpecDecoder& S = m->spec;
    BatchDecoder& B = m->sess();
    ad.take(q.pages());
    const auto t0 = clk::now();
    const int slot = ad.slots[0];
    S.init(T, B, kWideSeqs);
    const uint32_t tok = batch_prefill_slot(m, slot, req, q.budget, q.lp_n, q.hit());
    T.pages.map(B.slots[slot].table, (int)q.ctx);   // the positions of the last pass's drafts
    if (q.budget > 1) {
        const std::vector<uint32_t> pred(sp.prediction, sp.prediction + sp.n_prediction);
        const bool lookup = (sp.flags & AHA_SPEC_PROMPT_LOOKUP) != 0;
        const int lp_on = q.lp_n >= 0 ? q.lp_n + 1 : 0;
        S.set_ctl(slot, samp, pred, req.ids, lookup ? req.seq_len : 0, m->stop_ids, (int)q.budget, ngram, lp_on, B.d_states + slot,
                  B.d_hist + (size_t)slot * T.hist_cap, S.d_slot_lp + (size_t)slot * kSpecMaxRows, 0, lp_on ? B.d_lp_rec + slot : nullptr);
    }
    const double secs = seconds(clk::now() - t0), vision = m->last_vision_secs;
    ad.commit({tok}, {secs}, {vision}, slot_out, first_token, finished, usage);
    if (!*finished) { slot_req(m, slot).spec = true; slot_req(m, slot).R = R; }
}

// One step of every running request, the core of batch_step, batch_step_n and batch_step_spec: a decode step of the plain slots
// (BatchDecoder::step) or, beside a speculative request, one mixed launch (SpecDecoder::step) -- a decode step of the plain slots and a
// verify pass of every speculative slot.  Slot s delivers its tokens into tokens[s * stride ..] (stride kSpecMaxRows once a speculative
// request runs) and their count into n_tokens[s] when given; status[s] = 1 running, 2 finished.  The caller zeroes the outputs.  Finished
// slots are released.  -> the requests stepped
size_t session_step_core(aha_model* m, uint32_t* tokens, size_t stride, uint32_t* n_tokens, int32_t* status) {
    BatchDecoder& B = m->sess();
    Ctx& c = m->ctx;
    std::vector<int> plain, spec;
    for (int i = 0; i < m->session.width; ++i) if (slot_req(m, i).used) (slot_req(m, i).spec ? spec : plain).push_back(i);
    if (plain.empty() && spec.empty()) return 0;
    if (spec.empty()) B.step(plain);
    else m->spec.step(plain, spec);
    std::vector<uint32_t> h_tok((size_t)B.cap);
    std::vector<DecodeState> h_st(spec.empty() ? 0 : (size_t)B.cap);
    std::vector<SpecCtl> h_ctl(spec.empty() ? 0 : (size_t)kWideSeqs);
    AHA_CUDA_CHECK(cudaMemcpyAsync(h_tok.data(), B.d_tok, h_tok.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, c.stream));
    if (!spec.empty()) {
        AHA_CUDA_CHECK(cudaMemcpyAsync(h_st.data(), B.d_states, h_st.size() * sizeof(DecodeState), cudaMemcpyDeviceToHost, c.stream));
        AHA_CUDA_CHECK(cudaMemcpyAsync(h_ctl.data(), m->spec.d_ctl, h_ctl.size() * sizeof(SpecCtl), cudaMemcpyDeviceToHost, c.stream));
    }
    AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
    if (!spec.empty()) {
        for (int s : spec) {   // the tokens the pass emitted: history [produced, n_hist)
            const size_t E0 = slot_req(m, s).produced, n = (size_t)h_st[s].n_hist - E0;
            AHA_REQUIRE(n >= 1 && n <= (size_t)kSpecMaxRows, "batch_step_spec: a verify pass emitted no token");
            AHA_CUDA_CHECK(cudaMemcpyAsync(tokens + (size_t)s * stride, B.d_hist + (size_t)s * m->text.hist_cap + E0, n * sizeof(uint32_t),
                                           cudaMemcpyDeviceToHost, c.stream));
        }
        AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
    }
    // a request whose sampler failed (all-zero weights) poisons only the check below; the session is closed by the caller's error path
    for (int s : plain) {
        SlotRequest& r = slot_req(m, s);
        const uint32_t t = h_tok[s];
        tokens[(size_t)s * stride] = t;
        if (n_tokens) n_tokens[s] = 1;
        r.produced += 1;
        r.lp_valid = B.slots[s].lp > 0;
        r.last_n = 0;
        bool stop = r.produced >= r.budget;
        for (uint32_t e : m->stop_ids) if (e == t) stop = true;     // an EOS token is delivered, then the request ends (generate.rs:139-141)
        status[s] = stop ? 2 : 1;
    }
    for (int s : spec) {
        SlotRequest& r = slot_req(m, s);
        const SpecCtl& k = h_ctl[s];
        const size_t n = (size_t)h_st[s].n_hist - r.produced;
        n_tokens[s] = (uint32_t)n;
        r.produced += n;
        r.last_n = (int)n;
        r.lp_valid = B.slots[s].lp > 0;
        r.spec_stats = aha_spec_stats{k.passes, k.drafted, k.accepted, 0};
        status[s] = k.done ? 2 : 1;   // (the accept kernel applies EOS and max_tokens)
    }
    for (int i = 0; i < m->session.width; ++i) if (status[i] == 2) session_release(m, i);
    // sampler errors surface after the bookkeeping so that the slots stay consistent
    m->text.check_sample_error();
    return plain.size() + spec.size();
}
// batch_step / batch_step_n: tokens_out / status_out: [cap] entries, cap >= the session width (8 for batch_step)
size_t session_step(aha_model* m, uint32_t* tokens_out, int32_t* status_out, size_t cap, bool step8) {
    const int width = open_session(m).width;
    if (step8)
        AHA_REQUIRE(width <= kGemvBatchMax, "batch_step: tokens_out[8] cannot hold a session of " + std::to_string(width) + " slots: use aha_b200_batch_step_n");
    AHA_REQUIRE(cap >= (size_t)width, "batch_step_n: cap " + std::to_string(cap) + " is smaller than the session width " + std::to_string(width));
    for (size_t i = 0; i < cap; ++i) { status_out[i] = 0; tokens_out[i] = 0; }
    AHA_REQUIRE(!session_has_spec(m), std::string(step8 ? "batch_step" : "batch_step_n") +
                                          ": a speculative request is running: step the session with aha_b200_batch_step_spec");
    return session_step_core(m, tokens_out, 1, nullptr, status_out);
}
// batch_step_spec: tokens_out [cap][kSpecMaxRows], n_tokens / status [cap]
size_t session_step_spec(aha_model* m, uint32_t* tokens_out, uint32_t* n_tokens, int32_t* status_out, size_t cap) {
    const int width = open_session(m).width;
    AHA_REQUIRE(cap >= (size_t)width, "batch_step_spec: cap " + std::to_string(cap) + " is smaller than the session width " + std::to_string(width));
    for (size_t i = 0; i < cap * kSpecMaxRows; ++i) tokens_out[i] = 0;
    for (size_t i = 0; i < cap; ++i) { n_tokens[i] = 0; status_out[i] = 0; }
    return session_step_core(m, tokens_out, kSpecMaxRows, n_tokens, status_out);
}

// Per slot of the open session, `rows` records of the tokens its request delivered last (zero records elsewhere): rows 1 (batch_logprobs)
// the record of its last token, rows kSpecMaxRows (batch_logprobs_spec) one per token its last speculative pass delivered.
std::vector<aha_logprobs> session_records(aha_model* m, int rows) {
    const int width = m->session.width;
    BatchDecoder& B = m->sess();
    std::vector<aha_logprobs> last((size_t)width), pass, out((size_t)width * rows);
    if (B.d_lp_rec) AHA_CUDA_CHECK(cudaMemcpyAsync(last.data(), B.d_lp_rec, last.size() * sizeof(aha_logprobs), cudaMemcpyDeviceToHost, m->ctx.stream));
    if (rows > 1 && m->spec.d_slot_lp) {
        pass.resize((size_t)width * kSpecMaxRows);
        AHA_CUDA_CHECK(cudaMemcpyAsync(pass.data(), m->spec.d_slot_lp, pass.size() * sizeof(aha_logprobs), cudaMemcpyDeviceToHost, m->ctx.stream));
    }
    AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
    for (int i = 0; i < width; ++i) {
        const SlotRequest& r = slot_req(m, i);
        if (!r.lp_valid) continue;
        const int n = rows > 1 ? r.last_n : 0;
        if (n == 0) out[(size_t)i * rows] = last[i];
        else for (int k = 0; k < n; ++k) out[(size_t)i * rows + k] = pass[(size_t)i * kSpecMaxRows + k];
    }
    return out;
}

// A narrow session run to completion, the driver of generate_batch and generate_n: admit(slot, first, finished) admits the n requests (or
// choices) into a fresh session, then it steps until every one has finished.  Request i's tokens go to out_tokens[i * cap ..] and, when
// out_lp is given, their records to out_lp[i * cap ..]; its usage gets its completion time and token count.  Whatever happens, the handle
// is left as after clear_cache().
void narrow_session_run(aha_model* m, size_t n, uint32_t* out_tokens, aha_logprobs* out_lp, size_t cap, size_t* n_out, aha_usage* usage,
                        const std::function<void(int32_t* slot, uint32_t* first, int32_t* finished)>& admit) {
    session_open(m, 0);
    struct Close {
        aha_model* m;
        ~Close() { session_close(m); }
    } close{m};
    std::vector<int32_t> slot(n), fin(n);
    std::vector<uint32_t> first(n);
    admit(slot.data(), first.data(), fin.data());
    std::vector<aha_logprobs> rec;
    auto take = [&](size_t i, int s, uint32_t t) {
        out_tokens[i * cap + n_out[i]] = t;
        if (out_lp) out_lp[i * cap + n_out[i]] = rec[s];
        ++n_out[i];
    };
    if (out_lp) rec = session_records(m, 1);
    std::vector<int> req_of(kGemvBatchMax, -1);   // slot -> request
    for (size_t i = 0; i < n; ++i) {
        take(i, slot[i], first[i]);
        if (!fin[i]) req_of[slot[i]] = (int)i;
    }
    const auto t_dec = clk::now();
    uint32_t tok[kGemvBatchMax];
    int32_t status[kGemvBatchMax];
    while (session_step(m, tok, status, kGemvBatchMax, true) > 0) {
        if (out_lp) rec = session_records(m, 1);
        for (int s = 0; s < kGemvBatchMax; ++s) {
            if (!status[s]) continue;
            const int i = req_of[s];
            take((size_t)i, s, tok[s]);
            if (status[s] == 2 && usage) usage[i].completion_secs = seconds(clk::now() - t_dec);
        }
    }
    if (usage) for (size_t i = 0; i < n; ++i) usage[i].completion_tokens = (uint32_t)n_out[i];
}

// Static batching: a narrow session that admits the n requests one by one (each prefilled alone on its own page table) and steps until all
// have finished.  Every request follows generate_generic's rules on its own (first token never EOS-checked, an EOS token is pushed and ends
// THAT request, its own sampler / seed / repeat-penalty history) and so yields exactly the tokens aha_b200_generate would yield for it alone.
void generate_batch_impl(aha_model* m, const aha_batch_request* reqs, size_t n, uint32_t* out_tokens, size_t cap, size_t* n_out, aha_usage* usage) {
    TextModel& T = m->text;
    require_no_session(m);
    AHA_REQUIRE(n >= 1 && n <= (size_t)kGemvBatchMax, "generate_batch: 1 to 8 requests");
    size_t pages = 0;
    for (size_t i = 0; i < n; ++i) {
        AHA_REQUIRE(reqs[i].ids && reqs[i].seq_len >= 1, "generate_batch: every request needs input_ids");
        const size_t sample_len = token_budget(reqs[i].params);
        AHA_REQUIRE(cap >= sample_len, "out_tokens capacity (per request) is smaller than max_tokens");
        AHA_REQUIRE((reqs[i].params.flags & (AHA_GEN_CONTINUE_RNG | AHA_GEN_REUSE_PREFIX)) == 0, "generate_batch: CONTINUE_RNG / REUSE_PREFIX are per-handle states of the single-request calls");
        refuse_logprobs(reqs[i].params, "generate_batch", "a batch session (aha_b200_batch_open, aha_b200_batch_logprobs)");
        pages += (reqs[i].seq_len + sample_len + kPage - 1) / kPage;
        n_out[i] = 0;
    }
    AHA_REQUIRE(pages <= (size_t)T.num_pages, "the requests of the batch need " + std::to_string(pages * kPage) + " tokens of KV capacity, max_ctx is " + std::to_string(T.max_ctx));
    narrow_session_run(m, n, out_tokens, nullptr, cap, n_out, usage, [&](int32_t* slot, uint32_t* first, int32_t* fin) {
        for (size_t i = 0; i < n; ++i) session_add_many(m, reqs + i, 1, slot + i, first + i, fin + i, usage ? usage + i : nullptr, false);
    });
}

// n choices of one request (OpenAI `n`, 1..8): a narrow session, one batch_add_n, steps until every choice has finished.  Choice i yields
// exactly what aha_b200_generate yields for the request with its seed, and with AHA_GEN_LOGPROBS the records generate_logprobs yields.
void generate_n_impl(aha_model* m, const uint32_t* ids, size_t seq_len, const aha_mm* mm, const aha_gen_params& params, size_t n,
                     const uint64_t* seeds, uint32_t* out_tokens, aha_logprobs* out_lp, size_t cap, size_t* n_out, aha_usage* usage) {
    TextModel& T = m->text;
    const std::string who = "generate_n: ";
    require_no_session(m);
    AHA_REQUIRE(n >= 1 && n <= (size_t)kGemvBatchMax, who + "n must be 1 to 8 (more choices: batch_add_n on a wide session)");
    AHA_REQUIRE(cap >= token_budget(params), who + "out_tokens capacity (per choice) is smaller than max_tokens");
    const bool lp = logprob_request(params, T, who) >= 0;
    AHA_REQUIRE(!lp || out_lp, who + "AHA_GEN_LOGPROBS needs out_logprobs");
    for (size_t i = 0; i < n; ++i) n_out[i] = 0;
    const aha_batch_request req{ids, seq_len, mm, params};
    narrow_session_run(m, n, out_tokens, lp ? out_lp : nullptr, cap, n_out, usage, [&](int32_t* slot, uint32_t* first, int32_t* fin) {
        session_add_n(m, req, n, seeds, slot, first, fin, usage);
    });
}
}  // namespace

int aha_b200_batch_open(aha_model* m) { return guarded(m, [&] { session_open(m, 0); }); }

int aha_b200_batch_open_wide(aha_model* m, size_t max_seqs) {
    return guarded(m, [&] {
        AHA_REQUIRE(max_seqs >= 1 && max_seqs <= (size_t)kWideSeqs, "batch_open_wide: max_seqs must be 1 to 64");
        session_open(m, (int)max_seqs);
    });
}

int aha_b200_batch_add(aha_model* m, const aha_batch_request* req, int32_t* slot_out, uint32_t* first_token_out, int32_t* finished_out, aha_usage* usage) {
    return guarded(m, [&] {
        AHA_REQUIRE(req && slot_out && first_token_out && finished_out, "req, slot_out, first_token_out and finished_out are required");
        session_add_many(m, req, 1, slot_out, first_token_out, finished_out, usage, false);
    });
}

int aha_b200_batch_add_many(aha_model* m, const aha_batch_request* reqs, size_t n, int32_t* slots_out, uint32_t* first_tokens_out,
                            int32_t* finished_out, aha_usage* usage) {
    return guarded(m, [&] {
        AHA_REQUIRE(reqs && slots_out && first_tokens_out && finished_out, "reqs, slots_out, first_tokens_out and finished_out are required");
        session_add_many(m, reqs, n, slots_out, first_tokens_out, finished_out, usage, true);
    });
}

int aha_b200_batch_add_n(aha_model* m, const aha_batch_request* req, size_t n, const uint64_t* seeds, int32_t* slots_out, uint32_t* first_tokens_out,
                         int32_t* finished_out, aha_usage* usage) {
    return guarded(m, [&] {
        AHA_REQUIRE(req && slots_out && first_tokens_out && finished_out, "req, slots_out, first_tokens_out and finished_out are required");
        session_add_n(m, *req, n, seeds, slots_out, first_tokens_out, finished_out, usage);
    });
}

int aha_b200_generate_n(aha_model* m, const uint32_t* ids, size_t seq_len, const aha_mm* mm, const aha_gen_params* params, size_t n,
                        const uint64_t* seeds, uint32_t* out_tokens, aha_logprobs* out_logprobs, size_t cap, size_t* n_out, aha_usage* usage) {
    return guarded(m, [&] {
        AHA_REQUIRE(params && out_tokens && n_out, "params, out_tokens and n_out are required");
        generate_n_impl(m, ids, seq_len, mm, *params, n, seeds, out_tokens, out_logprobs, cap, n_out, usage);
    });
}

int aha_b200_batch_step(aha_model* m, uint32_t* tokens_out, int32_t* status_out, size_t* n_stepped_out) {
    return guarded(m, [&] {
        AHA_REQUIRE(tokens_out && status_out, "tokens_out[8] and status_out[8] are required");
        const size_t n = session_step(m, tokens_out, status_out, kGemvBatchMax, true);
        if (n_stepped_out) *n_stepped_out = n;
    });
}

int aha_b200_batch_step_n(aha_model* m, uint32_t* tokens_out, int32_t* status_out, size_t cap, size_t* n_stepped_out) {
    return guarded(m, [&] {
        AHA_REQUIRE(tokens_out && status_out, "tokens_out[cap] and status_out[cap] are required");
        const size_t n = session_step(m, tokens_out, status_out, cap, false);
        if (n_stepped_out) *n_stepped_out = n;
    });
}

int aha_b200_batch_logprobs(aha_model* m, aha_logprobs* out, size_t cap) {
    return guarded(m, [&] {
        const int width = open_session(m).width;
        AHA_REQUIRE(out, "batch_logprobs: out[cap] is required");
        AHA_REQUIRE(cap >= (size_t)width, "batch_logprobs: cap " + std::to_string(cap) + " is smaller than the session width " + std::to_string(width));
        const std::vector<aha_logprobs> h = session_records(m, 1);
        for (size_t i = 0; i < cap; ++i) out[i] = i < (size_t)width ? h[i] : aha_logprobs{};
    });
}

int aha_b200_batch_add_speculative(aha_model* m, const aha_batch_request* req, const aha_spec_params* spec, int32_t* slot_out,
                                   uint32_t* first_token_out, int32_t* finished_out, aha_usage* usage) {
    return guarded(m, [&] {
        AHA_REQUIRE(req && spec && slot_out && first_token_out && finished_out, "req, spec, slot_out, first_token_out and finished_out are required");
        session_add_spec(m, *req, *spec, slot_out, first_token_out, finished_out, usage);
    });
}

int aha_b200_batch_step_spec(aha_model* m, uint32_t* tokens_out, uint32_t* n_tokens_out, int32_t* status_out, size_t cap, size_t* n_stepped_out) {
    return guarded(m, [&] {
        AHA_REQUIRE(tokens_out && n_tokens_out && status_out, "tokens_out[cap][16], n_tokens_out[cap] and status_out[cap] are required");
        const size_t n = session_step_spec(m, tokens_out, n_tokens_out, status_out, cap);
        if (n_stepped_out) *n_stepped_out = n;
    });
}

int aha_b200_batch_logprobs_spec(aha_model* m, aha_logprobs* out, size_t cap) {
    return guarded(m, [&] {
        const int width = open_session(m).width;
        AHA_REQUIRE(out, "batch_logprobs_spec: out[cap][16] is required");
        AHA_REQUIRE(cap >= (size_t)width, "batch_logprobs_spec: cap " + std::to_string(cap) + " is smaller than the session width " + std::to_string(width));
        const std::vector<aha_logprobs> h = session_records(m, kSpecMaxRows);
        for (size_t i = 0; i < cap * kSpecMaxRows; ++i) out[i] = i < h.size() ? h[i] : aha_logprobs{};
    });
}

int aha_b200_batch_spec_stats(aha_model* m, aha_spec_stats* out, size_t cap) {
    return guarded(m, [&] {
        const int width = open_session(m).width;
        AHA_REQUIRE(out, "batch_spec_stats: out[cap] is required");
        AHA_REQUIRE(cap >= (size_t)width, "batch_spec_stats: cap " + std::to_string(cap) + " is smaller than the session width " + std::to_string(width));
        for (size_t i = 0; i < cap; ++i) out[i] = i < (size_t)width ? slot_req(m, (int)i).spec_stats : aha_spec_stats{};
    });
}

int aha_b200_batch_prefix_cache(aha_model* m, size_t max_tokens) {
    return guarded(m, [&] {
        PrefixIndex& X = open_session(m).prefix;
        TextModel& T = m->text;
        X.max_pages = max_tokens / kPage;
        if (!X.on()) { X.clear(T.pages); return; }
        while (X.blocks.size() > X.max_pages && X.evict_one(T.pages, {})) {}
    });
}

int aha_b200_batch_prefix_stats(aha_model* m, aha_prefix_stats* out, size_t* hits_out, size_t cap) {
    return guarded(m, [&] {
        const int width = open_session(m).width;
        AHA_REQUIRE(out, "batch_prefix_stats: out is required");
        AHA_REQUIRE(!hits_out || cap >= (size_t)width, "batch_prefix_stats: cap " + std::to_string(cap) + " is smaller than the session width " + std::to_string(width));
        const PrefixIndex& X = m->session.prefix;
        *out = aha_prefix_stats{};
        out->cached_pages = X.blocks.size();
        for (const auto& e : X.blocks) out->shared_pages += m->text.pages.refs[e.first] > 1;
        out->hit_tokens = X.hit_tokens; out->lookups = X.lookups; out->evicted_pages = X.evicted; out->max_pages = X.max_pages;
        out->free_pages = m->text.pages.free_count();
        if (hits_out) for (size_t i = 0; i < cap; ++i) hits_out[i] = i < (size_t)width ? slot_req(m, (int)i).hit : 0;
    });
}

int aha_b200_batch_swap_space(aha_model* m, size_t max_tokens) { return guarded(m, [&] { swap_space(m, max_tokens); }); }

int aha_b200_batch_cancel(aha_model* m, int32_t slot) { return guarded(m, [&] { session_cancel(m, slot); }); }

int aha_b200_batch_suspend(aha_model* m, int32_t slot, uint32_t* id_out) {
    return guarded(m, [&] {
        AHA_REQUIRE(id_out, "batch_suspend: id_out is required");
        *id_out = session_suspend(m, slot);
    });
}

int aha_b200_batch_resume(aha_model* m, uint32_t id, int32_t* slot_out) {
    return guarded(m, [&] {
        AHA_REQUIRE(slot_out, "batch_resume: slot_out is required");
        *slot_out = session_resume(m, id);
    });
}

int aha_b200_batch_discard(aha_model* m, uint32_t id) { return guarded(m, [&] { session_discard(m, id); }); }

int aha_b200_batch_swap_stats(aha_model* m, aha_swap_stats* out) {
    return guarded(m, [&] {
        AHA_REQUIRE(out, "batch_swap_stats: out is required");
        const aha_model::SwapArena& A = m->swap;
        *out = aha_swap_stats{};
        out->host_pages = A.pages;
        out->free_host_pages = A.free.size();
        out->suspended = m->suspended.size();
        out->pages_out = A.pages_out;
        out->pages_in = A.pages_in;
        out->bytes_out = A.pages_out * m->swap_page_bytes();
        out->bytes_in = A.pages_in * m->swap_page_bytes();
        out->suspend_secs = A.suspend_secs;
        out->resume_secs = A.resume_secs;
    });
}

int aha_b200_batch_close(aha_model* m) {
    return guarded(m, [&] { AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream)); session_close(m); });
}

int aha_b200_generate_batch(aha_model* m, const aha_batch_request* reqs, size_t n, uint32_t* out_tokens, size_t cap, size_t* n_out, aha_usage* usage) {
    return guarded(m, [&] {
        AHA_REQUIRE(reqs && out_tokens && n_out, "reqs, out_tokens and n_out are required");
        generate_batch_impl(m, reqs, n, out_tokens, cap, n_out, usage);
    });
}

int aha_b200_generate(aha_model* m, const uint32_t* ids, size_t seq_len, const aha_mm* mm, const aha_gen_params* params, uint32_t* out_tokens,
                      size_t cap, size_t* n_out, aha_usage* usage) {
    return guarded(m, [&] {
        AHA_REQUIRE(params && out_tokens && n_out, "params, out_tokens and n_out are required");
        AHA_REQUIRE(cap >= token_budget(*params), "out_tokens capacity is smaller than max_tokens");
        refuse_logprobs(*params, "generate", "aha_b200_generate_logprobs");
        if (usage) *usage = aha_usage{};
        size_t n = 0;
        GenSink sink{[&](uint32_t t, size_t i, const aha_logprobs*) { out_tokens[i] = t; n = i + 1; return false; }};
        generate_impl(m, ids, seq_len, mm, *params, sink, false, usage, nullptr);
        *n_out = n;
    });
}

int aha_b200_generate_speculative(aha_model* m, const uint32_t* ids, size_t seq_len, const aha_mm* mm, const aha_gen_params* params,
                                  const aha_spec_params* spec, uint32_t* out_tokens, aha_logprobs* out_logprobs, size_t cap, size_t* n_out,
                                  aha_usage* usage, aha_spec_stats* stats) {
    return guarded(m, [&] {
        AHA_REQUIRE(params && spec && out_tokens && n_out, "params, spec, out_tokens and n_out are required");
        AHA_REQUIRE(ids && seq_len >= 1, "input_ids must hold at least one token");
        if (usage) *usage = aha_usage{};
        *n_out = 0;
        generate_speculative_impl(m, ids, seq_len, mm, *params, *spec, out_tokens, out_logprobs, cap, n_out, usage, stats);
    });
}

int aha_b200_fsm_check(const aha_token_fsm* fsm, size_t vocab) {
    return guarded_host([&] { fsm_validate(fsm, vocab); });
}

int aha_b200_fsm_create(aha_model* m, const aha_token_fsm* fsm, uint32_t* id_out) {
    return guarded(m, [&] {
        AHA_REQUIRE(id_out, "fsm_create: id_out is required");
        fsm_validate(fsm, (size_t)m->text.cfg.V);
        AHA_REQUIRE(m->next_fsm_id != 0, "fsm_create: the handle has used every automaton id");
        aha_model::Fsm f;
        AHA_CUDA_CHECK(cudaMalloc(&f.mem, fsm_bytes(*fsm)));
        try {
            f.dev = fsm_upload(*fsm, f.mem);
        } catch (...) {
            cudaFree(f.mem);
            throw;
        }
        const uint32_t id = m->next_fsm_id++;
        m->fsms[id] = f;
        *id_out = id;
    });
}

int aha_b200_fsm_destroy(aha_model* m, uint32_t id) {
    return guarded(m, [&] {
        const auto it = m->fsms.find(id);
        AHA_REQUIRE(it != m->fsms.end(), "fsm_destroy: no token automaton has id " + std::to_string(id) + " on this handle");
        for (int i = 0; m->session.open && i < m->session.width; ++i)
            AHA_REQUIRE(!(slot_req(m, i).used && m->sess().slots[i].fsm_id == id),
                        "fsm_destroy: token automaton " + std::to_string(id) + " constrains the running request in slot " + std::to_string(i));
        for (const auto& e : m->suspended)
            AHA_REQUIRE(e.second.sampler.fsm_id != id,
                        "fsm_destroy: token automaton " + std::to_string(id) + " constrains suspended request " + std::to_string(e.first));
        for (const auto& r : m->rules)
            AHA_REQUIRE(r.second.fsm != id, "fsm_destroy: token automaton " + std::to_string(id) + " is named by logit-rules object " +
                                                std::to_string(r.first) + " (destroy that first)");
        AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
        AHA_CUDA_CHECK(cudaFree(it->second.mem));
        m->fsms.erase(it);
    });
}

int aha_b200_rules_check(const aha_logit_rules* r, size_t vocab) {
    return guarded_host([&] { rules_validate(r, vocab); });
}

int aha_b200_rules_create(aha_model* m, const aha_logit_rules* r, uint32_t* id_out) {
    return guarded(m, [&] {
        AHA_REQUIRE(id_out, "rules_create: id_out is required");
        rules_validate(r, (size_t)m->text.cfg.V);
        AHA_REQUIRE(r->fsm == 0 || m->fsms.count(r->fsm), "rules_create: no token automaton has id " + std::to_string(r->fsm) + " on this handle");
        AHA_REQUIRE(m->next_rules_id != 0, "rules_create: the handle has used every logit-rules id");
        aha_model::Rules x;
        x.fsm = r->fsm;
        if (r->n_bias) AHA_CUDA_CHECK(cudaMalloc(&x.mem, r->n_bias * (sizeof(uint32_t) + sizeof(float))));
        try {
            x.dev = rules_upload(*r, x.mem);
        } catch (...) {
            cudaFree(x.mem);
            throw;
        }
        const uint32_t id = m->next_rules_id++;
        m->rules[id] = x;
        *id_out = id;
    });
}

int aha_b200_rules_destroy(aha_model* m, uint32_t id) {
    return guarded(m, [&] {
        const auto it = m->rules.find(id);
        AHA_REQUIRE(it != m->rules.end(), "rules_destroy: no logit-rules object has id " + std::to_string(id) + " on this handle");
        for (int i = 0; m->session.open && i < m->session.width; ++i)
            AHA_REQUIRE(!(slot_req(m, i).used && m->sess().slots[i].rules_id == id),
                        "rules_destroy: logit-rules object " + std::to_string(id) + " applies to the running request in slot " + std::to_string(i));
        for (const auto& e : m->suspended)
            AHA_REQUIRE(e.second.sampler.rules_id != id,
                        "rules_destroy: logit-rules object " + std::to_string(id) + " applies to suspended request " + std::to_string(e.first));
        AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
        if (it->second.mem) AHA_CUDA_CHECK(cudaFree(it->second.mem));
        m->rules.erase(it);
    });
}

}  // extern "C"

namespace {
// One PEFT tensor name of the text stack: [base_model.model.]<prefix>layers.<l>.<self_attn.{q,k,v,o}_proj | mlp.{gate,up,down}_proj>.lora_{A,B}.weight
struct LoraName { int layer = 0, group = 0, sub = 0; bool b = false; };
bool parse_lora_name(const std::string& prefix, std::string n, LoraName& t) {
    const std::string bm = "base_model.model.", lp = prefix + "layers.";
    if (n.compare(0, bm.size(), bm) == 0) n = n.substr(bm.size());
    if (n.compare(0, lp.size(), lp) != 0) return false;
    size_t j = lp.size();
    while (j < n.size() && j - lp.size() < 6 && n[j] >= '0' && n[j] <= '9') ++j;
    if (j == lp.size() || j >= n.size() || n[j] != '.') return false;
    t.layer = std::stoi(n.substr(lp.size(), j - lp.size()));
    const std::string rest = n.substr(j + 1);
    static const struct { const char* name; int g, sub; } kTargets[] = {
        {"self_attn.q_proj", LORA_QKV, 0}, {"self_attn.k_proj", LORA_QKV, 1}, {"self_attn.v_proj", LORA_QKV, 2}, {"self_attn.o_proj", LORA_O, 0},
        {"mlp.gate_proj", LORA_GU, 0}, {"mlp.up_proj", LORA_GU, 1}, {"mlp.down_proj", LORA_DOWN, 0}};
    for (const auto& x : kTargets)
        for (int b = 0; b < 2; ++b)
            if (rest == std::string(x.name) + (b ? ".lora_B.weight" : ".lora_A.weight")) { t.group = x.g; t.sub = x.sub; t.b = b != 0; return true; }
    return false;
}

// Checks every tensor of an adapter (names, pairs, ranks, shapes, dtypes, fp16 range) and stages it as fp16 blocks in the pool layout of
// lora.cuh; nothing touches the device.
LoraAdapter lora_stage(const aha_model* m, const aha_tensor_desc* tensors, size_t n, float scale) {
    const TextModel& T = m->text;
    const TextCfg& cf = T.cfg;
    const std::string who = "lora_create: ";
    AHA_REQUIRE(T.tp_world == 1, who + "LoRA adapters are single-GPU (tp_world > 1 is not supported)");
    AHA_REQUIRE(std::isfinite(scale), who + "scale must be finite");
    AHA_REQUIRE(tensors && n >= 2, who + "an adapter needs at least one lora_A / lora_B pair");
    // (layer, group, sub) -> A, B
    std::map<std::array<int, 3>, std::array<const aha_tensor_desc*, 2>> pairs;
    int r = 0;
    for (size_t i = 0; i < n; ++i) {
        const aha_tensor_desc& d = tensors[i];
        const std::string name = d.name ? d.name : "";
        LoraName t;
        AHA_REQUIRE(parse_lora_name(T.wprefix, name, t), who + "tensor '" + name + "' is not a lora_A / lora_B weight of a q/k/v/o/gate/up/down "
                                                                  "projection of the text stack (DoRA and other PEFT methods are not supported)");
        AHA_REQUIRE(t.layer < cf.L, who + "tensor '" + name + "': the model has " + std::to_string(cf.L) + " layers");
        AHA_REQUIRE(d.dtype == AHA_F16 || d.dtype == AHA_BF16 || d.dtype == AHA_F32, who + "tensor '" + name + "' must be f16, bf16 or f32");
        AHA_REQUIRE(d.data && d.rank == 2, who + "tensor '" + name + "' must be a 2-D matrix");
        auto& slot = pairs[{t.layer, t.group, t.sub}][t.b ? 1 : 0];
        AHA_REQUIRE(!slot, who + "tensor '" + name + "' appears twice");
        slot = &d;
        const int rank = (int)(t.b ? d.shape[1] : d.shape[0]);
        AHA_REQUIRE(r == 0 || rank == r, who + "tensor '" + name + "' has rank " + std::to_string(rank) + ", the adapter's other tensors " + std::to_string(r));
        r = rank;
    }
    AHA_REQUIRE(r >= 1 && r <= kLoraMaxRank, who + "rank " + std::to_string(r) + " is outside 1 .. " + std::to_string(kLoraMaxRank));
    const int H = cf.H, q = T.nh_l * cf.hd, kv = T.nkv_l * cf.hd;
    auto dims = [&](int g, int sub, int& N, int& K) {   // the base projection of a target: out N, in K
        switch (g) {
            case LORA_QKV: N = sub == 0 ? q : kv; K = H; break;
            case LORA_O: N = H; K = q; break;
            case LORA_GU: N = T.I_l; K = H; break;
            default: N = H; K = T.I_l; break;
        }
    };
    std::set<int> subs[kLoraGroups];
    for (const auto& e : pairs) {
        const int g = e.first[1], sub = e.first[2];
        const aha_tensor_desc* A = e.second[0];
        const aha_tensor_desc* B = e.second[1];
        AHA_REQUIRE(A && B, who + "layer " + std::to_string(e.first[0]) + ": a lora_" + (A ? "A" : "B") + " weight without its lora_" + (A ? "B" : "A"));
        int N = 0, K = 0;
        dims(g, sub, N, K);
        AHA_REQUIRE(A->shape[0] == r && A->shape[1] == K, who + "tensor '" + std::string(A->name) + "' must be [" + std::to_string(r) + ", " +
                                                               std::to_string(K) + "] (rank x the projection's input)");
        AHA_REQUIRE(B->shape[0] == N && B->shape[1] == r, who + "tensor '" + std::string(B->name) + "' must be [" + std::to_string(N) + ", " +
                                                               std::to_string(r) + "] (the projection's output x rank)");
        subs[g].insert(sub);
    }
    LoraAdapter ad;
    ad.r = r;
    ad.scale = scale;
    const WeightTable wt(tensors, n);
    for (int g = 0; g < kLoraGroups; ++g) {
        ad.w[g] = ceil_div((int)subs[g].size() * r, kLoraAlign) * kLoraAlign;
        ad.A[g].assign(cf.L, {});
        ad.B[g].assign(cf.L, {});
    }
    for (const auto& e : pairs) {
        const int l = e.first[0], g = e.first[1], sub = e.first[2], w = ad.w[g];
        const int col = (int)std::distance(subs[g].begin(), subs[g].find(sub)) * r;   // the target's sub-block
        int N = 0, K = 0;
        dims(g, sub, N, K);
        const int Kg = T.lora.K[g], Ng = T.lora.N[g];
        std::vector<__half>& a = ad.A[g][l];
        std::vector<__half>& b = ad.B[g][l];
        if (a.empty()) { a.assign((size_t)w * Kg, __float2half_rn(0.f)); b.assign((size_t)Ng * w, __float2half_rn(0.f)); }
        wt.rows_to_half(e.second[0]->name, r, K, 0, r, 0, K, a.data() + (size_t)col * Kg, Kg);
        std::vector<__half> bs((size_t)N * r);
        wt.rows_to_half(e.second[1]->name, N, r, 0, N, 0, r, bs.data(), r);
        for (int i = 0; i < N; ++i) {   // the base row layout: q | k | v stacked, gate / up interleaved
            int row = i;
            if (g == LORA_QKV) row = sub == 0 ? i : (sub == 1 ? q + i : q + kv + i);
            if (g == LORA_GU) row = 2 * i + sub;
            std::copy(bs.begin() + (size_t)i * r, bs.begin() + (size_t)(i + 1) * r, b.begin() + (size_t)row * w + col);
        }
    }
    return ad;
}
}  // namespace

extern "C" {

int aha_b200_lora_create(aha_model* m, const aha_tensor_desc* tensors, size_t n, float scale, uint32_t* id_out) {
    return guarded(m, [&] {
        AHA_REQUIRE(id_out, "lora_create: id_out is required");
        AHA_REQUIRE(m->next_lora_id < (uint32_t)std::numeric_limits<int>::max(), "lora_create: the handle has used every adapter id");
        LoraAdapter ad = lora_stage(m, tensors, n, scale);
        ad.id = m->next_lora_id;
        LoraSet& L = m->text.lora;
        L.ads.push_back(std::move(ad));
        try {
            L.rebuild(m->ctx.stream);
        } catch (...) {
            L.ads.pop_back();
            L.rebuild(m->ctx.stream);
            throw;
        }
        for (BatchDecoder* B : {&m->batch, &m->wide_batch}) B->composition_changed();
        *id_out = m->next_lora_id++;
    });
}

int aha_b200_lora_destroy(aha_model* m, uint32_t id) {
    return guarded(m, [&] {
        LoraSet& L = m->text.lora;
        const int idx = L.index_of(id);
        AHA_REQUIRE(id != 0 && idx >= 0, "lora_destroy: no LoRA adapter has id " + std::to_string(id) + " on this handle");
        for (int i = 0; m->session.open && i < m->session.width; ++i)
            AHA_REQUIRE(!(slot_req(m, i).used && slot_req(m, i).lora == id),
                        "lora_destroy: adapter " + std::to_string(id) + " runs the request in slot " + std::to_string(i));
        for (const auto& e : m->suspended)
            AHA_REQUIRE(e.second.req.lora != id, "lora_destroy: adapter " + std::to_string(id) + " runs suspended request " + std::to_string(e.first));
        if (m->session.open && m->session.prefix.on()) m->session.prefix.drop(m->text.pages, id);
        L.ads.erase(L.ads.begin() + idx);
        L.rebuild(m->ctx.stream);
        for (BatchDecoder* B : {&m->batch, &m->wide_batch}) B->composition_changed();
    });
}

int aha_b200_batch_add_lora(aha_model* m, const aha_batch_request* reqs, const uint32_t* adapters, size_t n, int32_t* slots_out,
                            uint32_t* first_tokens_out, int32_t* finished_out, aha_usage* usage) {
    return guarded(m, [&] {
        const std::string who = "batch_add_lora: ";
        AHA_REQUIRE(reqs && adapters && slots_out && first_tokens_out && finished_out, "reqs, adapters, slots_out, first_tokens_out and finished_out are required");
        open_session(m);
        AHA_REQUIRE(m->session.wide, who + "LoRA requests need a wide session (aha_b200_batch_open_wide): a narrow session promises the ids of "
                                           "single-request runs, and its CUDA-core GEMV has no adapter tail");
        bool any = false;
        for (size_t i = 0; i < n; ++i) {
            AHA_REQUIRE(adapters[i] == 0 || m->text.lora.index_of(adapters[i]) >= 0,
                        who + "request " + std::to_string(i) + ": no LoRA adapter has id " + std::to_string(adapters[i]) + " on this handle");
            any = any || adapters[i] != 0;
        }
        AHA_REQUIRE(!any || !session_has_spec(m), who + "a speculative request is running: speculative requests and adapters do not share a session");
        session_add_many(m, reqs, n, slots_out, first_tokens_out, finished_out, usage, true, adapters);
    });
}

extern "C++" {
namespace {
// Host staging of the debug attention entries: a paged KV pool laid out like the model's ([page][K|V][kv_head][kPage][hd]), filled with NaN,
// into which each sequence's tokens 0 .. ctx - 1 are written through its page table.  Every slot no table references, and every slot past a
// context inside its last page, stays NaN: a kernel that reads pool memory its sequence does not own, even under a mask or with a zero
// probability, returns NaN.
struct HostPool {
    int nkv, hd;
    size_t page_stride;
    std::vector<float> data;
    HostPool(int n_pages, int nkv_, int hd_)
        : nkv(nkv_), hd(hd_), page_stride((size_t)2 * nkv_ * kPage * hd_), data((size_t)n_pages * page_stride, std::numeric_limits<float>::quiet_NaN()) {}
    int pages() const { return (int)(data.size() / page_stride); }
    // k, v: [ctx][nkv][hd]; table: ceil(ctx / kPage) distinct physical pages
    void put(const int* table, int ctx, const float* k, const float* v) {
        for (int p = 0; p < ceil_div(ctx, kPage); ++p)
            AHA_REQUIRE(table[p] >= 0 && table[p] < pages(), "page table entry " + std::to_string(table[p]) + " is outside the pool");
        for (int t = 0; t < ctx; ++t)
            for (int h = 0; h < nkv; ++h) {
                const size_t base = (size_t)table[t / kPage] * page_stride + (size_t)h * kPage * hd + (size_t)(t % kPage) * hd;
                std::memcpy(&data[base], k + ((size_t)t * nkv + h) * hd, hd * sizeof(float));
                std::memcpy(&data[base + (size_t)nkv * kPage * hd], v + ((size_t)t * nkv + h) * hd, hd * sizeof(float));
            }
    }
    // layer view of the device copy `d` through the device page table `d_table`
    KVSrc src(float* d, const int* d_table) const {
        KVSrc s;
        s.k = d; s.v = d + (size_t)nkv * kPage * hd; s.page_table = d_table; s.page_shift = kPageShift;
        s.page_stride = page_stride; s.tok_stride = hd; s.head_stride = (size_t)kPage * hd;
        return s;
    }
};
// copies and fills on the model's stream, ordered with the launches that follow
template <typename T>
T* upload_scratch(Scratch& mem, cudaStream_t st, const T* h, size_t n) {
    T* d = mem.alloc<T>(std::max<size_t>(n, 1));
    if (n) AHA_CUDA_CHECK(cudaMemcpyAsync(d, h, n * sizeof(T), cudaMemcpyHostToDevice, st));
    return d;
}
template <typename T>
void fill_nan(cudaStream_t st, T* d, size_t n) { AHA_CUDA_CHECK(cudaMemsetAsync(d, 0xff, n * sizeof(T), st)); }   // all-ones words: NaN
template <int HD>
void debug_attention_run(Ctx& c, const FlashArgs& fa, int nh, bool causal, const std::vector<std::pair<int, int>>& segs, const int* d_work, int n_work) {
    if (segs.empty()) { flash_dispatch<HD>(c, fa, nh, causal); return; }
    if (causal) {   // a packed prefill (embed_batch, batch_add_many)
        PrefillSegments sg;
        sg.segs = segs; sg.d_work = d_work; sg.n_work = n_work;
        flash_dispatch_segments(c, fa, nh, sg);
        return;
    }
    for (const auto& s : segs) {   // the ViT / audio encoder: one launch per segment, keys and queries both from the segment
        FlashArgs f = fa;
        f.Sq = f.Skv = s.second; f.q0 = f.kv0 = s.first;
        flash_dispatch<HD>(c, f, nh, false);
    }
}
template <int G>
void debug_decode_launch(cudaStream_t st, int B, int nkv, const DecodeAttnArgs& a0, const DecodeAttnArgs* d_table) {
    if (B == 1) decode_attn_kernel<128, G><<<dim3(kDecodeSplits, nkv), 256, 0, st>>>(a0);
    else decode_attn_batch_kernel<128, G><<<dim3(kDecodeSplits, nkv, B), 256, 0, st>>>(d_table);
}
}  // namespace
}  // extern "C++"

extern "C++" {
namespace {
// The verify attention over n requests on host data: request j has R[j] rows at positions pos0[j] .. pos0[j] + R[j] - 1 over its own page
// table `tables[j]` (ceil((pos0[j] + R[j]) / 32) pages of one NaN pool); its K / V are rows [kv_off[j], kv_off[j] + pos0[j] + R[j]) of k / v, its
// q / out rows start at q_off[j].  ctas: grid.x of the attention (every request's chunks are spread over it).
void debug_verify_run(aha_model* m, int n, const int* R, const int* pos0, const int* tables, int n_pool_pages, int nh, int nkv, const float* q,
                      const float* k, const float* v, float* out, int ctas) {
    constexpr int HD = 128;
    Ctx& c = m->ctx;
    AHA_REQUIRE(n >= 1 && n <= kWideSeqs, "debug_verify_attn: 1 to 64 requests");
    AHA_REQUIRE(nkv >= 1 && nh >= nkv && nh % nkv == 0 && nh <= 64, "debug_verify_attn: bad head counts");
    HostPool pool(n_pool_pages, nkv, HD);
    int rows = 0, max_ctx = 0;
    size_t kv_off = 0, t_off = 0;
    std::vector<int> tab_off(n), row0(n);
    for (int j = 0; j < n; ++j) {
        AHA_REQUIRE(R[j] >= 1 && R[j] <= kSpecMaxRows && pos0[j] >= 0, "debug_verify_attn: every request needs 1 to 16 rows at a position >= 0");
        const int ctx = pos0[j] + R[j];
        pool.put(tables + t_off, ctx, k + kv_off * nkv * HD, v + kv_off * nkv * HD);
        tab_off[j] = (int)t_off; row0[j] = rows;
        t_off += ceil_div(ctx, kPage); kv_off += ctx; rows += R[j];
        max_ctx = std::max(max_ctx, ctx);
    }
    AHA_REQUIRE(rows <= kWideSeqs, "debug_verify_attn: at most 64 rows in all");
    std::vector<DecodeState> st(rows);
    for (int j = 0; j < n; ++j) for (int r = 0; r < R[j]; ++r) st[row0[j] + r] = DecodeState{0, pos0[j] + r, 0, 0, 0, 0, {0, 0}};
    const int max_chunks = ceil_div(max_ctx, kSpecChunk);
    Scratch mem;
    float* d_pool = upload_scratch(mem, c.stream, pool.data.data(), pool.data.size());
    float* d_q = upload_scratch(mem, c.stream, q, (size_t)rows * nh * HD);
    float* d_out = mem.alloc<float>((size_t)rows * nh * HD);
    float* d_part = mem.alloc<float>((size_t)rows * nh * max_chunks * spec_part_stride(HD));
    const int* d_tables = upload_scratch(mem, c.stream, tables, t_off);
    std::vector<SpecReq> reqs(n);
    for (int j = 0; j < n; ++j) reqs[j] = SpecReq{nullptr, d_tables + tab_off[j], row0[j], R[j], pos0[j] + R[j]};
    const SpecReq* d_reqs = upload_scratch(mem, c.stream, reqs.data(), reqs.size());
    DecodeState* d_st = upload_scratch(mem, c.stream, st.data(), st.size());
    SpecAttnArgs a{};
    a.q = d_q; a.ldq = nh * HD;
    a.kv = pool.src(d_pool, nullptr);
    a.reqs = d_reqs; a.rows = d_st; a.partial = d_part; a.max_chunks = max_chunks; a.out = d_out; a.ldo = nh * HD;
    a.nh = nh; a.nkv = nkv; a.scaling = (float)(1.0 / std::sqrt((double)HD));
    AHA_CUDA_CHECK(cudaFuncSetAttribute(spec_verify_attn_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)spec_attn_smem_bytes<HD>()));
    spec_verify_attn_kernel<HD><<<dim3(std::max(1, std::min(ctas, max_chunks)), nkv, n), kSpecAttnThreads, spec_attn_smem_bytes<HD>(), c.stream>>>(a);
    spec_verify_merge_kernel<HD><<<dim3(nh, rows), HD, 0, c.stream>>>(a);
    AHA_CUDA_CHECK(cudaGetLastError());
    AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
    AHA_CUDA_CHECK(cudaMemcpy(out, d_out, (size_t)rows * nh * HD * sizeof(float), cudaMemcpyDeviceToHost));
}
}  // namespace
}  // extern "C++"

int aha_b200_debug_kv_swap(aha_model* m, size_t layers, size_t page_floats, size_t n_pool_pages, size_t n_host_pages, size_t n,
                           const int32_t* table_out, const int32_t* table_in, const int32_t* host_pages, const float* pool_in, float* host_out,
                           float* pool_out) {
    return guarded(m, [&] {
        AHA_REQUIRE(table_out && table_in && host_pages && pool_in && host_out && pool_out, "debug_kv_swap: every array is required");
        AHA_REQUIRE(layers >= 1 && page_floats >= 1, "debug_kv_swap: layers and page_floats must be positive");
        AHA_REQUIRE(n >= 1 && n <= n_pool_pages && n <= n_host_pages, "debug_kv_swap: 1 <= n <= the pool's and the arena's pages");
        for (size_t p = 0; p < n; ++p)
            AHA_REQUIRE(table_out[p] >= 0 && (size_t)table_out[p] < n_pool_pages && table_in[p] >= 0 && (size_t)table_in[p] < n_pool_pages &&
                        host_pages[p] >= 0 && (size_t)host_pages[p] < n_host_pages, "debug_kv_swap: page index out of range");
        Ctx& c = m->ctx;
        Scratch sc;
        const size_t pool_n = layers * n_pool_pages * page_floats, host_n = n_host_pages * layers * page_floats;
        float* pool = sc.alloc<float>(pool_n);
        struct Pinned {
            float* p = nullptr;
            ~Pinned() { if (p) cudaFreeHost(p); }
        } arena;
        AHA_CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&arena.p), host_n * sizeof(float), cudaHostAllocPortable));
        std::fill(arena.p, arena.p + host_n, std::numeric_limits<float>::quiet_NaN());
        AHA_CUDA_CHECK(cudaMemcpy(pool, pool_in, pool_n * sizeof(float), cudaMemcpyHostToDevice));
        const size_t layer_stride = n_pool_pages * page_floats;
        kv_swap(c, true, pool, layer_stride, page_floats, (int)layers, table_out, host_pages, arena.p, (int)n);
        AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
        std::memcpy(host_out, arena.p, host_n * sizeof(float));
        kv_swap(c, false, pool, layer_stride, page_floats, (int)layers, table_in, host_pages, arena.p, (int)n);
        AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
        AHA_CUDA_CHECK(cudaMemcpy(pool_out, pool, pool_n * sizeof(float), cudaMemcpyDeviceToHost));
    });
}

int aha_b200_debug_verify_attn(aha_model* m, size_t rows, size_t n_heads, size_t n_kv_heads, size_t pos0, const float* q, const float* k,
                               const float* v, float* out) {
    return guarded(m, [&] {
        AHA_REQUIRE(q && k && v && out, "q, k, v and out are required");
        AHA_REQUIRE(rows >= 1 && rows <= (size_t)kSpecMaxRows, "debug_verify_attn: rows must be 1 to " + std::to_string(kSpecMaxRows));
        AHA_REQUIRE(n_kv_heads >= 1 && n_heads >= n_kv_heads && n_heads % n_kv_heads == 0 && n_heads <= 64, "debug_verify_attn: bad head counts");
        const int R = (int)rows, p0 = (int)pos0;
        // a paged pool with the pages in reverse order and one page no table references
        const int np = ceil_div(p0 + R, kPage);
        std::vector<int> table(np);
        for (int p = 0; p < np; ++p) table[p] = np - p;
        // few CTAs, so that a CTA walks several chunks
        debug_verify_run(m, 1, &R, &p0, table.data(), np + 1, (int)n_heads, (int)n_kv_heads, q, k, v, out, 3);
    });
}

int aha_b200_debug_verify_attn_batch(aha_model* m, size_t n, const int32_t* rows, const int32_t* pos0, const int32_t* tables, size_t n_pool_pages,
                                     size_t n_heads, size_t n_kv_heads, const float* q, const float* k, const float* v, float* out) {
    return guarded(m, [&] {
        AHA_REQUIRE(rows && pos0 && tables && q && k && v && out, "rows, pos0, tables, q, k, v and out are required");
        AHA_REQUIRE(n >= 1 && n <= (size_t)kWideSeqs, "debug_verify_attn_batch: 1 to 64 requests");
        size_t t = 0;
        std::vector<char> seen(n_pool_pages, 0);
        for (size_t j = 0; j < n; ++j) {
            AHA_REQUIRE(rows[j] >= 1 && rows[j] <= kSpecMaxRows && pos0[j] >= 0, "debug_verify_attn_batch: every request needs 1 to 16 rows at a position >= 0");
            for (int p = 0; p < ceil_div(pos0[j] + rows[j], kPage); ++p, ++t) {
                AHA_REQUIRE(tables[t] >= 0 && (size_t)tables[t] < n_pool_pages && !seen[tables[t]], "debug_verify_attn_batch: the tables' pages must be distinct pages of the pool");
                seen[tables[t]] = 1;
            }
        }
        debug_verify_run(m, (int)n, rows, pos0, tables, (int)n_pool_pages, (int)n_heads, (int)n_kv_heads, q, k, v, out, 3);
    });
}

int aha_b200_debug_prefix_attention(aha_model* m, int impl, size_t n_heads, size_t n_kv_heads, const int32_t* segments, size_t n_segments,
                                    const int32_t* page_order, const float* q, const float* k, const float* v, float* out) {
    return guarded(m, [&] {
        AHA_REQUIRE(q && k && v && out && segments && n_segments >= 1, "q, k, v, out and at least one segment are required");
        AHA_REQUIRE(impl >= 0 && impl <= 2, "impl must be 0 (wgmma), 1 (SIMT) or 2 (mma.sync)");
        AHA_REQUIRE(n_kv_heads >= 1 && n_heads % n_kv_heads == 0 && n_heads <= 64, "debug_prefix_attention: bad head counts");
        constexpr int HD = 128;
        Ctx& c = m->ctx;
        const int nh = (int)n_heads, nkv = (int)n_kv_heads;
        // segment j: its queries follow the previous segment's, its keys (prefix, then one per query) follow the previous segment's keys
        PrefillSegments sg;
        std::vector<int> work;
        int Sq = 0, Skv = 0;
        for (size_t j = 0; j < n_segments; ++j) {
            const int pre = segments[2 * j], len = segments[2 * j + 1];
            AHA_REQUIRE(pre >= 0 && len >= 1 && Skv + pre + len <= (1 << 20), "debug_prefix_attention: segments need prefix >= 0 and rows >= 1");
            AHA_REQUIRE(Skv % 16 == 0, "debug_prefix_attention: every segment's keys must start on a multiple of 16 rows");
            sg.segs.emplace_back(Sq, len);
            sg.kv.emplace_back(Skv, pre + len);
            for (int q0 = 0; q0 < len; q0 += kFaBQ) work.insert(work.end(), {Sq, len, Skv, pre + len, q0});   // as plan_pack builds it
            Sq += len;
            Skv += pre + len;
        }
        const int np = ceil_div(Skv, kPage);
        std::vector<int> table(np);
        for (int p = 0; p < np; ++p) table[p] = page_order ? page_order[p] : p;
        std::vector<char> seen(*std::max_element(table.begin(), table.end()) + 1, 0);
        for (int p : table) { AHA_REQUIRE(p >= 0 && !seen[p], "page_order must hold distinct non-negative pages"); seen[p] = 1; }
        HostPool pool((int)seen.size(), nkv, HD);
        pool.put(table.data(), Skv, k, v);
        Scratch mem;
        FlashArgs fa;
        fa.q = upload_scratch(mem, c.stream, q, (size_t)Sq * nh * HD); fa.q_tok_stride = (size_t)nh * HD; fa.q_head_stride = HD;
        fa.kv = pool.src(upload_scratch(mem, c.stream, pool.data.data(), pool.data.size()), upload_scratch(mem, c.stream, table.data(), table.size()));
        const size_t n_out = (size_t)Sq * nh * HD;
        fa.out = mem.alloc<float>(n_out); fa.o_tok_stride = (size_t)nh * HD; fa.o_head_stride = HD;
        fill_nan(c.stream, fa.out, n_out);
        fa.Sq = Sq; fa.Skv = Skv; fa.q0 = 0; fa.kv0 = 0; fa.groups = nh / nkv; fa.scaling = (float)(1.0 / std::sqrt((double)HD));
        sg.d_work = upload_scratch(mem, c.stream, work.data(), work.size());
        sg.n_work = (int)(work.size() / kFaWork);
        const int saved = c.attn_impl;
        c.attn_impl = impl;
        try { flash_dispatch_segments(c, fa, nh, sg); } catch (...) { c.attn_impl = saved; throw; }
        c.attn_impl = saved;
        AHA_CUDA_CHECK(cudaGetLastError());
        AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
        AHA_CUDA_CHECK(cudaMemcpy(out, fa.out, n_out * sizeof(float), cudaMemcpyDeviceToHost));
    });
}

int aha_b200_debug_attention(aha_model* m, int impl, int head_dim, size_t n_heads, size_t n_kv_heads, size_t sq, size_t skv, int causal,
                             const int32_t* segments, size_t n_segments, const int32_t* page_order, int split_out, const float* q, const float* k,
                             const float* v, float* out) {
    return guarded(m, [&] {
        AHA_REQUIRE(q && k && v && out, "q, k, v and out are required");
        AHA_REQUIRE(impl >= 0 && impl <= 2, "impl must be 0 (wgmma), 1 (SIMT) or 2 (mma.sync)");
        AHA_REQUIRE(head_dim == 64 || head_dim == 128, "head_dim must be 64 or 128");
        AHA_REQUIRE(n_kv_heads >= 1 && n_heads % n_kv_heads == 0 && n_heads <= 64, "debug_attention: bad head counts");
        AHA_REQUIRE(sq >= 1 && skv >= 1 && skv <= (1u << 20), "debug_attention: bad lengths");
        AHA_REQUIRE(!causal || skv >= sq, "causal attention needs skv >= sq (skv - sq tokens already cached)");
        AHA_REQUIRE(!split_out || impl == 0, "the split hi / lo output is written by the wgmma kernel only");
        Ctx& c = m->ctx;
        const int hd = head_dim, nh = (int)n_heads, nkv = (int)n_kv_heads, Sq = (int)sq, Skv = (int)skv;
        std::vector<std::pair<int, int>> segs;
        std::vector<int> work;
        if (n_segments) {
            AHA_REQUIRE(segments && Sq == Skv, "segments split one sequence: sq == skv");
            AHA_REQUIRE(!causal || hd == 128, "packed causal segments are head_dim 128");
            int end = 0;
            for (size_t i = 0; i < n_segments; ++i) {
                const int s0 = segments[2 * i], len = segments[2 * i + 1];
                AHA_REQUIRE(s0 >= end && len >= 1 && s0 + len <= Sq, "segments must be non-empty, in order, disjoint and inside [0, sq)");
                segs.emplace_back(s0, len);
                for (int q0 = 0; q0 < len; q0 += kFaBQ) work.insert(work.end(), {s0, len, s0, len, q0});   // as plan_pack builds it
                end = s0 + len;
            }
        }
        Scratch mem;
        FlashArgs fa;
        fa.q = upload_scratch(mem, c.stream, q, (size_t)Sq * nh * hd); fa.q_tok_stride = (size_t)nh * hd; fa.q_head_stride = hd;
        if (causal) {   // the LLM prefill: K / V in a paged pool through the caller's page order
            const int np = ceil_div(Skv, kPage);
            std::vector<int> table(np);
            for (int p = 0; p < np; ++p) table[p] = page_order ? page_order[p] : p;
            std::vector<char> seen(*std::max_element(table.begin(), table.end()) + 1, 0);
            for (int p : table) { AHA_REQUIRE(p >= 0 && !seen[p], "page_order must hold distinct non-negative pages"); seen[p] = 1; }
            HostPool pool((int)seen.size(), nkv, hd);
            pool.put(table.data(), Skv, k, v);
            fa.kv = pool.src(upload_scratch(mem, c.stream, pool.data.data(), pool.data.size()), upload_scratch(mem, c.stream, table.data(), table.size()));
        } else {        // the encoders: contiguous [token][kv_head][hd], followed by a page of NaN tokens
            const size_t n = (size_t)Skv * nkv * hd, pad = (size_t)kPage * nkv * hd;
            float* dk = mem.alloc<float>(n + pad);
            float* dv = mem.alloc<float>(n + pad);
            fill_nan(c.stream, dk + n, pad); fill_nan(c.stream, dv + n, pad);
            AHA_CUDA_CHECK(cudaMemcpyAsync(dk, k, n * sizeof(float), cudaMemcpyHostToDevice, c.stream));
            AHA_CUDA_CHECK(cudaMemcpyAsync(dv, v, n * sizeof(float), cudaMemcpyHostToDevice, c.stream));
            fa.kv.k = dk; fa.kv.v = dv; fa.kv.page_table = nullptr; fa.kv.page_shift = 0; fa.kv.page_stride = 0;
            fa.kv.tok_stride = (size_t)nkv * hd; fa.kv.head_stride = hd;
        }
        const size_t n_out = (size_t)Sq * nh * hd;
        fa.out = mem.alloc<float>(n_out); fa.o_tok_stride = (size_t)nh * hd; fa.o_head_stride = hd;
        fill_nan(c.stream, fa.out, n_out);   // rows no segment covers stay NaN
        if (split_out) {
            fa.out_hi = mem.alloc<__half>(n_out); fa.out_lo = mem.alloc<__half>(n_out);
            fill_nan(c.stream, fa.out_hi, n_out); fill_nan(c.stream, fa.out_lo, n_out);
        }
        fa.Sq = Sq; fa.Skv = Skv; fa.q0 = 0; fa.kv0 = 0; fa.groups = nh / nkv; fa.scaling = (float)(1.0 / std::sqrt((double)hd));
        const int* d_work = upload_scratch(mem, c.stream, work.data(), work.size());
        const int saved = c.attn_impl;
        c.attn_impl = impl;
        try {
            if (hd == 64) debug_attention_run<64>(c, fa, nh, causal != 0, segs, d_work, (int)work.size() / kFaWork);
            else debug_attention_run<128>(c, fa, nh, causal != 0, segs, d_work, (int)work.size() / kFaWork);
        } catch (...) { c.attn_impl = saved; throw; }
        c.attn_impl = saved;
        AHA_CUDA_CHECK(cudaGetLastError());
        AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
        if (!split_out) {
            AHA_CUDA_CHECK(cudaMemcpy(out, fa.out, n_out * sizeof(float), cudaMemcpyDeviceToHost));
            return;
        }
        std::vector<__half> hi(n_out), lo(n_out);
        AHA_CUDA_CHECK(cudaMemcpy(hi.data(), fa.out_hi, n_out * sizeof(__half), cudaMemcpyDeviceToHost));
        AHA_CUDA_CHECK(cudaMemcpy(lo.data(), fa.out_lo, n_out * sizeof(__half), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < n_out; ++i) out[i] = __half2float(hi[i]) + __half2float(lo[i]);   // exact in fp32
    });
}

int aha_b200_debug_decode_attn(aha_model* m, size_t batch, size_t n_heads, size_t n_kv_heads, const float* qkv, const int32_t* pos,
                               const int32_t* rope_delta, const float* k_cache, const float* v_cache, const int32_t* tables, size_t n_pool_pages,
                               const float* q_norm, const float* k_norm, float eps, float rope_theta, float* out, float* out_repeat,
                               float* pool_out) {
    return guarded(m, [&] {
        AHA_REQUIRE(qkv && pos && rope_delta && tables && q_norm && k_norm && out, "qkv, pos, rope_delta, tables, the norm weights and out are required");
        AHA_REQUIRE(batch >= 1 && batch <= 64, "debug_decode_attn: batch must be 1 to 64");
        AHA_REQUIRE(n_kv_heads >= 1 && n_heads % n_kv_heads == 0, "debug_decode_attn: bad head counts");
        const int G = (int)(n_heads / n_kv_heads);
        AHA_REQUIRE(G == 1 || G == 2 || G == 4 || G == 6, "debug_decode_attn: GQA group must be 1, 2, 4 or 6");
        constexpr int HD = 128;
        Ctx& c = m->ctx;
        const int B = (int)batch, nh = (int)n_heads, nkv = (int)n_kv_heads, row = (nh + 2 * nkv) * HD;
        HostPool pool((int)n_pool_pages, nkv, HD);
        std::vector<char> used(n_pool_pages, 0);
        std::vector<int> t_off(B), c_off(B);
        int nt = 0, nc = 0;
        for (int b = 0; b < B; ++b) {
            AHA_REQUIRE(pos[b] >= 0, "debug_decode_attn: negative position");
            t_off[b] = nt; c_off[b] = nc;
            for (int p = 0; p < ceil_div(pos[b] + 1, kPage); ++p) {
                const int pg = tables[nt + p];
                AHA_REQUIRE(pg >= 0 && pg < (int)n_pool_pages && !used[pg], "tables must hold distinct pages of the pool");
                used[pg] = 1;
            }
            AHA_REQUIRE(pos[b] == 0 || (k_cache && v_cache), "k_cache and v_cache are required");
            if (pos[b]) pool.put(tables + nt, pos[b], k_cache + (size_t)nc * nkv * HD, v_cache + (size_t)nc * nkv * HD);
            nt += ceil_div(pos[b] + 1, kPage);
            nc += pos[b];
        }
        Scratch mem;
        float* d_pool = upload_scratch(mem, c.stream, pool.data.data(), pool.data.size());
        const int* d_tables = upload_scratch(mem, c.stream, tables, (size_t)nt);
        const float* d_qkv = upload_scratch(mem, c.stream, qkv, (size_t)B * row);
        const float* d_qw = upload_scratch(mem, c.stream, q_norm, HD);
        const float* d_kw = upload_scratch(mem, c.stream, k_norm, HD);
        const float* d_inv = upload_scratch(mem, c.stream, rope_inv_freq(rope_theta, HD).data(), HD / 2);
        std::vector<DecodeState> st(B);
        for (int b = 0; b < B; ++b) st[b] = DecodeState{0, pos[b], rope_delta[b], 0, 0, 0, {0, 0}};
        const DecodeState* d_st = upload_scratch(mem, c.stream, st.data(), st.size());
        const size_t part = (size_t)nh * kDecodeSplits * (HD + 2), n_out = (size_t)B * nh * HD;
        float* d_part = mem.alloc<float>((size_t)B * part);
        int* d_cnt = mem.alloc<int>((size_t)B * nkv);
        AHA_CUDA_CHECK(cudaMemsetAsync(d_cnt, 0, (size_t)B * nkv * sizeof(int), c.stream));
        float* d_out = mem.alloc<float>(n_out);
        std::vector<DecodeAttnArgs> args(B);
        for (int b = 0; b < B; ++b) {
            DecodeAttnArgs& d = args[b];
            d = DecodeAttnArgs{};
            d.qkv = d_qkv + (size_t)b * row; d.qw = d_qw; d.kw = d_kw; d.eps = eps; d.inv_freq = d_inv; d.st = d_st + b;
            d.kv = pool.src(d_pool, d_tables + t_off[b]);
            d.kbase = d_pool; d.vbase = const_cast<float*>(d.kv.v);
            d.partial = d_part + (size_t)b * part; d.counters = d_cnt + (size_t)b * nkv; d.out = d_out + (size_t)b * nh * HD;
            d.nh = nh; d.nkv = nkv; d.nsplit = kDecodeSplits; d.scaling = (float)(1.0 / std::sqrt((double)HD));
        }
        const DecodeAttnArgs* d_args = upload_scratch(mem, c.stream, args.data(), args.size());
        // Run 1 sees the pool as a decode step does: the new token's slot does not hold its K / V yet.  Run 2 (out_repeat) goes again on the
        // same partials and counters over the pool run 1 left, so a counter run 1 did not reset leaves its output NaN.
        for (int run = 0; run < (out_repeat ? 2 : 1); ++run) {
            fill_nan(c.stream, d_out, n_out);
            switch (G) {
                case 1: debug_decode_launch<1>(c.stream, B, nkv, args[0], d_args); break;
                case 2: debug_decode_launch<2>(c.stream, B, nkv, args[0], d_args); break;
                case 4: debug_decode_launch<4>(c.stream, B, nkv, args[0], d_args); break;
                default: debug_decode_launch<6>(c.stream, B, nkv, args[0], d_args); break;
            }
            AHA_CUDA_CHECK(cudaGetLastError());
            AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
            AHA_CUDA_CHECK(cudaMemcpy(run == 0 ? out : out_repeat, d_out, n_out * sizeof(float), cudaMemcpyDeviceToHost));
        }
        if (pool_out) AHA_CUDA_CHECK(cudaMemcpy(pool_out, d_pool, pool.data.size() * sizeof(float), cudaMemcpyDeviceToHost));
    });
}

int aha_b200_generate_logprobs(aha_model* m, const uint32_t* ids, size_t seq_len, const aha_mm* mm, const aha_gen_params* params,
                               uint32_t* out_tokens, aha_logprobs* out_logprobs, size_t cap, size_t* n_out, aha_usage* usage) {
    return guarded(m, [&] {
        AHA_REQUIRE(params && out_tokens && out_logprobs && n_out, "params, out_tokens, out_logprobs and n_out are required");
        AHA_REQUIRE(cap >= token_budget(*params), "out_tokens capacity is smaller than max_tokens");
        const int lp_n = logprob_request(*params, m->text, "generate_logprobs: ");
        AHA_REQUIRE(lp_n >= 0, "generate_logprobs: params.flags must carry AHA_GEN_LOGPROBS");
        if (usage) *usage = aha_usage{};
        size_t n = 0;
        GenSink sink{[&](uint32_t t, size_t i, const aha_logprobs* lp) { out_tokens[i] = t; out_logprobs[i] = *lp; n = i + 1; return false; }};
        generate_impl(m, ids, seq_len, mm, *params, sink, false, usage, nullptr, lp_n);
        *n_out = n;
    });
}

int aha_b200_generate_stream(aha_model* m, const uint32_t* ids, size_t seq_len, const aha_mm* mm, const aha_gen_params* params,
                             aha_token_callback on_token, void* user, aha_usage* usage) {
    return guarded(m, [&] {
        AHA_REQUIRE(params && on_token, "params and on_token are required");
        refuse_logprobs(*params, "generate_stream", "aha_b200_generate_stream_logprobs");
        if (usage) *usage = aha_usage{};
        GenSink sink{[&](uint32_t t, size_t i, const aha_logprobs*) { return on_token(user, t, (uint32_t)i) != 0; }};
        generate_impl(m, ids, seq_len, mm, *params, sink, true, usage, nullptr);
    });
}

int aha_b200_generate_stream_logprobs(aha_model* m, const uint32_t* ids, size_t seq_len, const aha_mm* mm, const aha_gen_params* params,
                                      aha_logprobs_callback on_token, void* user, aha_usage* usage) {
    return guarded(m, [&] {
        AHA_REQUIRE(params && on_token, "params and on_token are required");
        const int lp_n = logprob_request(*params, m->text, "generate_stream_logprobs: ");
        AHA_REQUIRE(lp_n >= 0, "generate_stream_logprobs: params.flags must carry AHA_GEN_LOGPROBS");
        if (usage) *usage = aha_usage{};
        GenSink sink{[&](uint32_t t, size_t i, const aha_logprobs* lp) { return on_token(user, t, (uint32_t)i, lp) != 0; }};
        generate_impl(m, ids, seq_len, mm, *params, sink, true, usage, nullptr, lp_n);
    });
}

int aha_b200_asr_generate(aha_model* m, const aha_asr_chunk* chunks, size_t n_chunks, const aha_gen_params* params, uint32_t* out_tokens, size_t cap,
                          size_t* n_out, aha_token_callback on_token, void* user, aha_usage* usage) {
    return guarded(m, [&] {
        AHA_REQUIRE(m->kind == aha_model::QWEN3_ASR, "asr_generate needs a qwen3_asr handle");
        AHA_REQUIRE(chunks && n_chunks >= 1 && params && out_tokens && n_out, "chunks, params, out_tokens and n_out are required");
        refuse_logprobs(*params, "asr_generate", "aha_b200_generate_logprobs on each chunk's prompt");
        AHA_REQUIRE((params->flags & AHA_GEN_CONSTRAINED) == 0, "asr_generate: AHA_GEN_CONSTRAINED is not supported on the ASR loop");
        AHA_REQUIRE((params->flags & AHA_GEN_LOGIT_RULES) == 0, "asr_generate: AHA_GEN_LOGIT_RULES is not supported on the ASR loop");
        if (usage) *usage = aha_usage{};
        // Qwen3AsrGenerateModel::generate (qwen3_asr/generate.rs:130-186): ONE LogitsProcessor for the whole request (its RNG
        // stream runs on across the chunks), no repeat penalty, every token -- the first included -- is EOS-checked, the KV
        // cache is cleared after every chunk, the token lists of the chunks are concatenated.
        size_t total = 0;
        for (size_t c = 0; c < n_chunks; ++c) {
            aha_gen_params p = *params;
            p.repeat_penalty = 1.0f;
            p.top_k = 0;                                  // get_logit_processor(Some(temperature), top_p, None, seed)
            p.flags |= AHA_GEN_EOS_ON_FIRST;
            if (c > 0) p.flags |= AHA_GEN_CONTINUE_RNG;
            AHA_REQUIRE(total + token_budget(p) <= cap, "out_tokens capacity is smaller than n_chunks * max_tokens");
            aha_mm mm{&chunks[c].input_features, 1};
            const size_t base = total;
            bool abort = false;
            GenSink sink{[&](uint32_t t, size_t i, const aha_logprobs*) {
                out_tokens[base + i] = t; total = base + i + 1;
                if (on_token && on_token(user, t, (uint32_t)(base + i)) != 0) abort = true;
                return abort;
            }};
            generate_impl(m, chunks[c].ids, chunks[c].seq_len, &mm, p, sink, on_token != nullptr, usage, nullptr);
            if (abort) break;
        }
        *n_out = total;
    });
}

int aha_b200_debug_sample(aha_model* m, int kernel, size_t rows, size_t V, const float* logits, size_t ld, const aha_gen_params* params,
                          const uint32_t* context, const uint32_t* n_context, const uint32_t* draw_index, int overwrite, const int32_t* act,
                          const int32_t* on, uint32_t* token_out, uint32_t* state_out, uint32_t* hist_out) {
    return aha_b200_debug_sample_fsm(m, kernel, rows, V, logits, ld, params, context, n_context, draw_index, overwrite, act, on, nullptr, nullptr,
                                     nullptr, token_out, state_out, hist_out, nullptr);
}

int aha_b200_debug_sample_fsm(aha_model* m, int kernel, size_t rows, size_t V, const float* logits, size_t ld, const aha_gen_params* params,
                              const uint32_t* context, const uint32_t* n_context, const uint32_t* draw_index, int overwrite, const int32_t* act,
                              const int32_t* on, const aha_token_fsm* fsm, const int32_t* constrained, const uint32_t* fsm_state_in,
                              uint32_t* token_out, uint32_t* state_out, uint32_t* hist_out, uint32_t* fsm_state_out) {
    return aha_b200_debug_sample_rules(m, kernel, rows, V, logits, ld, params, context, n_context, draw_index, overwrite, act, on, fsm, constrained,
                                       fsm_state_in, nullptr, nullptr, token_out, state_out, hist_out, fsm_state_out);
}

int aha_b200_debug_sample_rules(aha_model* m, int kernel, size_t rows, size_t V, const float* logits, size_t ld, const aha_gen_params* params,
                                const uint32_t* context, const uint32_t* n_context, const uint32_t* draw_index, int overwrite, const int32_t* act,
                                const int32_t* on, const aha_token_fsm* fsm, const int32_t* constrained, const uint32_t* fsm_state_in,
                                const aha_logit_rules* rules, const int32_t* ruled, uint32_t* token_out, uint32_t* state_out, uint32_t* hist_out,
                                uint32_t* fsm_state_out) {
    return guarded(m, [&] {
        AHA_REQUIRE(logits && params && n_context && draw_index && token_out && state_out && hist_out,
                    "logits, params, n_context, draw_index, token_out, state_out and hist_out are required");
        AHA_REQUIRE(kernel == 0 || kernel == 1, "kernel must be 0 (sample_kernel) or 1 (sample_rows_kernel)");
        AHA_REQUIRE(rows >= 1 && rows <= (size_t)kSampleMaxRows, "rows must be 1 to " + std::to_string(kSampleMaxRows));
        AHA_REQUIRE(V >= 1 && V <= (size_t)kSampleThreads * kSampleChunk, "V must be 1 to " + std::to_string(kSampleThreads * kSampleChunk));
        AHA_REQUIRE(ld == 0 || (ld >= V && ld <= (size_t)INT32_MAX), "ld must be 0 or V to 2^31 - 1");
        AHA_REQUIRE(kernel == 0 || (act && on), "sample_rows_kernel needs act and on");
        // row r runs as slot slot[r]: its own state, history, token and [V] scratch row
        std::vector<int> slot(rows);
        std::vector<char> used(kSampleMaxRows, 0);
        size_t n_ctx_total = 0, cap = 1;
        for (size_t r = 0; r < rows; ++r) {
            slot[r] = kernel == 0 ? (int)r : act[r];
            AHA_REQUIRE(slot[r] >= 0 && slot[r] < kSampleMaxRows && !used[slot[r]], "act must map the rows to distinct slots 0 to 63");
            used[slot[r]] = 1;
            AHA_REQUIRE(!overwrite || n_context[r] >= 1, "overwrite needs a context of at least one token (the pushed ArgMax token)");
            n_ctx_total += n_context[r];
            cap = std::max(cap, (size_t)n_context[r]);
        }
        AHA_REQUIRE(context || n_ctx_total == 0, "context is required");
        AHA_REQUIRE(!fsm || (constrained && fsm_state_in && fsm_state_out), "an automaton needs constrained, fsm_state_in and fsm_state_out");
        if (fsm) fsm_validate(fsm, V);
        for (size_t r = 0; fsm && r < rows; ++r)
            AHA_REQUIRE(!constrained[r] || fsm_state_in[r] < fsm->n_states, "row " + std::to_string(r) + ": fsm_state_in is not below n_states");
        AHA_REQUIRE(!rules || ruled, "logit rules need ruled");
        if (rules) {
            rules_validate(rules, V);
            AHA_REQUIRE(rules->fsm == 0, "the automaton of a debug call is passed as fsm, not named in rules");
        }
        Scratch mem;
        TokenFsmDev dev;
        if (fsm) dev = fsm_upload(*fsm, mem.alloc<char>(fsm_bytes(*fsm)));
        LogitRulesDev rdev;
        if (rules) rdev = rules_upload(*rules, mem.alloc<char>(std::max<size_t>(1, rules->n_bias * (sizeof(uint32_t) + sizeof(float)))));
        int* d_cnt = rules ? mem.alloc<int>(rows * V) : nullptr;       // row r's count row
        std::vector<SampleArgs> args(kSampleMaxRows, SampleArgs{});
        for (size_t r = 0; r < rows; ++r) {
            const Sampler s = make_sampler(params[r], (int)V, fsm && constrained[r] ? &dev : nullptr, rules && ruled[r] ? &rdev : nullptr);
            AHA_REQUIRE(s.active, "row " + std::to_string(r) + ": plain ArgMax needs no sampler (temperature < 1e-7 and no repeat penalty)");
            args[slot[r]] = s.args;
            if (s.counts) args[slot[r]].cnt = d_cnt + r * V;
        }
        cudaStream_t st = m->ctx.stream;
        if (d_cnt) AHA_CUDA_CHECK(cudaMemsetAsync(d_cnt, 0, rows * V * sizeof(int), st));
        const size_t n_logits = ld ? rows * ld : V;
        float* d_logits = mem.alloc<float>(n_logits);
        float* d_work = mem.alloc<float>(rows * V);
        DecodeState* d_st = mem.alloc<DecodeState>(rows);
        uint32_t* d_hist = mem.alloc<uint32_t>(rows * cap);
        uint32_t* d_tok = mem.alloc<uint32_t>(rows);
        int* d_err = mem.alloc<int>(1);
        std::vector<DecodeState> hs(rows);
        std::vector<uint32_t> hh(rows * cap, 0xffffffffu);
        for (size_t r = 0, off = 0; r < rows; off += n_context[r], ++r) {
            const uint32_t n = n_context[r];
            std::copy(context + off, context + off + n, hh.begin() + r * cap);
            hs[r] = DecodeState{n ? context[off + n - 1] : 0u, 0, 0, (int32_t)n, draw_index[r], fsm ? fsm_state_in[r] : 0u, {0, 0}};
            SampleArgs& a = args[slot[r]];
            a.logits = d_logits + r * ld; a.work = d_work + r * V;
            a.st = d_st + r; a.history = d_hist + r * cap; a.hist_cap = (int)cap; a.token_out = d_tok + r; a.error = d_err;
            a.overwrite = overwrite;
        }
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_logits, logits, n_logits * sizeof(float), cudaMemcpyHostToDevice, st));
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_st, hs.data(), rows * sizeof(DecodeState), cudaMemcpyHostToDevice, st));
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_hist, hh.data(), hh.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
        AHA_CUDA_CHECK(cudaMemsetAsync(d_tok, 0xff, rows * sizeof(uint32_t), st));
        AHA_CUDA_CHECK(cudaMemsetAsync(d_err, 0, sizeof(int), st));
        if (kernel == 0) {
            for (size_t r = 0; r < rows; ++r) sample_kernel<<<1, kSampleThreads, 0, st>>>(args[r]);
            m->ctx.cnt.kernels += rows;
        } else {
            SampleArgs* d_args = mem.alloc<SampleArgs>(kSampleMaxRows);
            int* d_on = mem.alloc<int>(kSampleMaxRows);
            int* d_act = mem.alloc<int>(rows);
            AHA_CUDA_CHECK(cudaMemcpyAsync(d_args, args.data(), kSampleMaxRows * sizeof(SampleArgs), cudaMemcpyHostToDevice, st));
            AHA_CUDA_CHECK(cudaMemcpyAsync(d_on, on, kSampleMaxRows * sizeof(int), cudaMemcpyHostToDevice, st));
            AHA_CUDA_CHECK(cudaMemcpyAsync(d_act, slot.data(), rows * sizeof(int), cudaMemcpyHostToDevice, st));
            sample_rows_kernel<<<(unsigned)rows, kSampleThreads, 0, st>>>(d_args, d_on, d_act, d_logits, (int)ld, overwrite);
            m->ctx.cnt.kernels++;
        }
        AHA_CUDA_CHECK(cudaGetLastError());
        int err = 0;
        AHA_CUDA_CHECK(cudaMemcpyAsync(token_out, d_tok, rows * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        AHA_CUDA_CHECK(cudaMemcpyAsync(hs.data(), d_st, rows * sizeof(DecodeState), cudaMemcpyDeviceToHost, st));
        AHA_CUDA_CHECK(cudaMemcpyAsync(hh.data(), d_hist, hh.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        AHA_CUDA_CHECK(cudaMemcpyAsync(&err, d_err, sizeof(int), cudaMemcpyDeviceToHost, st));
        std::vector<int> cnt_after(d_cnt ? rows * V : 0);
        if (d_cnt) AHA_CUDA_CHECK(cudaMemcpyAsync(cnt_after.data(), d_cnt, rows * V * sizeof(int), cudaMemcpyDeviceToHost, st));
        AHA_CUDA_CHECK(cudaStreamSynchronize(st));
        if (err) throw std::runtime_error(kSampleWeightsError);
        for (size_t i = 0; i < cnt_after.size(); ++i)
            AHA_REQUIRE(cnt_after[i] == 0, "row " + std::to_string(i / V) + ": the sampler left count " + std::to_string(cnt_after[i]) + " for token " +
                                               std::to_string(i % V) + " (count rows must be zero after every draw)");
        for (size_t r = 0; r < rows; ++r) {
            state_out[3 * r] = hs[r].token; state_out[3 * r + 1] = (uint32_t)hs[r].n_hist; state_out[3 * r + 2] = hs[r].n_draws;
            hist_out[r] = n_context[r] ? hh[r * cap + n_context[r] - 1] : 0xffffffffu;
            if (fsm) fsm_state_out[r] = hs[r].fsm_state;
        }
    });
}

int aha_b200_debug_logprobs(aha_model* m, const float* logits, size_t V, uint32_t token, uint32_t n_top, aha_logprobs* out) {
    return guarded(m, [&] {
        AHA_REQUIRE(logits && out, "logits and out are required");
        AHA_REQUIRE(V >= 1 && V <= (size_t)kLpMaxParts * kLpSlice, "V must be 1 to " + std::to_string(kLpMaxParts * kLpSlice));
        AHA_REQUIRE(n_top <= AHA_MAX_TOP_LOGPROBS && n_top <= V, "n_top must be at most 20 and at most V");
        AHA_REQUIRE(token < V, "token out of range");
        cudaStream_t st = m->ctx.stream;
        const int P = lp_parts((int)V);
        const int on = 1 + (int)n_top;
        const DecodeState ds{token, 0, 0, 0, 0, 0, {0, 0}};
        // scratch of this call only: [V] logits, the candidate lists, the on flag, the token, a state and the record
        const size_t o_part = V * sizeof(float), o_id = o_part + (size_t)P * kLpPartFloats * sizeof(float), o_on = o_id + (size_t)P * kLpMaxTop * sizeof(int);
        const size_t o_tok = o_on + 16, o_st = o_tok + 16, o_rec = o_st + sizeof(DecodeState), bytes = o_rec + sizeof(aha_logprobs);
        Scratch mem;
        char* b = mem.alloc<char>(bytes);
        AHA_CUDA_CHECK(cudaMemcpyAsync(b, logits, V * sizeof(float), cudaMemcpyHostToDevice, st));
        AHA_CUDA_CHECK(cudaMemcpyAsync(b + o_on, &on, sizeof(int), cudaMemcpyHostToDevice, st));
        AHA_CUDA_CHECK(cudaMemcpyAsync(b + o_tok, &token, sizeof(uint32_t), cudaMemcpyHostToDevice, st));
        AHA_CUDA_CHECK(cudaMemcpyAsync(b + o_st, &ds, sizeof(ds), cudaMemcpyHostToDevice, st));
        logprobs_rows(st, reinterpret_cast<float*>(b), (int)V, (int)V, 1, nullptr, reinterpret_cast<int*>(b + o_on), reinterpret_cast<float*>(b + o_part),
                      reinterpret_cast<int*>(b + o_id), reinterpret_cast<uint32_t*>(b + o_tok), reinterpret_cast<DecodeState*>(b + o_st), 1,
                      reinterpret_cast<aha_logprobs*>(b + o_rec), 0, 1);
        AHA_CUDA_CHECK(cudaGetLastError());
        m->ctx.cnt.kernels += 2;
        AHA_CUDA_CHECK(cudaMemcpyAsync(out, b + o_rec, sizeof(aha_logprobs), cudaMemcpyDeviceToHost, st));
        AHA_CUDA_CHECK(cudaStreamSynchronize(st));
    });
}

int aha_b200_decode_steps(aha_model* m, uint32_t first_token, size_t seqlen_offset, size_t n_steps, uint32_t* out_tokens, double* device_ms) {
    return guarded(m, [&] {
        TextModel& T = m->text;
        AHA_REQUIRE(first_token < (uint32_t)T.cfg.V, "token id out of range");
        AHA_REQUIRE(seqlen_offset + n_steps <= (size_t)T.max_ctx, "context exceeds max_ctx");
        require_no_session(m);
        m->cached_ids.clear();
        T.pages.map(T.table, (int)(seqlen_offset + n_steps));
        T.set_state(first_token, (int)seqlen_offset, decode_rope_delta(m), 0);
        if (n_steps > 0 && T.step_graph.size() == 0 && T.use_graph) {  // build the graph outside the timed region (pos is restored below)
            T.decode_step();
            T.set_state(first_token, (int)seqlen_offset, decode_rope_delta(m), 0);
        }
        const float ms = timed_ms(m, n_steps, [&](size_t) { T.decode_step(); });
        if (out_tokens) AHA_CUDA_CHECK(cudaMemcpy(out_tokens, T.d_history, n_steps * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        T.check_ll_abort();
        if (device_ms) *device_ms = ms;
    });
}

namespace {
void bench_score(aha_model* m, const std::string& w, int iters, double* avg_ms, uint64_t* bytes);   // the score_head timings, defined with scoring

// kernel timing "kv_fork:P:n": P pages of every layer copied from one table row to n - 1 others, over pool pages no sequence holds at the
// time (rows of a scratch table, row r taking pages r * P .. r * P + P - 1); bytes are the algorithmic read + writes, n * P pages
void bench_fork(aha_model* m, const std::string& w, int iters, double* avg_ms, uint64_t* bytes) {
    TextModel& T = m->text;
    int P = 0, n = 0;
    AHA_REQUIRE(std::sscanf(w.c_str(), "kv_fork:%d:%d", &P, &n) == 2 && P >= 1 && n >= 2 && n <= kForkMaxDst + 1,
                "the fork kernel is named kv_fork:P:n with P >= 1 pages and 2 <= n <= 64 choices");
    AHA_REQUIRE((size_t)P * n <= (size_t)T.num_pages, "kv_fork bench: P * n pages exceed the pool (max_ctx / 32 = " + std::to_string(T.num_pages) + ")");
    require_no_session(m);
    drop_cache(m);
    std::vector<int> h((size_t)n * T.num_pages, 0), dst;
    for (int r = 0; r < n; ++r) for (int p = 0; p < P; ++p) h[(size_t)r * T.num_pages + p] = r * P + p;
    for (int r = 1; r < n; ++r) dst.push_back(r);
    Scratch mem;
    int* tables = mem.alloc<int>(h.size());
    AHA_CUDA_CHECK(cudaMemcpy(tables, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice));
    auto launch = [&] { kv_fork(m->ctx, T.kv_pool, T.layer_stride, T.page_stride, T.cfg.L, tables, T.num_pages, 0, dst.data(), n - 1, P); };
    for (int i = 0; i < 3; ++i) launch();
    *avg_ms = timed_ms(m, (size_t)iters, [&](size_t) { launch(); }) / iters;
    *bytes = (uint64_t)n * P * T.cfg.L * T.page_stride * sizeof(float);
}
}  // namespace

int aha_b200_bench_kernel(aha_model* m, const char* which, int iters, double* avg_ms, uint64_t* bytes_per_launch) {
    return guarded(m, [&] {
        AHA_REQUIRE(which && iters > 0 && avg_ms && bytes_per_launch, "which, iters, avg_ms, bytes_per_launch are required");
        TextModel& T = m->text;
        const std::string w = which;
        cudaStream_t st = m->ctx.stream;
        const int L = T.cfg.L;
        if (w.rfind("score_", 0) == 0) { bench_score(m, w, iters, avg_ms, bytes_per_launch); return; }
        if (w.rfind("kv_fork:", 0) == 0) { bench_fork(m, w, iters, avg_ms, bytes_per_launch); return; }
        uint64_t bytes = 0;
        auto launch = [&](int i) {
            TextLayer& Y = T.layers[i % L];
            GemvArgs a{};
            if (w == "gemv_gate_up") { a.W = Y.gu.w; a.x = T.x1; a.norm_w = Y.ln2; a.eps = T.cfg.eps; a.out = T.h1; a.N = Y.gu.N; a.K = Y.gu.K; gemv(st, PRO_RMSNORM, GEPI_SWIGLU, a); bytes = 2ull * a.N * a.K; }
            else if (w == "gemv_qkv") { a.W = Y.qkv.w; a.x = T.x1; a.norm_w = Y.ln1; a.eps = T.cfg.eps; a.out = T.qkv1; a.N = Y.qkv.N; a.K = Y.qkv.K; gemv(st, PRO_RMSNORM, GEPI_STORE, a); bytes = 2ull * a.N * a.K; }
            else if (w == "gemv_down") { a.W = Y.down.w; a.x = T.h1; a.resid = T.x1; a.out = T.x1; a.N = Y.down.N; a.K = Y.down.K; gemv(st, PRO_NONE, GEPI_RESID, a); bytes = 2ull * a.N * a.K; }
            else if (w == "gemv_o") { a.W = Y.o.w; a.x = T.attn1; a.resid = T.x1; a.out = T.x1; a.N = Y.o.N; a.K = Y.o.K; gemv(st, PRO_NONE, GEPI_RESID, a); bytes = 2ull * a.N * a.K; }
            else if (w == "gemv_lm_head") { T.head(T.x1); bytes = 2ull * T.cfg.V * T.cfg.H; }
            else throw std::runtime_error("unknown kernel '" + w + "'");
            m->ctx.cnt.kernels++;
        };
        for (int i = 0; i < 3; ++i) launch(i);
        *avg_ms = timed_ms(m, (size_t)iters, [&](size_t i) { launch((int)i + 3); }) / iters;
        *bytes_per_launch = bytes;
    });
}

int aha_b200_mel_spectrogram(aha_model* m, const float* wave, size_t n_samples, float* mel_out, size_t mel_cap, size_t* n_frames) {
    return guarded(m, [&] {
        AHA_REQUIRE(m->kind == aha_model::QWEN3_ASR, "mel_spectrogram needs a qwen3_asr handle");
        AHA_REQUIRE(wave && mel_out && n_frames, "wave, mel_out and n_frames are required");
        const int frames = m->audio.mel_from_host(wave, n_samples);
        AHA_REQUIRE((size_t)frames * m->audio.cfg.mel <= mel_cap, "mel_out too small");
        AHA_CUDA_CHECK(cudaMemcpyAsync(mel_out, m->audio.d_mel, (size_t)frames * m->audio.cfg.mel * sizeof(float), cudaMemcpyDeviceToHost, m->ctx.stream));
        AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
        *n_frames = (size_t)frames;
    });
}

// u8 HWC -> normalised, frame-duplicated, merge-block-ordered patches.
__global__ void patchify_kernel(const uint8_t* __restrict__ img, int H, int W, int patch, int merge, int tpatch, float* __restrict__ out) {
    const int gw = W / patch, gh = H / patch;
    const int p = blockIdx.x;  // patch in merge-block order (single temporal group)
    const int mw = gw / merge;
    const int blk = p / (merge * merge), in = p % (merge * merge);
    const int row = (blk / mw) * merge + in / merge, col = (blk % mw) * merge + in % merge;
    (void)gh;
    const int feat = 3 * tpatch * patch * patch;
    for (int f = threadIdx.x; f < feat; f += blockDim.x) {
        const int c = f / (tpatch * patch * patch), rem = f % (patch * patch), py = rem / patch, px = rem % patch;
        const uint8_t v = img[((size_t)(row * patch + py) * W + (col * patch + px)) * 3 + c];
        // img_transform: f32(v) * (1/255), (x - 0.5) / 0.5   (img_utils.rs:272-294 with mean = std = 0.5).  Each step rounded on its own
        // (candle runs affine, broadcast_sub and broadcast_div as three kernels; a contracted v * (1/255) - 0.5 differs in the last bit)
        const float x = __fmul_rn((float)v, 1.0f / 255.0f);
        out[(size_t)p * feat + f] = __fdiv_rn(__fsub_rn(x, 0.5f), 0.5f);
    }
}

// process_videos for one video (qwen3vl/processor.rs:253-280 + process_vision_tensor :174-227): T frames u8 (T, H, W, 3) -> rescale, normalise,
// pad the frame count to a multiple of temporal_patch_size by repeating the last frame, merge-block patch order with features (c, frame in group, py, px)
__global__ void video_patchify_kernel(const uint8_t* __restrict__ frames, int T, int H, int W, int patch, int merge, int tpatch, float* __restrict__ out) {
    const int gw = W / patch, gh = H / patch;
    const int per = gh * gw;
    const int gt = blockIdx.x / per, p = blockIdx.x % per;   // temporal group, patch in merge-block order inside it
    const int mw = gw / merge;
    const int blk = p / (merge * merge), in = p % (merge * merge);
    const int row = (blk / mw) * merge + in / merge, col = (blk % mw) * merge + in % merge;
    const int pp = patch * patch, feat = 3 * tpatch * pp;
    for (int f = threadIdx.x; f < feat; f += blockDim.x) {
        const int c = f / (tpatch * pp), tt = (f / pp) % tpatch, rem = f % pp, py = rem / patch, px = rem % patch;
        const int frame = min(gt * tpatch + tt, T - 1);
        const uint8_t v = frames[(((size_t)frame * H + (row * patch + py)) * W + (col * patch + px)) * 3 + c];
        const float x = __fmul_rn((float)v, 1.0f / 255.0f);   // affine, broadcast_sub, broadcast_div: three separately rounded steps
        out[(size_t)blockIdx.x * feat + f] = __fdiv_rn(__fsub_rn(x, 0.5f), 0.5f);
    }
}

int aha_b200_video_preprocess(aha_model* m, const uint8_t* frames_thwc, size_t n_frames, size_t h, size_t w, float* pixel_values_out, size_t cap,
                              uint32_t grid_thw_out[3]) {
    return guarded(m, [&] {
        AHA_REQUIRE(m->kind == aha_model::QWEN3VL, "video_preprocess needs a qwen3vl handle");
        AHA_REQUIRE(frames_thwc && pixel_values_out && grid_thw_out && n_frames > 0 && h > 0 && w > 0, "frames, outputs and positive sizes are required");
        VisionModel& V = m->vision;
        const int ps = V.cfg.patch, mg = V.cfg.merge, tp = V.cfg.tpatch;
        AHA_REQUIRE(h % (ps * mg) == 0 && w % (ps * mg) == 0, "frame size must already be a multiple of patch_size*merge_size (video_smart_resize output)");
        const int gt = ((int)n_frames + tp - 1) / tp, gh = (int)h / ps, gw = (int)w / ps;
        const size_t N = (size_t)gt * gh * gw;
        AHA_REQUIRE(N <= (size_t)V.max_patches, "video needs " + std::to_string(N) + " patches, max_patches is " + std::to_string(V.max_patches));
        AHA_REQUIRE(N * V.patch_dim <= cap, "pixel_values_out too small");
        const size_t bytes = n_frames * h * w * 3;
        Scratch mem;
        uint8_t* d_in = mem.alloc<uint8_t>(bytes);
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_in, frames_thwc, bytes, cudaMemcpyHostToDevice, m->ctx.stream));
        video_patchify_kernel<<<(unsigned)N, 256, 0, m->ctx.stream>>>(d_in, (int)n_frames, (int)h, (int)w, ps, mg, tp, V.pix);
        m->ctx.cnt.kernels++;
        AHA_CUDA_CHECK(cudaMemcpyAsync(pixel_values_out, V.pix, N * V.patch_dim * sizeof(float), cudaMemcpyDeviceToHost, m->ctx.stream));
        AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
        grid_thw_out[0] = (uint32_t)gt; grid_thw_out[1] = (uint32_t)gh; grid_thw_out[2] = (uint32_t)gw;
    });
}

int aha_b200_image_patchify(aha_model* m, const uint8_t* img_hwc, size_t h, size_t w, float* pixel_values_out, size_t cap, uint32_t grid_thw_out[3]) {
    return guarded(m, [&] {
        AHA_REQUIRE(m->kind == aha_model::QWEN3VL, "image_patchify needs a qwen3vl handle");
        VisionModel& V = m->vision;
        const int ps = V.cfg.patch, mg = V.cfg.merge;
        AHA_REQUIRE(h % (ps * mg) == 0 && w % (ps * mg) == 0, "image size must already be a multiple of patch_size*merge_size (img_smart_resize output)");
        const int gh = (int)h / ps, gw = (int)w / ps, N = gh * gw;
        AHA_REQUIRE(N <= V.max_patches, "image exceeds max_patches");
        AHA_REQUIRE((size_t)N * V.patch_dim <= cap, "pixel_values_out too small");
        Scratch mem;
        uint8_t* d_img = mem.alloc<uint8_t>(h * w * 3);
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_img, img_hwc, h * w * 3, cudaMemcpyHostToDevice, m->ctx.stream));
        patchify_kernel<<<N, 256, 0, m->ctx.stream>>>(d_img, (int)h, (int)w, ps, mg, V.cfg.tpatch, V.pix);
        m->ctx.cnt.kernels++;
        AHA_CUDA_CHECK(cudaMemcpyAsync(pixel_values_out, V.pix, (size_t)N * V.patch_dim * sizeof(float), cudaMemcpyDeviceToHost, m->ctx.stream));
        AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
        grid_thw_out[0] = 1; grid_thw_out[1] = (uint32_t)gh; grid_thw_out[2] = (uint32_t)gw;
    });
}

extern "C++" {
namespace {
// resize (h, w, 3) u8 on the device -> (nh, nw, 3) u8 on the device; both buffers owned by the caller
void resize_on_device(aha_model* m, const uint8_t* d_in, int h, int w, uint8_t* d_out, int nh, int nw, float* d_tmp) {
    if (nh == h && nw == w) {   // imageops::resize copies when the dimensions already match
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_out, d_in, (size_t)h * w * 3, cudaMemcpyDeviceToDevice, m->ctx.stream));
        return;
    }
    AHA_REQUIRE(2.0f * std::max(1.0f, (float)h / nh) + 2 <= kResizeMaxTaps && 2.0f * std::max(1.0f, (float)w / nw) + 2 <= kResizeMaxTaps,
                "image downscale factor beyond the resize kernel's tap window (15x)");
    resize_vertical_kernel<<<nh, 256, 0, m->ctx.stream>>>(d_in, h, w, nh, d_tmp);
    resize_horizontal_kernel<<<nw, 256, 0, m->ctx.stream>>>(d_tmp, nh, w, nw, d_out);
    AHA_CUDA_CHECK(cudaGetLastError());
    m->ctx.cnt.kernels += 2;
}
}  // namespace
}  // extern "C++"

int aha_b200_img_smart_resize(uint32_t img_h, uint32_t img_w, uint32_t factor, uint32_t min_pixels, uint32_t max_pixels, uint32_t* out_h, uint32_t* out_w) {
    return guarded_host([&] {
        AHA_REQUIRE(out_h && out_w, "out_h and out_w are required");
        img_smart_resize(img_h, img_w, factor, min_pixels, max_pixels, *out_h, *out_w);
    });
}

int aha_b200_image_resize(aha_model* m, const uint8_t* img_hwc, size_t h, size_t w, size_t new_h, size_t new_w, uint8_t* out_hwc) {
    return guarded(m, [&] {
        AHA_REQUIRE(img_hwc && out_hwc && h > 0 && w > 0 && new_h > 0 && new_w > 0, "images and positive sizes are required");
        Scratch mem;
        uint8_t* d_in = mem.alloc<uint8_t>(h * w * 3);
        uint8_t* d_out = mem.alloc<uint8_t>(new_h * new_w * 3);
        float* d_tmp = mem.alloc<float>(new_h * w * 3);
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_in, img_hwc, h * w * 3, cudaMemcpyHostToDevice, m->ctx.stream));
        resize_on_device(m, d_in, (int)h, (int)w, d_out, (int)new_h, (int)new_w, d_tmp);
        AHA_CUDA_CHECK(cudaMemcpyAsync(out_hwc, d_out, new_h * new_w * 3, cudaMemcpyDeviceToHost, m->ctx.stream));
        AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
    });
}

int aha_b200_image_preprocess(aha_model* m, const uint8_t* img_hwc, size_t h, size_t w, uint32_t min_pixels, uint32_t max_pixels, float* pixel_values_out,
                              size_t cap, uint32_t grid_thw_out[3]) {
    return guarded(m, [&] {
        AHA_REQUIRE(m->kind == aha_model::QWEN3VL, "image_preprocess needs a qwen3vl handle");
        AHA_REQUIRE(img_hwc && pixel_values_out && grid_thw_out && h > 0 && w > 0, "image, outputs and positive sizes are required");
        VisionModel& V = m->vision;
        const int ps = V.cfg.patch, mg = V.cfg.merge;
        uint32_t rh = 0, rw = 0;
        img_smart_resize((uint32_t)h, (uint32_t)w, (uint32_t)(ps * mg), min_pixels, max_pixels, rh, rw);   // Qwen3VLProcessor::process_img
        const int gh = (int)rh / ps, gw = (int)rw / ps, N = gh * gw;
        AHA_REQUIRE(N <= V.max_patches, "image needs " + std::to_string(N) + " patches after img_smart_resize, max_patches is " + std::to_string(V.max_patches));
        AHA_REQUIRE((size_t)N * V.patch_dim <= cap, "pixel_values_out too small");
        Scratch mem;
        uint8_t* d_in = mem.alloc<uint8_t>(h * w * 3);
        uint8_t* d_rs = mem.alloc<uint8_t>((size_t)rh * rw * 3);
        float* d_tmp = mem.alloc<float>((size_t)rh * w * 3);
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_in, img_hwc, h * w * 3, cudaMemcpyHostToDevice, m->ctx.stream));
        resize_on_device(m, d_in, (int)h, (int)w, d_rs, (int)rh, (int)rw, d_tmp);
        patchify_kernel<<<N, 256, 0, m->ctx.stream>>>(d_rs, (int)rh, (int)rw, ps, mg, V.cfg.tpatch, V.pix);   // img_transform + frame duplication + 9-D permute
        m->ctx.cnt.kernels++;
        AHA_CUDA_CHECK(cudaMemcpyAsync(pixel_values_out, V.pix, (size_t)N * V.patch_dim * sizeof(float), cudaMemcpyDeviceToHost, m->ctx.stream));
        AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
        grid_thw_out[0] = 1; grid_thw_out[1] = (uint32_t)gh; grid_thw_out[2] = (uint32_t)gw;
    });
}

int aha_b200_expand_placeholders(const uint32_t* ids, size_t n, uint32_t token_id, const uint32_t* counts, size_t n_counts, uint32_t* out, size_t cap,
                                 size_t* n_out) {
    return guarded_host([&] {
        AHA_REQUIRE(ids && n_out && (counts || n_counts == 0), "ids and n_out are required");
        const std::vector<uint32_t> r = expand_placeholders(ids, n, token_id, counts, n_counts);
        *n_out = r.size();
        if (out) { AHA_REQUIRE(r.size() <= cap, "out too small"); std::memcpy(out, r.data(), r.size() * sizeof(uint32_t)); }
    });
}

int aha_b200_video_smart_resize(uint32_t num_frames, uint32_t height, uint32_t width, uint32_t temporal_factor, uint32_t factor, uint32_t min_pixels,
                                uint32_t max_pixels, uint32_t video_ratio, uint32_t* out_h, uint32_t* out_w) {
    return guarded_host([&] {
        AHA_REQUIRE(out_h && out_w, "out_h and out_w are required");
        video_smart_resize(num_frames, height, width, temporal_factor, factor, min_pixels, max_pixels, video_ratio, *out_h, *out_w);
    });
}

int aha_b200_video_sample_frames(uint32_t total_frames, uint32_t rate_num, uint32_t rate_den, uint32_t fps, uint32_t min_frames, uint32_t max_frames,
                                 uint32_t* nframes_out, uint32_t* indices_out, size_t cap, size_t* n_out) {
    return guarded_host([&] {
        AHA_REQUIRE(n_out, "n_out is required");
        uint32_t nframes = 0;
        const std::vector<uint32_t> idx = video_sample_frames(total_frames, rate_num, rate_den, fps, min_frames, max_frames, nframes);
        if (nframes_out) *nframes_out = nframes;
        *n_out = idx.size();
        if (indices_out) { AHA_REQUIRE(idx.size() <= cap, "indices_out too small"); std::memcpy(indices_out, idx.data(), idx.size() * sizeof(uint32_t)); }
    });
}

int aha_b200_video_timestamps(const uint32_t* frame_indices, size_t n, float fps, uint32_t t_merge_size, float* stamps_out, size_t cap, size_t* n_out) {
    return guarded_host([&] {
        AHA_REQUIRE(frame_indices && n_out, "frame_indices and n_out are required");
        const std::vector<float> st = video_timestamps(frame_indices, n, fps, t_merge_size);
        *n_out = st.size();
        if (stamps_out) { AHA_REQUIRE(st.size() <= cap, "stamps_out too small"); std::memcpy(stamps_out, st.data(), st.size() * sizeof(float)); }
    });
}

int aha_b200_format_timestamp(float seconds, char* out, size_t cap) {
    return guarded_host([&] {
        AHA_REQUIRE(out && cap > 0, "out is required");
        // format!("<{:.1} seconds>", t): both Rust and printf print the exactly rounded decimal (ties to even) of the f32 value
        const int n = std::snprintf(out, cap, "<%.1f seconds>", (double)seconds);
        AHA_REQUIRE(n > 0 && (size_t)n < cap, "out too small");
    });
}

int aha_b200_expand_video_placeholders(const uint32_t* ids, size_t n, uint32_t video_token_id, uint32_t vision_start_token_id, uint32_t vision_end_token_id,
                                       const uint32_t* video_grid_thw, size_t n_videos, uint32_t merge_size, const uint32_t* stamp_ids,
                                       const uint32_t* stamp_lens, size_t n_stamps, uint32_t* out, size_t cap, size_t* n_out) {
    return guarded_host([&] {
        AHA_REQUIRE(ids && n_out && (video_grid_thw || n_videos == 0) && (stamp_lens || n_stamps == 0), "ids, video_grid_thw, stamp_lens and n_out are required");
        const std::vector<uint32_t> r = expand_video_placeholders(ids, n, video_token_id, vision_start_token_id, vision_end_token_id, video_grid_thw, n_videos, merge_size,
                                                                  stamp_ids, stamp_lens, n_stamps);
        *n_out = r.size();
        if (out) { AHA_REQUIRE(r.size() <= cap, "out too small"); std::memcpy(out, r.data(), r.size() * sizeof(uint32_t)); }
    });
}

size_t aha_b200_feat_extract_output_length(size_t n_frames) { return feat_extract_output_length(n_frames); }

int aha_b200_float_range_normalize(float* wave, size_t n) {
    return guarded_host([&] { AHA_REQUIRE(wave || n == 0, "wave is required"); float_range_normalize(wave, n); });
}

int aha_b200_resample(aha_model* m, const float* wave, size_t n, int64_t orig_freq, int64_t new_freq, float* out, size_t cap, size_t* n_out) {
    return guarded(m, [&] {
        AHA_REQUIRE(n_out, "n_out is required");
        AHA_REQUIRE(wave || n == 0, "wave is required");
        if (orig_freq == new_freq) {   // resample(): the waveform itself
            AHA_REQUIRE(orig_freq > 0, "Frequencies must be positive");
            *n_out = n;
            if (!out) return;
            AHA_REQUIRE(cap >= n, "output buffer too small");
            std::memcpy(out, wave, n * sizeof(float));
            return;
        }
        const SincBank B = sinc_resample_bank(orig_freq, new_freq);
        const size_t len_out = sinc_resample_out_len(B, n);
        *n_out = len_out;
        if (!out) return;
        AHA_REQUIRE(cap >= len_out, "output buffer too small");
        if (len_out == 0) return;
        cudaStream_t st = m->ctx.stream;
        Scratch mem;
        float* d_w = mem.alloc<float>(std::max<size_t>(n, 1));
        float* d_t = mem.alloc<float>(B.taps.size());
        float* d_o = mem.alloc<float>(len_out);
        AHA_CUDA_CHECK(cudaMemcpyAsync(d_w, wave, n * sizeof(float), cudaMemcpyHostToDevice, st));
        const size_t smem = B.taps.size() * sizeof(float);
        const unsigned blocks = (unsigned)((len_out + 255) / 256);
        if (smem <= 96 * 1024) {   // the whole bank in shared memory
            AHA_CUDA_CHECK(cudaMemcpyAsync(d_t, B.taps.data(), smem, cudaMemcpyHostToDevice, st));
            if (smem > 48 * 1024) AHA_CUDA_CHECK(cudaFuncSetAttribute(sinc_resample_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            sinc_resample_kernel<true><<<blocks, 256, smem, st>>>(d_w, (long long)n, d_t, B.orig, B.fresh, B.width, B.K, d_o, (long long)len_out);
        } else {                   // 44.1 kHz and friends: hundreds of KB of taps, read from a transposed copy through the caches
            std::vector<float> tT(B.taps.size());
            for (int j = 0; j < B.fresh; ++j) for (int k = 0; k < B.K; ++k) tT[(size_t)k * B.fresh + j] = B.taps[(size_t)j * B.K + k];
            AHA_CUDA_CHECK(cudaMemcpyAsync(d_t, tT.data(), smem, cudaMemcpyHostToDevice, st));
            AHA_CUDA_CHECK(cudaStreamSynchronize(st));   // tT is a temporary
            sinc_resample_kernel<false><<<blocks, 256, 0, st>>>(d_w, (long long)n, d_t, B.orig, B.fresh, B.width, B.K, d_o, (long long)len_out);
        }
        AHA_CUDA_CHECK(cudaGetLastError());
        m->ctx.cnt.kernels++;
        AHA_CUDA_CHECK(cudaMemcpyAsync(out, d_o, len_out * sizeof(float), cudaMemcpyDeviceToHost, st));
        AHA_CUDA_CHECK(cudaStreamSynchronize(st));
    });
}

int aha_b200_sinc_resample_bank(int64_t orig_freq, int64_t new_freq, float* taps_out, size_t cap, int32_t dims_out[4]) {
    return guarded_host([&] {
        AHA_REQUIRE(dims_out, "dims_out is required");
        const SincBank B = sinc_resample_bank(orig_freq, new_freq);
        dims_out[0] = B.fresh; dims_out[1] = B.K; dims_out[2] = B.width; dims_out[3] = B.orig;
        if (!taps_out) return;
        AHA_REQUIRE(cap >= B.taps.size(), "output buffer too small");
        std::memcpy(taps_out, B.taps.data(), B.taps.size() * sizeof(float));
    });
}

int aha_b200_split_audio_into_chunks(size_t total_len, uint32_t sample_rate, float max_chunk_sec, size_t* lens_out, size_t cap, size_t* n_out) {
    return guarded_host([&] {
        AHA_REQUIRE(n_out && sample_rate > 0 && max_chunk_sec > 0.f, "n_out, a positive sample rate and chunk length are required");
        const std::vector<size_t> r = split_audio_into_chunks(total_len, sample_rate, max_chunk_sec);
        *n_out = r.size();
        if (lens_out) { AHA_REQUIRE(r.size() <= cap, "lens_out too small"); for (size_t i = 0; i < r.size(); ++i) lens_out[i] = r[i]; }
    });
}

int aha_b200_debug_gemm(aha_model* m, int impl, int epi, int act, int M, int N, int K, const float* x, const uint16_t* w, const float* bias,
                        const float* resid, float* out, int iters, double* device_ms) {
    return guarded(m, [&] {
        AHA_REQUIRE(x && w && out && M > 0 && N > 0 && K > 0, "x, w, out and positive sizes are required");
        AHA_REQUIRE(impl >= 1 && impl <= 7, "impl must be 1 (SIMT), 2 / 3 (wgmma 128 x 128 / 128 x 256), 4 (batch-1 GEMV), 5 / 6 (batched GEMV) or 7 (wide batched GEMV)");
        Ctx& c = m->ctx;
        const int Nout = epi == EPI_SWIGLU ? N / 2 : N;
        Scratch mem;
        float* dx = mem.alloc<float>((size_t)M * K);
        __half* dw = mem.alloc<__half>((size_t)N * K);
        float* dy = mem.alloc<float>((size_t)M * Nout);
        float *db = nullptr, *dr = nullptr;
        AHA_CUDA_CHECK(cudaMemcpy(dx, x, (size_t)M * K * 4, cudaMemcpyHostToDevice));
        AHA_CUDA_CHECK(cudaMemcpy(dw, w, (size_t)N * K * 2, cudaMemcpyHostToDevice));
        if (bias) { db = mem.alloc<float>(N); AHA_CUDA_CHECK(cudaMemcpy(db, bias, (size_t)N * 4, cudaMemcpyHostToDevice)); }
        if (epi == EPI_RESID) {
            AHA_REQUIRE(resid, "resid is required for the residual epilogue");
            dr = mem.alloc<float>((size_t)M * N); AHA_CUDA_CHECK(cudaMemcpy(dr, resid, (size_t)M * N * 4, cudaMemcpyHostToDevice));
        }
        LinearW W; W.w = dw; W.b = db; W.N = N; W.K = K;
        auto unit_gain = [&] {   // the gain of a unit RMSNorm prologue (the SwiGLU instantiations of the batched GEMVs carry one)
            std::vector<float> h1((size_t)K, 1.0f);
            float* ones = mem.alloc<float>(K);
            AHA_CUDA_CHECK(cudaMemcpy(ones, h1.data(), (size_t)K * 4, cudaMemcpyHostToDevice));
            return ones;
        };
        const size_t n = (size_t)std::max(iters, 0);
        float ms = 0.f;
        if (impl == 7) {   // the wide decode projection (gemv_wide.cuh): M <= 64 rows split into fp16 hi / lo operand rows, then the kernel
            AHA_REQUIRE(M <= kWideSeqs && (epi == EPI_STORE || epi == EPI_RESID || epi == EPI_SWIGLU), "wide batched GEMV: M <= 64, epilogue store / residual / SwiGLU");
            AHA_REQUIRE(gemv_wide_supported(N, K), "wide batched GEMV: N and K must be multiples of 64");
            const int gepi = epi == EPI_STORE ? GEPI_STORE : (epi == EPI_RESID ? GEPI_RESID : GEPI_SWIGLU);
            const size_t xh = (size_t)kWideSeqs * K;
            __half* hi = mem.alloc<__half>(xh);
            __half* lo = mem.alloc<__half>(xh);
            AHA_CUDA_CHECK(cudaMemset(hi, 0, xh * sizeof(__half))); AHA_CUDA_CHECK(cudaMemset(lo, 0, xh * sizeof(__half)));   // rows M..63 stay zero
            const size_t wsf = wide_ws_floats(N, K, c.num_sms);
            const int tiles = wide_plan(N, K, c.num_sms).tiles;
            float* ws = wsf ? mem.alloc<float>(wsf) : nullptr;
            int* cnt = mem.alloc<int>(tiles);
            AHA_CUDA_CHECK(cudaMemset(cnt, 0, (size_t)tiles * sizeof(int)));
            const float* ones = gepi == GEPI_SWIGLU ? unit_gain() : nullptr;   // (behind a unit-gain RMSNorm prologue, as impl 5)
            WideArgs a{};
            a.bias = db; a.resid = dr; a.ldr = N; a.out = dy; a.ldo = Nout; a.N = N; a.K = K; a.nb = M; a.ws = ws; a.counters = cnt;
            const CUtensorMap tm = make_tmap_f16(dw, (uint64_t)N, (uint64_t)K);
            auto run = [&] {
                if (ones) rmsnorm_split_kernel<<<M, 256, 0, c.stream>>>(dx, ones, 1e-6f, hi, lo, K);
                else split_f32_to_f16x2_kernel<<<(unsigned)(((size_t)M * K / 4 + 255) / 256), 256, 0, c.stream>>>(dx, K, hi, lo, M, K);
                gemv_wide(c.stream, gepi, tm, hi, lo, a, c.num_sms);
            };
            run();
            ms = timed_ms(m, n, [&](size_t) { run(); });
        } else if (impl == 4) {   // the batch-1 decode GEMV (gemv.cuh), once per activation row; epilogues and SwiGLU prologue as impl 5
            AHA_REQUIRE(epi == EPI_STORE || epi == EPI_RESID || epi == EPI_SWIGLU, "batch-1 GEMV: epilogue store / residual / SwiGLU");
            const int gepi = epi == EPI_STORE ? GEPI_STORE : (epi == EPI_RESID ? GEPI_RESID : GEPI_SWIGLU);
            const int pro = epi == EPI_SWIGLU ? PRO_RMSNORM : PRO_NONE;
            const float* ones = pro == PRO_RMSNORM ? unit_gain() : nullptr;
            auto run = [&] {
                for (int r = 0; r < M; ++r) {
                    GemvArgs a{};
                    a.W = dw; a.x = dx + (size_t)r * K; a.norm_w = ones; a.eps = ones ? 1e-6f : 0.f; a.bias = db;
                    a.resid = dr ? dr + (size_t)r * N : nullptr; a.out = dy + (size_t)r * Nout; a.N = N; a.K = K;
                    gemv(c.stream, pro, gepi, a);
                }
            };
            run();
            ms = timed_ms(m, n, [&](size_t) { run(); });
        } else if (impl == 5 || impl == 6) {   // the batched decode GEMV (gemv_batch.cuh; 6 = the cp.async ring version): M <= 8 activation rows against every weight row
            AHA_REQUIRE(M <= kGemvBatchMax && (epi == EPI_STORE || epi == EPI_RESID || epi == EPI_SWIGLU), "batched GEMV: M <= 8, epilogue store / residual / SwiGLU");
            GemvBatchArgs a{};
            a.W = dw; a.x = dx; a.ldx = K; a.bias = db; a.resid = dr; a.ldr = N; a.out = dy; a.ldo = Nout; a.N = N; a.K = K; a.nb = M; a.eps = 0.f;
            const int gepi = epi == EPI_STORE ? GEPI_STORE : (epi == EPI_RESID ? GEPI_RESID : GEPI_SWIGLU);
            const int pro = epi == EPI_SWIGLU ? PRO_RMSNORM : PRO_NONE;
            if (pro == PRO_RMSNORM) { a.norm_w = unit_gain(); a.eps = 1e-6f; }
            gemv_batch(c.stream, pro, gepi, a, impl == 6);
            ms = timed_ms(m, n, [&](size_t) { gemv_batch(c.stream, pro, gepi, a, impl == 6); });
        } else {
            const int saved = c.gemm_impl;
            c.gemm_impl = impl;
            try {
                linear_gemm(c, epi, dx, K, W, dr, N, dy, Nout, M, act);   // warm-up + correctness run
                ms = timed_ms(m, n, [&](size_t) { linear_gemm(c, epi, dx, K, W, dr, N, dy, Nout, M, act); });
            } catch (...) { c.gemm_impl = saved; throw; }
            c.gemm_impl = saved;
        }
        if (device_ms) *device_ms = ms;
        AHA_CUDA_CHECK(cudaMemcpy(out, dy, (size_t)M * Nout * 4, cudaMemcpyDeviceToHost));
    });
}

namespace {
// Qwen3Model::forward_hidden + l2_normalize for one text; result left in T.xn[0:H] and copied to `out`
void embed_one(aha_model* m, const uint32_t* ids, size_t S, float* out) {
    require_no_session(m);
    AHA_REQUIRE(m->kind == aha_model::QWEN3, "embeddings need a qwen3 handle (Qwen3-Embedding shares Qwen3Model)");
    AHA_REQUIRE(ids && S >= 1 && out, "ids, seq_len and out are required");
    TextModel& T = m->text;
    drop_cache(m);
    upload_ids(m, ids, S);
    std::vector<int> pos3((size_t)3 * S);
    for (int r = 0; r < 3; ++r) for (size_t i = 0; i < S; ++i) pos3[(size_t)r * S + i] = (int)i;
    upload_pos(m, pos3);
    T.prefill(T.table, (int)S, 0, false, nullptr, 0, {});
    const int H = T.cfg.H;
    rmsnorm_kernel<<<1, 256, 0, m->ctx.stream>>>(T.x + (size_t)(S - 1) * H, T.norm, T.cfg.eps, T.xn, H);
    l2_normalize_kernel<<<1, 256, 0, m->ctx.stream>>>(T.xn, T.xn + H, H);
    m->ctx.cnt.kernels += 2;
    AHA_CUDA_CHECK(cudaMemcpyAsync(out, T.xn + H, (size_t)H * sizeof(float), cudaMemcpyDeviceToHost, m->ctx.stream));
    AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
    drop_cache(m);   // clear_kv_cache()
}

// Qwen3Embedding::embed_multi (qwen3_embedding/mod.rs:38-48): embed_one for every text, computed as packed prefills.  The texts, in input
// order, are cut into packs of at most min(max_prefill, max_ctx) tokens.  A pack is one prefill in which every text attends only to itself
// and its positions restart at 0 (TextModel::prefill with PrefillSegments), so one pass over the weights serves many texts.  The last row of
// every text then goes through the final RMSNorm and l2_normalize kernels that embed_one uses.
void embed_batch(aha_model* m, const uint32_t* ids, const size_t* lens, size_t n, float* out) {
    AHA_REQUIRE(n >= 1, "embedding input cannot be empty");
    require_no_session(m);
    AHA_REQUIRE(m->kind == aha_model::QWEN3, "embeddings need a qwen3 handle (Qwen3-Embedding shares Qwen3Model)");
    AHA_REQUIRE(ids && lens && out, "ids, lens and out are required");
    TextModel& T = m->text;
    AHA_REQUIRE(T.tp_world == 1, "embed_batch is single-GPU (tp_world must be 1)");
    std::vector<const uint32_t*> text_ids(n);
    size_t total = 0;
    for (size_t j = 0; j < n; ++j) {
        const size_t S = lens[j];
        text_ids[j] = ids + total;
        AHA_REQUIRE(S >= 1, "empty input_ids");
        AHA_REQUIRE(S <= (size_t)T.max_prefill, "prompt of " + std::to_string(S) + " tokens exceeds max_prefill " + std::to_string(T.max_prefill));
        AHA_REQUIRE(S <= (size_t)T.max_ctx, "context of " + std::to_string(S) + " tokens exceeds max_ctx " + std::to_string(T.max_ctx));
        for (size_t i = 0; i < S; ++i) AHA_REQUIRE(ids[total + i] < (uint32_t)T.cfg.V, "token id out of range");
        total += S;
    }
    Ctx& c = m->ctx;
    alloc_pack_buffers(m);
    const size_t cap = (size_t)std::min(T.max_prefill, T.max_ctx);
    const int H = T.cfg.H;
    drop_cache(m);
    const std::vector<size_t> text_lens(lens, lens + n);
    for (size_t first = 0; first < n;) {
        // Texts start on multiples of 16 tokens: a segment's start is the innermost TMA coordinate of the attention kernel's V^T tiles, which
        // has to sit on a 16-byte boundary.  A text's KV tiles and query tiles stay the ones it runs alone (a 16-token round-up never crosses a
        // 64-token boundary).
        Pack p = plan_pack(text_ids, text_lens, first, 16, cap);
        upload_pack(m, p);
        T.prefill(T.table, (int)p.S, 0, false, nullptr, 0, {}, p.sg);
        const int np = (int)(p.last - first);
        gather_rows_kernel<<<np, 256, 0, c.stream>>>(m->d_pack_rows, T.x, T.xn, H);
        rmsnorm_kernel<<<np, 256, 0, c.stream>>>(T.xn, T.norm, T.cfg.eps, T.x, H);
        l2_normalize_kernel<<<np, 256, 0, c.stream>>>(T.x, T.xn, H);
        c.cnt.kernels += 3;
        AHA_CUDA_CHECK(cudaMemcpyAsync(out + first * H, T.xn, (size_t)np * H * sizeof(float), cudaMemcpyDeviceToHost, c.stream));
        AHA_CUDA_CHECK(cudaStreamSynchronize(c.stream));
        first = p.last;
    }
    drop_cache(m);
}

// ---- scoring: log p(ids[i] | ids[0 .. i)) for given text (aha_b200_score, aha_b200_score_batch) --------------------------------------------
// Record i of a text is the distribution at row i - 1 evaluated at ids[i].  The rows to score are gathered from TextModel::x right after the
// prefill that computed them and go through the final RMSNorm (rmsnorm_split_kernel with a row list), score_head_kernel and
// score_final_rows_kernel.  Scoring uses the prefill scratch and leaves the cache empty, like embed.
using ScoreBufs = aha_model::ScoreBufs;

// the buffers of M rows in one allocation at `base` (nullptr: only the size); returns the bytes they take
size_t score_bufs_carve(char* base, size_t M, int V, ScoreBufs& b) {
    const size_t P = (size_t)lp_parts(V);
    size_t off = 0;
    auto take = [&](auto*& ptr, size_t n) {
        using E = std::remove_reference_t<decltype(*ptr)>;
        off = (off + 255) & ~(size_t)255;
        if (base) ptr = reinterpret_cast<E*>(base + off);
        off += n * sizeof(E);
    };
    take(b.rows, M); take(b.tgt, M); take(b.index, M); take(b.tlogit, M);
    take(b.part, M * P * kLpPartFloats); take(b.part_id, M * P * kLpMaxTop); take(b.on, 1); take(b.rec, M);
    return off;
}

// what every scoring entry refuses
void score_require(aha_model* m, uint32_t n_top) {
    require_no_session(m);
    AHA_REQUIRE(m->kind != aha_model::QWEN3_ASR, "scoring needs a qwen3 or qwen3vl handle (Qwen3-ASR prompts carry audio)");
    const TextModel& T = m->text;
    AHA_REQUIRE(T.tp_world == 1, "scoring is single-GPU (tp_world must be 1)");
    AHA_REQUIRE(n_top <= AHA_MAX_TOP_LOGPROBS, "n_top " + std::to_string(n_top) + ": at most " + std::to_string(AHA_MAX_TOP_LOGPROBS) + " alternatives");
    AHA_REQUIRE(n_top <= (uint32_t)T.cfg.V, "n_top " + std::to_string(n_top) + " exceeds the vocabulary of " + std::to_string(T.cfg.V));
    AHA_REQUIRE(T.cfg.V <= kLpMaxParts * kLpSlice, "vocabulary too large for the log-probability kernels");
    AHA_REQUIRE(score_head_supported(T.cfg.H), "scoring needs hidden_size to be a multiple of 64");
}
// one text: 1 <= start < len <= max_ctx, ids inside the vocabulary and no multimodal placeholder (scoring takes text-only prompts)
void score_check_text(aha_model* m, const uint32_t* ids, size_t S, size_t start) {
    const TextModel& T = m->text;
    AHA_REQUIRE(start >= 1, "start must be at least 1 (token 0 has no prefix to be scored against)");
    AHA_REQUIRE(start < S, "start " + std::to_string(start) + " leaves nothing to score in a text of " + std::to_string(S) + " tokens");
    AHA_REQUIRE(S <= (size_t)T.max_ctx, "context of " + std::to_string(S) + " tokens exceeds max_ctx " + std::to_string(T.max_ctx));
    const auto mmt = mm_token_ids(m);
    for (size_t i = 0; i < S; ++i) {
        AHA_REQUIRE(ids[i] < (uint32_t)T.cfg.V, "token id out of range");
        for (uint32_t t : mmt) AHA_REQUIRE(ids[i] != t, "scoring takes text-only prompts: token " + std::to_string(i) + " is a multimodal placeholder");
    }
}
void alloc_score_buffers(aha_model* m) {
    if (m->score_ready) return;
    const TextModel& T = m->text;
    char* base = m->ctx.alloc<char>(score_bufs_carve(nullptr, (size_t)T.max_prefill, T.cfg.V, m->score));
    score_bufs_carve(base, (size_t)T.max_prefill, T.cfg.V, m->score);
    m->score_tm_w = make_tmap_f16_rows(T.lm_head, (uint64_t)T.cfg.V, (uint64_t)T.cfg.H, kShBN);
    m->score_ready = true;
}

// The head over M rows of x [., H] (d_rows: the gather list, nullptr = rows 0 .. M-1) with b.tgt / b.index set: final RMSNorm + split, then
// impl 0: score_head_kernel; impl 1 (tests, timing): gemm_tc EPI_STORE into `logits` [M][V] + logprob_partial_rows_kernel.  Then stage 2
// into b.rec.
void score_head_rows(aha_model* m, int impl, const float* x, const int* d_rows, int M, int n, const ScoreBufs& b, float* logits = nullptr) {
    TextModel& T = m->text;
    Ctx& c = m->ctx;
    const int H = T.cfg.H, V = T.cfg.V, P = lp_parts(V);
    const ActSplit a = act_split(c, 0, (size_t)M * H);
    rmsnorm_split_kernel<<<M, 256, 0, c.stream>>>(x, T.norm, T.cfg.eps, a.hi, a.lo, H, d_rows);
    if (impl == 0) {
        const ScoreHeadArgs s{M, V, H, n, b.tgt, b.part, b.part_id, b.tlogit};
        score_head_launch(c.stream, a.hi, a.lo, m->score_tm_w, s);
    } else {
        GemmTcArgs g{};
        g.C = logits; g.ldc = V; g.M = M; g.N = V; g.K = H; g.act = ACT_NONE;
        gemm_tc_launch<kShBN>(c.stream, EPI_STORE, a.hi, a.lo, m->score_tm_w, g);
        const int on = 1 + n;
        AHA_CUDA_CHECK(cudaMemcpyAsync(b.on, &on, sizeof(int), cudaMemcpyHostToDevice, c.stream));
        logprob_partial_rows_kernel<<<dim3(P, M), kLpThreads, 0, c.stream>>>(logits, V, V, nullptr, b.on, b.part, b.part_id);
        c.cnt.kernels++;
    }
    score_final_rows_kernel<<<M, kLpMaxParts, 0, c.stream>>>(b.part, b.part_id, P, n, b.tgt, impl == 0 ? b.tlogit : nullptr, logits, V, b.index, b.rec);
    c.cnt.kernels += 3;
    AHA_CUDA_CHECK(cudaGetLastError());
}

// the head over the listed rows of TextModel::x, scored at tgt with record indices idx; the records go to out[0 .. rows.size())
void score_gathered(aha_model* m, const std::vector<int>& rows, const std::vector<uint32_t>& tgt, const std::vector<uint32_t>& idx, int n, aha_logprobs* out) {
    const int M = (int)rows.size();
    if (M == 0) return;
    const ScoreBufs& b = m->score;
    cudaStream_t st = m->ctx.stream;
    AHA_CUDA_CHECK(cudaMemcpyAsync(b.rows, rows.data(), (size_t)M * sizeof(int), cudaMemcpyHostToDevice, st));
    AHA_CUDA_CHECK(cudaMemcpyAsync(b.tgt, tgt.data(), (size_t)M * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    AHA_CUDA_CHECK(cudaMemcpyAsync(b.index, idx.data(), (size_t)M * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    score_head_rows(m, 0, m->text.x, b.rows, M, n, b);
    AHA_CUDA_CHECK(cudaMemcpyAsync(out, b.rec, (size_t)M * sizeof(aha_logprobs), cudaMemcpyDeviceToHost, st));
    AHA_CUDA_CHECK(cudaStreamSynchronize(st));
}

// one checked text through the chunked prefill (forward_any's chunks: any length up to max_ctx); each chunk's scored rows go through the
// head right after its prefill.  Records from out[0] = the record of ids[start].
void score_text(aha_model* m, const uint32_t* ids, size_t S, size_t start, int n, aha_logprobs* out) {
    drop_cache(m);
    prefill_chunked(m, m->text.table, ids, S, 0, nullptr, false, false, false, [&](size_t done, size_t len) {
        const size_t j0 = std::max(start - 1, done), j1 = std::min(S - 1, done + len);   // rows j0 .. j1 - 1 of the text
        if (j0 >= j1) return;
        std::vector<int> rows;
        std::vector<uint32_t> tgt, idx;
        for (size_t j = j0; j < j1; ++j) { rows.push_back((int)(j - done)); tgt.push_back(ids[j + 1]); idx.push_back((uint32_t)(j + 1)); }
        score_gathered(m, rows, tgt, idx, n, out + (j0 + 1 - start));
    });
}

void score_one(aha_model* m, const uint32_t* ids, size_t S, size_t start, uint32_t n_top, aha_logprobs* out, size_t cap, size_t* n_out) {
    AHA_REQUIRE(ids && n_out, "ids and n_out are required");
    score_require(m, n_top);
    score_check_text(m, ids, S, start);
    AHA_REQUIRE(out && S - start <= cap, "out holds " + std::to_string(cap) + " records, the text needs " + std::to_string(S - start));
    *n_out = 0;
    alloc_score_buffers(m);
    score_text(m, ids, S, start, (int)n_top, out);
    drop_cache(m);
    *n_out = S - start;
}

// The texts, in input order, are cut into packs of at most min(max_prefill, max_ctx) tokens, as embed_batch cuts them.  A pack is one prefill
// (each text attends only to itself, its positions restart at 0), then one head launch over the scored rows of all its texts.  A text longer
// than a pack goes through score_text in its place.
void score_batch(aha_model* m, const uint32_t* ids, const size_t* lens, const size_t* starts, size_t n, uint32_t n_top, aha_logprobs* out, size_t cap,
                 size_t* n_out) {
    AHA_REQUIRE(ids && lens && n >= 1 && n_out, "ids, lens, n >= 1 and n_out are required");
    score_require(m, n_top);
    TextModel& T = m->text;
    std::vector<const uint32_t*> text_ids(n);
    const std::vector<size_t> text_lens(lens, lens + n);
    std::vector<size_t> st(n), first_rec(n);
    size_t total = 0, recs = 0;
    for (size_t j = 0; j < n; ++j) {
        text_ids[j] = ids + total;
        st[j] = starts ? starts[j] : 1;
        AHA_REQUIRE(lens[j] >= 1, "text " + std::to_string(j) + " is empty");
        score_check_text(m, text_ids[j], lens[j], st[j]);
        first_rec[j] = recs;
        recs += lens[j] - st[j];
        total += lens[j];
    }
    AHA_REQUIRE(out && recs <= cap, "out holds " + std::to_string(cap) + " records, the texts need " + std::to_string(recs));
    *n_out = 0;
    alloc_score_buffers(m);
    alloc_pack_buffers(m);
    const size_t pcap = (size_t)std::min(T.max_prefill, T.max_ctx);
    drop_cache(m);
    for (size_t first = 0; first < n;) {
        if (text_lens[first] > pcap) {
            score_text(m, text_ids[first], text_lens[first], st[first], (int)n_top, out + first_rec[first]);
            ++first;
            continue;
        }
        // 16-token starts, as in embed_batch: a text's attention tiles stay the ones it runs alone
        Pack p = plan_pack(text_ids, text_lens, first, 16, pcap);
        upload_pack(m, p);
        T.prefill(T.table, (int)p.S, 0, false, nullptr, 0, {}, p.sg);
        std::vector<int> rows;
        std::vector<uint32_t> tgt, idx;
        for (size_t j = p.first; j < p.last; ++j) {
            const size_t s0 = p.start[j - first];
            for (size_t i = st[j]; i < text_lens[j]; ++i) { rows.push_back((int)(s0 + i - 1)); tgt.push_back(text_ids[j][i]); idx.push_back((uint32_t)i); }
        }
        score_gathered(m, rows, tgt, idx, (int)n_top, out + first_rec[first]);
        first = p.last;
    }
    drop_cache(m);
    *n_out = recs;
}

// kernel timing (aha_b200_bench_kernel "score_head:M:n" / "score_twin:M:n"): the head over rows 0 .. M-1 of TextModel::x as the last
// prefill left them, every row scored at token 0
void bench_score(aha_model* m, const std::string& w, int iters, double* avg_ms, uint64_t* bytes) {
    TextModel& T = m->text;
    char kind[16] = {0};
    int M = 0, n = 0;
    AHA_REQUIRE(std::sscanf(w.c_str(), "score_%4[a-z]:%d:%d", kind, &M, &n) == 3 && (std::string(kind) == "head" || std::string(kind) == "twin"),
                "score kernels are named score_head:M:n or score_twin:M:n");
    const int impl = std::string(kind) == "head" ? 0 : 1;
    score_require(m, (uint32_t)std::max(n, 0));
    AHA_REQUIRE(M >= 1 && M <= T.max_prefill && n >= 0, "score bench: 1 <= M <= max_prefill");
    AHA_REQUIRE(impl == 0 || T.cfg.V % 2 == 0, "the gemm_tc twin needs an even vocabulary");
    alloc_score_buffers(m);
    const ScoreBufs& b = m->score;
    cudaStream_t st = m->ctx.stream;
    AHA_CUDA_CHECK(cudaMemsetAsync(b.tgt, 0, (size_t)M * sizeof(uint32_t), st));
    AHA_CUDA_CHECK(cudaMemsetAsync(b.index, 0, (size_t)M * sizeof(uint32_t), st));
    Scratch mem;
    float* logits = impl == 1 ? mem.alloc<float>((size_t)M * T.cfg.V) : nullptr;
    score_head_rows(m, impl, T.x, nullptr, M, n, b, logits);
    *avg_ms = timed_ms(m, (size_t)iters, [&](size_t) { score_head_rows(m, impl, T.x, nullptr, M, n, b, logits); }) / iters;
    *bytes = 2ull * T.cfg.V * T.cfg.H;
}
}  // namespace

int aha_b200_score(aha_model* m, const uint32_t* ids, size_t seq_len, size_t start, uint32_t n_top, aha_logprobs* out, size_t cap, size_t* n_out) {
    return guarded(m, [&] { score_one(m, ids, seq_len, start, n_top, out, cap, n_out); });
}

int aha_b200_score_batch(aha_model* m, const uint32_t* ids, const size_t* lens, const size_t* starts, size_t n, uint32_t n_top, aha_logprobs* out,
                         size_t cap, size_t* n_out) {
    return guarded(m, [&] { score_batch(m, ids, lens, starts, n, n_top, out, cap, n_out); });
}

int aha_b200_debug_score_head(aha_model* m, int impl, const float* hidden, size_t M, const uint32_t* targets, uint32_t n_top, aha_logprobs* out) {
    return guarded(m, [&] {
        AHA_REQUIRE(hidden && targets && out && M >= 1 && M <= 65535, "hidden, targets, out and 1 <= M <= 65535 are required");
        AHA_REQUIRE(impl == 0 || impl == 1, "impl must be 0 (score_head_kernel) or 1 (gemm_tc + logprob_partial_rows_kernel)");
        score_require(m, n_top);
        const TextModel& T = m->text;
        const int H = T.cfg.H, V = T.cfg.V;
        for (size_t r = 0; r < M; ++r) AHA_REQUIRE(targets[r] < (uint32_t)V, "target id out of range");
        AHA_REQUIRE(impl == 0 || V % 2 == 0, "the gemm_tc twin needs an even vocabulary");
        alloc_score_buffers(m);
        cudaStream_t st = m->ctx.stream;
        // scratch of this call only: the hidden rows, the buffers of M rows and (twin) the logits block
        ScoreBufs b;
        const size_t o_x = (score_bufs_carve(nullptr, M, V, b) + 255) & ~(size_t)255;
        const size_t o_lg = (o_x + M * H * sizeof(float) + 255) & ~(size_t)255;
        Scratch mem;
        char* base = mem.alloc<char>(o_lg + (impl == 1 ? M * (size_t)V * sizeof(float) : 0));
        score_bufs_carve(base, M, V, b);
        float* x = reinterpret_cast<float*>(base + o_x);
        std::vector<uint32_t> idx(M);
        for (size_t r = 0; r < M; ++r) idx[r] = (uint32_t)r;
        AHA_CUDA_CHECK(cudaMemcpyAsync(x, hidden, M * H * sizeof(float), cudaMemcpyHostToDevice, st));
        AHA_CUDA_CHECK(cudaMemcpyAsync(b.tgt, targets, M * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
        AHA_CUDA_CHECK(cudaMemcpyAsync(b.index, idx.data(), M * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
        score_head_rows(m, impl, x, nullptr, (int)M, (int)n_top, b, impl == 1 ? reinterpret_cast<float*>(base + o_lg) : nullptr);
        AHA_CUDA_CHECK(cudaMemcpyAsync(out, b.rec, M * sizeof(aha_logprobs), cudaMemcpyDeviceToHost, st));
        AHA_CUDA_CHECK(cudaStreamSynchronize(st));
    });
}

int aha_b200_embed(aha_model* m, const uint32_t* ids, size_t seq_len, float* out) {
    return guarded(m, [&] { embed_one(m, ids, seq_len, out); });
}

int aha_b200_embed_batch(aha_model* m, const uint32_t* ids, const size_t* lens, size_t n, float* out) {
    return guarded(m, [&] { embed_batch(m, ids, lens, n, out); });
}

int aha_b200_rerank(aha_model* m, const uint32_t* query_ids, size_t query_len, const uint32_t* doc_ids, const size_t* doc_lens, size_t n_docs,
                    float* scores_out) {
    return guarded(m, [&] {
        AHA_REQUIRE(doc_ids && doc_lens && scores_out && n_docs >= 1, "documents are required (embedding input cannot be empty)");
        const int H = m->text.cfg.H;
        std::vector<float> q(H), d(H);
        embed_one(m, query_ids, query_len, q.data());
        size_t off = 0;
        for (size_t i = 0; i < n_docs; ++i) {
            embed_one(m, doc_ids + off, doc_lens[i], d.data());
            off += doc_lens[i];
            float acc = 0.f;   // (1,H) x (H,1) in fp32, like the reference's matmul of two host-side f32 tensors
            for (int k = 0; k < H; ++k) acc += q[k] * d[k];
            scores_out[i] = acc;
        }
    });
}

int aha_b200_nccl_unique_id(uint8_t out[128]) {
    return guarded_host([&] {
        AHA_REQUIRE(out != nullptr, "out is required");
        NcclApi& n = NcclApi::get();
        NcclApi::unique_id id;
        n.check(n.GetUniqueId(&id), "ncclGetUniqueId");
        std::memcpy(out, &id, 128);
    });
}

int aha_b200_rope_index_mm(const uint32_t* ids, size_t seq_len, const uint32_t* grid_thw, size_t n_images, const uint32_t* video_grid_thw, size_t n_videos,
                           uint32_t spatial_merge_size, uint32_t image_token_id, uint32_t video_token_id, uint32_t vision_start_token_id, int32_t* pos3_out,
                           int32_t* rope_delta_out) {
    return guarded_host([&] {
        AHA_REQUIRE(ids != nullptr && seq_len > 0 && pos3_out != nullptr && rope_delta_out != nullptr, "ids, pos3_out and rope_delta_out are required");
        AHA_REQUIRE(n_images == 0 || grid_thw != nullptr, "grid_thw is required when n_images > 0");
        AHA_REQUIRE(n_videos == 0 || video_grid_thw != nullptr, "video_grid_thw is required when n_videos > 0");
        AHA_REQUIRE(spatial_merge_size > 0 && seq_len < (size_t)1 << 30, "bad spatial_merge_size / seq_len");
        std::vector<std::array<int, 3>> grid(n_images), frames;
        for (size_t i = 0; i < n_images; ++i) grid[i] = {(int)grid_thw[3 * i], (int)grid_thw[3 * i + 1], (int)grid_thw[3 * i + 2]};
        for (size_t i = 0; i < n_videos; ++i)
            for (uint32_t t = 0; t < video_grid_thw[3 * i]; ++t) frames.push_back({1, (int)video_grid_thw[3 * i + 1], (int)video_grid_thw[3 * i + 2]});
        std::vector<int> pos3;
        int delta = 0;
        get_rope_index(ids, (int)seq_len, grid, frames, (int)spatial_merge_size, (int)image_token_id, (int)video_token_id, (int)vision_start_token_id, pos3, delta);
        for (size_t i = 0; i < pos3.size(); ++i) pos3_out[i] = pos3[i];
        *rope_delta_out = delta;
    });
}
int aha_b200_rope_index(const uint32_t* ids, size_t seq_len, const uint32_t* grid_thw, size_t n_images, uint32_t spatial_merge_size,
                        uint32_t image_token_id, uint32_t vision_start_token_id, int32_t* pos3_out, int32_t* rope_delta_out) {
    return aha_b200_rope_index_mm(ids, seq_len, grid_thw, n_images, nullptr, 0, spatial_merge_size, image_token_id, 0xffffffffu, vision_start_token_id, pos3_out,
                                  rope_delta_out);
}

void aha_b200_destroy(aha_model* m) {
    if (!m) return;
    cudaSetDevice(m->ctx.device);
    if (m->ctx.stream) cudaStreamSynchronize(m->ctx.stream);
    m->text.destroy();
    m->batch.graphs.clear();
    m->wide_batch.graphs.clear();
    m->spec.destroy();
    for (auto& f : m->fsms) cudaFree(f.second.mem);
    for (auto& r : m->rules) cudaFree(r.second.mem);
    m->ctx.free_all();
    if (m->h_pin) cudaFreeHost(m->h_pin);
    if (m->h_lp_pin) cudaFreeHost(m->h_lp_pin);
    if (m->swap.host) cudaFreeHost(m->swap.host);
    if (m->ev0) cudaEventDestroy(m->ev0);
    if (m->ev1) cudaEventDestroy(m->ev1);
    for (auto& e : m->ev_tok) if (e) cudaEventDestroy(e);
    if (m->ctx.stream) cudaStreamDestroy(m->ctx.stream);
    delete m;
}

const char* aha_b200_last_error(aha_model* m) {
    if (m) return m->last_error.c_str();
    std::lock_guard<std::mutex> lk(g_err_mu);
    static thread_local std::string copy;
    copy = g_create_error;
    return copy.c_str();
}

void* aha_b200_stream(aha_model* m) { return m ? (void*)m->ctx.stream : nullptr; }

int aha_b200_get_stats(aha_model* m, aha_stats* out) {
    return guarded(m, [&] {
        AHA_REQUIRE(out, "out is required");
        out->kernel_launches = m->ctx.cnt.kernels;
        out->graph_launches = m->ctx.cnt.graphs;
        out->kernels_per_decode_step = m->text.step_graph_kernels;
        out->weight_bytes = m->ctx.alloc_bytes;
        out->kv_bytes_per_token = (uint64_t)m->text.cfg.L * 2 * m->text.nkv_l * m->text.cfg.hd * sizeof(float);
        out->decode_bytes_per_step_fixed = m->text.decode_weight_bytes;
    });
}
int aha_b200_reset_stats(aha_model* m) {
    return guarded(m, [&] { m->ctx.cnt = Counters{}; });
}
int aha_b200_set_trace(aha_model* m, int on) {
    return guarded(m, [&] {
        m->text.set_trace(on != 0);
        if (m->kind == aha_model::QWEN3VL) m->vision.set_trace(on != 0);
        if (m->kind == aha_model::QWEN3_ASR) m->audio.set_trace(on != 0);
    });
}
int aha_b200_debug_read(aha_model* m, const char* what, int index, float* out, size_t cap, size_t* n) {
    return guarded(m, [&] {
        AHA_REQUIRE(what && out && n, "what, out and n are required");
        const std::string w = what;
        const float* src = nullptr;
        size_t cnt = 0;
        TextModel& T = m->text;
        if (w == "hidden") {
            AHA_REQUIRE(T.trace_buf && index >= 0 && index < T.cfg.L, "hidden trace not available");
            src = T.trace_buf + (size_t)index * T.max_prefill * T.cfg.H; cnt = (size_t)T.trace_S * T.cfg.H;
        } else if (w == "vit") {
            AHA_REQUIRE(m->kind == aha_model::QWEN3VL && m->vision.trace_buf && index >= 0 && index <= m->vision.cfg.depth, "vit trace not available");
            src = m->vision.trace_buf + (size_t)index * m->vision.max_patches * m->vision.cfg.H; cnt = (size_t)m->vision.last_N * m->vision.cfg.H;
        } else if (w == "image_embeds") {
            AHA_REQUIRE(m->kind == aha_model::QWEN3VL, "image_embeds needs a qwen3vl handle");
            const int ne = m->vision.last_N / (m->vision.cfg.merge * m->vision.cfg.merge);
            src = index <= 0 ? m->vision.image_embeds : m->vision.ds_out.at(index - 1); cnt = (size_t)ne * m->vision.cfg.out_hidden;
        } else if (w == "audio") {
            AHA_REQUIRE(m->kind == aha_model::QWEN3_ASR && m->audio.trace_buf && index >= 0 && index <= m->audio.cfg.layers, "audio trace not available");
            src = m->audio.trace_buf + (size_t)index * m->audio.max_tokens * m->audio.cfg.d_model; cnt = (size_t)m->audio.last_tokens * m->audio.cfg.d_model;
        } else if (w == "audio_embeds") {
            AHA_REQUIRE(m->kind == aha_model::QWEN3_ASR, "audio_embeds needs a qwen3_asr handle");
            src = m->audio.audio_embeds; cnt = (size_t)m->audio.last_tokens * m->audio.cfg.out_dim;
        } else if (w == "fused_trace") {  // globaltimer stamps (ns, relative to the first) of CTA 0; index 0 = consumer, 1 = producer
            AHA_REQUIRE(T.d_ftrace && (index == 0 || index == 1) && cap >= 4096, "fused trace not available");
            std::vector<unsigned long long> h(4096);
            AHA_CUDA_CHECK(cudaMemcpy(h.data(), T.d_ftrace + (size_t)index * 4096, 4096 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
            size_t k = 0;
            for (; k < 4096 && h[k]; ++k) out[k] = (float)(double)(h[k] - h[0]);
            *n = k; return;
        } else if (w == "fused_cta_trace") {  // barrier arrival stamps of CTA `index` (ns relative to CTA 0's first), [255] = %smid
            AHA_REQUIRE(T.d_ftrace && index >= 0 && index < 256 && cap >= 256, "fused trace not available");
            std::vector<unsigned long long> h(256);
            unsigned long long base = 0;
            AHA_CUDA_CHECK(cudaMemcpy(&base, T.d_ftrace + 8192, sizeof(base), cudaMemcpyDeviceToHost));
            AHA_CUDA_CHECK(cudaMemcpy(h.data(), T.d_ftrace + 8192 + (size_t)index * 256, 256 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
            for (size_t k = 0; k < 255; ++k) out[k] = h[k] ? (float)((double)h[k] - (double)base) : -1e30f;
            out[255] = (float)h[255];
            *n = 256; return;
        } else if (w == "fused_stage_trace") {  // AHA_STAGE_TRACE builds: 4 stamps per ring stage of the traced CTA, ns relative to the earliest stamp (0 = missing)
            AHA_REQUIRE(T.d_ftrace && cap >= 4 * 8192, "fused trace not available");
            std::vector<unsigned long long> h(4 * 8192);
            AHA_CUDA_CHECK(cudaMemcpy(h.data(), T.d_ftrace + 8192, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
            unsigned long long base = ~0ull;
            for (auto v : h) if (v && v < base) base = v;
            for (size_t k = 0; k < h.size(); ++k) out[k] = h[k] ? (float)((double)(h[k] - base) + 1.0) : 0.f;
            AHA_CUDA_CHECK(cudaMemset(T.d_ftrace + 8192, 0, h.size() * sizeof(unsigned long long)));
            *n = h.size(); return;
        } else if (w == "fused_sync_trace") {  // AHA_STAGE_TRACE builds, dbg bit10: [0, 4096) = 8 words per grid barrier, [4096, 8192) = 4 per activation load
            AHA_REQUIRE(T.d_ftrace && cap >= 8192, "fused trace not available");
            std::vector<unsigned long long> h(8192);
            AHA_CUDA_CHECK(cudaMemcpy(h.data(), T.d_ftrace + 8192 + 32768, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
            unsigned long long base = ~0ull;
            for (auto v : h) if (v > 1000000000000ull && v < base) base = v;
            for (size_t k = 0; k < h.size(); ++k) out[k] = h[k] > 1000000000000ull ? (float)((double)(h[k] - base) + 1.0) : (float)h[k];   // small values are counts
            AHA_CUDA_CHECK(cudaMemset(T.d_ftrace + 8192 + 32768, 0, h.size() * sizeof(unsigned long long)));
            *n = h.size(); return;
        } else if (w == "logits") {   // logits of the last prefill / decode step (what the step's argmax was taken over)
            AHA_REQUIRE(T.tp_world == 1, "logits: the tensor-parallel ranks hold vocabulary shards");
            src = T.logits; cnt = (size_t)T.cfg.V;
        } else if (w == "batch_graphs") {   // step graphs captured in the open batch session (wide: at most one per running count)
            AHA_REQUIRE(cap >= 1, "out too small");
            out[0] = (float)(m->sess().graphs.size() + (m->session.wide ? m->spec.steps.size() : 0)); *n = 1; return;
        } else if (w == "spec_graphs") {    // pass graphs of speculative requests (one per row count R)
            AHA_REQUIRE(cap >= 1, "out too small");
            out[0] = (float)m->spec.graphs.size(); *n = 1; return;
        } else if (w == "rope_delta") {
            AHA_REQUIRE(cap >= 1, "out too small");
            out[0] = (float)m->rope_delta; *n = 1; return;
        } else {
            throw std::runtime_error("unknown debug tensor '" + w + "'");
        }
        AHA_REQUIRE(cnt <= cap, "out too small");
        AHA_CUDA_CHECK(cudaMemcpyAsync(out, src, cnt * sizeof(float), cudaMemcpyDeviceToHost, m->ctx.stream));
        AHA_CUDA_CHECK(cudaStreamSynchronize(m->ctx.stream));
        *n = cnt;
    });
}

}  // extern "C"
