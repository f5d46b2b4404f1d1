// aha_b200.hpp -- header-only C++17 host mirror of aha's model-executor seam on top of the C ABI (aha_b200.h).
//
// The reference's host side is compiled code (Rust).  Its seam is
//     trait InferenceModel { forward_initial, forward_step, clear_cache, stop_token_ids }
//         (src/models/common/mod.rs:25-45)
// driven by generate_generic (src/models/common/generate.rs:115-159) through a GenerationContext
// (generate.rs:21-68) and sample_and_push (generate.rs:70-86, sample.rs:13-60).  This header restates exactly that
// surface in C++ -- same names, same argument meaning, same error behaviour (errors are values in Rust, exceptions
// here; nothing crosses the C ABI as an exception) -- so a C++ host can drive the library the way `aha run` drives
// its models, and so the Rust shim of INTEGRATION.md has a compiled twin that is exercised by the tests.
//
//   aha::InferenceModel            the trait
//   aha::B200Model                 impl InferenceModel over an aha_model* handle (owns it; move-only)
//   aha::GenerationContext         offsets / sampling parameters of one request
//   aha::generate_generic          the reference's host loop over the trait (one forward_step call per token)
//   aha::B200Model::generate       the same request with the decode loop on the device (aha_b200_generate)
#pragma once
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <optional>
#include <stdexcept>
#include <string>
#include <unordered_set>
#include <utility>
#include <vector>

#include "aha_b200.h"

namespace aha {

struct Error : std::runtime_error {
    using std::runtime_error::runtime_error;
};

// MultiModalData (src/models/common/mod.rs:14-22): positional tensors, see aha_mm in aha_b200.h.
struct MultiModalData {
    std::vector<aha_tensor_desc> data_vec;
    static aha_tensor_desc absent() { return aha_tensor_desc{nullptr, AHA_F32, 0, {0}, nullptr}; }
    static aha_tensor_desc tensor(const void* data, int32_t dtype, std::initializer_list<int64_t> shape) {
        aha_tensor_desc d{nullptr, dtype, (int32_t)shape.size(), {0}, data};
        int i = 0;
        for (int64_t s : shape) d.shape[i++] = s;
        return d;
    }
    // Qwen3-VL: [pixel_values (N, 1536) f32, image_grid_thw (n, 3) u32, -, -, -]  (qwen3vl/generate.rs:88-94)
    static MultiModalData image(const float* pixel_values, int64_t n_patches, int64_t patch_dim, const uint32_t* grid_thw, int64_t n_images) {
        MultiModalData m;
        m.data_vec = {tensor(pixel_values, AHA_F32, {n_patches, patch_dim}), tensor(grid_thw, AHA_U32, {n_images, 3}), absent(), absent(), absent()};
        return m;
    }
    // Qwen3-ASR: [input_features (n_mels, T) f32]  (qwen3_asr/model.rs:405-411)
    static MultiModalData audio(const float* mel, int64_t n_mels, int64_t n_frames) {
        MultiModalData m;
        m.data_vec = {tensor(mel, AHA_F32, {n_mels, n_frames})};
        return m;
    }
    aha_mm view() const { return aha_mm{data_vec.data(), data_vec.size()}; }
};

// trait InferenceModel (src/models/common/mod.rs:25-45).  Logits come back as (1, 1, V) in the
// reference and are cast to f32 by the caller (generate.rs:75): here they are V floats.
class InferenceModel {
public:
    virtual ~InferenceModel() = default;
    virtual std::vector<float> forward_initial(const std::vector<uint32_t>& input_ids, size_t seqlen_offset, const MultiModalData* data) = 0;
    virtual std::vector<float> forward_step(const std::vector<uint32_t>& input_ids, size_t seqlen_offset) = 0;
    virtual void clear_cache() = 0;
    virtual std::vector<uint32_t> stop_token_ids() const = 0;
    // The ArgMax sampler fused behind the same calls: the token instead of 600 KB of logits (used by generate_generic
    // when the request is greedy without repeat penalty).  Default: argmax of the logits on the host.
    virtual uint32_t forward_initial_argmax(const std::vector<uint32_t>& ids, size_t off, const MultiModalData* data) { return argmax(forward_initial(ids, off, data)); }
    virtual uint32_t forward_step_argmax(const std::vector<uint32_t>& ids, size_t off) { return argmax(forward_step(ids, off)); }
    static uint32_t argmax(const std::vector<float>& v) {   // Sampling::ArgMax: first maximal index
        size_t b = 0;
        for (size_t i = 1; i < v.size(); ++i) if (v[i] > v[b]) b = i;
        return (uint32_t)b;
    }
};

struct Usage {   // generate.rs:126-145
    uint32_t prompt_tokens = 0, completion_tokens = 0;
    double prompt_secs = 0, completion_secs = 0, vision_secs = 0;
};

// GenerationContext (generate.rs:21-68) for the deterministic sampler.  temperature < 1e-7 (or unset) selects
// Sampling::ArgMax (sample.rs:13); anything else needs candle's LogitsProcessor RNG and is rejected, like the library.
struct GenerationContext {
    float repeat_penalty = 1.0f;   // sample.rs:46: 1.0 = off
    size_t repeat_last_n = 64;     // generate.rs:47
    size_t seqlen_offset = 0;
    size_t seq_len = 0;
    size_t sample_len = 1024;      // generate.rs:408-409
    GenerationContext(std::optional<float> temperature, std::optional<float> repeat_penalty_, std::optional<size_t> repeat_last_n_,
                      size_t initial_seq_len, size_t max_tokens)
        : repeat_penalty(repeat_penalty_.value_or(1.0f)), repeat_last_n(repeat_last_n_.value_or(64)), seq_len(initial_seq_len), sample_len(max_tokens) {
        if (temperature && *temperature >= 1e-7f) throw Error("non-greedy sampling is not implemented (candle LogitsProcessor RNG)");
    }
    bool plain_argmax() const { return repeat_penalty == 1.0f || repeat_last_n == 0; }
    std::vector<uint32_t> prepare_for_next_token(uint32_t token) {   // generate.rs:60-67
        seqlen_offset += seq_len;
        seq_len = 1;
        return {token};
    }
};

// candle_transformers::utils::apply_repeat_penalty over the last repeat_last_n generated tokens (sample.rs:40-60).
inline void apply_repeat_penalty(std::vector<float>& logits, float penalty, const std::vector<uint32_t>& generated, size_t last_n) {
    const size_t start = generated.size() > last_n ? generated.size() - last_n : 0;
    std::unordered_set<uint32_t> seen(generated.begin() + (std::ptrdiff_t)start, generated.end());
    for (uint32_t t : seen)
        if (t < logits.size()) logits[t] = logits[t] >= 0.f ? logits[t] / penalty : logits[t] * penalty;
}

// generate_generic (generate.rs:115-159) minus tokenizer / response building: prefill + first sample, then one
// forward_step per token; the first token is never EOS-checked, an EOS token is pushed before the break, the cache is
// cleared at the end.  Returns the generated ids.
inline std::vector<uint32_t> generate_generic(InferenceModel& model, const std::vector<uint32_t>& input_ids, const MultiModalData* data,
                                              GenerationContext ctx, Usage* usage = nullptr) {
    using clock = std::chrono::steady_clock;
    std::vector<uint32_t> generated;
    const std::vector<uint32_t> eos = model.stop_token_ids();
    auto is_eos = [&](uint32_t t) { for (uint32_t e : eos) if (e == t) return true; return false; };
    auto sample_and_push = [&](bool initial, const std::vector<uint32_t>& ids) {   // generate.rs:70-86
        uint32_t tok;
        if (ctx.plain_argmax()) {
            tok = initial ? model.forward_initial_argmax(ids, ctx.seqlen_offset, data) : model.forward_step_argmax(ids, ctx.seqlen_offset);
        } else {
            std::vector<float> logits = initial ? model.forward_initial(ids, ctx.seqlen_offset, data) : model.forward_step(ids, ctx.seqlen_offset);
            apply_repeat_penalty(logits, ctx.repeat_penalty, generated, ctx.repeat_last_n);
            tok = InferenceModel::argmax(logits);
        }
        generated.push_back(tok);
        return tok;
    };
    auto t0 = clock::now();
    uint32_t tok = sample_and_push(true, input_ids);
    const double prompt_secs = std::chrono::duration<double>(clock::now() - t0).count();
    std::vector<uint32_t> ids = ctx.prepare_for_next_token(tok);
    t0 = clock::now();
    for (size_t i = 1; i < ctx.sample_len; ++i) {
        tok = sample_and_push(false, ids);
        if (is_eos(tok)) break;
        ids = ctx.prepare_for_next_token(tok);
    }
    const double completion_secs = std::chrono::duration<double>(clock::now() - t0).count();
    model.clear_cache();
    if (usage) {
        usage->prompt_tokens = (uint32_t)input_ids.size();
        usage->completion_tokens = (uint32_t)generated.size();
        usage->prompt_secs = prompt_secs;
        usage->completion_secs = completion_secs;
    }
    return generated;
}

// impl InferenceModel for this library: XModel::new(cfg, VarBuilder, eos_ids) == the constructor.
class B200Model final : public InferenceModel {
public:
    B200Model(const std::string& kind, const std::string& config_json, const std::vector<aha_tensor_desc>& weights,
              const std::vector<uint32_t>& eos_ids = {}, const aha_options* opts = nullptr) {
        if (aha_b200_create(kind.c_str(), config_json.c_str(), weights.data(), weights.size(), eos_ids.data(), eos_ids.size(), opts, &h_) != 0) {
            const char* msg = aha_b200_last_error(nullptr);
            throw Error(msg ? msg : "aha_b200_create failed");
        }
    }
    ~B200Model() override { if (h_) aha_b200_destroy(h_); }
    B200Model(const B200Model&) = delete;
    B200Model& operator=(const B200Model&) = delete;
    B200Model(B200Model&& o) noexcept : h_(std::exchange(o.h_, nullptr)), vocab_(o.vocab_) {}
    B200Model& operator=(B200Model&& o) noexcept {
        if (this != &o) { if (h_) aha_b200_destroy(h_); h_ = std::exchange(o.h_, nullptr); vocab_ = o.vocab_; }
        return *this;
    }
    void set_vocab_size(size_t v) { vocab_ = v; }   // logits length (config.json vocab_size); needed by the logits-returning calls

    std::vector<float> forward_initial(const std::vector<uint32_t>& ids, size_t off, const MultiModalData* data) override {
        std::vector<float> logits(need_vocab());
        const aha_mm mm = data ? data->view() : aha_mm{nullptr, 0};
        check(aha_b200_forward_initial(h_, ids.data(), ids.size(), off, data ? &mm : nullptr, logits.data(), nullptr));
        return logits;
    }
    std::vector<float> forward_step(const std::vector<uint32_t>& ids, size_t off) override {
        std::vector<float> logits(need_vocab());
        check(aha_b200_forward_step(h_, ids.data(), ids.size(), off, logits.data(), nullptr));
        return logits;
    }
    uint32_t forward_initial_argmax(const std::vector<uint32_t>& ids, size_t off, const MultiModalData* data) override {
        uint32_t tok = 0;
        const aha_mm mm = data ? data->view() : aha_mm{nullptr, 0};
        check(aha_b200_forward_initial(h_, ids.data(), ids.size(), off, data ? &mm : nullptr, nullptr, &tok));
        return tok;
    }
    uint32_t forward_step_argmax(const std::vector<uint32_t>& ids, size_t off) override {
        uint32_t tok = 0;
        check(aha_b200_forward_step(h_, ids.data(), ids.size(), off, nullptr, &tok));
        return tok;
    }
    void clear_cache() override { check(aha_b200_clear_cache(h_)); }
    std::vector<uint32_t> stop_token_ids() const override {
        std::vector<uint32_t> out(aha_b200_stop_token_ids(h_, nullptr, 0));
        if (!out.empty()) aha_b200_stop_token_ids(h_, out.data(), out.size());
        return out;
    }
    // Token automata of constrained requests (aha_b200_fsm_create): the id goes into generate() / BatchRequest::fsm_id.
    uint32_t fsm_create(const aha_token_fsm& fsm) {
        uint32_t id = 0;
        check(aha_b200_fsm_create(h_, &fsm, &id));
        return id;
    }
    void fsm_destroy(uint32_t id) { check(aha_b200_fsm_destroy(h_, id)); }
    // Logit-rules objects (OpenAI presence_penalty / frequency_penalty / logit_bias, aha_b200_rules_create): the id goes into generate() /
    // BatchRequest::rules_id.  An automaton named in the object (aha_logit_rules::fsm) constrains the request too.
    uint32_t rules_create(const aha_logit_rules& rules) {
        uint32_t id = 0;
        check(aha_b200_rules_create(h_, &rules, &id));
        return id;
    }
    void rules_destroy(uint32_t id) { check(aha_b200_rules_destroy(h_, id)); }
    // LoRA adapters (aha_b200_lora_create): PEFT-named lora_A / lora_B tensors and lora_alpha / r; the id goes into batch_add_lora.
    uint32_t lora_create(const std::vector<aha_tensor_desc>& tensors, float scale) {
        uint32_t id = 0;
        check(aha_b200_lora_create(h_, tensors.data(), tensors.size(), scale, &id));
        return id;
    }
    void lora_destroy(uint32_t id) { check(aha_b200_lora_destroy(h_, id)); }
    // The whole request with the decode loop on the device (generate_generic semantics, aha_b200_generate).
    // reuse_prefix (new design; the reference clears the cache after every request, generate.rs:147): keep the K/V of this request and
    // prefill only what follows the prefix the prompt shares with the cache -- same tokens, shorter time to the first one.
    // fsm_id (non-zero): every token is drawn from the tokens that automaton allows (AHA_GEN_CONSTRAINED).
    // rules_id (non-zero): the logit rules of that object apply to every draw (AHA_GEN_LOGIT_RULES); give at most one of the two ids.
    std::vector<uint32_t> generate(const std::vector<uint32_t>& ids, const MultiModalData* data, const GenerationContext& ctx, Usage* usage = nullptr,
                                   bool reuse_prefix = false, uint32_t fsm_id = 0, uint32_t rules_id = 0) {
        aha_gen_params p{};
        p.temperature = 0.f; p.repeat_penalty = ctx.repeat_penalty; p.repeat_last_n = (int32_t)ctx.repeat_last_n; p.max_tokens = (uint32_t)ctx.sample_len;
        if (reuse_prefix) p.flags |= AHA_GEN_REUSE_PREFIX;
        if (fsm_id) { p.flags |= AHA_GEN_CONSTRAINED; p.reserved = fsm_id; }
        if (rules_id) { p.flags |= AHA_GEN_LOGIT_RULES; p.reserved = rules_id; }
        std::vector<uint32_t> out(ctx.sample_len);
        size_t n = 0;
        aha_usage u{};
        const aha_mm mm = data ? data->view() : aha_mm{nullptr, 0};
        check(aha_b200_generate(h_, ids.data(), ids.size(), data ? &mm : nullptr, &p, out.data(), out.size(), &n, &u));
        out.resize(n);
        if (usage) *usage = Usage{u.prompt_tokens, u.completion_tokens, u.prompt_secs, u.completion_secs, u.vision_secs};
        return out;
    }
    // Static batching (aha_b200_generate_batch): up to 8 requests decoded in lockstep; result i is what generate() returns for request i alone.
    struct BatchRequest { std::vector<uint32_t> ids; const MultiModalData* data = nullptr; GenerationContext ctx; uint32_t fsm_id = 0; uint32_t rules_id = 0; };
    std::vector<std::vector<uint32_t>> generate_batch(const std::vector<BatchRequest>& reqs, std::vector<Usage>* usage = nullptr) {
        const size_t n = reqs.size();
        std::vector<aha_batch_request> r(n);
        std::vector<aha_mm> mms(n);
        size_t cap = 1;
        for (size_t i = 0; i < n; ++i) {
            if (reqs[i].data) mms[i] = reqs[i].data->view();
            r[i].ids = reqs[i].ids.data(); r[i].seq_len = reqs[i].ids.size(); r[i].mm = reqs[i].data ? &mms[i] : nullptr;
            r[i].params = aha_gen_params{};
            r[i].params.repeat_penalty = reqs[i].ctx.repeat_penalty; r[i].params.repeat_last_n = (int32_t)reqs[i].ctx.repeat_last_n;
            r[i].params.max_tokens = (uint32_t)reqs[i].ctx.sample_len;
            if (reqs[i].fsm_id) { r[i].params.flags |= AHA_GEN_CONSTRAINED; r[i].params.reserved = reqs[i].fsm_id; }
            if (reqs[i].rules_id) { r[i].params.flags |= AHA_GEN_LOGIT_RULES; r[i].params.reserved = reqs[i].rules_id; }
            cap = std::max(cap, reqs[i].ctx.sample_len);
        }
        std::vector<uint32_t> out(n * cap);
        std::vector<size_t> n_out(n);
        std::vector<aha_usage> us(n);
        check(aha_b200_generate_batch(h_, r.data(), n, out.data(), cap, n_out.data(), us.data()));
        std::vector<std::vector<uint32_t>> res(n);
        for (size_t i = 0; i < n; ++i) res[i].assign(out.begin() + (std::ptrdiff_t)(i * cap), out.begin() + (std::ptrdiff_t)(i * cap + n_out[i]));
        if (usage) {
            usage->clear();
            for (const aha_usage& u : us) usage->push_back(Usage{u.prompt_tokens, u.completion_tokens, u.prompt_secs, u.completion_secs, u.vision_secs});
        }
        return res;
    }
    // OpenAI `n` (aha_b200_generate_n): n (1..8) choices of one request, the prompt prefilled once; choice i is what generate() with the
    // same params returns for seed seeds[i] (seeds empty: params.seed + i).  params carries the sampler (temperature, top_k, top_p, ...).
    std::vector<std::vector<uint32_t>> generate_n(const std::vector<uint32_t>& ids, const MultiModalData* data, const aha_gen_params& params, size_t n,
                                                  const std::vector<uint64_t>& seeds = {}, std::vector<Usage>* usage = nullptr) {
        if (!seeds.empty() && seeds.size() != n) throw Error("generate_n: seeds must be empty or hold n seeds");
        const size_t cap = std::max<size_t>(params.max_tokens, 1);
        std::vector<uint32_t> out(n * cap);
        std::vector<size_t> n_out(n);
        std::vector<aha_usage> us(n);
        const aha_mm mm = data ? data->view() : aha_mm{nullptr, 0};
        check(aha_b200_generate_n(h_, ids.data(), ids.size(), data ? &mm : nullptr, &params, n, seeds.empty() ? nullptr : seeds.data(), out.data(),
                                  nullptr, cap, n_out.data(), us.data()));
        std::vector<std::vector<uint32_t>> res(n);
        for (size_t i = 0; i < n; ++i) res[i].assign(out.begin() + (std::ptrdiff_t)(i * cap), out.begin() + (std::ptrdiff_t)(i * cap + n_out[i]));
        if (usage) {
            usage->clear();
            for (const aha_usage& u : us) usage->push_back(Usage{u.prompt_tokens, u.completion_tokens, u.prompt_secs, u.completion_secs, u.vision_secs});
        }
        return res;
    }
    // Speculative decoding of one greedy request (aha_b200_generate_speculative): verify passes of max_draft + 1 rows drafted from
    // `prediction` and, with prompt_lookup, from the prompt and the output so far.  The ids do not depend on the drafts.
    std::vector<uint32_t> generate_speculative(const std::vector<uint32_t>& ids, const MultiModalData* data, const GenerationContext& ctx,
                                               const std::vector<uint32_t>& prediction, bool prompt_lookup = false, uint32_t max_draft = 7,
                                               uint32_t ngram = 0, Usage* usage = nullptr, aha_spec_stats* stats = nullptr) {
        aha_gen_params p{};
        p.temperature = 0.f; p.repeat_penalty = ctx.repeat_penalty; p.repeat_last_n = (int32_t)ctx.repeat_last_n; p.max_tokens = (uint32_t)ctx.sample_len;
        aha_spec_params s{};
        s.prediction = prediction.empty() ? nullptr : prediction.data(); s.n_prediction = prediction.size();
        s.max_draft = max_draft; s.ngram = ngram; s.flags = prompt_lookup ? AHA_SPEC_PROMPT_LOOKUP : 0u;
        std::vector<uint32_t> out(std::max<size_t>(ctx.sample_len, 1));
        size_t n = 0;
        aha_usage u{};
        const aha_mm mm = data ? data->view() : aha_mm{nullptr, 0};
        check(aha_b200_generate_speculative(h_, ids.data(), ids.size(), data ? &mm : nullptr, &p, &s, out.data(), nullptr, out.size(), &n, &u, stats));
        out.resize(n);
        if (usage) *usage = Usage{u.prompt_tokens, u.completion_tokens, u.prompt_secs, u.completion_secs, u.vision_secs};
        return out;
    }
    // A greedy speculative request into the open wide session (aha_b200_batch_add_speculative), stepped by batch_step_spec.
    struct Admitted { int32_t slot; uint32_t first_token; bool finished; };
    Admitted batch_add_speculative(const std::vector<uint32_t>& ids, const MultiModalData* data, const GenerationContext& ctx,
                                   const std::vector<uint32_t>& prediction, bool prompt_lookup = false, uint32_t max_draft = 7, uint32_t ngram = 0) {
        const aha_mm mm = data ? data->view() : aha_mm{nullptr, 0};
        aha_batch_request r{};
        r.ids = ids.data(); r.seq_len = ids.size(); r.mm = data ? &mm : nullptr;
        r.params.repeat_penalty = ctx.repeat_penalty; r.params.repeat_last_n = (int32_t)ctx.repeat_last_n; r.params.max_tokens = (uint32_t)ctx.sample_len;
        aha_spec_params s{};
        s.prediction = prediction.empty() ? nullptr : prediction.data(); s.n_prediction = prediction.size();
        s.max_draft = max_draft; s.ngram = ngram; s.flags = prompt_lookup ? AHA_SPEC_PROMPT_LOOKUP : 0u;
        Admitted a{-1, 0, false};
        int32_t fin = 0;
        check(aha_b200_batch_add_speculative(h_, &r, &s, &a.slot, &a.first_token, &fin, nullptr));
        a.finished = fin != 0;
        return a;
    }
    // Requests into the open wide session, request i running adapter adapters[i] (0: the base model); all or nothing.
    std::vector<Admitted> batch_add_lora(const std::vector<aha_batch_request>& reqs, const std::vector<uint32_t>& adapters) {
        if (adapters.size() != reqs.size()) throw std::runtime_error("batch_add_lora: one adapter id per request");
        const size_t n = reqs.size();
        std::vector<int32_t> slots(n), fin(n);
        std::vector<uint32_t> first(n);
        check(aha_b200_batch_add_lora(h_, reqs.data(), adapters.data(), n, slots.data(), first.data(), fin.data(), nullptr));
        std::vector<Admitted> out(n);
        for (size_t i = 0; i < n; ++i) out[i] = Admitted{slots[i], first[i], fin[i] != 0};
        return out;
    }
    // One step of every running request of the open session (aha_b200_batch_step_spec), `width` = the session width: per slot its status
    // (0 idle, 1 continues, 2 finished) and the tokens it delivered (1 for a plain request, 1 .. max_draft + 1 for a speculative one).
    struct SlotStep { int32_t status; std::vector<uint32_t> tokens; };
    std::vector<SlotStep> batch_step_spec(size_t width) {
        std::vector<uint32_t> tok(width * AHA_SPEC_MAX_ROWS), n_tok(width);
        std::vector<int32_t> status(width);
        check(aha_b200_batch_step_spec(h_, tok.data(), n_tok.data(), status.data(), width, nullptr));
        std::vector<SlotStep> res(width);
        for (size_t i = 0; i < width; ++i) {
            res[i].status = status[i];
            res[i].tokens.assign(tok.begin() + (std::ptrdiff_t)(i * AHA_SPEC_MAX_ROWS), tok.begin() + (std::ptrdiff_t)(i * AHA_SPEC_MAX_ROWS + n_tok[i]));
        }
        return res;
    }
    size_t last_prefix_hit() const { return aha_b200_last_prefix_hit(h_); }
    // The open batch session's prefix cache (aha_b200_batch_prefix_cache / _stats): on with max_tokens > 0, off (its pages released) with 0.
    // batch_prefix_stats' hits: per slot of the session (width entries), the prompt tokens its running request took from the cache.
    void batch_prefix_cache(size_t max_tokens) { check(aha_b200_batch_prefix_cache(h_, max_tokens)); }
    aha_prefix_stats batch_prefix_stats(std::vector<size_t>* hits = nullptr, size_t width = 64) const {
        aha_prefix_stats st{};
        if (hits) hits->assign(width, 0);
        check(aha_b200_batch_prefix_stats(h_, &st, hits ? hits->data() : nullptr, hits ? width : 0));
        return st;
    }
    // Cancel, suspend and resume requests of the open session (aha_b200_batch_swap_space / _cancel / _suspend / _resume / _discard):
    // batch_suspend returns the suspended request's id, batch_resume the slot it went back into.
    void batch_swap_space(size_t max_tokens) { check(aha_b200_batch_swap_space(h_, max_tokens)); }
    void batch_cancel(int32_t slot) { check(aha_b200_batch_cancel(h_, slot)); }
    uint32_t batch_suspend(int32_t slot) {
        uint32_t id = 0;
        check(aha_b200_batch_suspend(h_, slot, &id));
        return id;
    }
    int32_t batch_resume(uint32_t id) {
        int32_t slot = -1;
        check(aha_b200_batch_resume(h_, id, &slot));
        return slot;
    }
    void batch_discard(uint32_t id) { check(aha_b200_batch_discard(h_, id)); }
    aha_swap_stats batch_swap_stats() const {
        aha_swap_stats st{};
        check(aha_b200_batch_swap_stats(h_, &st));
        return st;
    }
    // Prefill continuation (aha_b200_forward_extend): further prompt tokens against the `off` tokens already in the cache.
    std::vector<float> forward_extend(const std::vector<uint32_t>& ids, size_t off) {
        std::vector<float> logits(need_vocab());
        check(aha_b200_forward_extend(h_, ids.data(), ids.size(), off, logits.data(), nullptr));
        return logits;
    }
    aha_model* handle() const { return h_; }

private:
    void check(int rc) const { if (rc != 0) throw Error(aha_b200_last_error(h_)); }
    size_t need_vocab() const {
        if (!vocab_) throw Error("set_vocab_size() first: the logits-returning calls need the vocabulary size");
        return vocab_;
    }
    aha_model* h_ = nullptr;
    size_t vocab_ = 0;
};

// How many leading tokens of `ids` a cache holding `cached` supplies (the rule behind AHA_GEN_REUSE_PREFIX, aha_b200_prefix_match).
inline size_t prefix_match(const std::vector<uint32_t>& cached, const std::vector<uint32_t>& ids, const std::vector<uint32_t>& mm_token_ids = {},
                           bool same_mm = true) {
    return aha_b200_prefix_match(cached.data(), cached.size(), ids.data(), ids.size(), mm_token_ids.data(), mm_token_ids.size(), same_mm ? 1 : 0);
}

// Qwen3VLModel::get_rope_index on the host (aha_b200_rope_index): (3, S) position ids and rope_delta.
inline std::pair<std::vector<int32_t>, int32_t> rope_index(const std::vector<uint32_t>& ids, const std::vector<uint32_t>& grid_thw, uint32_t spatial_merge_size,
                                                           uint32_t image_token_id, uint32_t vision_start_token_id) {
    std::vector<int32_t> pos(3 * ids.size());
    int32_t delta = 0;
    if (aha_b200_rope_index(ids.data(), ids.size(), grid_thw.data(), grid_thw.size() / 3, spatial_merge_size, image_token_id, vision_start_token_id,
                            pos.data(), &delta) != 0)
        throw Error(aha_b200_last_error(nullptr));
    return {std::move(pos), delta};
}

}  // namespace aha
