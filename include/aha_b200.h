/*
 * aha_b200.h -- C ABI of libaha_b200.so: an H100-native (sm_90a) prefill + decode path for
 * Qwen3 / Qwen3-VL / Qwen3-ASR that drops in behind jhqxxx/aha's model-executor seam.
 *
 * The reference has no FFI; its seam is the Rust trait
 *     trait InferenceModel { forward_initial, forward_step, clear_cache, stop_token_ids }
 *     (src/models/common/mod.rs:25-45)
 * consumed by generate_generic* (src/models/common/generate.rs:87-368) and, for ASR,
 * the inherent `forward` (src/models/qwen3_asr/generate.rs:153-155).
 * Each entry point below names the reference item it replaces.  INTEGRATION.md shows the Rust shim
 * (`impl InferenceModel for B200Model`) a maintainer would add.
 *
 * Rules of the ABI:
 *   - plain C types only; every call returns 0 on success, non-zero on error; the message is
 *     available from aha_b200_last_error(); nothing throws or aborts across the boundary;
 *   - the library owns all device memory (weights, paged KV pool, workspaces, CUDA graphs) behind the
 *     opaque handle; the caller owns every host buffer it passes; no host pointer is retained past
 *     a call (weights are copied to HBM during aha_b200_create);
 *   - a handle is NOT re-entrant (aha serialises requests behind a write lock,
 *     src/server/api.rs:31,117,131) but IS thread-migratable: every entry binds
 *     the CUDA device itself, no thread-local state;
 *   - there is no CPU fallback: if no sm_90 device is present, create fails.
 */
#ifndef AHA_B200_H
#define AHA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AHA_B200_ABI_VERSION 3

typedef struct aha_model aha_model;

/* candle DType subset carried across the boundary */
enum { AHA_F32 = 0, AHA_F16 = 1, AHA_BF16 = 2, AHA_U32 = 3, AHA_I64 = 4, AHA_U8 = 5 };

/* A contiguous row-major host tensor (what a candle Tensor flattens to). */
typedef struct aha_tensor_desc {
    const char* name;      /* checkpoint tensor name (weights) or NULL */
    int32_t dtype;         /* AHA_* */
    int32_t rank;
    int64_t shape[8];
    const void* data;      /* host pointer */
} aha_tensor_desc;

/* MultiModalData (src/models/common/mod.rs:14-22), positional like data_vec:
 * Qwen3-VL: [pixel_values, image_grid_thw, pixel_values_video, video_grid_thw, cache_position]
 *           (src/models/qwen3vl/generate.rs:88-94; length checked model.rs:1292-1296)
 * Qwen3-ASR: [input_features]  (src/models/qwen3_asr/model.rs:405-411)
 * An absent entry is a desc with data == NULL.  n must be 5 (VL) or 1 (ASR). */
typedef struct aha_mm {
    const aha_tensor_desc* data_vec;
    size_t n;
} aha_mm;

typedef struct aha_options {
    int32_t device;        /* CUDA ordinal (reference: Device::new_cuda(0), src/utils/mod.rs:36) */
    int32_t tp_rank;       /* tensor-parallel rank / world (new design, SURVEY 8e); 0/1 = single GPU */
    int32_t tp_world;
    int32_t max_ctx;       /* KV capacity in tokens (0 = 8192) */
    int32_t max_prefill;   /* largest S accepted by forward_initial (0 = max_ctx) */
    int32_t max_patches;   /* largest ViT patch count (0 = 16384); Qwen3-VL only */
    int32_t max_frames;    /* largest mel frame count (0 = 3000); Qwen3-ASR only */
    int32_t use_graph;     /* 1 = replay the decode step from a CUDA graph (default), 0 = eager launches */
    int32_t decode_impl;   /* 0 = auto (persistent fused step kernel where the model shape allows: grid-barrier version on one GPU,
                            * hybrid version under tensor parallelism), 1 = per-op kernels under a CUDA graph (validation twin),
                            * 3 = fused, grid-barrier version (single GPU only), 4 = fused hybrid (grid barriers inside the layer, tagged
                            * packets for the two residual-stream exchanges).  2 is refused. */
    int32_t gemm_impl;     /* 0 = auto, 1 = SIMT fp32, 2 = wgmma 128x128 tiles (split-fp16, fp32-exact), 3 = wgmma 128x256 tiles */
    const void* tp_comm;   /* opaque: ncclUniqueId bytes (128) when tp_world > 1, else NULL */
    int32_t reserved[8];   /* reserved[0]: prefill attention, 0 = tensor cores (wgmma kernel; split-fp16), 1 = fp32 SIMT twin, 2 = mma.sync kernel everywhere */
} aha_options;

typedef struct aha_gen_params {      /* ChatCompletionParameters subset used by generate_generic / GenerationContext::new (generate.rs:32-52) */
    float temperature;     /* < 1e-7 => Sampling::ArgMax (sample.rs:13), else softmax(logits / temperature) is sampled on the device */
    float repeat_penalty;  /* 1.0 = off (sample.rs:46); applied to the distinct tokens among the last repeat_last_n generated ones */
    int32_t repeat_last_n; /* default 64 (generate.rs:47); 0 = off */
    uint32_t max_tokens;   /* sample_len, already resolved by the caller (default 1024, generate.rs:408-409); 0 and 1 both yield one token */
    uint64_t seed;         /* StdRng::seed_from_u64(seed) (default 299792458 / 34562 for ASR) */
    float top_p;           /* <= 0 = None; with top_k: Sampling::TopKThenTopP, without: TopP */
    int32_t top_k;         /* <= 0 = None; <= 1024 on the device sampler */
    uint32_t flags;        /* AHA_GEN_* */
    uint32_t reserved;
} aha_gen_params;
#define AHA_GEN_EOS_ON_FIRST 1u  /* the first token ends the request too if it is a stop id (the ASR loop, qwen3_asr/generate.rs:152-168) */
#define AHA_GEN_CONTINUE_RNG 2u  /* keep drawing from the previous request's random stream (one LogitsProcessor across audio chunks) */
#define AHA_GEN_REUSE_PREFIX 4u  /* KV reuse across requests (SURVEY 8f rank 4; the reference clears the cache after every request, generate.rs:147):
                                  * leave this request's K/V in the paged cache and, at its start, prefill only what follows the longest prefix
                                  * the prompt shares with the cache (same token ids and the same multimodal tensors).  Tokens are unchanged. */
#define AHA_GEN_LOGPROBS 8u      /* one aha_logprobs record per generated token (OpenAI `logprobs`): aha_b200_generate_logprobs,
                                  * aha_b200_generate_stream_logprobs and batch sessions (aha_b200_batch_logprobs); the other entries refuse it */
#define AHA_GEN_TOP_LOGPROBS(n) ((uint32_t)(n) << 8)   /* OpenAI `top_logprobs`: n alternatives per record, in bits 8-15 of flags and up.
                                  * Not masked: a count above AHA_MAX_TOP_LOGPROBS (or above the vocabulary) is refused, never wrapped.
                                  * Needs AHA_GEN_LOGPROBS. */
#define AHA_MAX_TOP_LOGPROBS 20

/* The log-probability record of one generated token (new design; the reference's responses carry `logprobs: None`).
 *   logprob = x[token] - (M + log sum_j exp(x[j] - M)), x = the fp32 logits row the step computed, M = its maximum: the model's own
 *   distribution, taken BEFORE repeat penalty, temperature, top-k and top-p, so greedy and sampled requests report comparable numbers
 *   (a sampled token that top-k would have excluded still has a finite value);
 *   top_ids / top_logprobs[0 .. n_top): the n_top largest entries of x, by raw logit descending, ties by ascending id.  A greedy request
 *   without repeat penalty has token == top_ids[0] and logprob == top_logprobs[0] bit for bit.  Entries from n_top on are zero;
 *   index: the token's position in the request's output (0 = the first token, computed from the prefill logits);
 *   valid: 1 for a record, 0 for an aha_b200_batch_logprobs slot that holds none.
 * Computed on the device by one pair of kernels for every path, so a request's records are bit-identical whichever path computes them
 * from the same logits.  Single GPU only (tp_world > 1 is refused). */
typedef struct aha_logprobs {
    uint32_t token;
    uint32_t index;
    float logprob;
    uint32_t n_top;
    uint32_t top_ids[AHA_MAX_TOP_LOGPROBS];
    float top_logprobs[AHA_MAX_TOP_LOGPROBS];
    uint32_t valid;
    uint32_t reserved;
} aha_logprobs;

/* generate_stream: called once per generated token, in order, as soon as its step has completed (the device keeps running a few
 * steps ahead); a non-zero return ends the request (the reference's stream is dropped when the client goes away). */
typedef int (*aha_token_callback)(void* user, uint32_t token, uint32_t index);
/* generate_stream_logprobs: the same, with the token's record (valid for the duration of the call) */
typedef int (*aha_logprobs_callback)(void* user, uint32_t token, uint32_t index, const aha_logprobs* lp);

typedef struct aha_asr_chunk {       /* one AudioData of Qwen3AsrProcessor::process_info (qwen3_asr/processor.rs:181-184) */
    const uint32_t* ids;             /* prompt with the <|audio_pad|> run already expanded */
    size_t seq_len;
    aha_tensor_desc input_features;  /* log-mel (num_mel_bins, frames) */
} aha_asr_chunk;

typedef struct aha_usage {           /* Usage timing split (generate.rs:126-145) */
    uint32_t prompt_tokens;
    uint32_t completion_tokens;
    double prompt_secs;              /* forward_initial + first sample */
    double completion_secs;          /* the decode loop */
    double vision_secs;              /* device time of the ViT / audio tower inside prompt_secs */
} aha_usage;

typedef struct aha_stats {
    uint64_t kernel_launches;        /* kernels launched by this handle since create / last reset */
    uint64_t graph_launches;
    uint64_t kernels_per_decode_step;/* kernel nodes inside one decode-step graph */
    uint64_t weight_bytes;           /* bytes of weights resident in HBM */
    uint64_t kv_bytes_per_token;
    uint64_t decode_bytes_per_step_fixed; /* algorithmic weight bytes read per decode step */
} aha_stats;

/* XModel::new(cfg, VarBuilder, eos_ids) inside XGenerateModel::init
 * (src/models/qwen3/generate.rs:22-50, qwen3vl/generate.rs:33-63,
 *  qwen3_asr/generate.rs:51-87).  kind = "qwen3" | "qwen3vl" | "qwen3_asr"; config_json is the
 * checkpoint's config.json text; weights are the safetensors tensors by name. */
int aha_b200_create(const char* kind, const char* config_json,
                    const aha_tensor_desc* weights, size_t n_weights,
                    const uint32_t* eos_ids, size_t n_eos,
                    const aha_options* opts, aha_model** out);

/* InferenceModel::forward_initial (src/models/common/mod.rs:28-35;
 * Qwen3-VL model.rs:1285-1311; Qwen3-ASR model.rs:394-411).  ids: (1,S) u32.
 * logits_out: V floats or NULL; argmax_out: first-max index or NULL (ArgMax sampler on device). */
int aha_b200_forward_initial(aha_model* m, const uint32_t* ids, size_t seq_len, size_t seqlen_offset,
                             const aha_mm* mm, float* logits_out, uint32_t* argmax_out);

/* InferenceModel::forward_step (src/models/common/mod.rs:37-38). */
int aha_b200_forward_step(aha_model* m, const uint32_t* ids, size_t seq_len, size_t seqlen_offset,
                          float* logits_out, uint32_t* argmax_out);

/* Prefill continuation (new design -- the reference's (S, S) causal mask makes a multi-token call with a non-empty cache fail,
 * qwen3/model.rs:164-175): seq_len >= 1 further prompt tokens against a cache that holds exactly seqlen_offset tokens, with the
 * (S, offset + S) causal mask.  Text tokens only (multimodal rows belong to forward_initial; Qwen3-VL positions continue as
 * index + rope_delta, model.rs:1250-1264).  forward_initial(ids[0..a]) + forward_extend(ids[a..S], a) produces the logits of
 * forward_initial(ids[0..S]).  It is what aha_b200_generate runs after a prefix-cache hit, and what a prompt longer than
 * aha_options.max_prefill is cut into. */
int aha_b200_forward_extend(aha_model* m, const uint32_t* ids, size_t seq_len, size_t seqlen_offset,
                            float* logits_out, uint32_t* argmax_out);

/* Prompt tokens the last aha_b200_generate / _generate_stream call took from the cache instead of prefilling them
 * (0 without AHA_GEN_REUSE_PREFIX).  usage.prompt_tokens keeps counting the whole prompt, as the reference reports it. */
size_t aha_b200_last_prefix_hit(aha_model* m);

/* The rule behind AHA_GEN_REUSE_PREFIX, host only: the longest prefix of ids[0..n) whose K/V a cache holding cached[0..n_cached) can
 * supply = the common prefix, at most n - 1 (the last prompt token is always run), and 0 unless the multimodal tensors are the same
 * (same_mm) and every placeholder token (mm_token_ids: <|image_pad|>, <|video_pad|>, <|audio_pad|>) of both sequences lies inside it. */
size_t aha_b200_prefix_match(const uint32_t* cached, size_t n_cached, const uint32_t* ids, size_t n,
                             const uint32_t* mm_token_ids, size_t n_mm_tokens, int same_mm);
/* 64-bit fingerprint of a request's MultiModalData (dtype, shape and bytes of every present entry; 0 = no tensor).  Host only. */
uint64_t aha_b200_mm_fingerprint(const aha_mm* mm);

/* InferenceModel::clear_cache (mod.rs:41; Qwen3-VL also resets rope_deltas, model.rs:1279-1282). */
int aha_b200_clear_cache(aha_model* m);

/* InferenceModel::stop_token_ids (mod.rs:44).  Returns the count; writes up to cap ids. */
size_t aha_b200_stop_token_ids(aha_model* m, uint32_t* out, size_t cap);

/* generate_generic (src/models/common/generate.rs:115-159) with the ArgMax sampler:
 * prefill, then the decode loop entirely on the device (token feedback without host round trips),
 * first token never EOS-checked, EOS token pushed before the break, cache cleared at the end. */
int aha_b200_generate(aha_model* m, const uint32_t* ids, size_t seq_len, const aha_mm* mm,
                      const aha_gen_params* params, uint32_t* out_tokens, size_t cap, size_t* n_out,
                      aha_usage* usage);

/* Static batching (new design, SURVEY 8f rank 4: the reference serves one request at a time, server/api.rs:117): up to 8 independent
 * requests on one handle, each prefilled on its own page table of the shared paged KV pool, then decoded in LOCKSTEP -- one pass over the
 * weights per step serves every sequence.  Each request obeys generate_generic on its own (own sampler / seed / repeat penalty, an EOS
 * token ends that request only) and returns exactly the tokens aha_b200_generate returns for it alone.  out_tokens: [n][cap], n_out: [n],
 * usage: [n] or NULL.  The sum of ceil((seq_len + max_tokens) / 32) pages over the requests must fit max_ctx.  Single GPU. */
typedef struct aha_batch_request {
    const uint32_t* ids;
    size_t seq_len;
    const aha_mm* mm;                /* NULL for text-only models / prompts */
    aha_gen_params params;
} aha_batch_request;
int aha_b200_generate_batch(aha_model* m, const aha_batch_request* reqs, size_t n, uint32_t* out_tokens, size_t cap,
                            size_t* n_out, aha_usage* usage);

/* Continuous batching on the same slots and the same lockstep step (new design): requests join and leave a running batch BETWEEN steps.
 *   batch_open                      clear_cache, enter batch mode (the single-request entries are refused until batch_close / clear_cache)
 *   batch_add(req)                  prefill the request into a free slot (its own page table; pages come from the shared pool and go back the
 *                                   moment the request finishes) -> slot id, its first token, finished = 1 if that was also its last one
 *   batch_step(tokens[8], status[8]) one decode step for every running request: status 0 = slot idle, 1 = token delivered, request continues,
 *                                   2 = token delivered and it was the request's last (EOS or max_tokens): the slot is free again
 *   batch_close                     drop everything
 * Each request still yields exactly the ids aha_b200_generate yields for it alone, whenever it joins and whatever runs beside it. */
int aha_b200_batch_open(aha_model* m);
int aha_b200_batch_add(aha_model* m, const aha_batch_request* req, int32_t* slot_out, uint32_t* first_token_out,
                       int32_t* finished_out, aha_usage* usage /* prompt side only; may be NULL */);
/* Continuous batching: admit n requests at once.  Text-only requests that fit are packed into shared prefills (each attends only to
 * itself); a request with multimodal tensors, or one longer than max_prefill, is prefilled alone exactly as batch_add does it.
 * All or nothing: if the requests do not all fit (free slots, free KV pages) or one is malformed, nothing is admitted and the session
 * is unchanged.  Slots are assigned in input order, lowest free slot first (what n batch_add calls would assign, except that a request
 * finished at admission keeps its slot until the call returns).
 * Each request yields the ids its own generate_generic run yields; for prompts of 32 tokens or more (every prompt with gemm_impl 1)
 * exactly the ids batch_add gives it.  slots_out / first_tokens_out / finished_out: [n]; usage: [n] or NULL (prompt side only). */
int aha_b200_batch_add_many(aha_model* m, const aha_batch_request* reqs, size_t n, int32_t* slots_out,
                            uint32_t* first_tokens_out, int32_t* finished_out, aha_usage* usage);
int aha_b200_batch_step(aha_model* m, uint32_t* tokens_out /* [8] */, int32_t* status_out /* [8] */, size_t* n_stepped_out /* may be NULL */);
int aha_b200_batch_close(aha_model* m);
/* Wide continuous batching: a session of max_seqs (1..64) slots whose decode step runs every projection and the lm_head on the tensor
 * cores (wgmma, each weight streamed once per step for all running requests).  Requires no open session, a single GPU, and a model whose
 * projections all have row and column counts that are multiples of 64 (every Qwen3 / Qwen3-VL / Qwen3-ASR text stack); anything else is
 * refused with a message.  Requests are admitted with batch_add / batch_add_many (packing included) and the session ends with
 * batch_close or clear_cache, as for batch_open.  aha_options.gemm_impl still selects the admission prefill's GEMM; AHA_BATCH_GEMV does not
 * apply.  Buffers for 64 sequences are allocated on the first wide session of a handle and kept.
 * Results: every request yields the ids of its own generate_generic run.  They are bit-identical whichever slot it holds, whatever runs
 * beside it and at whatever step it joins, given the same admission entry (batch_add and batch_add_many differ below 32 prompt tokens).
 * They need NOT equal aha_b200_generate's ids or a narrow session's in the last bits: the tensor-core sums run in another order than the
 * CUDA-core GEMV's.  The narrow session (batch_open) keeps its own kernels and its bit-equality with single-request runs. */
int aha_b200_batch_open_wide(aha_model* m, size_t max_seqs);
/* batch_step over cap entries (cap >= the session width; works on narrow sessions too).  batch_step refuses a session wider than 8. */
int aha_b200_batch_step_n(aha_model* m, uint32_t* tokens_out /* [cap] */, int32_t* status_out /* [cap] */, size_t cap,
                          size_t* n_stepped_out /* may be NULL */);
/* Log-probabilities in a batch session (narrow or wide): a request asks with AHA_GEN_LOGPROBS [| AHA_GEN_TOP_LOGPROBS(n)] in its
 * params.flags.  out[slot] (cap >= the session width) receives the record of the last token the slot's request delivered -- by
 * batch_add, batch_add_many or the last step, including the step that finished it -- until another request takes the slot.  Slots whose
 * request did not ask, or that never held one, get valid = 0.  A step computes records only while a running request asks, so a session
 * without such requests launches exactly the kernels it launched before. */
int aha_b200_batch_logprobs(aha_model* m, aha_logprobs* out /* [cap] */, size_t cap);

/* WhisperFeatureExtractor::call (src/models/feature_extractor/
 * feature_extraction_whisper.rs:65-115): wave (n) f32 host -> log-mel (n_mels, n_frames) f32 host.
 * Returns frames through *n_frames.  Qwen3-ASR handles only. */
/* generate_stream_generic (common/generate.rs:231-368) minus tokenizer / SSE framing: tokens are delivered through on_token. */
int aha_b200_generate_stream(aha_model* m, const uint32_t* ids, size_t seq_len, const aha_mm* mm,
                             const aha_gen_params* params, aha_token_callback on_token, void* user, aha_usage* usage);
/* aha_b200_generate / _generate_stream with one aha_logprobs record per generated token (params.flags must carry AHA_GEN_LOGPROBS;
 * AHA_GEN_TOP_LOGPROBS(n) adds n alternatives).  out_logprobs: [cap] records, out_logprobs[i] belongs to out_tokens[i].  Tokens are
 * exactly those of aha_b200_generate.  The records travel with the tokens, a burst at a time (the streaming variant: each behind its
 * own step).  A handle allocates the record buffer the first time a request asks.  generate, generate_stream, generate_batch and
 * asr_generate refuse the flag. */
int aha_b200_generate_logprobs(aha_model* m, const uint32_t* ids, size_t seq_len, const aha_mm* mm, const aha_gen_params* params,
                               uint32_t* out_tokens, aha_logprobs* out_logprobs, size_t cap, size_t* n_out, aha_usage* usage);
int aha_b200_generate_stream_logprobs(aha_model* m, const uint32_t* ids, size_t seq_len, const aha_mm* mm, const aha_gen_params* params,
                                      aha_logprobs_callback on_token, void* user, aha_usage* usage);

/* Speculative decoding of one request (new design; the reference decodes one token per forward_step and ignores
 * ChatCompletionParameters.prediction, src/params/chat.rs:102-105).  After the normal prefill and first token the request runs in verify
 * passes of R = max_draft + 1 rows through one weight stream: row 0 is the last emitted token, rows 1..R-1 are drafted tokens at the
 * following positions.  A pass emits the longest run of drafts that the request's own sampler reproduces, plus the sampler's next token.
 *   Drafts: for n = min(ngram, emitted) down to 1, the last n emitted tokens are looked up first in `prediction` (OpenAI "Predicted
 *   Outputs": text the answer will largely repeat), then, with AHA_SPEC_PROMPT_LOOKUP, in the prompt followed by the tokens emitted so
 *   far.  The most recent occurrence that is followed by at least one token wins, and the up to max_draft tokens after it are the drafts.
 *   Exact: row r is sampled with draw index n_draws + r and the repeat-penalty context "history followed by drafts 1..r", which is what a
 *   sequential decode does with the same logits, so ids and records do not depend on the drafts, max_draft or use_graph.  A wrong draft
 *   costs time, never the answer.
 *   Numerics: the first token equals aha_b200_generate's.  The tokens after it follow the model as wide batch sessions do (tensor-core
 *   projections): they need NOT equal aha_b200_generate's in the last bits.
 *   Cost: every pass costs R rows, so a request whose drafts are rarely accepted runs SLOWER than aha_b200_generate.
 *   EOS inside an accepted run ends the request after the EOS token; max_tokens cuts a run.  KV pages for seq_len + max_tokens + max_draft
 *   tokens are mapped up front; a request that does not fit max_ctx is refused.  Single GPU, no open batch session, models whose
 *   projections tile by 64 with head_dim 128; Qwen3-ASR handles and AHA_GEN_REUSE_PREFIX / _CONTINUE_RNG / _EOS_ON_FIRST are refused.
 * out_logprobs: [cap] records when params.flags carries AHA_GEN_LOGPROBS, else may be NULL.  stats may be NULL. */
#define AHA_SPEC_PROMPT_LOOKUP 1u    /* also draft from the prompt and the tokens generated so far */
typedef struct aha_spec_params {
    const uint32_t* prediction;      /* the caller's predicted output (token ids), or NULL */
    size_t n_prediction;
    uint32_t max_draft;              /* 1..15 drafted tokens per pass (R = max_draft + 1 rows) */
    uint32_t ngram;                  /* longest suffix looked up, 1..8; 0 = default (3) */
    uint32_t flags;                  /* AHA_SPEC_PROMPT_LOOKUP */
    uint32_t reserved[3];
} aha_spec_params;
typedef struct aha_spec_stats {
    uint32_t passes;                 /* verify passes run */
    uint32_t drafted;                /* drafted tokens over all passes */
    uint32_t accepted;               /* drafted tokens that were emitted */
    uint32_t reserved;
} aha_spec_stats;
int aha_b200_generate_speculative(aha_model* m, const uint32_t* ids, size_t seq_len, const aha_mm* mm, const aha_gen_params* params,
                                  const aha_spec_params* spec, uint32_t* out_tokens, aha_logprobs* out_logprobs, size_t cap,
                                  size_t* n_out, aha_usage* usage, aha_spec_stats* stats);

/* Qwen3AsrGenerateModel::generate / generate_stream (qwen3_asr/generate.rs:130-268): per-chunk loop, stop on either EOS id
 * (the handle's stop ids), KV cache cleared per chunk, one sampler for the whole request.  on_token may be NULL. */
int aha_b200_asr_generate(aha_model* m, const aha_asr_chunk* chunks, size_t n_chunks, const aha_gen_params* params,
                          uint32_t* out_tokens, size_t cap, size_t* n_out, aha_token_callback on_token, void* user,
                          aha_usage* usage);

int aha_b200_mel_spectrogram(aha_model* m, const float* wave, size_t n_samples,
                             float* mel_out, size_t mel_cap, size_t* n_frames);

/* img_transform + process_vision_tensor (src/utils/img_utils.rs:272-294,
 * src/models/qwen3vl/processor.rs:174-251): u8 HWC image whose size already satisfies
 * img_smart_resize -> pixel_values (grid_t*grid_h*grid_w, 3*2*16*16) f32 host + grid_thw[3]. */
int aha_b200_image_patchify(aha_model* m, const uint8_t* img_hwc, size_t h, size_t w,
                            float* pixel_values_out, size_t cap, uint32_t grid_thw_out[3]);

/* Qwen3Embedding::embed_one (src/models/qwen3_embedding/mod.rs:50-64): forward_hidden over the ids
 * (offset 0), last-token hidden state after the final RMSNorm, L2-normalised (x / sqrt(sum x^2 + 1e-6),
 * src/models/common/modules.rs:1287-1294); the cache is cleared afterwards.  out: hidden_size floats.  "qwen3" handles. */
/* ---- processors (host side of Qwen3VLProcessor / Qwen3AsrProcessor; the *_resize / *_preprocess entries run on the GPU) ---- */
/* img_smart_resize (src/utils/img_utils.rs:297-331): (h, w) -> multiples of `factor` inside the pixel budget.  Host only. */
int aha_b200_img_smart_resize(uint32_t img_h, uint32_t img_w, uint32_t factor, uint32_t min_pixels, uint32_t max_pixels,
                              uint32_t* out_h, uint32_t* out_w);
/* DynamicImage::resize_exact(w, h, FilterType::CatmullRom) of an RGB8 image (qwen3vl/processor.rs:167) */
int aha_b200_image_resize(aha_model* m, const uint8_t* img_hwc, size_t h, size_t w, size_t new_h, size_t new_w, uint8_t* out_hwc);
/* Qwen3VLProcessor::process_img + process_vision_tensor for one image of ANY size (qwen3vl/processor.rs:151-251):
 * img_smart_resize -> CatmullRom resize -> img_transform -> frame duplication -> merge-block patch order */
int aha_b200_image_preprocess(aha_model* m, const uint8_t* img_hwc, size_t h, size_t w, uint32_t min_pixels, uint32_t max_pixels,
                              float* pixel_values_out, size_t cap, uint32_t grid_thw_out[3]);
/* <|image_pad|> / <|audio_pad|> expansion on token ids (qwen3vl/processor.rs:386-399, qwen3_asr/processor.rs:93-97): the i-th
 * occurrence of token_id becomes counts[i] copies.  out may be NULL to query n_out.  Host only. */
int aha_b200_expand_placeholders(const uint32_t* ids, size_t n, uint32_t token_id, const uint32_t* counts, size_t n_counts,
                                 uint32_t* out, size_t cap, size_t* n_out);
/* ---- video half of Qwen3VLProcessor (qwen3vl/processor.rs:253-307, 404-437, 447-571).  Decoding and scaling the file is ffmpeg's job in the
 * reference (a cargo feature) and stays with the caller; everything computed around it is here. ---- */
/* video_smart_resize (utils/video_utils.rs:9-59): frame size for a clip of num_frames frames inside the pixel budget; video_ratio = 16 as
 * get_video_data passes it (0 = None).  Host only. */
int aha_b200_video_smart_resize(uint32_t num_frames, uint32_t height, uint32_t width, uint32_t temporal_factor, uint32_t factor,
                                uint32_t min_pixels, uint32_t max_pixels, uint32_t video_ratio, uint32_t* out_h, uint32_t* out_w);
/* Frame sampling of get_video_data (processor.rs:481-491, 526-527): stream of total_frames frames at rate_num/rate_den per second, `fps` samples per
 * second clamped to [min_frames, max_frames] (the processor's 2, 4, 768) -> nframes (what video_smart_resize is given) and the kept indices
 * (every round(total/nframes)-th frame).  indices_out may be NULL to query n_out.  Host only. */
int aha_b200_video_sample_frames(uint32_t total_frames, uint32_t rate_num, uint32_t rate_den, uint32_t fps, uint32_t min_frames,
                                 uint32_t max_frames, uint32_t* nframes_out, uint32_t* indices_out, size_t cap, size_t* n_out);
/* calculate_timestamps (processor.rs:282-307): one stamp (seconds) per group of t_merge_size sampled frames.  Host only. */
int aha_b200_video_timestamps(const uint32_t* frame_indices, size_t n, float fps, uint32_t t_merge_size, float* stamps_out, size_t cap,
                              size_t* n_out);
/* format!("<{:.1} seconds>", stamp) (processor.rs:419): the text the caller tokenises for each frame group.  Host only. */
int aha_b200_format_timestamp(float seconds, char* out, size_t cap);
/* Qwen3VLProcessor::process_videos for one clip (processor.rs:253-280): n_frames RGB24 frames (T, H, W, 3) already at the size
 * video_smart_resize chose -> rescale + normalise + process_vision_tensor (last frame repeated up to a multiple of temporal_patch_size)
 * -> pixel_values_video (grid_t*grid_h*grid_w, 3*2*16*16) f32 host + video_grid_thw[3].  Runs on the GPU. */
int aha_b200_video_preprocess(aha_model* m, const uint8_t* frames_thwc, size_t n_frames, size_t h, size_t w,
                              float* pixel_values_out, size_t cap, uint32_t grid_thw_out[3]);
/* <|video_pad|> expansion of process_info (processor.rs:404-437) on token ids: video i becomes grid_t runs of
 * [stamp text ids, <|vision_start|>, h*w/merge^2 x <|video_pad|>, <|vision_end|>], replacing the first
 * <|vision_start|><|video_pad|><|vision_end|> triple if the prompt holds one, else the first lone <|video_pad|>.  stamp_ids/stamp_lens:
 * the tokenised "<x.x seconds>" strings of all frame groups of all videos, back to back.  out may be NULL to query n_out.  Host only. */
int aha_b200_expand_video_placeholders(const uint32_t* ids, size_t n, uint32_t video_token_id, uint32_t vision_start_token_id,
                                       uint32_t vision_end_token_id, const uint32_t* video_grid_thw, size_t n_videos,
                                       uint32_t merge_size, const uint32_t* stamp_ids, const uint32_t* stamp_lens, size_t n_stamps,
                                       uint32_t* out, size_t cap, size_t* n_out);
/* get_feat_extract_output_lengths (qwen3_asr/processor.rs:187-195).  Host only. */
size_t aha_b200_feat_extract_output_length(size_t n_frames);
/* float_range_normalize (common/modules.rs:1353-1368), in place.  Host only. */
int aha_b200_float_range_normalize(float* wave, size_t n);
/* resample_simple (utils/audio_utils.rs:66-255: windowed-sinc polyphase filter, lowpass width 6, rolloff 0.99, Hann), the
 * step load_audio_with_resample (audio_utils.rs:636-650) applies to bring a decoded mono waveform to the model's 16 kHz.  The filter bank
 * is built on the host in the reference's f32 arithmetic, the strided convolution runs on the GPU.  out may be NULL to query n_out
 * (= min(ceil(new * n / orig), frames * new) samples).  Equal frequencies return the waveform unchanged, like the reference. */
int aha_b200_resample(aha_model* m, const float* wave, size_t n, int64_t orig_freq, int64_t new_freq, float* out, size_t cap, size_t* n_out);
/* get_sinc_resample_kernel (audio_utils.rs:66-151) alone: taps_out[new/g][2*width + orig/g]; dims_out = {new/g, taps per phase, width, orig/g}.
 * taps_out may be NULL to query dims_out.  Host only. */
int aha_b200_sinc_resample_bank(int64_t orig_freq, int64_t new_freq, float* taps_out, size_t cap, int32_t dims_out[4]);
/* split_audio_into_chunks (utils/audio_utils.rs:1743-1760): chunk lengths in samples.  Host only. */
int aha_b200_split_audio_into_chunks(size_t total_len, uint32_t sample_rate, float max_chunk_sec, size_t* lens_out, size_t cap,
                                     size_t* n_out);

int aha_b200_embed(aha_model* m, const uint32_t* ids, size_t seq_len, float* out);
/* Qwen3Embedding::embed_multi (src/models/qwen3_embedding/mod.rs:38-48): embed_one for every text, computed as packed prefills.
 * ids: the n texts back to back; lens[n]: their lengths; out: [n][hidden_size] unit vectors, in input order.  "qwen3" handles,
 * single GPU.  The cache is cleared before and after, like aha_b200_embed. */
int aha_b200_embed_batch(aha_model* m, const uint32_t* ids, const size_t* lens, size_t n, float* out);
/* Qwen3Reranker::rerank (src/models/qwen3_reranker/mod.rs:23-31): cosine score of the query embedding
 * against each document embedding (cosine_similarity_no_l2 on unit vectors).  doc_ids holds the documents back to back,
 * doc_lens[n_docs] their lengths; scores_out: n_docs floats. */
int aha_b200_rerank(aha_model* m, const uint32_t* query_ids, size_t query_len, const uint32_t* doc_ids, const size_t* doc_lens,
                    size_t n_docs, float* scores_out);

/* Scoring given text (new design; the reference has no prompt log-probabilities): OpenAI `echo` + `logprobs`, evaluation harnesses
 * (lm-eval loglikelihood and is_greedy), perplexity, label likelihoods.
 * Log-probability of every given token from position `start` on: record i - start holds token ids[i], index i,
 * logprob = log p(ids[i] | ids[0..i)) and the n_top alternatives at that position (aha_logprobs semantics: raw model distribution,
 * (logit desc, id asc)).  1 <= start < seq_len <= max_ctx; prompts longer than max_prefill run as continuation chunks.  "qwen3" and
 * "qwen3vl" handles with text-only ids (Qwen3-VL positions of a text-only prompt), single GPU, no open batch session, n_top <= 20 and
 * <= V, cap >= seq_len - start.  Everything is refused before any device work.  The cache is cleared before and after, like
 * aha_b200_embed. */
int aha_b200_score(aha_model* m, const uint32_t* ids, size_t seq_len, size_t start, uint32_t n_top, aha_logprobs* out, size_t cap,
                   size_t* n_out);
/* The same for n texts packed into shared prefills (each text attends only to itself); starts == NULL means 1 for every text.  Records
 * text by text in input order, `index` relative to the text; *n_out = sum of (lens[j] - starts[j]).  A text longer than
 * min(max_prefill, max_ctx) is scored alone inside the same call. */
int aha_b200_score_batch(aha_model* m, const uint32_t* ids, const size_t* lens, const size_t* starts, size_t n, uint32_t n_top,
                         aha_logprobs* out, size_t cap, size_t* n_out);

/* Tensor parallelism (new design; the reference has none): rank 0 creates a 128-byte ncclUniqueId, the host side
 * distributes it (bench.py broadcasts it between the per-GPU processes) and every rank passes it in aha_options.tp_comm together
 * with tp_rank / tp_world.  Heads and MLP rows are sharded; the only exchange steps are all-reduce(sum) after
 * o_proj and down_proj. */
int aha_b200_nccl_unique_id(uint8_t out[128]);

void aha_b200_destroy(aha_model* m);

/* Host-only helper (no device work, usable without a GPU): Qwen3VLModel::get_rope_index, image branch
 * (src/models/qwen3vl/model.rs:901-1133) -- the M-RoPE position ids of a prompt whose image
 * placeholders follow <|vision_start|>.  grid_thw: n_images x 3 (t, h, w in patches).  pos3_out: [3][seq_len] (t, h, w rows),
 * rope_delta_out: max position + 1 - seq_len.  This is the routine aha_b200_forward_initial runs on the first call. */
int aha_b200_rope_index(const uint32_t* ids, size_t seq_len, const uint32_t* grid_thw, size_t n_images, uint32_t spatial_merge_size,
                        uint32_t image_token_id, uint32_t vision_start_token_id, int32_t* pos3_out, int32_t* rope_delta_out);

/* The same with the video branch (model.rs:907-925, 973-981): every row (t, h, w) of video_grid_thw stands for t runs of
 * <|vision_start|><|video_pad|>... in the prompt, each positioned as a (1, h, w) grid. */
int aha_b200_rope_index_mm(const uint32_t* ids, size_t seq_len, const uint32_t* grid_thw, size_t n_images, const uint32_t* video_grid_thw, size_t n_videos,
                           uint32_t spatial_merge_size, uint32_t image_token_id, uint32_t video_token_id, uint32_t vision_start_token_id, int32_t* pos3_out,
                           int32_t* rope_delta_out);

/* Last error message of the handle (or of the failed create / handle-less call when m == NULL). */
const char* aha_b200_last_error(aha_model* m);

/* --- introspection used by tests / bench (not part of the reference seam) --- */
int aha_b200_abi_version(void);
/* cudaStream_t the handle launches on (for CUDA-event timing on the launching stream). */
void* aha_b200_stream(aha_model* m);
int aha_b200_get_stats(aha_model* m, aha_stats* out);
int aha_b200_reset_stats(aha_model* m);
/* Copy an internal activation to the host: what = "hidden" (text hidden states after layer `index`
 * of the last forward_initial, S*H floats; requires aha_b200_set_trace(m,1)), "vit" (ViT hidden after
 * block `index`), "image_embeds", "audio_embeds", "rope_delta" (1 float), "batch_graphs" (1 float: step graphs
 * captured in the open batch session: at most one per running count, two where requests asking for log-probabilities ran),
 * "spec_graphs" (1 float: pass graphs of speculative requests, at most one per row count). */
int aha_b200_set_trace(aha_model* m, int on);
int aha_b200_debug_read(aha_model* m, const char* what, int index, float* out, size_t cap, size_t* n);
/* Run n decode steps back to back on the device (graph replays, token feedback on device) without any
 * host synchronisation inside; used by bench.py to time the device-resident `value`. */
int aha_b200_decode_steps(aha_model* m, uint32_t first_token, size_t seqlen_offset, size_t n_steps,
                          uint32_t* out_tokens /* n_steps, host, may be NULL */,
                          double* device_ms /* CUDA-event time of the n_steps on the launching stream, may be NULL */);
/* Time one kernel of the decode step in isolation (CUDA events on the launching stream), cycling over the
 * layers' weights so that consecutive launches never hit L2.  which = "gemv_gate_up" | "gemv_qkv" |
 * "gemv_down" | "gemv_o" | "gemv_lm_head" | "decode_attn", or the scoring head over rows 0 .. M-1 of the last prefill with n
 * alternatives: "score_head:M:n" (score_head_kernel) | "score_twin:M:n" (gemm_tc + logprob_partial_rows_kernel), each with its final
 * RMSNorm and stage 2.  bytes_per_launch = algorithmic bytes (the score entries: the lm_head's). */
/* the device sampler on a given logits row (tests): context = tokens generated so far, draw_index = draws already consumed */
int aha_b200_debug_sample(aha_model* m, const float* logits, const aha_gen_params* params, const uint32_t* context,
                          size_t n_context, uint32_t draw_index, uint32_t* token_out);
/* the log-probability kernels on a given logits row of V entries (tests): `token` is taken as the row's final token, index 0 */
int aha_b200_debug_logprobs(aha_model* m, const float* logits, size_t V, uint32_t token, uint32_t n_top, aha_logprobs* out);
int aha_b200_bench_kernel(aha_model* m, const char* which, int iters, double* avg_ms, uint64_t* bytes_per_launch);
/* tests: the scoring head alone on given pre-norm hidden rows [M][H] (final RMSNorm, head, records; row r scored at targets[r], index r);
 * impl 0 = score_head_kernel, 1 = the gemm_tc + row-kernel twin (a [M][V] logits block, then the generation path's stage-1 kernel) */
int aha_b200_debug_score_head(aha_model* m, int impl, const float* hidden, size_t M, const uint32_t* targets, uint32_t n_top,
                              aha_logprobs* out);
/* the verify attention of speculative decoding on host data (tests): `rows` query rows at positions pos0 .. pos0 + rows - 1 over K / V of
 * pos0 + rows positions (laid out on a paged pool with the pages in reverse order), head_dim 128.  q, out: [rows][n_heads][128] (q
 * normalised and rotated); k, v: [pos0 + rows][n_kv_heads][128].  Row r attends to positions 0 .. pos0 + r. */
int aha_b200_debug_verify_attn(aha_model* m, size_t rows, size_t n_heads, size_t n_kv_heads, size_t pos0, const float* q, const float* k,
                               const float* v, float* out);
/* Run ONE Linear layer y = epilogue(x W^T + b) through the library's GEMM dispatch on host data (unit tests of the
 * wgmma and SIMT kernels against numpy): impl 1 = SIMT fp32, 2 / 3 = wgmma split-fp16 (128x128 / 128x256 tiles), 5 = the batched decode GEMV (M <= 8; its SwiGLU
 * instantiation runs with a unit-gain RMSNorm prologue), 6 = the same with the cp.async weight ring, 7 = the wide batched decode GEMV
 * (wgmma, M <= 64, N and K multiples of 64; epilogues and SwiGLU prologue as impl 5); epi 0 = store, 1 = residual
 * add (resid [M,N]), 2 = activation (act: 1 silu, 2 gelu-erf, 3 gelu-tanh), 3 = SwiGLU on interleaved columns
 * (out [M,N/2]).  x [M,K] f32, w [N,K] f16 bits, bias [N] f32 or NULL.  device_ms: CUDA-event time of `iters` runs. */
int aha_b200_debug_gemm(aha_model* m, int impl, int epi, int act, int M, int N, int K, const float* x, const uint16_t* w,
                        const float* bias, const float* resid, float* out, int iters, double* device_ms);

#ifdef __cplusplus
}
#endif
#endif /* AHA_B200_H */
