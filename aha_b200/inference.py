"""Host-side mirror of aha's model-executor seam for the B200 path.

`B200Model` has the methods of `trait InferenceModel`
(src/models/common/mod.rs:25-45): forward_initial, forward_step, clear_cache,
stop_token_ids -- same names, argument meaning and error behaviour (errors are raised, never
swallowed) -- and `generate` = generate_generic (src/models/common/generate.rs:115-159).
Everything here is plumbing around libaha_b200.so; no arithmetic happens in Python."""
import ctypes as C
import json

import numpy as np

from . import _lib as L


class B200Error(RuntimeError):
    pass


class MultiModalData:
    """common/mod.rs:14-22 -- positional list of optional tensors."""

    def __init__(self, data_vec):
        self.data_vec = list(data_vec)


def nccl_unique_id():
    """128-byte ncclUniqueId created by the calling rank (rank 0); broadcast it to the other ranks."""
    lib = L.load()
    buf = (C.c_uint8 * 128)()
    if lib.aha_b200_nccl_unique_id(buf) != 0:
        raise B200Error(lib.aha_b200_last_error(None).decode())
    return bytes(buf)


def rope_index(ids, grid_thw, config, video_grid_thw=None):
    """M-RoPE position ids (3, S) int32 and rope_delta of a Qwen3-VL prompt -- the host routine forward_initial runs
    (Qwen3VLModel::get_rope_index, src/models/qwen3vl/model.rs:901-1133), image and video branches.  No device work."""
    lib = L.load()
    ids = np.ascontiguousarray(np.asarray(ids).reshape(-1), dtype=np.uint32)
    grid = np.ascontiguousarray(np.asarray(grid_thw if grid_thw is not None else [], dtype=np.uint32).reshape(-1, 3))
    vgrid = np.ascontiguousarray(np.asarray(video_grid_thw if video_grid_thw is not None else [], dtype=np.uint32).reshape(-1, 3))
    pos = np.empty((3, ids.size), np.int32)
    delta = C.c_int32(0)
    u32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint32))
    rc = lib.aha_b200_rope_index_mm(u32(ids), ids.size, u32(grid), grid.shape[0], u32(vgrid), vgrid.shape[0],
                                    int(config["vision_config"]["spatial_merge_size"]), int(config["image_token_id"]),
                                    int(config.get("video_token_id", 0xffffffff)), int(config["vision_start_token_id"]),
                                    pos.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(delta))
    if rc != 0:
        raise B200Error(lib.aha_b200_last_error(None).decode())
    return pos, int(delta.value)


def prefix_match(cached_ids, ids, mm_token_ids=(), same_mm=True):
    """The rule behind generate(reuse_prefix=True), host only: how many leading tokens of `ids` a KV cache holding `cached_ids`
    can supply (see aha_b200_prefix_match in include/aha_b200.h)."""
    lib = L.load()
    a = np.ascontiguousarray(np.asarray(cached_ids, dtype=np.uint32).reshape(-1))
    b = np.ascontiguousarray(np.asarray(ids, dtype=np.uint32).reshape(-1))
    t = np.ascontiguousarray(np.asarray(list(mm_token_ids), dtype=np.uint32).reshape(-1))
    u32 = lambda x: x.ctypes.data_as(C.POINTER(C.c_uint32))
    return int(lib.aha_b200_prefix_match(u32(a), a.size, u32(b), b.size, u32(t), t.size, 1 if same_mm else 0))


def rules_check(presence_penalty=0.0, frequency_penalty=0.0, logit_bias=None, vocab_size=None):
    """Check a logit-rules object (OpenAI presence_penalty, frequency_penalty, logit_bias) the way rules_create checks it, over a
    vocabulary of vocab_size tokens (host only, aha_b200_rules_check).  Raises B200Error."""
    lib = L.load()
    r, _keep = L.logit_rules(presence_penalty, frequency_penalty, logit_bias)
    if lib.aha_b200_rules_check(C.byref(r), int(vocab_size)) != 0:
        raise B200Error(lib.aha_b200_last_error(None).decode())


def fsm_check(offsets, tokens, next, start=0, vocab_size=None):
    """Check a token automaton (CSR: state s allows tokens[offsets[s]:offsets[s + 1]], next[j] follows tokens[j]) the way
    fsm_create checks it, over a vocabulary of vocab_size tokens (host only, aha_b200_fsm_check).  Raises B200Error."""
    lib = L.load()
    f, _keep = L.token_fsm(offsets, tokens, next, start)
    if lib.aha_b200_fsm_check(C.byref(f), int(vocab_size)) != 0:
        raise B200Error(lib.aha_b200_last_error(None).decode())


def mm_fingerprint(data):
    """64-bit fingerprint of a MultiModalData list (0 = no tensor): what decides whether two requests carry the same images / audio."""
    lib = L.load()
    mm, _keep = B200Model._mm(None, data)
    return int(lib.aha_b200_mm_fingerprint(C.byref(mm))) if mm is not None else 0


class B200Model:
    def __init__(self, kind, config, weights, eos_ids=(), device=0, max_ctx=8192, max_prefill=0, max_patches=0,
                 max_frames=0, use_graph=True, decode_impl=0, gemm_impl=0, attn_impl=0, tp_rank=0, tp_world=1, tp_unique_id=None):
        self._lib = L.load()
        self.kind = kind
        self.config = config
        cfg_json = json.dumps(config).encode()
        names = list(weights.keys())
        arrs = [weights[n] if (isinstance(weights[n], np.ndarray) and weights[n].flags["C_CONTIGUOUS"]) else np.ascontiguousarray(weights[n])
                for n in names]   # (a BF16-tagged view must keep its subclass)
        descs = (L.TensorDesc * len(names))(*[L.make_desc(a, n) for a, n in zip(arrs, names)])
        eos = np.asarray(list(eos_ids), dtype=np.uint32)
        opts = L.Options(device=device, tp_rank=tp_rank, tp_world=tp_world, max_ctx=max_ctx, max_prefill=max_prefill,
                         max_patches=max_patches, max_frames=max_frames, use_graph=1 if use_graph else 0,
                         decode_impl=decode_impl, gemm_impl=gemm_impl)
        opts.reserved[0] = attn_impl
        if tp_world > 1:
            if tp_unique_id is None or len(tp_unique_id) != 128:
                raise ValueError("tp_world > 1 needs the 128-byte NCCL unique id (nccl_unique_id() on rank 0, then broadcast)")
            self._tp_id = (C.c_uint8 * 128)(*bytes(tp_unique_id))
            opts.tp_comm = C.cast(self._tp_id, C.c_void_p)
        h = C.c_void_p()
        rc = self._lib.aha_b200_create(kind.encode(), cfg_json, descs, len(names),
                                       eos.ctypes.data_as(C.POINTER(C.c_uint32)), len(eos), C.byref(opts), C.byref(h))
        if rc != 0:
            raise B200Error(self._lib.aha_b200_last_error(None).decode())
        self._h = h
        tc = config if kind == "qwen3" else (config["text_config"] if kind == "qwen3vl" else config["thinker_config"]["text_config"])
        self.vocab_size = tc["vocab_size"]
        self.hidden_size = tc["hidden_size"]

    # ------------------------------------------------------------------ helpers
    def _check(self, rc):
        if rc != 0:
            raise B200Error(self._lib.aha_b200_last_error(self._h).decode())

    def _mm(self, data):
        if data is None:
            return None, None
        vec = data.data_vec if isinstance(data, MultiModalData) else list(data)
        keep, descs = [], []
        for t in vec:
            if t is None:
                d = L.TensorDesc()
                d.data = None
            else:
                a = np.ascontiguousarray(t)
                if a.dtype == np.int32:
                    a = a.astype(np.int64)
                keep.append(a)
                d = L.make_desc(a)
            descs.append(d)
        arr = (L.TensorDesc * len(descs))(*descs)
        mm = L.MM(arr, len(descs))
        return mm, (keep, arr)

    @staticmethod
    def _ids(input_ids):
        return np.ascontiguousarray(np.asarray(input_ids, dtype=np.uint32).reshape(-1))

    # ------------------------------------------------------------------ InferenceModel
    def forward_initial(self, input_ids, seqlen_offset, data=None, want_logits=True):
        """-> logits (1,1,V) float32 (like the reference's Tensor) and sets self.last_argmax."""
        ids = self._ids(input_ids)
        mm, _keep = self._mm(data)
        logits = np.empty(self.vocab_size, np.float32) if want_logits else None
        am = C.c_uint32(0)
        self._check(self._lib.aha_b200_forward_initial(
            self._h, ids.ctypes.data_as(C.POINTER(C.c_uint32)), ids.size, int(seqlen_offset),
            C.byref(mm) if mm is not None else None,
            logits.ctypes.data_as(C.POINTER(C.c_float)) if want_logits else None, C.byref(am)))
        self.last_argmax = int(am.value)
        return logits.reshape(1, 1, -1) if want_logits else None

    def forward_step(self, input_ids, seqlen_offset, want_logits=True):
        ids = self._ids(input_ids)
        logits = np.empty(self.vocab_size, np.float32) if want_logits else None
        am = C.c_uint32(0)
        self._check(self._lib.aha_b200_forward_step(
            self._h, ids.ctypes.data_as(C.POINTER(C.c_uint32)), ids.size, int(seqlen_offset),
            logits.ctypes.data_as(C.POINTER(C.c_float)) if want_logits else None, C.byref(am)))
        self.last_argmax = int(am.value)
        return logits.reshape(1, 1, -1) if want_logits else None

    def forward_extend(self, input_ids, seqlen_offset, want_logits=True):
        """Prefill continuation (new design; the reference's (S, S) mask rejects S > 1 with a non-empty cache): further prompt
        tokens against the `seqlen_offset` tokens already in the cache -> logits of the last one."""
        ids = self._ids(input_ids)
        logits = np.empty(self.vocab_size, np.float32) if want_logits else None
        am = C.c_uint32(0)
        self._check(self._lib.aha_b200_forward_extend(
            self._h, ids.ctypes.data_as(C.POINTER(C.c_uint32)), ids.size, int(seqlen_offset),
            logits.ctypes.data_as(C.POINTER(C.c_float)) if want_logits else None, C.byref(am)))
        self.last_argmax = int(am.value)
        return logits.reshape(1, 1, -1) if want_logits else None

    def last_prefix_hit(self):
        """Prompt tokens the last generate call took from the KV cache (reuse_prefix=True) instead of prefilling them."""
        return int(self._lib.aha_b200_last_prefix_hit(self._h))

    def clear_cache(self):
        self._check(self._lib.aha_b200_clear_cache(self._h))

    def stop_token_ids(self):
        n = self._lib.aha_b200_stop_token_ids(self._h, None, 0)
        out = (C.c_uint32 * max(n, 1))()
        self._lib.aha_b200_stop_token_ids(self._h, out, n)
        return [int(out[i]) for i in range(n)]

    # ------------------------------------------------------------------ generate_generic / generate_stream_generic
    @staticmethod
    def _gen_params(max_tokens, temperature, top_p, top_k, repeat_penalty, repeat_last_n, seed, flags=0, fsm=None, rules=None):
        """fsm: the id of a token automaton (fsm_create) that constrains the request (AHA_GEN_CONSTRAINED), or None.
        rules: the id of a logit-rules object (rules_create, AHA_GEN_LOGIT_RULES), or None.  params.reserved holds one id: with both,
        the library refuses the request (an automaton goes into the rules object instead)."""
        if fsm is not None:
            flags |= L.GEN_CONSTRAINED
        if rules is not None:
            flags |= L.GEN_LOGIT_RULES
        return L.GenParams(temperature=temperature or 0.0, repeat_penalty=repeat_penalty, repeat_last_n=repeat_last_n,
                           max_tokens=max_tokens, seed=seed, top_p=top_p or 0.0, top_k=top_k or 0, flags=flags,
                           reserved=int(rules) if rules is not None else (0 if fsm is None else int(fsm)))

    @staticmethod
    def _usage(u):
        return dict(prompt_tokens=u.prompt_tokens, completion_tokens=u.completion_tokens, prompt_secs=u.prompt_secs,
                    completion_secs=u.completion_secs, vision_secs=u.vision_secs)

    def generate(self, input_ids, data=None, max_tokens=1024, temperature=0.0, top_p=None, top_k=None, repeat_penalty=1.0,
                 repeat_last_n=64, seed=299792458, flags=0, reuse_prefix=False, logprobs=False, top_logprobs=0, fsm=None, rules=None):
        """-> (generated ids, usage dict).  temperature < 1e-7: ArgMax; else the device sampler (TopK / TopKThenTopP / TopP /
        All exactly as get_logit_processor picks them from temperature, top_p, top_k).  reuse_prefix: keep this request's K/V
        and prefill only what follows the prefix shared with the cache (multi-turn chats; same tokens as without it).
        logprobs=True (aha_b200_generate_logprobs): -> (ids, usage, records), one record dict per token (token, index, logprob,
        top_ids, top_logprobs with top_logprobs alternatives; raw model log-probabilities, before penalty and temperature).
        fsm: the id of a token automaton (fsm_create); every token is drawn from the tokens its current state allows.
        rules: the id of a logit-rules object (rules_create): logit bias, frequency and presence penalties on every draw."""
        ids = self._ids(input_ids)
        mm, _keep = self._mm(data)
        if reuse_prefix:
            flags |= L.GEN_REUSE_PREFIX
        flags |= L.logprob_flags(logprobs, top_logprobs, self.vocab_size)
        p = self._gen_params(max_tokens, temperature, top_p, top_k, repeat_penalty, repeat_last_n, seed, flags, fsm, rules)
        cap = max(max_tokens, 1)
        out = (C.c_uint32 * cap)()
        n = C.c_size_t(0)
        u = L.Usage()
        ids_p, mm_p = ids.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(mm) if mm is not None else None
        if logprobs:
            recs = (L.Logprobs * cap)()
            self._check(self._lib.aha_b200_generate_logprobs(self._h, ids_p, ids.size, mm_p, C.byref(p), out, recs, cap, C.byref(n), C.byref(u)))
            return [int(out[i]) for i in range(n.value)], self._usage(u), [L.logprobs_record(recs[i]) for i in range(n.value)]
        self._check(self._lib.aha_b200_generate(self._h, ids_p, ids.size, mm_p, C.byref(p), out, cap, C.byref(n), C.byref(u)))
        return [int(out[i]) for i in range(n.value)], self._usage(u)

    def generate_speculative(self, input_ids, data=None, prediction=None, prompt_lookup=False, max_draft=7, ngram=3, max_tokens=1024,
                             temperature=0.0, top_p=None, top_k=None, repeat_penalty=1.0, repeat_last_n=64, seed=299792458, flags=0,
                             logprobs=False, top_logprobs=0, rules=None):
        """Speculative decoding of one request (aha_b200_generate_speculative): verify passes of max_draft + 1 rows, drafted from
        `prediction` (token ids the answer will largely repeat) and, with prompt_lookup, from the prompt and the output so far.
        -> (ids, usage, stats) with stats = dict(passes, drafted, accepted); (ids, usage, stats, records) with logprobs=True.
        The ids and records do not depend on the drafts; they follow the model as wide batch sessions do.  rules: a logit-rules id whose
        object names no automaton."""
        ids = self._ids(input_ids)
        mm, _keep = self._mm(data)
        sp, _pred = L.spec_params(prediction, prompt_lookup, max_draft, ngram, self.vocab_size)
        flags |= L.logprob_flags(logprobs, top_logprobs, self.vocab_size)
        p = self._gen_params(max_tokens, temperature, top_p, top_k, repeat_penalty, repeat_last_n, seed, flags, rules=rules)
        cap = max(max_tokens, 1)
        out = (C.c_uint32 * cap)()
        recs = (L.Logprobs * cap)() if logprobs else None
        n = C.c_size_t(0)
        u = L.Usage()
        st = L.SpecStats()
        self._check(self._lib.aha_b200_generate_speculative(
            self._h, ids.ctypes.data_as(C.POINTER(C.c_uint32)), ids.size, C.byref(mm) if mm is not None else None, C.byref(p), C.byref(sp),
            out, recs, cap, C.byref(n), C.byref(u), C.byref(st)))
        toks = [int(out[i]) for i in range(n.value)]
        stats = dict(passes=int(st.passes), drafted=int(st.drafted), accepted=int(st.accepted))
        if logprobs:
            return toks, self._usage(u), stats, [L.logprobs_record(recs[i]) for i in range(n.value)]
        return toks, self._usage(u), stats

    def debug_verify_attn(self, q, k, v, pos0):
        """The verify attention of speculative decoding on host data: q [R][nh][128] at positions pos0 .. pos0 + R - 1,
        k / v [pos0 + R][nkv][128] -> [R][nh][128]."""
        q = np.ascontiguousarray(q, np.float32)
        k = np.ascontiguousarray(k, np.float32)
        v = np.ascontiguousarray(v, np.float32)
        R, nh, hd = q.shape
        nkv = k.shape[1]
        if hd != 128 or k.shape != (pos0 + R, nkv, 128) or v.shape != k.shape:
            raise ValueError("q [R][nh][128], k and v [pos0 + R][nkv][128]")
        out = np.empty_like(q)
        f = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
        self._check(self._lib.aha_b200_debug_verify_attn(self._h, R, nh, nkv, int(pos0), f(q), f(k), f(v), f(out)))
        return out

    def debug_verify_attn_batch(self, qs, ks, vs, pos0s, tables, n_pool_pages):
        """The verify attention over several requests in one launch (aha_b200_debug_verify_attn_batch): request j has q qs[j]
        [R_j][nh][128] at positions pos0s[j] .. pos0s[j] + R_j - 1 over k / v ks[j], vs[j] [pos0s[j] + R_j][nkv][128] on the page table
        tables[j] (ceil((pos0s[j] + R_j) / 32) distinct pages of a NaN pool of n_pool_pages) -> [out_j [R_j][nh][128], ...]."""
        qs = [np.ascontiguousarray(q, np.float32) for q in qs]
        nh, nkv = qs[0].shape[1], np.shape(ks[0])[1]
        rows = np.ascontiguousarray([q.shape[0] for q in qs], np.int32)
        p0 = np.ascontiguousarray(pos0s, np.int32)
        for j, q in enumerate(qs):
            want = (int(p0[j]) + q.shape[0], nkv, 128)
            if q.shape[1:] != (nh, 128) or np.shape(ks[j]) != want or np.shape(vs[j]) != want or np.size(tables[j]) != -(-want[0] // 32):
                raise ValueError(f"request {j}: q [R][nh][128], k and v [pos0 + R][nkv][128], a table of ceil((pos0 + R) / 32) pages")
        q = np.ascontiguousarray(np.concatenate(qs), np.float32)
        k = np.ascontiguousarray(np.concatenate(ks), np.float32)
        v = np.ascontiguousarray(np.concatenate(vs), np.float32)
        tb = np.ascontiguousarray(np.concatenate([np.asarray(t, np.int32).reshape(-1) for t in tables]), np.int32)
        out = np.empty_like(q)
        f = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
        i32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))
        self._check(self._lib.aha_b200_debug_verify_attn_batch(self._h, len(qs), i32(rows), i32(p0), i32(tb), int(n_pool_pages), nh, nkv,
                                                               f(q), f(k), f(v), f(out)))
        return np.split(out, np.cumsum(rows)[:-1])

    def debug_attention(self, q, k, v, impl, causal, segments=None, page_order=None, split_out=False):
        """The prefill attention on host data (aha_b200_debug_attention): q [Sq][nh][hd], k / v [Skv][nkv][hd] with hd 64 or 128 ->
        [Sq][nh][hd].  impl 0 = wgmma, 1 = SIMT, 2 = mma.sync.  causal: query i sees keys 0 .. Skv - Sq + i, K / V on a paged pool
        (logical page p at physical page page_order[p]).  segments: [(start, len), ...] attending only to themselves (Sq == Skv).
        split_out: the wgmma kernel's fp16 hi + lo output, summed."""
        q = np.ascontiguousarray(q, np.float32)
        k = np.ascontiguousarray(k, np.float32)
        v = np.ascontiguousarray(v, np.float32)
        Sq, nh, hd = q.shape
        Skv, nkv = k.shape[:2]
        if k.shape != (Skv, nkv, hd) or v.shape != k.shape:
            raise ValueError("q [Sq][nh][hd], k and v [Skv][nkv][hd]")
        seg = np.ascontiguousarray(np.asarray(segments if segments is not None else [], np.int32).reshape(-1, 2))
        po = None if page_order is None else np.ascontiguousarray(page_order, np.int32)
        if po is not None and po.size != -(-Skv // 32):
            raise ValueError("page_order needs one entry per 32-token page")
        out = np.empty_like(q)
        f = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
        i32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32)) if a is not None and a.size else None
        self._check(self._lib.aha_b200_debug_attention(self._h, int(impl), hd, nh, nkv, Sq, Skv, 1 if causal else 0, i32(seg), len(seg),
                                                       i32(po), 1 if split_out else 0, f(q), f(k), f(v), f(out)))
        return out

    def debug_prefix_attention(self, q, k, v, impl, segments, page_order=None):
        """Packed prefill attention over segments with cached prefixes on host data (aha_b200_debug_prefix_attention): segments
        [(prefix, rows), ...]; q [sum rows][nh][128], k / v [sum (prefix + rows)][nkv][128] laid out segment by segment -> [sum rows][nh][128].
        impl 0 = wgmma varlen kernel, 1 = SIMT, 2 = mma.sync."""
        q = np.ascontiguousarray(q, np.float32)
        k = np.ascontiguousarray(k, np.float32)
        v = np.ascontiguousarray(v, np.float32)
        seg = np.ascontiguousarray(np.asarray(segments, np.int32).reshape(-1, 2))
        Sq, nh, hd = q.shape
        Skv, nkv = k.shape[:2]
        if hd != 128 or Sq != int(seg[:, 1].sum()) or Skv != int(seg.sum()) or k.shape != (Skv, nkv, 128) or v.shape != k.shape:
            raise ValueError("q [sum rows][nh][128], k and v [sum (prefix + rows)][nkv][128]")
        po = None if page_order is None else np.ascontiguousarray(page_order, np.int32)
        if po is not None and po.size != -(-Skv // 32):
            raise ValueError("page_order needs one entry per 32-token page")
        out = np.empty_like(q)
        f = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
        i32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32)) if a is not None and a.size else None
        self._check(self._lib.aha_b200_debug_prefix_attention(self._h, int(impl), nh, nkv, i32(seg), len(seg), i32(po), f(q), f(k), f(v), f(out)))
        return out

    def debug_decode_attn(self, qkv, pos, rope_delta, k_cache, v_cache, tables, n_pool_pages, q_norm, k_norm, n_heads, n_kv_heads,
                          eps=1e-6, rope_theta=1e6):
        """The decode attention on host data (aha_b200_debug_decode_attn) for B sequences: qkv [B][(nh + 2 nkv) * 128] raw
        projections, pos / rope_delta [B], k_cache / v_cache lists of [pos[b]][nkv][128], tables a list of B page tables
        (ceil((pos[b] + 1) / 32) distinct pages of a pool of n_pool_pages).  -> (out [B][nh][128] of a run on the pool as a decode step
        finds it, out of a second run on the same partials and counters, pool after the call [n_pool_pages][2][nkv][32][128])."""
        qkv = np.ascontiguousarray(qkv, np.float32)
        B = qkv.shape[0]
        if qkv.shape != (B, (n_heads + 2 * n_kv_heads) * 128) or len(pos) != B or len(rope_delta) != B or len(tables) != B:
            raise ValueError("qkv [B][(nh + 2 nkv) * 128]; pos, rope_delta, k_cache, v_cache and tables one per sequence")
        for b in range(B):
            if np.shape(tables[b]) != (-(-(int(pos[b]) + 1) // 32),) or np.shape(k_cache[b]) != (pos[b], n_kv_heads, 128) or \
                    np.shape(v_cache[b]) != np.shape(k_cache[b]):
                raise ValueError(f"sequence {b}: k_cache / v_cache [pos][nkv][128], table of ceil((pos + 1) / 32) pages")
        kc = np.ascontiguousarray(np.concatenate([np.reshape(x, (-1, n_kv_heads, 128)) for x in k_cache]), np.float32)
        vc = np.ascontiguousarray(np.concatenate([np.reshape(x, (-1, n_kv_heads, 128)) for x in v_cache]), np.float32)
        tb = np.ascontiguousarray(np.concatenate([np.asarray(t, np.int32) for t in tables]), np.int32)
        p = np.ascontiguousarray(pos, np.int32)
        rd = np.ascontiguousarray(rope_delta, np.int32)
        qn = np.ascontiguousarray(q_norm, np.float32)
        kn = np.ascontiguousarray(k_norm, np.float32)
        out = np.empty((B, n_heads, 128), np.float32)
        again = np.empty_like(out)
        pool = np.empty((n_pool_pages, 2, n_kv_heads, 32, 128), np.float32)
        f = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
        i32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))
        self._check(self._lib.aha_b200_debug_decode_attn(self._h, B, n_heads, n_kv_heads, f(qkv), i32(p), i32(rd), f(kc), f(vc), i32(tb),
                                                         n_pool_pages, f(qn), f(kn), float(eps), float(rope_theta), f(out), f(again),
                                                         f(pool)))
        return out, again, pool

    def generate_batch(self, requests):
        """Static batching (aha_b200_generate_batch): requests = [dict(input_ids=..., data=None, max_tokens=..., temperature=..., top_p=...,
        top_k=..., repeat_penalty=..., repeat_last_n=..., seed=..., fsm=..., rules=...), ...] (at most 8) decoded in lockstep on this handle.
        -> [(generated ids, usage dict), ...]: per request exactly what generate() returns for it alone."""
        n = len(requests)
        arr, _keep = self._batch_requests(requests)
        cap = max([1] + [r.get("max_tokens", 1024) for r in requests])
        out = (C.c_uint32 * (n * cap))()
        n_out = (C.c_size_t * n)()
        us = (L.Usage * n)()
        self._check(self._lib.aha_b200_generate_batch(self._h, arr, n, out, cap, n_out, us))
        return [([int(out[i * cap + j]) for j in range(n_out[i])], self._usage(us[i])) for i in range(n)]

    def _batch_requests(self, requests):
        """request dicts -> (aha_batch_request array, the buffers it points into)"""
        arr = (L.BatchRequest * max(len(requests), 1))()
        keep = []
        for i, r in enumerate(requests):
            ids = self._ids(r["input_ids"])
            mm, k = self._mm(r.get("data"))
            keep += [ids, mm, k]
            arr[i].ids = ids.ctypes.data_as(C.POINTER(C.c_uint32))
            arr[i].seq_len = ids.size
            arr[i].mm = C.pointer(mm) if mm is not None else None
            flags = r.get("flags", 0) | L.logprob_flags(r.get("logprobs", False), r.get("top_logprobs", 0), self.vocab_size)
            arr[i].params = self._gen_params(r.get("max_tokens", 1024), r.get("temperature", 0.0), r.get("top_p"), r.get("top_k"),
                                             r.get("repeat_penalty", 1.0), r.get("repeat_last_n", 64), r.get("seed", 299792458), flags,
                                             r.get("fsm"), r.get("rules"))
        return arr, keep

    # ---- constrained decoding: token automata on the handle
    def fsm_create(self, offsets, tokens, next, start=0):
        """Copy a token automaton to the device (aha_b200_fsm_create) -> its id, the `fsm` argument of the generation entries.
        State s allows tokens[offsets[s]:offsets[s + 1]] (strictly ascending, at least one) and next[j] is the state after tokens[j]."""
        f, _keep = L.token_fsm(offsets, tokens, next, start)
        i = C.c_uint32(0)
        self._check(self._lib.aha_b200_fsm_create(self._h, C.byref(f), C.byref(i)))
        return int(i.value)

    def fsm_destroy(self, fsm):
        """Free a token automaton (refused while a running batch slot uses it or a logit-rules object names it)."""
        self._check(self._lib.aha_b200_fsm_destroy(self._h, int(fsm)))

    # ---- LoRA adapters: many fine-tunes of the base model in one wide session
    def lora_create(self, tensors, scale):
        """Load one adapter (aha_b200_lora_create) -> its id, the adapter of batch_add_lora.  tensors: {PEFT name: array [r, K] (lora_A) or
        [N, r] (lora_B)}, f16 / bf16 / f32, as in adapter_model.safetensors; scale: lora_alpha / r (lora_alpha / sqrt(r) for rsLoRA)."""
        names = list(tensors.keys())
        arrs = [tensors[n] if (isinstance(tensors[n], np.ndarray) and tensors[n].flags["C_CONTIGUOUS"]) else np.ascontiguousarray(tensors[n])
                for n in names]
        descs = (L.TensorDesc * max(len(names), 1))(*[L.make_desc(a, n) for a, n in zip(arrs, names)])
        i = C.c_uint32(0)
        self._check(self._lib.aha_b200_lora_create(self._h, descs, len(names), float(scale), C.byref(i)))
        return int(i.value)

    def lora_destroy(self, adapter):
        """Free an adapter (refused while a running or suspended request uses it); its prefix-cache pages are dropped."""
        self._check(self._lib.aha_b200_lora_destroy(self._h, int(adapter)))

    def batch_add_lora(self, requests, adapters, return_usage=False):
        """batch_add_many with request i running adapter adapters[i] (0: the base model); wide sessions only.  All or nothing.
        -> [(slot, first token, finished), ...] in input order, and with return_usage=True also the prompt-side usage dicts."""
        n = len(requests)
        ad = np.ascontiguousarray(np.asarray(adapters, dtype=np.uint32).reshape(-1))
        if ad.size != n:
            raise ValueError(f"adapters must hold one id per request ({n}), got {ad.size}")
        arr, _keep = self._batch_requests(requests)
        slots, toks, fins = (C.c_int32 * max(n, 1))(), (C.c_uint32 * max(n, 1))(), (C.c_int32 * max(n, 1))()
        us = (L.Usage * max(n, 1))()
        self._check(self._lib.aha_b200_batch_add_lora(self._h, arr, ad.ctypes.data_as(C.POINTER(C.c_uint32)), n, slots, toks, fins, us))
        res = [(int(slots[i]), int(toks[i]), bool(fins[i])) for i in range(n)]
        return (res, [self._usage(us[i]) for i in range(n)]) if return_usage else res

    # ---- OpenAI presence_penalty / frequency_penalty / logit_bias: logit-rules objects on the handle
    def rules_create(self, presence_penalty=0.0, frequency_penalty=0.0, logit_bias=None, fsm=None):
        """A logit-rules object (aha_b200_rules_create) -> its id, the `rules` argument of the generation entries.  Penalties in [-2, 2];
        logit_bias: {token id (int or decimal string): bias in [-100, 100]} or (id, bias) pairs; fsm: a token automaton id (fsm_create)
        that constrains the request too."""
        r, _keep = L.logit_rules(presence_penalty, frequency_penalty, logit_bias, fsm)
        i = C.c_uint32(0)
        self._check(self._lib.aha_b200_rules_create(self._h, C.byref(r), C.byref(i)))
        return int(i.value)

    def rules_destroy(self, rules):
        """Free a logit-rules object (refused while a running batch slot uses it)."""
        self._check(self._lib.aha_b200_rules_destroy(self._h, int(rules)))

    # ---- continuous batching: requests join / leave a running batch between steps (aha_b200_batch_open / _add / _step / _close)
    def batch_open(self):
        self._check(self._lib.aha_b200_batch_open(self._h))
        self._batch_width = 8

    def batch_open_wide(self, max_seqs):
        """A session of max_seqs (1..64) slots stepped on the tensor cores; admission, stepping and closing as for batch_open."""
        self._check(self._lib.aha_b200_batch_open_wide(self._h, int(max_seqs)))
        self._batch_width = int(max_seqs)

    def batch_add(self, input_ids, data=None, max_tokens=1024, temperature=0.0, top_p=None, top_k=None, repeat_penalty=1.0, repeat_last_n=64,
                  seed=299792458, flags=0, logprobs=False, top_logprobs=0, fsm=None, rules=None):
        """Prefill one request into a free slot -> (slot, first token, finished).  logprobs / top_logprobs: batch_logprobs() holds the
        record of each token it delivers."""
        flags |= L.logprob_flags(logprobs, top_logprobs, self.vocab_size)
        ids = self._ids(input_ids)
        mm, _keep = self._mm(data)
        req = L.BatchRequest()
        req.ids = ids.ctypes.data_as(C.POINTER(C.c_uint32))
        req.seq_len = ids.size
        req.mm = C.pointer(mm) if mm is not None else None
        req.params = self._gen_params(max_tokens, temperature, top_p, top_k, repeat_penalty, repeat_last_n, seed, flags, fsm, rules)
        slot, fin, tok = C.c_int32(-1), C.c_int32(0), C.c_uint32(0)
        u = L.Usage()
        self._check(self._lib.aha_b200_batch_add(self._h, C.byref(req), C.byref(slot), C.byref(tok), C.byref(fin), C.byref(u)))
        return int(slot.value), int(tok.value), bool(fin.value)

    def batch_add_many(self, requests, return_usage=False):
        """Admit several requests (dicts as for generate_batch) in one call, the text-only ones packed into shared prefills; all or
        nothing.  -> [(slot, first token, finished), ...] in input order, and with return_usage=True also the prompt-side usage dicts."""
        n = len(requests)
        arr, _keep = self._batch_requests(requests)
        slots, toks, fins = (C.c_int32 * max(n, 1))(), (C.c_uint32 * max(n, 1))(), (C.c_int32 * max(n, 1))()
        us = (L.Usage * max(n, 1))()
        self._check(self._lib.aha_b200_batch_add_many(self._h, arr, n, slots, toks, fins, us))
        res = [(int(slots[i]), int(toks[i]), bool(fins[i])) for i in range(n)]
        return (res, [self._usage(us[i]) for i in range(n)]) if return_usage else res

    @staticmethod
    def _seeds(n, seeds):
        """per-choice seeds -> (uint64 array or None, the pointer argument)"""
        if seeds is None:
            return None, None
        s = np.ascontiguousarray(np.asarray(seeds, dtype=np.uint64).reshape(-1))
        if s.size != n:
            raise ValueError(f"seeds must hold n = {n} seeds, got {s.size}")
        return s, s.ctypes.data_as(C.POINTER(C.c_uint64))

    def batch_add_n(self, input_ids, n, seeds=None, data=None, max_tokens=1024, temperature=0.0, top_p=None, top_k=None, repeat_penalty=1.0,
                    repeat_last_n=64, seed=299792458, flags=0, logprobs=False, top_logprobs=0, return_usage=False, fsm=None, rules=None):
        """OpenAI `n` (aha_b200_batch_add_n): n choices of one request in the n lowest free slots, the prompt prefilled once and its K/V
        copied into every other choice's own pages.  Choice i samples with seeds[i] (None: seed + i) and yields exactly what batch_add
        yields for the request with that seed.  All or nothing.  -> [(slot, first token, finished), ...] per choice, and with
        return_usage=True also the prompt-side usage dicts."""
        n = int(n)
        flags |= L.logprob_flags(logprobs, top_logprobs, self.vocab_size)
        ids = self._ids(input_ids)
        mm, _keep = self._mm(data)
        _s, seeds_p = self._seeds(n, seeds)
        req = L.BatchRequest()
        req.ids = ids.ctypes.data_as(C.POINTER(C.c_uint32))
        req.seq_len = ids.size
        req.mm = C.pointer(mm) if mm is not None else None
        req.params = self._gen_params(max_tokens, temperature, top_p, top_k, repeat_penalty, repeat_last_n, seed, flags, fsm, rules)
        k = max(n, 1)
        slots, toks, fins, us = (C.c_int32 * k)(), (C.c_uint32 * k)(), (C.c_int32 * k)(), (L.Usage * k)()
        self._check(self._lib.aha_b200_batch_add_n(self._h, C.byref(req), n, seeds_p, slots, toks, fins, us))
        res = [(int(slots[i]), int(toks[i]), bool(fins[i])) for i in range(n)]
        return (res, [self._usage(us[i]) for i in range(n)]) if return_usage else res

    def generate_n(self, input_ids, n, seeds=None, data=None, max_tokens=1024, temperature=0.0, top_p=None, top_k=None, repeat_penalty=1.0,
                   repeat_last_n=64, seed=299792458, flags=0, logprobs=False, top_logprobs=0, fsm=None, rules=None):
        """OpenAI `n` in one call (aha_b200_generate_n, 1 <= n <= 8): the prompt prefilled once, the choices decoded in lockstep.
        -> [(ids, usage), ...] per choice, [(ids, usage, records), ...] with logprobs=True; choice i is exactly what generate()
        returns for seeds[i] (None: seed + i)."""
        n = int(n)
        ids = self._ids(input_ids)
        mm, _keep = self._mm(data)
        _s, seeds_p = self._seeds(n, seeds)
        flags |= L.logprob_flags(logprobs, top_logprobs, self.vocab_size)
        p = self._gen_params(max_tokens, temperature, top_p, top_k, repeat_penalty, repeat_last_n, seed, flags, fsm, rules)
        cap, k = max(max_tokens, 1), max(n, 1)
        out = (C.c_uint32 * (k * cap))()
        recs = (L.Logprobs * (k * cap))() if logprobs else None
        n_out, us = (C.c_size_t * k)(), (L.Usage * k)()
        self._check(self._lib.aha_b200_generate_n(self._h, ids.ctypes.data_as(C.POINTER(C.c_uint32)), ids.size,
                                                  C.byref(mm) if mm is not None else None, C.byref(p), n, seeds_p, out, recs, cap, n_out, us))
        res = []
        for i in range(n):
            toks = [int(out[i * cap + j]) for j in range(n_out[i])]
            if logprobs:
                res.append((toks, self._usage(us[i]), [L.logprobs_record(recs[i * cap + j]) for j in range(n_out[i])]))
            else:
                res.append((toks, self._usage(us[i])))
        return res

    def batch_step(self):
        """One decode step of every running request -> {slot: (token, finished)} (empty when nothing is running)."""
        w = getattr(self, "_batch_width", 8)
        if w > 8:
            toks, status, n = (C.c_uint32 * w)(), (C.c_int32 * w)(), C.c_size_t(0)
            self._check(self._lib.aha_b200_batch_step_n(self._h, toks, status, w, C.byref(n)))
            return {i: (int(toks[i]), status[i] == 2) for i in range(w) if status[i] != 0}
        toks = (C.c_uint32 * 8)()
        status = (C.c_int32 * 8)()
        n = C.c_size_t(0)
        self._check(self._lib.aha_b200_batch_step(self._h, toks, status, C.byref(n)))
        return {i: (int(toks[i]), status[i] == 2) for i in range(8) if status[i] != 0}

    def batch_logprobs(self):
        """-> {slot: record} for the slots whose request asked for log-probabilities: the record of the last token each delivered (by
        batch_add, batch_add_many or the last batch_step, including the step that finished it)."""
        w = getattr(self, "_batch_width", 8)
        recs = (L.Logprobs * w)()
        self._check(self._lib.aha_b200_batch_logprobs(self._h, recs, w))
        return {i: L.logprobs_record(recs[i]) for i in range(w) if recs[i].valid}

    def batch_add_speculative(self, input_ids, data=None, prediction=None, prompt_lookup=False, max_draft=7, ngram=3, max_tokens=1024,
                              temperature=0.0, top_p=None, top_k=None, repeat_penalty=1.0, repeat_last_n=64, seed=299792458, flags=0,
                              logprobs=False, top_logprobs=0, rules=None, return_usage=False):
        """Admit a speculative request into the open wide session (aha_b200_batch_add_speculative): admitted as batch_add admits it, then
        every batch_step_spec runs one verify pass of max_draft + 1 rows for it (drafts as for generate_speculative).  -> (slot, first token,
        finished), and with return_usage=True also the prompt-side usage dict."""
        ids = self._ids(input_ids)
        mm, _keep = self._mm(data)
        sp, _pred = L.spec_params(prediction, prompt_lookup, max_draft, ngram, self.vocab_size)
        flags |= L.logprob_flags(logprobs, top_logprobs, self.vocab_size)
        req = L.BatchRequest()
        req.ids = ids.ctypes.data_as(C.POINTER(C.c_uint32))
        req.seq_len = ids.size
        req.mm = C.pointer(mm) if mm is not None else None
        req.params = self._gen_params(max_tokens, temperature, top_p, top_k, repeat_penalty, repeat_last_n, seed, flags, rules=rules)
        slot, fin, tok = C.c_int32(-1), C.c_int32(0), C.c_uint32(0)
        u = L.Usage()
        self._check(self._lib.aha_b200_batch_add_speculative(self._h, C.byref(req), C.byref(sp), C.byref(slot), C.byref(tok), C.byref(fin),
                                                             C.byref(u)))
        res = (int(slot.value), int(tok.value), bool(fin.value))
        return (res, self._usage(u)) if return_usage else res

    def batch_step_spec(self):
        """One step of every running request (aha_b200_batch_step_spec) -> {slot: (tokens, finished)}: one token for a plain request,
        1 .. max_draft + 1 for a speculative one (empty when nothing is running)."""
        w = getattr(self, "_batch_width", 8)
        R = L.SPEC_MAX_ROWS
        toks, n_tok, status, n = (C.c_uint32 * (w * R))(), (C.c_uint32 * w)(), (C.c_int32 * w)(), C.c_size_t(0)
        self._check(self._lib.aha_b200_batch_step_spec(self._h, toks, n_tok, status, w, C.byref(n)))
        return {i: ([int(toks[i * R + k]) for k in range(n_tok[i])], status[i] == 2) for i in range(w) if status[i] != 0}

    def batch_logprobs_spec(self):
        """-> {slot: [record, ...]} for the slots whose request asked for log-probabilities: the records of every token each delivered in
        the last batch_step_spec (or at admission)."""
        w = getattr(self, "_batch_width", 8)
        R = L.SPEC_MAX_ROWS
        recs = (L.Logprobs * (w * R))()
        self._check(self._lib.aha_b200_batch_logprobs_spec(self._h, recs, w))
        out = {}
        for i in range(w):
            got = [L.logprobs_record(recs[i * R + k]) for k in range(R) if recs[i * R + k].valid]
            if got:
                out[i] = got
        return out

    def batch_spec_stats(self):
        """-> {slot: dict(passes, drafted, accepted)} for the slots whose (running or last) request was speculative."""
        w = getattr(self, "_batch_width", 8)
        st = (L.SpecStats * w)()
        self._check(self._lib.aha_b200_batch_spec_stats(self._h, st, w))
        return {i: dict(passes=int(st[i].passes), drafted=int(st[i].drafted), accepted=int(st[i].accepted)) for i in range(w) if st[i].passes}

    def batch_close(self):
        self._check(self._lib.aha_b200_batch_close(self._h))

    def batch_prefix_cache(self, max_tokens):
        """Turn the open session's prefix cache on (aha_b200_batch_prefix_cache): admitted text-only prompts leave their full 32-token
        pages in an index that keeps up to max_tokens / 32 of them alive, and later requests that start with those pages share them and
        prefill only what follows.  0 turns it off and releases the pages only the index holds."""
        self._check(self._lib.aha_b200_batch_prefix_cache(self._h, int(max_tokens)))

    def batch_prefix_stats(self):
        """-> (stats dict: cached_pages, shared_pages, hit_tokens, lookups, evicted_pages, max_pages, free_pages; {slot: prompt tokens its running
        request took from the cache} for every slot with a request that hit)."""
        w = getattr(self, "_batch_width", 8)
        st, hits = L.PrefixStats(), (C.c_size_t * w)()
        self._check(self._lib.aha_b200_batch_prefix_stats(self._h, C.byref(st), hits, w))
        return {name: int(getattr(st, name)) for name, _ in L.PrefixStats._fields_}, {i: int(hits[i]) for i in range(w) if hits[i]}

    # ---- cancel, suspend and resume requests of the open session (swap preemption)
    def batch_swap_space(self, max_tokens):
        """Size the handle's pinned host arena to max_tokens / 32 host pages (aha_b200_batch_swap_space; 0 frees it).  It outlives sessions;
        resizing is refused while a request is suspended."""
        n = L.swap_int("max_tokens", max_tokens, 0, 2 ** 63 - 1)
        self._check(self._lib.aha_b200_batch_swap_space(self._h, n))

    def batch_cancel(self, slot):
        """End the request in `slot` now, as if it had finished (a client went away): its pages and the slot are free at once, and
        batch_logprobs shows no record for it."""
        slot = L.swap_int("slot", slot, 0, 63)
        self._check(self._lib.aha_b200_batch_cancel(self._h, slot))

    def batch_suspend(self, slot):
        """Copy the request in `slot` to the swap arena and free its slot and pages -> its id (>= 1), for batch_resume / batch_discard."""
        slot, i = L.swap_int("slot", slot, 0, 63), C.c_uint32(0)
        self._check(self._lib.aha_b200_batch_suspend(self._h, slot, C.byref(i)))
        return int(i.value)

    def batch_resume(self, id):
        """Put a suspended request back into the lowest free slot -> that slot.  It delivers its next token at the next step, exactly the
        token it would have delivered uninterrupted."""
        id, s = L.swap_int("id", id, 1, 2 ** 32 - 1), C.c_int32(-1)
        self._check(self._lib.aha_b200_batch_resume(self._h, id, C.byref(s)))
        return int(s.value)

    def batch_discard(self, id):
        """Free a suspended request without resuming it."""
        id = L.swap_int("id", id, 1, 2 ** 32 - 1)
        self._check(self._lib.aha_b200_batch_discard(self._h, id))

    def batch_swap_stats(self):
        """-> dict(host_pages, free_host_pages, suspended, pages_out, pages_in, bytes_out, bytes_in, suspend_secs, resume_secs)"""
        st = L.SwapStats()
        self._check(self._lib.aha_b200_batch_swap_stats(self._h, C.byref(st)))
        return {name: (float if name.endswith("secs") else int)(getattr(st, name)) for name, _ in L.SwapStats._fields_}

    def debug_kv_swap(self, pool, table_out, table_in, host_pages, n_host_pages):
        """The page copies of suspend / resume on host data (aha_b200_debug_kv_swap): pool [layers][n_pool_pages][page_floats]; logical page p goes out from
        pool page table_out[p] to host page host_pages[p] and back into pool page table_in[p] -> (arena [n_host_pages][layers][page_floats]
        after the way out, pool after the way back)."""
        pool = np.ascontiguousarray(pool, np.float32)
        if pool.ndim != 3:
            raise ValueError("pool must be [layers][n_pool_pages][page_floats]")
        layers, n_pool, pf = pool.shape
        to, ti, hp = (np.ascontiguousarray(np.asarray(a, np.int32).reshape(-1)) for a in (table_out, table_in, host_pages))
        if not to.size == ti.size == hp.size:
            raise ValueError("table_out, table_in and host_pages must have one entry per page")
        host = np.empty((int(n_host_pages), layers, pf), np.float32)
        out = np.empty_like(pool)
        f = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
        i32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))
        self._check(self._lib.aha_b200_debug_kv_swap(self._h, layers, pf, n_pool, int(n_host_pages), to.size, i32(to), i32(ti), i32(hp), f(pool),
                                                     f(host), f(out)))
        return host, out

    def generate_stream(self, input_ids, on_token, data=None, max_tokens=1024, temperature=0.0, top_p=None, top_k=None,
                        repeat_penalty=1.0, repeat_last_n=64, seed=299792458, reuse_prefix=False, logprobs=False, top_logprobs=0, fsm=None,
                        rules=None):
        """generate_stream_generic: on_token(token, index) is called per generated token as its step completes; a truthy
        return value ends the request.  logprobs=True: on_token(token, index, record).  -> usage dict."""
        ids = self._ids(input_ids)
        mm, _keep = self._mm(data)
        flags = (L.GEN_REUSE_PREFIX if reuse_prefix else 0) | L.logprob_flags(logprobs, top_logprobs, self.vocab_size)
        p = self._gen_params(max_tokens, temperature, top_p, top_k, repeat_penalty, repeat_last_n, seed, flags, fsm, rules)
        err = []

        def _cb(_user, token, index, *lp):
            try:
                args = (int(token), int(index)) + ((L.logprobs_record(lp[0].contents),) if lp else ())
                return 1 if on_token(*args) else 0
            except Exception as e:  # never unwind through the C ABI
                err.append(e)
                return 1
        u = L.Usage()
        ids_p, mm_p = ids.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(mm) if mm is not None else None
        if logprobs:
            cb = L.LOGPROBS_CALLBACK(_cb)
            self._check(self._lib.aha_b200_generate_stream_logprobs(self._h, ids_p, ids.size, mm_p, C.byref(p), cb, None, C.byref(u)))
        else:
            cb = L.TOKEN_CALLBACK(_cb)
            self._check(self._lib.aha_b200_generate_stream(self._h, ids_p, ids.size, mm_p, C.byref(p), cb, None, C.byref(u)))
        if err:
            raise err[0]
        return self._usage(u)

    def asr_generate(self, chunks, max_tokens=1024, temperature=0.0, top_p=None, seed=34562, on_token=None):
        """Qwen3AsrGenerateModel::generate: chunks = [(ids, mel), ...] (one AudioData each).  -> (ids of all chunks, usage)."""
        keep = []
        arr = (L.AsrChunk * len(chunks))()
        for i, (ids, mel) in enumerate(chunks):
            ids = self._ids(ids)
            mel = np.ascontiguousarray(mel, np.float32)
            keep += [ids, mel]
            arr[i].ids = ids.ctypes.data_as(C.POINTER(C.c_uint32))
            arr[i].seq_len = ids.size
            arr[i].input_features = L.make_desc(mel)
        p = self._gen_params(max_tokens, temperature, top_p, None, 1.0, 64, seed)
        cap = max(max_tokens, 1) * len(chunks)
        out = (C.c_uint32 * cap)()
        n = C.c_size_t(0)
        u = L.Usage()
        cb = L.TOKEN_CALLBACK((lambda _u, t, i: 1 if on_token(int(t), int(i)) else 0) if on_token else 0)
        self._check(self._lib.aha_b200_asr_generate(self._h, arr, len(chunks), C.byref(p), out, cap, C.byref(n), cb, None, C.byref(u)))
        return [int(out[i]) for i in range(n.value)], self._usage(u)

    def debug_sample(self, logits, context=(), draw_index=0, temperature=0.0, top_p=None, top_k=None, repeat_penalty=1.0,
                     repeat_last_n=64, seed=299792458):
        """The device sampler (sample_kernel) on a given logits row of any length (tests) -> token."""
        params = dict(temperature=temperature, top_p=top_p, top_k=top_k, repeat_penalty=repeat_penalty, repeat_last_n=repeat_last_n, seed=seed)
        return int(self.debug_sample_rows(logits, [params], [context], draw_index)["token"][0])

    def debug_sample_rows(self, logits, params, contexts=None, draw_index=0, overwrite=False, kernel=0, act=None, on=None, fsm=None,
                          constrained=None, fsm_states=None, rules=None, ruled=None):
        """The device sampler on given logits, one call for len(params) rows (1 to 64; tests).
        logits: [V] (every row reads it) or [rows, ld] with V = ld.  params: per row a dict of generate()'s sampling keywords
        (temperature, top_p, top_k, repeat_penalty, repeat_last_n, seed).  contexts: per row the tokens generated so far;
        draw_index: per row (or one for all) the draws already consumed.  overwrite: the last context token stands for the ArgMax token a
        decode step pushed; the sampled token replaces it.  kernel 0: sample_kernel per row; 1: sample_rows_kernel, row r as slot act[r]
        (default r), on: [64] flags per slot (default all on).
        fsm: (offsets, tokens, next) of a token automaton (aha_b200_debug_sample_fsm); the rows with constrained[r] (default all) are
        constrained by it from state fsm_states[r] (default 0).
        rules: dict(presence_penalty, frequency_penalty, logit_bias) (aha_b200_debug_sample_rules), applied by the rows with ruled[r]
        (default all); the call checks that every row's count row is zero again afterwards.
        -> dict of uint32 arrays [rows]: token (0xffffffff where the row did not sample), state_token, n_hist, n_draws (the DecodeState
        after the call), last_hist (the last history word, 0xffffffff without a context) and, with fsm, fsm_state (after the call)."""
        rows = len(params)
        lg = np.ascontiguousarray(logits, np.float32)
        V, ld = (lg.size, 0) if lg.ndim == 1 else (lg.shape[1], lg.shape[1])
        if lg.ndim not in (1, 2) or (lg.ndim == 2 and lg.shape[0] != rows):
            raise ValueError(f"logits must be [V] or [{rows}, V], got {lg.shape}")
        ps = (L.GenParams * rows)()
        for r, q in enumerate(params):
            q = dict(dict(temperature=0.0, top_p=None, top_k=None, repeat_penalty=1.0, repeat_last_n=64, seed=299792458), **q)
            ps[r] = self._gen_params(1, q["temperature"], q["top_p"], q["top_k"], q["repeat_penalty"], q["repeat_last_n"], q["seed"])
        ctxs = [np.asarray(c, np.uint32).reshape(-1) for c in (contexts if contexts is not None else [()] * rows)]
        if len(ctxs) != rows:
            raise ValueError(f"{len(ctxs)} contexts for {rows} rows")
        cat = np.ascontiguousarray(np.concatenate(ctxs + [np.zeros(0, np.uint32)]))
        n_ctx = np.array([c.size for c in ctxs], np.uint32)
        draws = np.ascontiguousarray(np.broadcast_to(np.asarray(draw_index, np.uint32), (rows,)))
        act = np.ascontiguousarray(np.arange(rows) if act is None else act, np.int32)
        on = np.ascontiguousarray(np.ones(64) if on is None else on, np.int32)
        if act.size != rows or on.size != 64:
            raise ValueError("act needs one slot per row and on one flag per slot (64)")
        tok, state, hist = np.zeros(rows, np.uint32), np.zeros((rows, 3), np.uint32), np.zeros(rows, np.uint32)
        u32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint32))
        i32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))
        lg_p = lg.ctypes.data_as(C.POINTER(C.c_float))
        if fsm is None and rules is None:
            self._check(self._lib.aha_b200_debug_sample(self._h, int(kernel), rows, V, lg_p, ld, ps, u32(cat), u32(n_ctx), u32(draws),
                                                        1 if overwrite else 0, i32(act), i32(on), u32(tok), u32(state), u32(hist)))
            return dict(token=tok, state_token=state[:, 0].copy(), n_hist=state[:, 1].copy(), n_draws=state[:, 2].copy(), last_hist=hist)
        f, _keep = L.token_fsm(*fsm) if fsm is not None else (None, None)
        con = np.ascontiguousarray(np.broadcast_to(np.asarray(True if constrained is None else constrained, np.int32), (rows,)))
        fin = np.ascontiguousarray(np.broadcast_to(np.asarray(0 if fsm_states is None else fsm_states, np.uint32), (rows,)))
        fout = np.zeros(rows, np.uint32)
        if rules is None:
            self._check(self._lib.aha_b200_debug_sample_fsm(self._h, int(kernel), rows, V, lg_p, ld, ps, u32(cat), u32(n_ctx), u32(draws),
                                                            1 if overwrite else 0, i32(act), i32(on), C.byref(f), i32(con), u32(fin), u32(tok),
                                                            u32(state), u32(hist), u32(fout)))
        else:
            rl, _rkeep = L.logit_rules(**rules)
            rd = np.ascontiguousarray(np.broadcast_to(np.asarray(True if ruled is None else ruled, np.int32), (rows,)))
            self._check(self._lib.aha_b200_debug_sample_rules(self._h, int(kernel), rows, V, lg_p, ld, ps, u32(cat), u32(n_ctx), u32(draws),
                                                              1 if overwrite else 0, i32(act), i32(on), C.byref(f) if f is not None else None,
                                                              i32(con), u32(fin), C.byref(rl), i32(rd), u32(tok), u32(state), u32(hist), u32(fout)))
        out = dict(token=tok, state_token=state[:, 0].copy(), n_hist=state[:, 1].copy(), n_draws=state[:, 2].copy(), last_hist=hist)
        if fsm is not None:
            out["fsm_state"] = fout
        return out

    def debug_logprobs(self, logits, token, n_top=0):
        """The log-probability kernels on a given logits row of any length (tests) -> record dict."""
        lg = np.ascontiguousarray(logits, np.float32).reshape(-1)
        r = L.Logprobs()
        self._check(self._lib.aha_b200_debug_logprobs(self._h, lg.ctypes.data_as(C.POINTER(C.c_float)), lg.size, int(token), int(n_top),
                                                      C.byref(r)))
        return L.logprobs_record(r)

    # ------------------------------------------------------------------ Qwen3-Embedding / Qwen3-Reranker
    def embed(self, input_ids):
        """Qwen3Embedding::embed_one on token ids -> unit vector (hidden_size,) float32."""
        ids = self._ids(input_ids)
        out = np.empty(self.hidden_size, np.float32)
        self._check(self._lib.aha_b200_embed(self._h, ids.ctypes.data_as(C.POINTER(C.c_uint32)), ids.size,
                                             out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    def embed_batch(self, list_of_ids):
        """Qwen3Embedding::embed_multi on token ids -> unit vectors (n, hidden_size) float32 in input order, the texts packed into
        shared prefills (each text attends only to itself)."""
        texts = [self._ids(t) for t in list_of_ids]
        cat = np.ascontiguousarray(np.concatenate(texts)) if texts else np.zeros(0, np.uint32)
        lens = (C.c_size_t * max(len(texts), 1))(*[t.size for t in texts])
        out = np.empty((len(texts), self.hidden_size), np.float32)
        self._check(self._lib.aha_b200_embed_batch(self._h, cat.ctypes.data_as(C.POINTER(C.c_uint32)), lens, len(texts),
                                                   out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    # ------------------------------------------------------------------ scoring given text
    def score(self, input_ids, start=1, top=0):
        """Log-probability of every token of input_ids from position `start` on (aha_b200_score): entry k is token input_ids[start + k]
        under the model given the tokens before it.  -> dict of numpy arrays: tokens (n,) uint32, logprobs (n,) float32 and, with top > 0,
        top_ids (n, top) uint32 and top_logprobs (n, top) float32 (the top alternatives at each position, by logit desc, id asc)."""
        ids = self._ids(input_ids)
        n = max(ids.size - int(start), 0)
        recs = np.zeros(max(n, 1), L.LOGPROBS_DTYPE)
        got = C.c_size_t()
        self._check(self._lib.aha_b200_score(self._h, ids.ctypes.data_as(C.POINTER(C.c_uint32)), ids.size, int(start), int(top),
                                             recs.ctypes.data_as(C.POINTER(L.Logprobs)), n, C.byref(got)))
        return L.score_arrays(recs[:got.value], top)

    def score_batch(self, list_of_ids, starts=None, top=0):
        """score() for many texts packed into shared prefills (aha_b200_score_batch) -> one dict of arrays per text, in input order.
        starts: one start per text (None: 1 for every text)."""
        texts = [self._ids(t) for t in list_of_ids]
        if starts is not None and len(starts) != len(texts):
            raise ValueError(f"{len(starts)} starts for {len(texts)} texts")
        st = [1] * len(texts) if starts is None else [int(s) for s in starts]
        counts = [max(t.size - s, 0) for t, s in zip(texts, st)]
        cat = np.ascontiguousarray(np.concatenate(texts)) if texts else np.zeros(0, np.uint32)
        lens = (C.c_size_t * max(len(texts), 1))(*[t.size for t in texts])
        c_starts = (C.c_size_t * max(len(texts), 1))(*st)
        recs = np.zeros(max(sum(counts), 1), L.LOGPROBS_DTYPE)
        got = C.c_size_t()
        self._check(self._lib.aha_b200_score_batch(self._h, cat.ctypes.data_as(C.POINTER(C.c_uint32)), lens, c_starts, len(texts), int(top),
                                                   recs.ctypes.data_as(C.POINTER(L.Logprobs)), sum(counts), C.byref(got)))
        bounds = np.cumsum([0] + counts)
        return [L.score_arrays(recs[bounds[j]:bounds[j + 1]], top) for j in range(len(texts))]

    def debug_score_head(self, hidden, targets, top=0, impl=0):
        """The scoring head alone on pre-norm hidden rows [M, H] (tests): impl 0 = score_head_kernel, 1 = the gemm_tc + row-kernel twin.
        -> dict of arrays as score(), row r scored at targets[r]."""
        x = np.ascontiguousarray(hidden, np.float32).reshape(-1, self.hidden_size)
        tg = np.ascontiguousarray(targets, np.uint32).reshape(-1)
        if tg.size != x.shape[0]:
            raise ValueError("one target per row")
        recs = np.zeros(x.shape[0], L.LOGPROBS_DTYPE)
        self._check(self._lib.aha_b200_debug_score_head(self._h, int(impl), x.ctypes.data_as(C.POINTER(C.c_float)), x.shape[0],
                                                        tg.ctypes.data_as(C.POINTER(C.c_uint32)), int(top),
                                                        recs.ctypes.data_as(C.POINTER(L.Logprobs))))
        return L.score_arrays(recs, top)

    def rerank(self, query_ids, documents_ids):
        """Qwen3Reranker::rerank on token ids -> cosine scores (n_docs,) float32."""
        q = self._ids(query_ids)
        docs = [self._ids(d) for d in documents_ids]
        cat = np.ascontiguousarray(np.concatenate(docs)) if docs else np.zeros(0, np.uint32)
        lens = (C.c_size_t * max(len(docs), 1))(*[d.size for d in docs])
        out = np.empty(len(docs), np.float32)
        self._check(self._lib.aha_b200_rerank(self._h, q.ctypes.data_as(C.POINTER(C.c_uint32)), q.size,
                                              cat.ctypes.data_as(C.POINTER(C.c_uint32)), lens, len(docs),
                                              out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    # ------------------------------------------------------------------ frontends
    def mel_spectrogram(self, wave):
        wave = np.ascontiguousarray(wave, dtype=np.float32).reshape(-1)
        n_mels = self.config["thinker_config"]["audio_config"]["num_mel_bins"]
        cap = n_mels * (wave.size // 160 + 2)
        out = np.empty(cap, np.float32)
        nf = C.c_size_t(0)
        self._check(self._lib.aha_b200_mel_spectrogram(self._h, wave.ctypes.data_as(C.POINTER(C.c_float)), wave.size,
                                                       out.ctypes.data_as(C.POINTER(C.c_float)), cap, C.byref(nf)))
        return out[: n_mels * nf.value].reshape(n_mels, nf.value).copy()

    def image_patchify(self, img_u8_hwc):
        img = np.ascontiguousarray(img_u8_hwc, dtype=np.uint8)
        h, w, _ = img.shape
        vc = self.config["vision_config"]
        feat = vc["in_channels"] * vc["temporal_patch_size"] * vc["patch_size"] ** 2
        n = (h // vc["patch_size"]) * (w // vc["patch_size"])
        out = np.empty((n, feat), np.float32)
        grid = (C.c_uint32 * 3)()
        self._check(self._lib.aha_b200_image_patchify(self._h, img.ctypes.data_as(C.POINTER(C.c_uint8)), h, w,
                                                      out.ctypes.data_as(C.POINTER(C.c_float)), out.size, grid))
        return out, np.array([[grid[0], grid[1], grid[2]]], dtype=np.uint32)

    def video_preprocess(self, frames_u8_thwc):
        """Qwen3VLProcessor::process_videos for one clip: RGB24 frames (T, H, W, 3) at their video_smart_resize size ->
        (pixel_values_video, video_grid_thw)."""
        fr = np.ascontiguousarray(frames_u8_thwc, dtype=np.uint8)
        t, h, w, _ = fr.shape
        vc = self.config["vision_config"]
        tp = vc["temporal_patch_size"]
        feat = vc["in_channels"] * tp * vc["patch_size"] ** 2
        n = ((t + tp - 1) // tp) * (h // vc["patch_size"]) * (w // vc["patch_size"])
        out = np.empty((n, feat), np.float32)
        grid = (C.c_uint32 * 3)()
        self._check(self._lib.aha_b200_video_preprocess(self._h, fr.ctypes.data_as(C.POINTER(C.c_uint8)), t, h, w,
                                                        out.ctypes.data_as(C.POINTER(C.c_float)), out.size, grid))
        return out, np.array([[grid[0], grid[1], grid[2]]], dtype=np.uint32)

    def image_resize(self, img_u8_hwc, new_h, new_w):
        """DynamicImage::resize_exact(new_w, new_h, CatmullRom) on the GPU."""
        img = np.ascontiguousarray(img_u8_hwc, dtype=np.uint8)
        h, w, _ = img.shape
        out = np.empty((new_h, new_w, 3), np.uint8)
        self._check(self._lib.aha_b200_image_resize(self._h, img.ctypes.data_as(C.POINTER(C.c_uint8)), h, w, new_h, new_w,
                                                    out.ctypes.data_as(C.POINTER(C.c_uint8))))
        return out

    def resample(self, wave, orig_freq, new_freq):
        """resample_simple (audio_utils.rs:245-255) of a mono f32 waveform on the GPU: windowed-sinc polyphase filter, width 6, rolloff 0.99."""
        w = np.ascontiguousarray(wave, np.float32).reshape(-1)
        n = C.c_size_t(0)
        fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
        self._check(self._lib.aha_b200_resample(self._h, fp(w), w.size, int(orig_freq), int(new_freq), None, 0, C.byref(n)))
        out = np.empty(n.value, np.float32)
        self._check(self._lib.aha_b200_resample(self._h, fp(w), w.size, int(orig_freq), int(new_freq), fp(out), out.size, C.byref(n)))
        return out[:n.value]

    def image_preprocess(self, img_u8_hwc, min_pixels=65536, max_pixels=16777216):
        """Qwen3VLProcessor::process_img + process_vision_tensor for an image of any size -> (pixel_values, grid_thw)."""
        img = np.ascontiguousarray(img_u8_hwc, dtype=np.uint8)
        h, w, _ = img.shape
        vc = self.config["vision_config"]
        from . import processors
        rh, rw = processors.img_smart_resize(h, w, vc["patch_size"] * vc["spatial_merge_size"], min_pixels, max_pixels)
        feat = vc["in_channels"] * vc["temporal_patch_size"] * vc["patch_size"] ** 2
        out = np.empty(((rh // vc["patch_size"]) * (rw // vc["patch_size"]), feat), np.float32)
        grid = (C.c_uint32 * 3)()
        self._check(self._lib.aha_b200_image_preprocess(self._h, img.ctypes.data_as(C.POINTER(C.c_uint8)), h, w, min_pixels, max_pixels,
                                                        out.ctypes.data_as(C.POINTER(C.c_float)), out.size, grid))
        return out, np.array([[grid[0], grid[1], grid[2]]], dtype=np.uint32)

    # ------------------------------------------------------------------ introspection (tests / bench)
    def decode_steps(self, first_token, seqlen_offset, n_steps, want_tokens=True, timed=False):
        """n_steps graph replays with on-device token feedback; timed=True also returns the CUDA-event ms."""
        out = (C.c_uint32 * max(n_steps, 1))() if want_tokens else None
        ms = C.c_double(0.0)
        self._check(self._lib.aha_b200_decode_steps(self._h, int(first_token), int(seqlen_offset), int(n_steps), out,
                                                    C.byref(ms)))
        toks = [int(out[i]) for i in range(n_steps)] if want_tokens else None
        return (toks, ms.value) if timed else toks

    def bench_kernel(self, which, iters=200):
        ms = C.c_double(0.0)
        nb = C.c_uint64(0)
        self._check(self._lib.aha_b200_bench_kernel(self._h, which.encode(), int(iters), C.byref(ms), C.byref(nb)))
        return ms.value, int(nb.value)

    def debug_gemm(self, x, w16, bias=None, resid=None, impl=2, epi=0, act=0, iters=0):
        """y = epilogue(x @ w16.T + bias) through the library's GEMM (impl 1 = SIMT, 2 / 3 = wgmma 128x128 / 128x256 tiles) or a decode
        projection kernel (4 = the batch-1 GEMV once per row, 5 / 6 = the batched GEMV, registers / cp.async ring, M <= 8, 7 = the wide
        batched GEMV, M <= 64; their SwiGLU epilogue runs behind a unit-gain RMSNorm prologue). -> (y, ms)"""
        x = np.ascontiguousarray(x, np.float32)
        w16 = np.ascontiguousarray(w16, np.float16)
        M, K = x.shape
        N = w16.shape[0]
        out = np.empty((M, N // 2 if epi == 3 else N), np.float32)
        fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float)) if a is not None else None
        b = np.ascontiguousarray(bias, np.float32) if bias is not None else None
        r = np.ascontiguousarray(resid, np.float32) if resid is not None else None
        ms = C.c_double(0.0)
        self._check(self._lib.aha_b200_debug_gemm(self._h, impl, epi, act, M, N, K, fp(x), w16.ctypes.data_as(C.POINTER(C.c_uint16)),
                                                  fp(b), fp(r), fp(out), iters, C.byref(ms)))
        return out, ms.value

    def stream_ptr(self):
        return int(self._lib.aha_b200_stream(self._h) or 0)

    def stats(self):
        s = L.Stats()
        self._check(self._lib.aha_b200_get_stats(self._h, C.byref(s)))
        return {k: int(getattr(s, k)) for k, _ in L.Stats._fields_}

    def reset_stats(self):
        self._check(self._lib.aha_b200_reset_stats(self._h))

    def set_trace(self, on=True):
        self._check(self._lib.aha_b200_set_trace(self._h, 1 if on else 0))

    def debug_read(self, what, index, cap):
        out = np.empty(cap, np.float32)
        n = C.c_size_t(0)
        self._check(self._lib.aha_b200_debug_read(self._h, what.encode(), int(index),
                                                  out.ctypes.data_as(C.POINTER(C.c_float)), cap, C.byref(n)))
        return out[: n.value].copy()

    def close(self):
        if getattr(self, "_h", None):
            self._lib.aha_b200_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
