"""ctypes bindings of include/aha_b200.h.  No torch types cross this boundary."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libaha_b200.so")

AHA_F32, AHA_F16, AHA_BF16, AHA_U32, AHA_I64, AHA_U8 = range(6)
_NP2AHA = {np.dtype(np.float32): AHA_F32, np.dtype(np.float16): AHA_F16, np.dtype(np.uint32): AHA_U32,
           np.dtype(np.int64): AHA_I64, np.dtype(np.uint8): AHA_U8}


class TensorDesc(C.Structure):
    _fields_ = [("name", C.c_char_p), ("dtype", C.c_int32), ("rank", C.c_int32), ("shape", C.c_int64 * 8),
                ("data", C.c_void_p)]


class MM(C.Structure):
    _fields_ = [("data_vec", C.POINTER(TensorDesc)), ("n", C.c_size_t)]


class Options(C.Structure):
    _fields_ = [("device", C.c_int32), ("tp_rank", C.c_int32), ("tp_world", C.c_int32), ("max_ctx", C.c_int32),
                ("max_prefill", C.c_int32), ("max_patches", C.c_int32), ("max_frames", C.c_int32),
                ("use_graph", C.c_int32), ("decode_impl", C.c_int32), ("gemm_impl", C.c_int32),
                ("tp_comm", C.c_void_p), ("reserved", C.c_int32 * 8)]


class GenParams(C.Structure):
    _fields_ = [("temperature", C.c_float), ("repeat_penalty", C.c_float), ("repeat_last_n", C.c_int32),
                ("max_tokens", C.c_uint32), ("seed", C.c_uint64), ("top_p", C.c_float), ("top_k", C.c_int32),
                ("flags", C.c_uint32), ("reserved", C.c_uint32)]


GEN_EOS_ON_FIRST, GEN_CONTINUE_RNG, GEN_REUSE_PREFIX, GEN_LOGPROBS, GEN_CONSTRAINED, GEN_LOGIT_RULES = 1, 2, 4, 8, 16, 32
MAX_TOP_LOGPROBS = 20
TOKEN_CALLBACK = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint32, C.c_uint32)


def gen_top_logprobs(n):
    """AHA_GEN_TOP_LOGPROBS(n): the count in bits 8 and up of flags, unmasked (an out-of-range count is refused, never wrapped)."""
    return (int(n) << 8) & 0xFFFFFFFF


def logprob_flags(logprobs=False, top_logprobs=0, vocab_size=None):
    """flags bits of an OpenAI-style (logprobs, top_logprobs) pair, checked the way the library checks them."""
    if isinstance(top_logprobs, bool) or not isinstance(top_logprobs, (int, np.integer)):
        raise TypeError(f"top_logprobs must be an int, not {type(top_logprobs).__name__}")
    n = int(top_logprobs)
    if not logprobs:
        if n:
            raise ValueError("top_logprobs needs logprobs=True")
        return 0
    if n < 0 or n > MAX_TOP_LOGPROBS:
        raise ValueError(f"top_logprobs must be 0 to {MAX_TOP_LOGPROBS}, got {n}")
    if vocab_size is not None and n > vocab_size:
        raise ValueError(f"top_logprobs {n} exceeds the vocabulary of {vocab_size}")
    return GEN_LOGPROBS | gen_top_logprobs(n)


class TokenFsm(C.Structure):
    _fields_ = [("n_states", C.c_uint32), ("start", C.c_uint32), ("offsets", C.POINTER(C.c_uint64)), ("tokens", C.POINTER(C.c_uint32)),
                ("next", C.POINTER(C.c_uint32))]


def token_fsm(offsets, tokens, next, start=0):
    """(TokenFsm, arrays it points into) of a token automaton in CSR form: state s allows tokens[offsets[s]:offsets[s + 1]] (ascending)
    and next[j] is the state after tokens[j].  The library checks the rest (aha_b200_fsm_check)."""
    off = np.ascontiguousarray(np.asarray(offsets, np.int64).reshape(-1).astype(np.uint64))
    tok = np.ascontiguousarray(np.asarray(tokens, np.int64).reshape(-1).astype(np.uint32))
    nxt = np.ascontiguousarray(np.asarray(next, np.int64).reshape(-1).astype(np.uint32))
    if off.size < 1 or tok.size != nxt.size:
        raise ValueError("offsets needs n_states + 1 entries, and tokens and next one entry per transition each")
    ptr = lambda a, t: a.ctypes.data_as(C.POINTER(t)) if a.size else None
    f = TokenFsm(n_states=off.size - 1, start=int(start), offsets=ptr(off, C.c_uint64), tokens=ptr(tok, C.c_uint32), next=ptr(nxt, C.c_uint32))
    return f, (off, tok, nxt)


class LogitRules(C.Structure):
    _fields_ = [("presence_penalty", C.c_float), ("frequency_penalty", C.c_float), ("bias_ids", C.POINTER(C.c_uint32)),
                ("bias_values", C.POINTER(C.c_float)), ("n_bias", C.c_size_t), ("fsm", C.c_uint32), ("reserved", C.c_uint32 * 3)]


def logit_rules(presence_penalty=0.0, frequency_penalty=0.0, logit_bias=None, fsm=None):
    """(LogitRules, arrays it points into).  logit_bias: OpenAI's map of token id (int or decimal string) -> bias, or (id, bias) pairs;
    fsm: the id of a token automaton on the handle, or None.  The library checks ranges and ids (aha_b200_rules_check)."""
    items = list((logit_bias or {}).items()) if isinstance(logit_bias, dict) else list(logit_bias or [])
    ids = np.ascontiguousarray(np.array([int(k) for k, _ in items], np.int64).astype(np.uint32))
    vals = np.ascontiguousarray(np.array([float(v) for _, v in items], np.float32))
    ptr = lambda a, t: a.ctypes.data_as(C.POINTER(t)) if a.size else None
    r = LogitRules(presence_penalty=float(presence_penalty), frequency_penalty=float(frequency_penalty), bias_ids=ptr(ids, C.c_uint32),
                   bias_values=ptr(vals, C.c_float), n_bias=ids.size, fsm=0 if fsm is None else int(fsm))
    return r, (ids, vals)


class Logprobs(C.Structure):
    _fields_ = [("token", C.c_uint32), ("index", C.c_uint32), ("logprob", C.c_float), ("n_top", C.c_uint32),
                ("top_ids", C.c_uint32 * MAX_TOP_LOGPROBS), ("top_logprobs", C.c_float * MAX_TOP_LOGPROBS),
                ("valid", C.c_uint32), ("reserved", C.c_uint32)]


def logprobs_record(r):
    """aha_logprobs -> dict(token, index, logprob, top_ids, top_logprobs); the float32 values are kept exactly."""
    n = int(r.n_top)
    return dict(token=int(r.token), index=int(r.index), logprob=np.float32(r.logprob),
                top_ids=[int(r.top_ids[i]) for i in range(n)], top_logprobs=[np.float32(r.top_logprobs[i]) for i in range(n)])


# aha_logprobs as a numpy record: the scoring entries fill arrays of them in one call (no Python object per record)
LOGPROBS_DTYPE = np.dtype([("token", "<u4"), ("index", "<u4"), ("logprob", "<f4"), ("n_top", "<u4"), ("top_ids", "<u4", (MAX_TOP_LOGPROBS,)),
                           ("top_logprobs", "<f4", (MAX_TOP_LOGPROBS,)), ("valid", "<u4"), ("reserved", "<u4")])
assert LOGPROBS_DTYPE.itemsize == C.sizeof(Logprobs)


def score_arrays(recs, top):
    """records of a scoring call -> dict(tokens, logprobs[, top_ids [n, top], top_logprobs [n, top]]) of numpy arrays"""
    d = dict(tokens=recs["token"].copy(), logprobs=recs["logprob"].copy())
    if top:
        d["top_ids"] = recs["top_ids"][:, :top].copy()
        d["top_logprobs"] = recs["top_logprobs"][:, :top].copy()
    return d


LOGPROBS_CALLBACK = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(Logprobs))


SPEC_PROMPT_LOOKUP = 1
SPEC_MAX_ROWS = 16
SPEC_MAX_DRAFT = 15
SPEC_MAX_NGRAM = 8


class SpecParams(C.Structure):
    _fields_ = [("prediction", C.POINTER(C.c_uint32)), ("n_prediction", C.c_size_t), ("max_draft", C.c_uint32), ("ngram", C.c_uint32),
                ("flags", C.c_uint32), ("reserved", C.c_uint32 * 3)]


class SpecStats(C.Structure):
    _fields_ = [("passes", C.c_uint32), ("drafted", C.c_uint32), ("accepted", C.c_uint32), ("reserved", C.c_uint32)]


def spec_params(prediction=None, prompt_lookup=False, max_draft=7, ngram=3, vocab_size=None):
    """(SpecParams, prediction array to keep alive) of a speculative request, checked the way the library checks them."""
    for name, v, lo, hi in (("max_draft", max_draft, 1, SPEC_MAX_DRAFT), ("ngram", ngram, 0, SPEC_MAX_NGRAM)):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
            raise TypeError(f"{name} must be an int, not {type(v).__name__}")
        if not lo <= int(v) <= hi:
            raise ValueError(f"{name} must be {lo} to {hi}, got {int(v)}")
    pred = np.zeros(0, np.uint32)
    if prediction is not None:
        p = np.asarray(prediction).reshape(-1)
        if p.size and not np.issubdtype(p.dtype, np.integer):
            raise TypeError("prediction must hold token ids (integers)")
        if p.size and (p.min() < 0 or (vocab_size is not None and p.max() >= vocab_size)):
            raise ValueError("prediction token id out of range")
        pred = np.ascontiguousarray(p.astype(np.uint32))
    sp = SpecParams(prediction=pred.ctypes.data_as(C.POINTER(C.c_uint32)) if pred.size else None, n_prediction=pred.size,
                    max_draft=int(max_draft), ngram=int(ngram), flags=SPEC_PROMPT_LOOKUP if prompt_lookup else 0)
    return sp, pred


class AsrChunk(C.Structure):
    _fields_ = [("ids", C.POINTER(C.c_uint32)), ("seq_len", C.c_size_t), ("input_features", TensorDesc)]


class BatchRequest(C.Structure):
    _fields_ = [("ids", C.POINTER(C.c_uint32)), ("seq_len", C.c_size_t), ("mm", C.POINTER(MM)), ("params", GenParams)]


class Usage(C.Structure):
    _fields_ = [("prompt_tokens", C.c_uint32), ("completion_tokens", C.c_uint32), ("prompt_secs", C.c_double),
                ("completion_secs", C.c_double), ("vision_secs", C.c_double)]


class Stats(C.Structure):
    _fields_ = [("kernel_launches", C.c_uint64), ("graph_launches", C.c_uint64),
                ("kernels_per_decode_step", C.c_uint64), ("weight_bytes", C.c_uint64),
                ("kv_bytes_per_token", C.c_uint64), ("decode_bytes_per_step_fixed", C.c_uint64)]


class PrefixStats(C.Structure):
    _fields_ = [("cached_pages", C.c_uint64), ("shared_pages", C.c_uint64), ("hit_tokens", C.c_uint64), ("lookups", C.c_uint64),
                ("evicted_pages", C.c_uint64), ("max_pages", C.c_uint64), ("free_pages", C.c_uint64)]


class SwapStats(C.Structure):
    _fields_ = [("host_pages", C.c_uint64), ("free_host_pages", C.c_uint64), ("suspended", C.c_uint64), ("pages_out", C.c_uint64),
                ("pages_in", C.c_uint64), ("bytes_out", C.c_uint64), ("bytes_in", C.c_uint64), ("suspend_secs", C.c_double),
                ("resume_secs", C.c_double)]


def swap_int(name, v, lo, hi):
    """v as an int in [lo, hi], refused the way the swap entries' arguments are: TypeError for a non-int (bool included), ValueError out of range"""
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
        raise TypeError(f"{name} must be an int, not {type(v).__name__}")
    if not lo <= int(v) <= hi:
        raise ValueError(f"{name} must be {lo} to {hi}, got {int(v)}")
    return int(v)


# every symbol include/aha_b200.h declares: name -> (restype, argtypes)
_P = C.c_void_p
_U32P = C.POINTER(C.c_uint32)
_F32P = C.POINTER(C.c_float)
_I32P = C.POINTER(C.c_int32)
SYMBOLS = {
    "aha_b200_abi_version": (C.c_int, []),
    "aha_b200_create": (C.c_int, [C.c_char_p, C.c_char_p, C.POINTER(TensorDesc), C.c_size_t, _U32P, C.c_size_t,
                                  C.POINTER(Options), C.POINTER(_P)]),
    "aha_b200_forward_initial": (C.c_int, [_P, _U32P, C.c_size_t, C.c_size_t, C.POINTER(MM), _F32P, _U32P]),
    "aha_b200_forward_step": (C.c_int, [_P, _U32P, C.c_size_t, C.c_size_t, _F32P, _U32P]),
    "aha_b200_forward_extend": (C.c_int, [_P, _U32P, C.c_size_t, C.c_size_t, _F32P, _U32P]),
    "aha_b200_last_prefix_hit": (C.c_size_t, [_P]),
    "aha_b200_prefix_match": (C.c_size_t, [_U32P, C.c_size_t, _U32P, C.c_size_t, _U32P, C.c_size_t, C.c_int]),
    "aha_b200_mm_fingerprint": (C.c_uint64, [C.POINTER(MM)]),
    "aha_b200_clear_cache": (C.c_int, [_P]),
    "aha_b200_stop_token_ids": (C.c_size_t, [_P, _U32P, C.c_size_t]),
    "aha_b200_generate": (C.c_int, [_P, _U32P, C.c_size_t, C.POINTER(MM), C.POINTER(GenParams), _U32P, C.c_size_t,
                                    C.POINTER(C.c_size_t), C.POINTER(Usage)]),
    "aha_b200_generate_logprobs": (C.c_int, [_P, _U32P, C.c_size_t, C.POINTER(MM), C.POINTER(GenParams), _U32P, C.POINTER(Logprobs),
                                             C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(Usage)]),
    "aha_b200_generate_stream_logprobs": (C.c_int, [_P, _U32P, C.c_size_t, C.POINTER(MM), C.POINTER(GenParams), LOGPROBS_CALLBACK, C.c_void_p,
                                                    C.POINTER(Usage)]),
    "aha_b200_batch_logprobs": (C.c_int, [_P, C.POINTER(Logprobs), C.c_size_t]),
    "aha_b200_generate_speculative": (C.c_int, [_P, _U32P, C.c_size_t, C.POINTER(MM), C.POINTER(GenParams), C.POINTER(SpecParams), _U32P,
                                                C.POINTER(Logprobs), C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(Usage), C.POINTER(SpecStats)]),
    "aha_b200_debug_verify_attn": (C.c_int, [_P, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, _F32P, _F32P, _F32P, _F32P]),
    "aha_b200_debug_verify_attn_batch": (C.c_int, [_P, C.c_size_t, _I32P, _I32P, _I32P, C.c_size_t, C.c_size_t, C.c_size_t, _F32P, _F32P, _F32P,
                                                   _F32P]),
    "aha_b200_batch_add_speculative": (C.c_int, [_P, C.POINTER(BatchRequest), C.POINTER(SpecParams), C.POINTER(C.c_int32), _U32P,
                                                 C.POINTER(C.c_int32), C.POINTER(Usage)]),
    "aha_b200_batch_step_spec": (C.c_int, [_P, _U32P, _U32P, C.POINTER(C.c_int32), C.c_size_t, C.POINTER(C.c_size_t)]),
    "aha_b200_batch_logprobs_spec": (C.c_int, [_P, C.POINTER(Logprobs), C.c_size_t]),
    "aha_b200_batch_spec_stats": (C.c_int, [_P, C.POINTER(SpecStats), C.c_size_t]),
    "aha_b200_debug_attention": (C.c_int, [_P, C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, _I32P, C.c_size_t,
                                           _I32P, C.c_int, _F32P, _F32P, _F32P, _F32P]),
    "aha_b200_debug_decode_attn": (C.c_int, [_P, C.c_size_t, C.c_size_t, C.c_size_t, _F32P, _I32P, _I32P, _F32P, _F32P, _I32P, C.c_size_t,
                                             _F32P, _F32P, C.c_float, C.c_float, _F32P, _F32P, _F32P]),
    "aha_b200_debug_logprobs": (C.c_int, [_P, _F32P, C.c_size_t, C.c_uint32, C.c_uint32, C.POINTER(Logprobs)]),
    "aha_b200_generate_batch": (C.c_int, [_P, C.POINTER(BatchRequest), C.c_size_t, _U32P, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(Usage)]),
    "aha_b200_batch_open": (C.c_int, [_P]),
    "aha_b200_batch_add": (C.c_int, [_P, C.POINTER(BatchRequest), C.POINTER(C.c_int32), _U32P, C.POINTER(C.c_int32), C.POINTER(Usage)]),
    "aha_b200_batch_add_many": (C.c_int, [_P, C.POINTER(BatchRequest), C.c_size_t, C.POINTER(C.c_int32), _U32P, C.POINTER(C.c_int32),
                                          C.POINTER(Usage)]),
    "aha_b200_batch_add_n": (C.c_int, [_P, C.POINTER(BatchRequest), C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_int32), _U32P,
                                       C.POINTER(C.c_int32), C.POINTER(Usage)]),
    "aha_b200_generate_n": (C.c_int, [_P, _U32P, C.c_size_t, C.POINTER(MM), C.POINTER(GenParams), C.c_size_t, C.POINTER(C.c_uint64), _U32P,
                                      C.POINTER(Logprobs), C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(Usage)]),
    "aha_b200_batch_step": (C.c_int, [_P, _U32P, C.POINTER(C.c_int32), C.POINTER(C.c_size_t)]),
    "aha_b200_batch_close": (C.c_int, [_P]),
    "aha_b200_batch_prefix_cache": (C.c_int, [_P, C.c_size_t]),
    "aha_b200_batch_prefix_stats": (C.c_int, [_P, C.POINTER(PrefixStats), C.POINTER(C.c_size_t), C.c_size_t]),
    "aha_b200_batch_swap_space": (C.c_int, [_P, C.c_size_t]),
    "aha_b200_batch_cancel": (C.c_int, [_P, C.c_int32]),
    "aha_b200_batch_suspend": (C.c_int, [_P, C.c_int32, _U32P]),
    "aha_b200_batch_resume": (C.c_int, [_P, C.c_uint32, _I32P]),
    "aha_b200_batch_discard": (C.c_int, [_P, C.c_uint32]),
    "aha_b200_batch_swap_stats": (C.c_int, [_P, C.POINTER(SwapStats)]),
    "aha_b200_debug_kv_swap": (C.c_int, [_P, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, _I32P, _I32P, _I32P, _F32P, _F32P,
                                         _F32P]),
    "aha_b200_debug_prefix_attention": (C.c_int, [_P, C.c_int, C.c_size_t, C.c_size_t, _I32P, C.c_size_t, _I32P, _F32P, _F32P, _F32P, _F32P]),
    "aha_b200_batch_open_wide": (C.c_int, [_P, C.c_size_t]),
    "aha_b200_batch_step_n": (C.c_int, [_P, _U32P, C.POINTER(C.c_int32), C.c_size_t, C.POINTER(C.c_size_t)]),
    "aha_b200_generate_stream": (C.c_int, [_P, _U32P, C.c_size_t, C.POINTER(MM), C.POINTER(GenParams), TOKEN_CALLBACK, C.c_void_p,
                                           C.POINTER(Usage)]),
    "aha_b200_asr_generate": (C.c_int, [_P, C.POINTER(AsrChunk), C.c_size_t, C.POINTER(GenParams), _U32P, C.c_size_t,
                                        C.POINTER(C.c_size_t), TOKEN_CALLBACK, C.c_void_p, C.POINTER(Usage)]),
    "aha_b200_debug_sample": (C.c_int, [_P, C.c_int, C.c_size_t, C.c_size_t, _F32P, C.c_size_t, C.POINTER(GenParams), _U32P, _U32P, _U32P,
                                        C.c_int, _I32P, _I32P, _U32P, _U32P, _U32P]),
    "aha_b200_debug_sample_fsm": (C.c_int, [_P, C.c_int, C.c_size_t, C.c_size_t, _F32P, C.c_size_t, C.POINTER(GenParams), _U32P, _U32P, _U32P,
                                            C.c_int, _I32P, _I32P, C.POINTER(TokenFsm), _I32P, _U32P, _U32P, _U32P, _U32P, _U32P]),
    "aha_b200_debug_sample_rules": (C.c_int, [_P, C.c_int, C.c_size_t, C.c_size_t, _F32P, C.c_size_t, C.POINTER(GenParams), _U32P, _U32P, _U32P,
                                              C.c_int, _I32P, _I32P, C.POINTER(TokenFsm), _I32P, _U32P, C.POINTER(LogitRules), _I32P, _U32P, _U32P,
                                              _U32P, _U32P]),
    "aha_b200_rules_check": (C.c_int, [C.POINTER(LogitRules), C.c_size_t]),
    "aha_b200_rules_create": (C.c_int, [_P, C.POINTER(LogitRules), _U32P]),
    "aha_b200_rules_destroy": (C.c_int, [_P, C.c_uint32]),
    "aha_b200_fsm_check": (C.c_int, [C.POINTER(TokenFsm), C.c_size_t]),
    "aha_b200_fsm_create": (C.c_int, [_P, C.POINTER(TokenFsm), _U32P]),
    "aha_b200_fsm_destroy": (C.c_int, [_P, C.c_uint32]),
    "aha_b200_lora_create": (C.c_int, [_P, C.POINTER(TensorDesc), C.c_size_t, C.c_float, _U32P]),
    "aha_b200_lora_destroy": (C.c_int, [_P, C.c_uint32]),
    "aha_b200_batch_add_lora": (C.c_int, [_P, C.POINTER(BatchRequest), _U32P, C.c_size_t, C.POINTER(C.c_int32), _U32P, C.POINTER(C.c_int32),
                                          C.POINTER(Usage)]),
    "aha_b200_mel_spectrogram": (C.c_int, [_P, _F32P, C.c_size_t, _F32P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "aha_b200_image_patchify": (C.c_int, [_P, C.POINTER(C.c_uint8), C.c_size_t, C.c_size_t, _F32P, C.c_size_t, _U32P]),
    "aha_b200_img_smart_resize": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, _U32P, _U32P]),
    "aha_b200_image_resize": (C.c_int, [_P, C.POINTER(C.c_uint8), C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.POINTER(C.c_uint8)]),
    "aha_b200_image_preprocess": (C.c_int, [_P, C.POINTER(C.c_uint8), C.c_size_t, C.c_size_t, C.c_uint32, C.c_uint32, _F32P, C.c_size_t, _U32P]),
    "aha_b200_expand_placeholders": (C.c_int, [_U32P, C.c_size_t, C.c_uint32, _U32P, C.c_size_t, _U32P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "aha_b200_video_smart_resize": (C.c_int, [C.c_uint32] * 8 + [_U32P, _U32P]),
    "aha_b200_video_sample_frames": (C.c_int, [C.c_uint32] * 6 + [_U32P, _U32P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "aha_b200_video_timestamps": (C.c_int, [_U32P, C.c_size_t, C.c_float, C.c_uint32, _F32P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "aha_b200_format_timestamp": (C.c_int, [C.c_float, C.c_char_p, C.c_size_t]),
    "aha_b200_video_preprocess": (C.c_int, [_P, C.POINTER(C.c_uint8), C.c_size_t, C.c_size_t, C.c_size_t, _F32P, C.c_size_t, _U32P]),
    "aha_b200_expand_video_placeholders": (C.c_int, [_U32P, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, _U32P, C.c_size_t, C.c_uint32, _U32P, _U32P,
                                                     C.c_size_t, _U32P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "aha_b200_feat_extract_output_length": (C.c_size_t, [C.c_size_t]),
    "aha_b200_float_range_normalize": (C.c_int, [_F32P, C.c_size_t]),
    "aha_b200_resample": (C.c_int, [_P, _F32P, C.c_size_t, C.c_int64, C.c_int64, _F32P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "aha_b200_sinc_resample_bank": (C.c_int, [C.c_int64, C.c_int64, _F32P, C.c_size_t, C.POINTER(C.c_int32)]),
    "aha_b200_split_audio_into_chunks": (C.c_int, [C.c_size_t, C.c_uint32, C.c_float, C.POINTER(C.c_size_t), C.c_size_t, C.POINTER(C.c_size_t)]),
    "aha_b200_embed": (C.c_int, [_P, _U32P, C.c_size_t, _F32P]),
    "aha_b200_embed_batch": (C.c_int, [_P, _U32P, C.POINTER(C.c_size_t), C.c_size_t, _F32P]),
    "aha_b200_score": (C.c_int, [_P, _U32P, C.c_size_t, C.c_size_t, C.c_uint32, C.POINTER(Logprobs), C.c_size_t, C.POINTER(C.c_size_t)]),
    "aha_b200_score_batch": (C.c_int, [_P, _U32P, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.c_size_t, C.c_uint32, C.POINTER(Logprobs),
                                       C.c_size_t, C.POINTER(C.c_size_t)]),
    "aha_b200_debug_score_head": (C.c_int, [_P, C.c_int, _F32P, C.c_size_t, _U32P, C.c_uint32, C.POINTER(Logprobs)]),
    "aha_b200_rerank": (C.c_int, [_P, _U32P, C.c_size_t, _U32P, C.POINTER(C.c_size_t), C.c_size_t, _F32P]),
    "aha_b200_nccl_unique_id": (C.c_int, [C.POINTER(C.c_uint8)]),
    "aha_b200_rope_index": (C.c_int, [_U32P, C.c_size_t, _U32P, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32,
                                      C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "aha_b200_rope_index_mm": (C.c_int, [_U32P, C.c_size_t, _U32P, C.c_size_t, _U32P, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                         C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "aha_b200_destroy": (None, [_P]),
    "aha_b200_last_error": (C.c_char_p, [_P]),
    "aha_b200_stream": (_P, [_P]),
    "aha_b200_get_stats": (C.c_int, [_P, C.POINTER(Stats)]),
    "aha_b200_reset_stats": (C.c_int, [_P]),
    "aha_b200_set_trace": (C.c_int, [_P, C.c_int]),
    "aha_b200_debug_read": (C.c_int, [_P, C.c_char_p, C.c_int, _F32P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "aha_b200_decode_steps": (C.c_int, [_P, C.c_uint32, C.c_size_t, C.c_size_t, _U32P, C.POINTER(C.c_double)]),
    "aha_b200_debug_gemm": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _F32P, C.POINTER(C.c_uint16), _F32P, _F32P, _F32P,
                                      C.c_int, C.POINTER(C.c_double)]),
    "aha_b200_bench_kernel": (C.c_int, [_P, C.c_char_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]),
}

_lib = None


def load():
    """Load libaha_b200.so (built in-tree by aha_b200.build).  Fails loudly: there is no fallback path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: run `python -m aha_b200.build` (nvcc, sm_90a). "
                          "aha_b200 has no CPU / PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the header and the library drift apart
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class BF16(np.ndarray):
    """uint16 array whose elements are bfloat16 bit patterns (numpy has no bf16 dtype): `arr.view(BF16)` marks it for make_desc."""


def to_bf16(x):
    """float32 -> bfloat16 bits (round to nearest even), tagged as BF16."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16).view(BF16)


def make_desc(arr, name=None):
    """TensorDesc for a C-contiguous numpy array (the caller keeps `arr` alive)."""
    if isinstance(arr, BF16):
        d = make_desc(arr.view(np.ndarray).view(np.float16), name)     # same bytes; only the dtype tag differs
        d.dtype = AHA_BF16
        return d
    if arr.dtype not in _NP2AHA:
        raise TypeError(f"unsupported dtype {arr.dtype}")
    if not arr.flags["C_CONTIGUOUS"]:
        raise ValueError("tensor must be C-contiguous")
    d = TensorDesc()
    d.name = name.encode() if name is not None else None
    d.dtype = _NP2AHA[arr.dtype]
    d.rank = arr.ndim
    for i, s in enumerate(arr.shape):
        d.shape[i] = s
    d.data = arr.ctypes.data
    return d
