"""Speculative decoding of single requests (aha_b200_generate_speculative, B200Model.generate_speculative).

Verify passes of max_draft + 1 rows must produce the request's oracle ids (as wide batch sessions do), ids and records that do not
depend on the drafts, max_draft or graphs, and the pass counts the draft rule (tests/spec_ref.py) predicts.  The verify attention is
checked on host data through debug_verify_attn."""
import ctypes as C

import numpy as np
import pytest

from attn_ref import attention
from conftest import make_model, make_oracle
from spec_ref import simulate
from test_batch_wide_gpu import SAMPLERS, _check_oracle_ids

pytestmark = pytest.mark.gpu


def _ids(n, V, seed):
    from aha_b200 import synth
    return synth.synth_text_ids(n, V - 8, seed)


def _key(r):
    return (r["token"], r["index"], np.float32(r["logprob"]).tobytes(), tuple(r["top_ids"]),
            b"".join(np.float32(v).tobytes() for v in r["top_logprobs"]))


# ------------------------------------------------------------------------------------------------------------ verify attention

@pytest.fixture(scope="module")
def tiny():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=2048)
    yield cfg, w, m
    m.close()


@pytest.mark.parametrize("G", [1, 2, 4, 6])
@pytest.mark.parametrize("R", [1, 2, 8, 16])
def test_verify_attention_against_float64(tiny, G, R):
    m = tiny[2]
    nkv = 2
    rng = np.random.default_rng(100 * G + R)
    for pos0 in (0, 30, 63, 64, 130, 300):     # contexts ending inside, on and across page (32) and chunk (64) boundaries
        q = rng.standard_normal((R, G * nkv, 128)).astype(np.float32)
        k = rng.standard_normal((pos0 + R, nkv, 128)).astype(np.float32)
        v = rng.standard_normal((pos0 + R, nkv, 128)).astype(np.float32)
        got = m.debug_verify_attn(q, k, v, pos0)
        assert np.abs(got - attention(q, k, v, causal=True)).max() <= 1e-5, pos0   # row r sees positions 0 .. pos0 + r
        for r in {0, R // 2, R - 1}:            # row r alone (R = 1 at its position) gives the same bits
            alone = m.debug_verify_attn(q[r:r + 1], k[:pos0 + r + 1], v[:pos0 + r + 1], pos0 + r)
            assert np.array_equal(alone[0], got[r]), (pos0, r)


# ------------------------------------------------------------------------------------------------------------ oracle ids

def _requests(V, seed, n, budget):
    reqs = []
    for i, kw in enumerate([{}] + SAMPLERS[1:] + [dict(repeat_penalty=1.3, repeat_last_n=16)]):
        kw = dict(kw)
        if kw.get("temperature"):
            kw["seed"] = seed + i
        reqs.append(dict(input_ids=_ids(n + 7 * i, V, seed + i), max_tokens=budget, **kw))
    return reqs


def _spec(m, r, **kw):
    args = {k: v for k, v in r.items()}
    args.update(kw)
    return m.generate_speculative(**args)


@pytest.mark.parametrize("preset,budget", [("tiny", 40), ("tiny-g1", 40), ("tiny-g4", 40), ("mid", 10)])
def test_oracle_ids(preset, budget):
    cfg, w, m = make_model("qwen3", preset, max_ctx=1024)
    o = make_oracle("qwen3", cfg, w)
    try:
        reqs = _requests(cfg["vocab_size"], 7, 20, budget)
        out = [_spec(m, r, prompt_lookup=True, max_draft=7)[0] for r in reqs]
        _check_oracle_ids(o, reqs, out)
    finally:
        m.close()


def test_oracle_ids_qwen3vl_image():
    from aha_b200 import synth
    from oracle.qwen3vl import process_image
    cfg, w, m = make_model("qwen3vl", "tiny", max_ctx=1024, max_patches=1024)
    o = make_oracle("qwen3vl", cfg, w)
    try:
        pv, grid = process_image(synth.synth_image(256, 320, 1))
        ids = synth.vl_prompt_ids(cfg, grid, 16)
        data = [pv, grid, None, None, None]
        reqs = [dict(input_ids=ids, data=data, max_tokens=24, **kw) for kw in
                ({}, dict(temperature=0.8, top_k=20, top_p=0.9, repeat_penalty=1.2, repeat_last_n=16, seed=5))]
        out = [_spec(m, r, prompt_lookup=True, max_draft=4)[0] for r in reqs]
        _check_oracle_ids(o, reqs, out)
        assert m.debug_read("rope_delta", 0, 1)[0] == 0            # the request cleared its cache and rope_delta
    finally:
        m.close()


# ------------------------------------------------------------------------------------------------------------ invariance + stats

@pytest.fixture(scope="module")
def pair():
    """two handles on the same weights: CUDA graphs and eager launches"""
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=2048)
    _, _, e = make_model("qwen3", "tiny", max_ctx=2048, use_graph=False)
    yield cfg, m, e
    m.close()
    e.close()


def _variants(ref, V, rng):
    ins = list(ref[:10]) + [int(rng.integers(0, V))] + list(ref[10:])
    dele = list(ref[:6]) + list(ref[9:])
    sub = [int(rng.integers(0, V)) if i % 5 == 3 else t for i, t in enumerate(ref)]
    edited = [t for i, t in enumerate(sub) if i % 11 != 7][:20] + ins[20:]
    rand = [int(x) for x in rng.integers(0, V, 60)]
    return dict(none=None, exact=list(ref), inserted=ins, deleted=dele, substituted=sub, edited=edited, random=rand)


@pytest.mark.parametrize("samp", [{}, dict(repeat_penalty=1.3, repeat_last_n=16), dict(temperature=0.9, top_k=40, top_p=0.9, seed=3)])
def test_ids_and_records_do_not_depend_on_the_drafts(pair, samp):
    cfg, m, e = pair
    V = cfg["vocab_size"]
    prompt = _ids(150, V, 21)
    base = dict(input_ids=prompt, max_tokens=48, logprobs=True, top_logprobs=5, **samp)
    ref_ids, _, _, ref_rec = m.generate_speculative(max_draft=1, **base)
    n = len(ref_ids)
    assert [r["index"] for r in ref_rec] == list(range(n))
    rng = np.random.default_rng(5)
    for name, pred in _variants(ref_ids, V, rng).items():
        for lookup in (False, True):
            for md in (1, 4, 7, 15):
                for h in (m, e):
                    ids, usage, stats, rec = h.generate_speculative(prediction=pred, prompt_lookup=lookup, max_draft=md, **base)
                    assert ids == ref_ids, (name, lookup, md, h is e)
                    assert [_key(r) for r in rec] == [_key(r) for r in ref_rec], (name, lookup, md, h is e)
                    want = simulate(ref_ids, pred, list(prompt) if lookup else None, md, 3)
                    assert (stats["passes"], stats["drafted"], stats["accepted"]) == want, (name, lookup, md)
                    assert usage["completion_tokens"] == n and usage["prompt_tokens"] == 150
    # records without alternatives and no records at all give the same ids
    assert m.generate_speculative(prediction=ref_ids, max_draft=7, **dict(base, logprobs=False, top_logprobs=0))[0] == ref_ids


def test_stats_exact_prediction_and_no_source(pair):
    cfg, m, _ = pair
    V = cfg["vocab_size"]
    r = dict(input_ids=_ids(90, V, 4), max_tokens=64)
    ids, _, st = m.generate_speculative(**r)
    n = len(ids)
    assert st == dict(passes=n - 1, drafted=0, accepted=0)
    for md in (4, 7, 15):
        got, _, st = m.generate_speculative(prediction=ids, max_draft=md, **r)
        assert got == ids
        passes, drafted, accepted = simulate(ids, ids, None, md, 3)
        assert st == dict(passes=passes, drafted=drafted, accepted=accepted)
        assert st["accepted"] > 0 and st["passes"] < n - 1


# ------------------------------------------------------------------------------------------------------------ edges

def test_eos_inside_an_accepted_run_and_max_tokens_mid_pass():
    from aha_b200 import B200Model, synth
    cfg = synth.get_config("qwen3", "tiny")
    w = synth.make_weights("qwen3", cfg, 0)
    m = B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"]], max_ctx=1024)
    try:
        r = dict(input_ids=_ids(60, cfg["vocab_size"], 8), max_tokens=40, temperature=1.0, top_k=50, seed=2)   # sampled: no greedy loop
        full, _, _ = m.generate_speculative(**r)
    finally:
        m.close()
    k = next(i for i in range(5, len(full)) if full[i] not in full[1:i])          # a token emitted for the first time at k >= 5
    m = B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"], full[k]], max_ctx=1024)
    try:
        ids, usage, st = m.generate_speculative(prediction=full, max_draft=15, **r)
        assert ids == full[:k + 1] and usage["completion_tokens"] == k + 1      # the EOS token is pushed, then the request ends
        assert st == dict(zip(("passes", "drafted", "accepted"), simulate(full[:k + 1], full, None, 15, 3)))
    finally:
        m.close()
    m = B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"]], max_ctx=1024)
    try:
        for mt in (1, 2, 5, 9, 13):
            ids, usage, st = m.generate_speculative(prediction=full, max_draft=7, **dict(r, max_tokens=mt))
            assert ids == full[:mt] and usage["completion_tokens"] == mt, mt
            assert st["passes"] == simulate(full[:mt], full, None, 7, 3)[0]
    finally:
        m.close()


def _raw(m, ids, params=None, spec=None, cap=None, n_pred=0):
    from aha_b200 import _lib as L
    ids = np.ascontiguousarray(ids, np.uint32)
    p = params or L.GenParams(temperature=0.0, repeat_penalty=1.0, repeat_last_n=64, max_tokens=8, seed=1)
    s = spec or L.SpecParams(max_draft=4)
    cap = cap if cap is not None else max(p.max_tokens, 1)
    out = (C.c_uint32 * max(cap, 1))()
    n = C.c_size_t(0)
    rc = m._lib.aha_b200_generate_speculative(m._h, ids.ctypes.data_as(C.POINTER(C.c_uint32)), ids.size, None, C.byref(p), C.byref(s), out,
                                              None, cap, C.byref(n), None, None)
    return rc, m._lib.aha_b200_last_error(m._h).decode()


def test_refusals(tiny):
    from aha_b200 import B200Error, _lib as L
    cfg, w, m = tiny
    ids = _ids(20, cfg["vocab_size"], 1)
    gp = lambda **kw: L.GenParams(**dict(dict(temperature=0.0, repeat_penalty=1.0, repeat_last_n=64, max_tokens=8, seed=1), **kw))
    for md in (0, 16):
        rc, err = _raw(m, ids, spec=L.SpecParams(max_draft=md))
        assert rc and "max_draft must be 1 to 15" in err
    rc, err = _raw(m, ids, spec=L.SpecParams(max_draft=4, ngram=9))
    assert rc and "ngram must be" in err
    for f in (L.GEN_REUSE_PREFIX, L.GEN_CONTINUE_RNG, L.GEN_EOS_ON_FIRST):
        rc, err = _raw(m, ids, params=gp(flags=f))
        assert rc and "not supported with speculative decoding" in err, f
    rc, err = _raw(m, ids, params=gp(max_tokens=20), cap=10)
    assert rc and "capacity" in err
    rc, err = _raw(m, ids, params=gp(flags=L.GEN_LOGPROBS))
    assert rc and "needs out_logprobs" in err
    with pytest.raises(B200Error, match="exceeds max_ctx"):
        m.generate_speculative(_ids(2000, cfg["vocab_size"], 2), max_tokens=42, max_draft=7)     # 2000 + 42 + 7 > 2048
    m.batch_open_wide(4)
    try:
        with pytest.raises(B200Error, match="batch session is open"):
            m.generate_speculative(ids, max_tokens=8)
    finally:
        m.batch_close()
    _, _, asr = make_model("qwen3_asr", "tiny", max_ctx=512)
    try:
        with pytest.raises(B200Error, match="Qwen3-ASR"):
            asr.generate_speculative(ids, max_tokens=8)
    finally:
        asr.close()
    from aha_b200 import B200Model, synth
    c1000 = dict(synth.get_config("qwen3", "tiny"), vocab_size=1000)      # a vocabulary the wide lm_head cannot tile
    odd = B200Model("qwen3", c1000, synth.make_weights("qwen3", c1000, 0), eos_ids=[999], max_ctx=512)
    try:
        with pytest.raises(B200Error, match="multiples of 64"):
            odd.generate_speculative(ids, max_tokens=8)
    finally:
        odd.close()


def test_handle_after_speculative_requests():
    """A plain generate afterwards equals a fresh handle's, a wide session can still fill the KV pool, and there is at most one pass graph
    per row count."""
    from aha_b200 import B200Model, synth
    cfg = synth.get_config("qwen3", "tiny")
    w = synth.make_weights("qwen3", cfg, 0)
    V = cfg["vocab_size"]
    mk = lambda: B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"]], max_ctx=1024)
    r = dict(input_ids=_ids(70, V, 30), max_tokens=30, temperature=0.8, top_k=30, seed=9)
    fresh = mk()
    try:
        want = fresh.generate(**r)[0]
        want_wide = _fill_wide(fresh, V)
    finally:
        fresh.close()
    m = mk()
    try:
        for md in (1, 4, 7, 15, 4, 7):
            m.generate_speculative(prompt_lookup=True, max_draft=md, **r)
        assert m.debug_read("spec_graphs", 0, 1)[0] == 4
        assert m.generate(**r)[0] == want
        assert _fill_wide(m, V) == want_wide
        m.generate_speculative(prompt_lookup=True, max_draft=7, **r)
        assert m.debug_read("spec_graphs", 0, 1)[0] == 4
    finally:
        m.close()


def _fill_wide(m, V):
    """8 requests whose pages take the whole pool (1024 tokens = 32 pages of 32): every one admitted, ids of all"""
    m.batch_open_wide(8)
    try:
        reqs = [dict(input_ids=_ids(100, V, 40 + i), max_tokens=28) for i in range(8)]     # 128 tokens = 4 pages each
        res = m.batch_add_many(reqs)
        out = {s: [t] for s, t, _ in res}
        while True:
            step = m.batch_step()
            if not step:
                break
            for s, (t, _) in step.items():
                out[s].append(t)
        return [out[s] for s, _, _ in res]
    finally:
        m.batch_close()
