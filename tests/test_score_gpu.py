"""Scoring given text (aha_b200_score / _score_batch, score_head.cuh): the fused head against float64 and against its gemm_tc twin, exact
ties across sub-tile, slice and vocabulary edges, score() against the oracle (short, chunked and Qwen3-VL text prompts), packed batches
bit-identical to one call per text, agreement with the records of generation, the handle state afterwards and every refusal."""
import ctypes as C

import numpy as np
import pytest

import score_ref as R
from aha_b200 import B200Error, B200Model, synth
from aha_b200 import _lib as L
from conftest import make_model, make_oracle

pytestmark = pytest.mark.gpu

ORACLE_TOL = 2e-3      # twice the 1e-3 logit budget
HEAD_TOL = 1e-4


def _model(kind, preset, seed=0, overrides=None, **kw):
    cfg = synth.get_config(kind, preset)
    tc = cfg if kind == "qwen3" else cfg["text_config"]
    tc.update(overrides or {})
    if tc["eos_token_id"] >= tc["vocab_size"]:
        tc["eos_token_id"] = tc["vocab_size"] - 1
    w = synth.make_weights(kind, cfg, seed)
    return cfg, w, B200Model(kind, cfg, w, eos_ids=[tc["eos_token_id"]], **kw)


def _text(n, V, seed, avoid=()):
    return synth.synth_text_ids(n, min(V, 1000), seed, avoid).astype(np.uint32)


def _hidden(M, H, lm_head, rng):
    """pre-norm rows: half plain noise (flat distributions), half a scaled lm_head row plus noise (one clear winner, then near ties)"""
    x = rng.standard_normal((M, H)).astype(np.float32)
    pick = rng.integers(0, lm_head.shape[0], M)
    x[::2] += 10.0 * np.asarray(lm_head[pick[::2]], np.float32)
    return x


def _same(a, b):
    return all(np.array_equal(a[k], b[k]) for k in a) and a.keys() == b.keys()


# ------------------------------------------------------------------------------------------------------------- the head alone

HEAD_CONFIGS = {
    "V1000": ("qwen3", "tiny", dict(vocab_size=1000)),
    "V1024": ("qwen3", "tiny", None),
    "V4096": ("qwen3", "mid", None),
    "V151936": ("qwen3", "q0.6", dict(num_hidden_layers=1)),
}


@pytest.fixture(scope="module", params=list(HEAD_CONFIGS))
def head_model(request):
    kind, preset, ov = HEAD_CONFIGS[request.param]
    cfg, w, m = _model(kind, preset, overrides=ov, max_ctx=1024, max_prefill=512)
    lm = w["lm_head.weight"] if "lm_head.weight" in w else w["model.embed_tokens.weight"]
    yield cfg, w, m, np.asarray(lm, np.float32), np.asarray(w["model.norm.weight"], np.float32)
    m.close()


@pytest.mark.parametrize("M", [1, 31, 128, 129, 300])
def test_head_against_float64_and_twin(head_model, M):
    cfg, w, m, lm, norm = head_model
    V, H = cfg["vocab_size"], cfg["hidden_size"]
    rng = np.random.default_rng(M + V)
    x = _hidden(M, H, lm, rng)
    tgt = rng.integers(0, V, M).astype(np.uint32)
    tgt[1::3] = np.argmax(x[1::3] @ lm.T, axis=1)          # some rows scored at their most likely token
    ref = R.log_softmax(R.head64(x, norm, cfg["rms_norm_eps"], lm))
    want = ref[np.arange(M), tgt]
    for n in (0, 1, 5, 20):
        fused = m.debug_score_head(x, tgt, n, impl=0)
        twin = m.debug_score_head(x, tgt, n, impl=1)
        for got in (fused, twin):
            assert np.array_equal(got["tokens"], tgt)
            assert np.abs(got["logprobs"] - want).max() <= HEAD_TOL, n
            if n:
                R.check_top(got["top_ids"], got["top_logprobs"], ref, HEAD_TOL)
        assert np.abs(fused["logprobs"] - twin["logprobs"]).max() <= 1e-5      # the same logits: only the exp-sum order differs
        if n:
            assert np.array_equal(fused["top_ids"], twin["top_ids"])
            d_f = fused["top_logprobs"] - fused["logprobs"][:, None]
            d_t = twin["top_logprobs"] - twin["logprobs"][:, None]
            assert np.abs(d_f - d_t).max() <= 2e-6
        assert _same(fused, m.debug_score_head(x, tgt, n, impl=0))          # deterministic


def test_head_rows_independent_of_the_batch(head_model):
    """a row's record does not depend on M, its place in the tile or the rows beside it"""
    cfg, w, m, lm, norm = head_model
    V, H = cfg["vocab_size"], cfg["hidden_size"]
    rng = np.random.default_rng(5)
    x = _hidden(300, H, lm, rng)
    tgt = rng.integers(0, V, 300).astype(np.uint32)
    full = m.debug_score_head(x, tgt, 5)
    perm = rng.permutation(300)
    shuffled = m.debug_score_head(x[perm], tgt[perm], 5)
    for k in full:
        assert np.array_equal(shuffled[k], full[k][perm])
    for r in (0, 127, 128, 299):
        one = m.debug_score_head(x[r:r + 1], tgt[r:r + 1], 5)
        for k in full:
            assert np.array_equal(one[k][0], full[k][r])


def test_exact_ties_in_ascending_id_order():
    """duplicated lm_head rows on both sides of a 256-column sub-tile, a 2048-column slice and the vocabulary edge: equal logits, ids ascending"""
    cfg, w, m = _model("qwen3", "tiny-untied", overrides=dict(vocab_size=4000), max_ctx=512, max_prefill=256)
    try:
        lm = np.array(w["lm_head.weight"], copy=True)
        dup = [255, 256, 2047, 2048, 3999]
        base = np.asarray(lm[dup[0]], np.float32)
        m.close()
        w = dict(w)
        lm[dup] = lm[dup[0]]
        w["lm_head.weight"] = lm
        m = B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"]], max_ctx=512, max_prefill=256)
        rng = np.random.default_rng(3)
        x = (40.0 * base[None] + rng.standard_normal((130, cfg["hidden_size"])).astype(np.float32) * 0.01)
        tgt = np.full(130, 2048, np.uint32)
        for impl in (0, 1):
            for n in (5, 20):
                got = m.debug_score_head(x, tgt, n, impl=impl)
                assert (got["top_ids"][:, :5] == np.array(dup)).all(), got["top_ids"][0]
                assert (got["top_logprobs"][:, :5] == got["top_logprobs"][:, :1]).all()
                assert np.array_equal(got["logprobs"], got["top_logprobs"][:, 3])
    finally:
        m.close()


# ------------------------------------------------------------------------------------------------------------- score() vs the oracle

ORACLE_CONFIGS = {
    "tiny": ("qwen3", "tiny", None),
    "tiny-untied": ("qwen3", "tiny-untied", None),
    "tiny-g4": ("qwen3", "tiny-g4", None),
    "mid": ("qwen3", "mid", None),
    "V1000": ("qwen3", "tiny", dict(vocab_size=1000)),
    "vl-tiny": ("qwen3vl", "tiny", None),
}


def _vl_avoid(cfg):
    return tuple(cfg.get(k, -1) for k in ("image_token_id", "video_token_id", "vision_start_token_id", "vision_end_token_id"))


@pytest.mark.parametrize("name", list(ORACLE_CONFIGS))
def test_score_matches_oracle(name):
    kind, preset, ov = ORACLE_CONFIGS[name]
    cfg, w, m = _model(kind, preset, overrides=ov, max_ctx=1024, max_prefill=512)
    try:
        o = make_oracle(kind, cfg, w)
        V = (cfg if kind == "qwen3" else cfg["text_config"])["vocab_size"]
        ids = _text(150, V, 11, _vl_avoid(cfg))
        got = m.score(ids, top=5)
        ref, want = R.score(kind, o, ids)
        assert np.array_equal(got["tokens"], ids[1:])
        assert np.abs(got["logprobs"] - want).max() <= ORACLE_TOL
        R.check_top(got["top_ids"], got["top_logprobs"], ref, ORACLE_TOL)
        for start in (2, 77, 149):
            tail = m.score(ids, start=start, top=5)
            for k in got:
                assert np.array_equal(tail[k], got[k][start - 1:]), (start, k)
    finally:
        m.close()


@pytest.mark.parametrize("max_prefill", [80, 96])
def test_long_prompt_in_chunks(max_prefill):
    """S > max_prefill: continuation chunks whose boundaries fall inside pages (32 tokens) and 64-token tiles, or on a page edge"""
    cfg, w, m = _model("qwen3", "tiny", max_ctx=1024, max_prefill=max_prefill)
    try:
        o = make_oracle("qwen3", cfg, w)
        ids = _text(333, cfg["vocab_size"], 12)
        got = m.score(ids, top=3)
        ref, want = R.score("qwen3", o, ids)
        assert np.abs(got["logprobs"] - want).max() <= ORACLE_TOL
        R.check_top(got["top_ids"], got["top_logprobs"], ref, ORACLE_TOL)
        tail = m.score(ids, start=200, top=3)
        assert np.abs(tail["logprobs"] - want[199:]).max() <= ORACLE_TOL
    finally:
        m.close()


# ------------------------------------------------------------------------------------------------------------- score_batch

LENS = [2, 5, 31, 32, 33, 63, 64, 65, 127, 128, 129, 200]


@pytest.fixture(scope="module")
def tiny():
    cfg, w, m = _model("qwen3", "tiny", max_ctx=1024, max_prefill=512)
    yield cfg, w, m
    m.close()


def _batch_texts(V, lens, seed):
    return [_text(n, V, seed + i) for i, n in enumerate(lens)]


def _check_batch(m, texts, got, starts=None, exact_below_32=False, top=5):
    for j, t in enumerate(texts):
        s = 1 if starts is None else starts[j]
        want = m.score(t, start=s, top=top)
        if t.size >= 32 or exact_below_32:
            assert _same(got[j], want), (j, t.size)
        else:   # alone: the SIMT GEMMs (fewer than 32 rows); packed: the wgmma GEMMs
            assert np.array_equal(got[j]["tokens"], want["tokens"])
            assert np.abs(got[j]["logprobs"] - want["logprobs"]).max() <= 1e-4


def test_score_batch_equals_score(tiny):
    cfg, w, m = tiny
    texts = _batch_texts(cfg["vocab_size"], LENS, 20)
    got = m.score_batch(texts, top=5)
    _check_batch(m, texts, got)
    starts = [1, 4, 30, 1, 2, 60, 63, 1, 100, 127, 5, 199]
    _check_batch(m, texts, m.score_batch(texts, starts=starts, top=5), starts)
    plain = m.score_batch(texts)
    for j in range(len(texts)):
        assert plain[j].keys() == {"tokens", "logprobs"} and np.array_equal(plain[j]["logprobs"], got[j]["logprobs"])


def test_score_batch_on_qwen3vl():
    """the packed path on a Qwen3-VL handle: per-segment M-RoPE positions of text-only prompts, segment-causal prefill"""
    cfg, w, m = _model("qwen3vl", "tiny", max_ctx=1024, max_prefill=512, max_patches=1024)
    try:
        V = cfg["text_config"]["vocab_size"]
        texts = [_text(n, V, 100 + i, _vl_avoid(cfg)) for i, n in enumerate([33, 40, 64, 100, 129])]
        starts = [1, 20, 1, 50, 3]
        got = m.score_batch(texts, starts=starts, top=5)
        _check_batch(m, texts, got, starts)
        ref, want = R.score("qwen3vl", make_oracle("qwen3vl", cfg, w), texts[3], start=50)
        assert np.abs(got[3]["logprobs"] - want).max() <= ORACLE_TOL
        R.check_top(got[3]["top_ids"], got[3]["top_logprobs"], ref, ORACLE_TOL)
    finally:
        m.close()


def test_score_batch_invariant_to_order_and_packing(tiny):
    cfg, w, m = tiny
    texts = _batch_texts(cfg["vocab_size"], LENS, 30)
    full = m.score_batch(texts, top=5)
    perm = np.random.default_rng(1).permutation(len(texts))
    shuffled = m.score_batch([texts[i] for i in perm], top=5)
    for k, i in enumerate(perm):
        assert _same(shuffled[k], full[i])
    split = m.score_batch(texts[:5], top=5) + m.score_batch(texts[5:], top=5)
    for a, b in zip(split, full):
        assert _same(a, b)


def test_score_batch_text_longer_than_a_pack():
    cfg, w, m = _model("qwen3", "tiny", max_ctx=1024, max_prefill=128)
    try:
        o = make_oracle("qwen3", cfg, w)
        texts = _batch_texts(cfg["vocab_size"], [40, 300, 70, 90, 129], 40)
        got = m.score_batch(texts, starts=[1, 150, 1, 1, 1])
        _check_batch(m, texts, got, starts=[1, 150, 1, 1, 1], top=0)
        ref, want = R.score("qwen3", o, texts[1], start=150)
        assert np.abs(got[1]["logprobs"] - want).max() <= ORACLE_TOL
    finally:
        m.close()


def test_score_batch_simt_gemm_bit_identical_for_every_length():
    cfg, w, m = _model("qwen3", "tiny", max_ctx=1024, max_prefill=512, gemm_impl=1)
    try:
        texts = _batch_texts(cfg["vocab_size"], [2, 3, 9, 17, 31, 40], 50)
        _check_batch(m, texts, m.score_batch(texts, top=5), exact_below_32=True)
    finally:
        m.close()


def test_score_batch_launches_fewer_kernels(tiny):
    cfg, w, m = tiny
    texts = _batch_texts(cfg["vocab_size"], [48] * 8, 60)
    m.reset_stats()
    m.score_batch(texts)
    packed = m.stats()["kernel_launches"]
    m.reset_stats()
    for t in texts:
        m.score(t)
    alone = m.stats()["kernel_launches"]
    assert packed < alone, (packed, alone)


# ------------------------------------------------------------------------------------------------------------- agreement with generation

@pytest.mark.parametrize("mode", [dict(), dict(temperature=0.8, top_p=0.9, seed=7)], ids=["greedy", "sampled"])
def test_score_agrees_with_generation_records(tiny, mode):
    cfg, w, m = tiny
    prompt = _text(40, cfg["vocab_size"], 70)
    toks, _, recs = m.generate(prompt, max_tokens=12, logprobs=True, top_logprobs=5, **mode)
    seq = np.concatenate([prompt, np.asarray(toks, np.uint32)])
    got = m.score(seq, start=len(prompt), top=5)
    assert list(got["tokens"]) == toks
    for k, r in enumerate(recs):
        assert abs(float(got["logprobs"][k]) - float(r["logprob"])) <= 1e-3
        lp = np.asarray(r["top_logprobs"], np.float64)
        for j in range(5):
            if (j == 0 or lp[j - 1] - lp[j] > 1e-3) and (j == 4 or lp[j] - lp[j + 1] > 1e-3):
                assert got["top_ids"][k, j] == r["top_ids"][j]
        if lp[0] - lp[1] > 1e-3:
            assert (got["top_ids"][k, 0] == toks[k]) == (r["top_ids"][0] == toks[k])
            if not mode:
                assert got["top_ids"][k, 0] == toks[k]


# ------------------------------------------------------------------------------------------------------------- handle state, refusals

def test_handle_state_after_scoring():
    cfg, w, m = _model("qwen3", "tiny", max_ctx=2048, max_prefill=512)
    cfg2, w2, fresh = _model("qwen3", "tiny", max_ctx=2048, max_prefill=512)
    try:
        V = cfg["vocab_size"]
        prompt = _text(30, V, 80)
        want, _ = fresh.generate(prompt, max_tokens=10)
        m.score(_text(700, V, 81), top=5)
        assert m.generate(prompt, max_tokens=10)[0] == want
        m.score_batch(_batch_texts(V, [50, 600, 20], 82), top=3)
        assert m.generate(prompt, max_tokens=10)[0] == want
        # a batch session can still fill the whole 64-page pool: eight requests of 8 pages each
        m.batch_open()
        try:
            res = m.batch_add_many([dict(input_ids=_text(200, V, 90 + i), max_tokens=56) for i in range(8)])
            assert [r[0] for r in res] == list(range(8))
            assert len(m.batch_step()) == 8
        finally:
            m.batch_close()
    finally:
        m.close()
        fresh.close()


def test_refusals_leave_the_handle_usable(tiny):
    cfg, w, m = tiny
    V = cfg["vocab_size"]
    ids = _text(20, V, 90)
    want = m.score(ids, top=2)
    bad_id = ids.copy()
    bad_id[3] = V
    cases = [
        (lambda: m.score(ids, start=0), "start must be at least 1"),
        (lambda: m.score(ids, start=20), "leaves nothing to score"),
        (lambda: m.score(bad_id), "token id out of range"),
        (lambda: m.score(_text(1025, V, 91)), "exceeds max_ctx"),
        (lambda: m.score(ids, top=21), "at most 20"),
        (lambda: m.score_batch([ids, bad_id]), "token id out of range"),
        (lambda: m.score_batch([ids, ids], starts=[1, 0]), "start must be at least 1"),
        (lambda: m.debug_score_head(np.zeros((2, cfg["hidden_size"]), np.float32), [0, V]), "target id out of range"),
    ]
    for fn, msg in cases:
        with pytest.raises(B200Error, match=msg):
            fn()
    recs = np.zeros(4, L.LOGPROBS_DTYPE)
    n = C.c_size_t()
    rc = m._lib.aha_b200_score(m._h, ids.ctypes.data_as(C.POINTER(C.c_uint32)), ids.size, 1, 0, recs.ctypes.data_as(C.POINTER(L.Logprobs)), 4,
                               C.byref(n))
    assert rc != 0 and b"records" in m._lib.aha_b200_last_error(m._h)
    m.batch_open()
    try:
        with pytest.raises(B200Error, match="batch session is open"):
            m.score(ids)
        with pytest.raises(B200Error, match="batch session is open"):
            m.score_batch([ids])
    finally:
        m.batch_close()
    assert _same(m.score(ids, top=2), want)


def test_refusals_of_handle_kinds():
    cfg, w, m = make_model("qwen3vl", "tiny", max_ctx=1024, max_patches=1024)
    try:
        ids = _text(20, cfg["text_config"]["vocab_size"], 92, _vl_avoid(cfg))
        ids[5] = cfg["image_token_id"]
        with pytest.raises(B200Error, match="text-only"):
            m.score(ids)
    finally:
        m.close()
    cfg, w, m = make_model("qwen3_asr", "tiny", max_ctx=1024, max_frames=400)
    try:
        with pytest.raises(B200Error, match="qwen3 or qwen3vl"):
            m.score(_text(20, 900, 93))
    finally:
        m.close()


def test_bench_kernel_entries(head_model):
    cfg, w, m, lm, norm = head_model
    m.score(_text(200, cfg["vocab_size"], 94))
    for name in ("score_head:128:0", "score_head:128:5", "score_twin:128:5"):
        ms, _ = m.bench_kernel(name, 3)
        assert ms > 0
