"""Packed Qwen3 embeddings (aha_b200_embed_batch / B200Model.embed_batch): many texts in one prefill, attention causal inside each
text, positions restarting at 0 per text.  Against the oracle's embed_multi, and bit-for-bit against one embed() per text."""
import numpy as np
import pytest

from conftest import TOL, make_model, make_oracle

pytestmark = pytest.mark.gpu

# segment starts land off the 32-token page, 64-token KV-tile and 128-query-tile boundaries
LENS = [1, 5, 31, 32, 33, 63, 64, 65, 127, 128, 129, 200]


def _texts(lens, vocab, seed):
    from aha_b200 import synth
    return [synth.synth_text_ids(n, vocab - 8, seed + i) for i, n in enumerate(lens)]


def _oracle_embed(cfg, w, texts):
    from oracle.qwen3_embedding import Qwen3Embedding
    return Qwen3Embedding(cfg, w).embed_multi(texts)


@pytest.fixture(scope="module")
def tiny():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=2048)
    texts = _texts(LENS, cfg["vocab_size"], 100)
    yield cfg, w, m, texts, _oracle_embed(cfg, w, texts)
    m.close()


def _check_oracle(got, want):
    assert got.shape == want.shape and got.dtype == np.float32
    assert np.abs(np.linalg.norm(got, axis=1) - 1.0).max() < 1e-4
    err = np.abs(got - want).max(axis=1)
    assert err.max() <= 1e-5, err


@pytest.mark.parametrize("preset", ["tiny", "tiny-g1", "tiny-g4", "mid"])
def test_embed_batch_matches_oracle(preset):
    cfg, w, m = make_model("qwen3", preset, max_ctx=2048)
    try:
        texts = _texts(LENS, cfg["vocab_size"], 7)
        _check_oracle(m.embed_batch(texts), _oracle_embed(cfg, w, texts))
    finally:
        m.close()


def _check_against_embed(m, texts, got, exact_below_32):
    for t, g in zip(texts, got):
        want = m.embed(t)
        if t.size >= 32 or exact_below_32:
            assert np.array_equal(g, want), t.size
        else:   # alone: the SIMT GEMM (fewer than 32 rows); packed: the wgmma GEMM
            assert np.abs(g - want).max() <= 1e-5, t.size


def test_embed_batch_bit_equal_to_embed(tiny):
    cfg, w, m, texts, want = tiny
    _check_against_embed(m, texts, m.embed_batch(texts), exact_below_32=False)


def test_embed_batch_bit_equal_to_embed_mid():
    cfg, w, m = make_model("qwen3", "mid", max_ctx=2048)
    try:
        texts = _texts(LENS, cfg["vocab_size"], 9)
        _check_against_embed(m, texts, m.embed_batch(texts), exact_below_32=False)
    finally:
        m.close()


def test_embed_batch_bit_equal_to_embed_simt_gemm():
    """gemm_impl=1: every GEMM is the SIMT kernel whatever the row count, so every length matches embed() exactly."""
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=2048, gemm_impl=1)
    try:
        texts = _texts(LENS, cfg["vocab_size"], 100)
        _check_against_embed(m, texts, m.embed_batch(texts), exact_below_32=True)
    finally:
        m.close()


def test_embed_batch_permutation_is_exact(tiny):
    cfg, w, m, texts, want = tiny
    base = m.embed_batch(texts)
    perm = np.random.default_rng(3).permutation(len(texts))
    got = m.embed_batch([texts[i] for i in perm])
    assert np.array_equal(got, base[perm])


def test_embed_batch_split_over_packs_is_exact(tiny):
    """10 texts of 100 tokens through max_prefill=256 (five packs of two) == the same texts in one pack."""
    cfg, w, m, _, _ = tiny
    texts = _texts([100] * 10, cfg["vocab_size"], 200)
    one = m.embed_batch(texts)
    _, _, small = make_model("qwen3", "tiny", max_ctx=2048, max_prefill=256)
    try:
        assert np.array_equal(small.embed_batch(texts), one)
    finally:
        small.close()


@pytest.mark.parametrize("attn_impl", [1, 2])
def test_embed_batch_attention_twins(tiny, attn_impl):
    """The SIMT (1) and mma.sync (2) attention kernels run the pack one segment at a time."""
    cfg, w, _, texts, want = tiny
    _, _, m = make_model("qwen3", "tiny", max_ctx=2048, attn_impl=attn_impl)
    try:
        _check_oracle(m.embed_batch(texts), want)
    finally:
        m.close()


def test_embed_batch_errors(tiny):
    from aha_b200 import B200Error
    cfg, w, m, texts, want = tiny
    V = cfg["vocab_size"]
    with pytest.raises(B200Error, match="embedding input cannot be empty"):
        m.embed_batch([])
    with pytest.raises(B200Error, match="empty input_ids"):
        m.embed_batch([texts[1], np.zeros(0, np.uint32)])
    with pytest.raises(B200Error, match="token id out of range"):
        m.embed_batch([texts[1], np.array([1, V], np.uint32)])
    m.batch_open()
    try:
        with pytest.raises(B200Error, match="batch session is open"):
            m.embed_batch(texts[:2])
    finally:
        m.batch_close()
    _, _, small = make_model("qwen3", "tiny", max_ctx=2048, max_prefill=64)
    try:
        with pytest.raises(B200Error, match="exceeds max_prefill"):
            small.embed_batch([texts[1], texts[-1]])
    finally:
        small.close()
    vcfg, _, vl = make_model("qwen3vl", "tiny", max_ctx=256, max_patches=256)
    try:
        with pytest.raises(B200Error, match="embeddings need a qwen3 handle"):
            vl.embed_batch([np.array([1, 2, 3], np.uint32)])
    finally:
        vl.close()
    _check_oracle(m.embed_batch(texts), want)   # the handle stays usable after every error


def test_embed_batch_leaves_the_handle_clean(tiny):
    """After embed_batch the handle prefills and generates like the oracle, and the cache was dropped: a reuse_prefix request
    that follows finds nothing to reuse."""
    from oracle.generate import GenerationContext, generate_generic
    cfg, w, m, texts, _ = tiny
    o = make_oracle("qwen3", cfg, w)
    p = _texts([40], cfg["vocab_size"], 300)[0]
    m.generate(p, max_tokens=5, reuse_prefix=True)
    m.embed_batch(texts)
    m.generate(p, max_tokens=5, reuse_prefix=True)
    assert m.last_prefix_hit() == 0
    m.clear_cache()
    got = m.forward_initial(p, 0)[0, 0]
    want = o.forward_initial(p.reshape(1, -1), 0)[0, 0]
    assert np.abs(got - want).max() <= TOL
    m.embed_batch(texts)
    o.clear_cache()
    ctx = GenerationContext(temperature=0.0, initial_seq_len=p.size, max_tokens=20)
    ref, _, _ = generate_generic(o, p.reshape(1, -1), None, ctx)
    out, _ = m.generate(p, max_tokens=20)
    assert out == ref
