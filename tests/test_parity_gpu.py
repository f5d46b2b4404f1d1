"""Parity of the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs.
Tolerance: max |logit difference| <= 1e-3 (north_star), greedy ids bit-exact wherever the oracle's
top-1/top-2 gap exceeds the measured error."""
import numpy as np
import pytest

from conftest import TOL, make_model, make_oracle, top2_gap

pytestmark = pytest.mark.gpu


def _ids(n, vocab, seed):
    from aha_b200 import synth
    return synth.synth_text_ids(n, vocab - 8, seed)


@pytest.fixture(scope="module")
def q3():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=512)
    yield cfg, w, m, make_oracle("qwen3", cfg, w)
    m.close()


@pytest.mark.parametrize("S", [1, 2, 31, 63, 64, 65, 130, 257])
def test_qwen3_prefill_logits(q3, S):
    cfg, w, m, o = q3
    ids = _ids(S, cfg["vocab_size"], S)
    m.clear_cache(); o.clear_cache()
    got = m.forward_initial(ids, 0)[0, 0]
    want = o.forward_initial(ids.reshape(1, -1), 0)[0, 0]
    err = np.abs(got - want).max()
    assert err <= TOL, err
    if top2_gap(want) > 10 * err:
        assert m.last_argmax == int(np.argmax(want))


def test_qwen3_per_layer_hidden(q3):
    cfg, w, m, o = q3
    ids = _ids(40, cfg["vocab_size"], 11)
    m.clear_cache(); o.clear_cache()
    m.set_trace(True)
    o.trace = []
    m.forward_initial(ids, 0)
    o.forward_initial(ids.reshape(1, -1), 0)
    for l in range(cfg["num_hidden_layers"]):
        got = m.debug_read("hidden", l, 40 * cfg["hidden_size"]).reshape(40, -1)
        assert np.abs(got - o.trace[l][0]).max() <= 1e-4
    m.set_trace(False)
    o.trace = None


def test_qwen3_teacher_forced_decode(q3):
    cfg, w, m, o = q3
    S, n = 37, 70  # crosses two 32-token page boundaries
    ids = _ids(S + n, cfg["vocab_size"], 3)
    m.clear_cache(); o.clear_cache()
    m.forward_initial(ids[:S], 0)
    o.forward_initial(ids[:S].reshape(1, -1), 0)
    worst = 0.0
    for i in range(n):
        got = m.forward_step(ids[S + i:S + i + 1], S + i)[0, 0]
        want = o.forward_step(ids[S + i:S + i + 1].reshape(1, 1), S + i)[0, 0]
        err = np.abs(got - want).max()
        worst = max(worst, err)
        assert err <= TOL, (i, err)
        if top2_gap(want) > 10 * max(err, 1e-6):
            assert m.last_argmax == int(np.argmax(want)), i
    print("teacher-forced worst abs logit err", worst)


def test_qwen3_greedy_generate_matches_oracle(q3):
    from oracle.generate import GenerationContext, generate_generic
    cfg, w, m, o = q3
    ids = _ids(21, cfg["vocab_size"], 5)
    m.clear_cache(); o.clear_cache()
    ctx = GenerationContext(temperature=0.0, initial_seq_len=21, max_tokens=40)
    want, _, _ = generate_generic(o, ids.reshape(1, -1), None, ctx)
    got, usage = m.generate(ids, max_tokens=40)
    assert got == want
    assert usage["prompt_tokens"] == 21 and usage["completion_tokens"] == len(want)


def test_qwen3_decode_implementations_agree(q3):
    """fused persistent kernel (default: grid-barrier version; 3 = the same, asked for; 4 = hybrid version) == per-op kernels under
    a CUDA graph == per-op eager launches."""
    cfg, w, m, o = q3
    others = [make_model("qwen3", "tiny", max_ctx=512, decode_impl=1)[2],
              make_model("qwen3", "tiny", max_ctx=512, decode_impl=1, use_graph=False)[2],
              make_model("qwen3", "tiny", max_ctx=512, decode_impl=3)[2],
              make_model("qwen3", "tiny", max_ctx=512, decode_impl=4)[2]]
    try:
        ids = _ids(50, cfg["vocab_size"], 8)
        m.clear_cache()
        m.forward_initial(ids, 0)
        a = m.decode_steps(5, 50, 40)
        la = m.forward_step(np.array([9], np.uint32), 90)[0, 0]
        assert m.stats()["kernels_per_decode_step"] == 1          # the fused step is a single launch
        for k, m2 in enumerate(others):
            m2.forward_initial(ids, 0)
            b = m2.decode_steps(5, 50, 40)
            assert a == b, k
            lb = m2.forward_step(np.array([9], np.uint32), 90)[0, 0]
            assert np.abs(la - lb).max() <= 1e-5, k
        assert others[0].stats()["kernels_per_decode_step"] > 100 or cfg["num_hidden_layers"] < 20
    finally:
        for m2 in others:
            m2.close()


@pytest.mark.parametrize("impl", [1, 3, 4])
def test_qwen3_long_context_decode(impl):
    """decode far past the prompt: many KV pages, every split of the attention busy."""
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=2048, decode_impl=impl)
    try:
        o = make_oracle("qwen3", cfg, w)
        S = 700
        ids = _ids(S + 3, cfg["vocab_size"], 21)
        m.forward_initial(ids[:S], 0)
        o.forward_initial(ids[:S].reshape(1, -1), 0)
        for i in range(3):
            got = m.forward_step(ids[S + i:S + i + 1], S + i)[0, 0]
            want = o.forward_step(ids[S + i:S + i + 1].reshape(1, 1), S + i)[0, 0]
            assert np.abs(got - want).max() <= TOL
    finally:
        m.close()


@pytest.mark.parametrize("impl", [1, 3, 4])
def test_qwen3_production_row_shapes(impl):
    """Qwen3-VL-2B text-stack row shapes (H=2048, I=6144; 2 layers): the 4-row / 1-row tensor-core stage paths of the
    fused kernel (impl 3, 4) and the per-op kernels (impl 1) against the oracle, teacher-forced over page boundaries."""
    cfg, w, m = make_model("qwen3", "mid", max_ctx=512, decode_impl=impl)
    try:
        o = make_oracle("qwen3", cfg, w)
        S, n = 90, 40
        ids = _ids(S + n, cfg["vocab_size"], 13)
        got = m.forward_initial(ids[:S], 0)[0, 0]
        want = o.forward_initial(ids[:S].reshape(1, -1), 0)[0, 0]
        assert np.abs(got - want).max() <= TOL
        worst = 0.0
        for i in range(n):
            got = m.forward_step(ids[S + i:S + i + 1], S + i)[0, 0]
            want = o.forward_step(ids[S + i:S + i + 1].reshape(1, 1), S + i)[0, 0]
            err = np.abs(got - want).max()
            worst = max(worst, err)
            assert err <= TOL, (i, err)
            if top2_gap(want) > 10 * max(err, 1e-6):
                assert m.last_argmax == int(np.argmax(want)), i
        print(f"impl {impl}: worst abs logit err over {n} decode steps {worst:.2e}")
    finally:
        m.close()


def test_qwen3_untied_lm_head():
    cfg, w, m = make_model("qwen3", "tiny-untied", max_ctx=128)
    try:
        o = make_oracle("qwen3", cfg, w)
        ids = _ids(17, cfg["vocab_size"], 2)
        got = m.forward_initial(ids, 0)[0, 0]
        want = o.forward_initial(ids.reshape(1, -1), 0)[0, 0]
        assert np.abs(got - want).max() <= TOL
    finally:
        m.close()


def test_qwen3_embedding_and_reranker(q3):
    from oracle.qwen3_embedding import Qwen3Embedding, Qwen3Reranker
    cfg, w, m, o = q3
    oe = Qwen3Embedding(cfg, w)
    for n in (1, 17, 80):
        ids = _ids(n, cfg["vocab_size"], 40 + n)
        got, want = m.embed(ids), oe.embed_one(ids)
        assert abs(float(np.linalg.norm(got)) - 1.0) < 1e-4
        assert np.abs(got - want).max() <= 1e-5
    q = _ids(9, cfg["vocab_size"], 1)
    docs = [_ids(n, cfg["vocab_size"], 50 + n) for n in (5, 33, 12)]
    got = m.rerank(q, docs)
    want = Qwen3Reranker(cfg, w).rerank(q, docs)
    assert np.abs(got - want).max() <= 1e-5
    assert m.forward_initial(_ids(4, cfg["vocab_size"], 1), 0).shape == (1, 1, cfg["vocab_size"])   # handle still serves decoding


def test_error_behaviour(q3):
    from aha_b200 import B200Error
    cfg, w, m, o = q3
    m.clear_cache()
    with pytest.raises(B200Error, match="token id out of range"):
        m.forward_initial(np.array([cfg["vocab_size"]], np.uint32), 0)
    with pytest.raises(B200Error, match="at least one token"):
        m.forward_initial(np.array([], np.uint32), 0)
    m.forward_initial(_ids(4, cfg["vocab_size"], 1), 0)
    with pytest.raises(B200Error, match="seq_len > 1 with seqlen_offset > 0"):
        m.forward_step(_ids(3, cfg["vocab_size"], 1), 4)
    with pytest.raises(B200Error, match="max_ctx"):
        m.forward_step(np.array([1], np.uint32), 512)
    assert m.stop_token_ids() == [cfg["eos_token_id"]]
    # the handle stays usable after an error
    m.clear_cache()
    assert m.forward_initial(_ids(4, cfg["vocab_size"], 1), 0).shape == (1, 1, cfg["vocab_size"])


def test_removed_decode_impl_is_refused_at_create():
    """decode_impl 2 is not a decode path: create fails and the message names the values that are."""
    from aha_b200 import B200Error
    with pytest.raises(B200Error, match=r"decode_impl must be 0 \(auto\), 1 \(per-op kernels\), 3 \(fused, grid barriers\) or 4 "):
        make_model("qwen3", "tiny", max_ctx=512, decode_impl=2)


def test_clear_cache_resets_state(q3):
    cfg, w, m, o = q3
    ids = _ids(33, cfg["vocab_size"], 4)
    m.clear_cache()
    a = m.forward_initial(ids, 0)[0, 0].copy()
    m.forward_step(np.array([3], np.uint32), 33)
    m.clear_cache()
    b = m.forward_initial(ids, 0)[0, 0]
    assert np.array_equal(a, b)  # deterministic and independent of earlier requests


# ----------------------------------------------------------------------------- Qwen3-VL
@pytest.fixture(scope="module")
def vl():
    cfg, w, m = make_model("qwen3vl", "tiny", max_ctx=1024, max_patches=2048)
    yield cfg, w, m, make_oracle("qwen3vl", cfg, w)
    m.close()


def _vl_inputs(cfg, sizes, n_text, seed=1):
    from aha_b200 import synth
    from oracle.qwen3vl import process_image
    pvs, grids = [], []
    for i, (h, w_) in enumerate(sizes):
        pv, g = process_image(synth.synth_image(h, w_, seed + i))
        pvs.append(pv); grids.append(g)
    pv = np.concatenate(pvs, 0); grid = np.concatenate(grids, 0)
    ids = np.concatenate([synth.synth_text_ids(3, 1000, 9), synth.vl_prompt_ids(cfg, grid, n_text)]).astype(np.uint32)
    return pv, grid, ids


@pytest.mark.parametrize("sizes", [[(256, 320)], [(256, 256), (320, 256)]])
def test_vl_prefill_and_decode(vl, sizes):
    cfg, w, m, o = vl
    pv, grid, ids = _vl_inputs(cfg, sizes, 9)
    m.clear_cache(); o.clear_cache()
    got = m.forward_initial(ids, 0, [pv, grid, None, None, None])[0, 0]
    want = o.forward_initial(ids.reshape(1, -1), 0, [pv, grid, None, None, None])[0, 0]
    assert np.abs(got - want).max() <= TOL
    assert int(m.debug_read("rope_delta", 0, 1)[0]) == o.rope_deltas
    S = len(ids)
    for i, t in enumerate([5, 17, 400]):
        got = m.forward_step(np.array([t], np.uint32), S + i)[0, 0]
        want = o.forward_step(np.array([[t]]), S + i)[0, 0]
        assert np.abs(got - want).max() <= TOL


def test_vl_vision_tower_blocks(vl):
    cfg, w, m, o = vl
    pv, grid, ids = _vl_inputs(cfg, [(256, 320)], 4)
    m.clear_cache(); o.clear_cache()
    m.set_trace(True)
    o.visual.trace = []
    m.forward_initial(ids, 0, [pv, grid, None, None, None])
    emb, deep = o.visual.forward(pv, grid)
    Hv, N = cfg["vision_config"]["hidden_size"], pv.shape[0]
    for i, (name, x) in enumerate(o.visual.trace):
        got = m.debug_read("vit", i, N * Hv).reshape(N, Hv)
        assert np.abs(got - x).max() <= 1e-4, name
    got = m.debug_read("image_embeds", 0, emb.size).reshape(emb.shape)
    assert np.abs(got - emb).max() <= 1e-4
    for k, d in enumerate(deep):
        got = m.debug_read("image_embeds", k + 1, d.size).reshape(d.shape)
        assert np.abs(got - d).max() <= 1e-4
    m.set_trace(False)
    o.visual.trace = None


@pytest.mark.parametrize("attn_impl,gemm_impl", [(0, 0), (1, 1), (2, 0)])
def test_vl_head_dim_72_tower(attn_impl, gemm_impl):
    """The Qwen3-VL-8B / 32B tower shape class: head_dim 72 (laid out in zero-padded 128-wide head slots) and an intermediate size that
    is not a multiple of 64 (zero-padded rows / columns): every block output, the merged embeddings and the prefill logits against the
    oracle, on the tensor-core kernels and on the exact fp32 twins."""
    cfg, w, m = make_model("qwen3vl", "tiny-hd72", max_ctx=1024, max_patches=2048, attn_impl=attn_impl, gemm_impl=gemm_impl)
    try:
        o = make_oracle("qwen3vl", cfg, w)
        pv, grid, ids = _vl_inputs(cfg, [(256, 320), (160, 96)], 5)
        m.set_trace(True)
        o.visual.trace = []
        got = m.forward_initial(ids, 0, [pv, grid, None, None, None])[0, 0]
        want = o.forward_initial(ids.reshape(1, -1), 0, [pv, grid, None, None, None])[0, 0]
        Hv, N = cfg["vision_config"]["hidden_size"], pv.shape[0]
        for i, (name, x) in enumerate(o.visual.trace):
            g = m.debug_read("vit", i, N * Hv).reshape(N, Hv)
            assert np.abs(g - x).max() <= 1e-4, name
        assert np.abs(got - want).max() <= TOL
    finally:
        m.close()


def test_vl_attention_implementations_agree(vl):
    """ViT attention: wgmma kernel (default for head_dim 64) == mma.sync kernel == fp32 SIMT twin on a two-image (varlen) prompt
    whose segment lengths are not multiples of the 128-query / 64-key tiles."""
    cfg, w, m, o = vl
    pv, grid, ids = _vl_inputs(cfg, [(256, 320), (352, 288)], 5)
    m.clear_cache()
    m.forward_initial(ids, 0, [pv, grid, None, None, None])
    n = pv.shape[0] // 4 * cfg["vision_config"]["out_hidden_size"]
    base = m.debug_read("image_embeds", 0, n)
    o.clear_cache()
    want, _ = o.visual.forward(pv, grid)
    assert np.abs(base - want.reshape(-1)).max() <= 1e-4
    for impl in (1, 2):
        _, _, m2 = make_model("qwen3vl", "tiny", max_ctx=1024, max_patches=2048, attn_impl=impl)
        try:
            m2.forward_initial(ids, 0, [pv, grid, None, None, None])
            other = m2.debug_read("image_embeds", 0, n)
            assert np.abs(base - other).max() <= 1e-4, impl
        finally:
            m2.close()


@pytest.mark.parametrize("S", [1, 63, 64, 65, 200, 257, 500])
def test_llm_prefill_attention_implementations_agree(q3, S):
    """Causal GQA prefill over the paged KV cache (head_dim 128): wgmma kernel (default) == mma.sync kernel == fp32 SIMT twin == oracle,
    at prompt lengths around the 128-query / 64-key tile edges."""
    cfg, w, m, o = q3
    ids = _ids(S, cfg["vocab_size"], 31 + S)
    m.clear_cache(); o.clear_cache()
    base = m.forward_initial(ids, 0)[0, 0]
    want = o.forward_initial(ids.reshape(1, -1), 0)[0, 0]
    o.clear_cache()
    assert np.abs(base - want).max() <= TOL
    for impl in (1, 2):
        _, _, m2 = make_model("qwen3", "tiny", max_ctx=1024, attn_impl=impl)
        try:
            other = m2.forward_initial(ids, 0)[0, 0]
            assert np.abs(base - other).max() <= 1e-4, impl
        finally:
            m2.close()


def _video_inputs(cfg, n_frames, h, w_, seed):
    from aha_b200 import synth
    from oracle.qwen3vl import img_transform, process_vision_tensor
    frames = np.stack([img_transform(synth.synth_image(h, w_, seed + i), (0.5, 0.5, 0.5), (0.5, 0.5, 0.5)) for i in range(n_frames)])
    return process_vision_tensor(frames)     # pixel_values_video (t*h*w, 1536), video_grid_thw [[t, h/16, w/16]]


@pytest.mark.parametrize("with_image", [False, True])
def test_vl_video_prefill_and_decode(vl, with_image):
    """The video branch of Qwen3VLModel::forward (model.rs:1169-1225): pixel_values_video / video_grid_thw through the same tower, scattered at
    the <|video_pad|> positions, joint deepstack injection with the image embeddings, M-RoPE with one (1, h, w) grid per frame group."""
    from aha_b200 import synth
    cfg, w, m, o = vl
    pvv, vgrid = _video_inputs(cfg, 4, 64, 96, 11)               # 4 frames -> 2 temporal steps of 4 x 6 patches
    parts = [synth.synth_text_ids(3, 1000, 9), synth.vl_video_prompt_ids(cfg, vgrid)]
    pv = grid = None
    if with_image:
        pv, grid, img_ids = _vl_inputs(cfg, [(128, 96)], 0)
        parts = [img_ids] + parts
    ids = np.concatenate(parts + [synth.synth_text_ids(6, 1000, 4)]).astype(np.uint32)
    m.clear_cache(); o.clear_cache()
    got = m.forward_initial(ids, 0, [pv, grid, pvv, vgrid, None])[0, 0]
    want = o.forward_initial(ids.reshape(1, -1), 0, [pv, grid, pvv, vgrid, None])[0, 0]
    assert np.abs(got - want).max() <= TOL
    assert int(m.debug_read("rope_delta", 0, 1)[0]) == o.rope_deltas
    S = len(ids)
    for i, t in enumerate([5, 17]):
        got = m.forward_step(np.array([t], np.uint32), S + i)[0, 0]
        want = o.forward_step(np.array([[t]]), S + i)[0, 0]
        assert np.abs(got - want).max() <= TOL
    bad = np.concatenate([ids, [cfg["video_token_id"]]]).astype(np.uint32)
    m.clear_cache()
    with pytest.raises(Exception, match="n_image_token num"):
        m.forward_initial(bad, 0, [pv, grid, pvv, vgrid, None])
    m.clear_cache()


def test_vl_text_only_prompt(vl):
    cfg, w, m, o = vl
    ids = _ids(12, 1000, 3)
    m.clear_cache(); o.clear_cache()
    got = m.forward_initial(ids, 0, [None, None, None, None, None])[0, 0]
    want = o.forward_initial(ids.reshape(1, -1), 0, [None, None, None, None, None])[0, 0]
    assert np.abs(got - want).max() <= TOL


def test_vl_errors(vl):
    from aha_b200 import B200Error
    cfg, w, m, o = vl
    pv, grid, ids = _vl_inputs(cfg, [(256, 320)], 4)
    m.clear_cache()
    with pytest.raises(B200Error, match="must have pixel_values"):
        m.forward_initial(ids, 0, [pv, grid])
    bad = ids.copy(); bad[5] = 7  # one placeholder fewer
    with pytest.raises(B200Error, match="not equal to image_embed len"):
        m.forward_initial(bad, 0, [pv, grid, None, None, None])


def test_vl_image_patchify(vl):
    from aha_b200 import synth
    from oracle.qwen3vl import process_image
    cfg, w, m, o = vl
    img = synth.synth_image(256, 320, 7)
    pv, grid = m.image_patchify(img)
    wpv, wgrid = process_image(img)
    assert grid.tolist() == wgrid.tolist()
    assert np.array_equal(pv, wpv)    # affine, sub, div rounded one by one like the reference: bit-exact


# ----------------------------------------------------------------------------- Qwen3-ASR
@pytest.fixture(scope="module")
def asr():
    cfg, w, m = make_model("qwen3_asr", "tiny", max_ctx=512, max_frames=600)
    yield cfg, w, m, make_oracle("qwen3_asr", cfg, w)
    m.close()


@pytest.mark.parametrize("seconds", [1.0, 2.5, 3.07])
def test_asr_mel_frontend(asr, seconds):
    from aha_b200 import synth
    from oracle.audio import WhisperFeatureExtractor
    cfg, w, m, o = asr
    wave = synth.synth_audio(seconds)
    want = WhisperFeatureExtractor().call(wave[None], 16000)[0]
    got = m.mel_spectrogram(wave)
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= 1e-3


@pytest.mark.parametrize("seconds", [1.0, 2.5])
def test_asr_prefill_and_decode(asr, seconds):
    from aha_b200 import synth
    from oracle.audio import WhisperFeatureExtractor, get_feat_extract_output_lengths
    cfg, w, m, o = asr
    mel = WhisperFeatureExtractor().call(synth.synth_audio(seconds)[None], 16000)[0]
    ids = synth.asr_prompt_ids(cfg, get_feat_extract_output_lengths(mel.shape[1]))
    m.clear_cache(); o.clear_cache()
    m.set_trace(True)
    o.audio.trace = []
    got = m.forward_initial(ids, 0, [mel])[0, 0]
    want = o.forward_initial(ids.reshape(1, -1), 0, [mel])[0, 0]
    D = cfg["thinker_config"]["audio_config"]["d_model"]
    for i, (name, x) in enumerate(o.audio.trace):
        g = m.debug_read("audio", i, x.size).reshape(x.shape)
        assert np.abs(g - x).max() <= 1e-4, name
    assert np.abs(got - want).max() <= TOL
    S = len(ids)
    got = m.forward_step(np.array([9], np.uint32), S)[0, 0]
    want = o.forward_step(np.array([[9]]), S)[0, 0]
    assert np.abs(got - want).max() <= TOL
    m.set_trace(False)
    o.audio.trace = None


def test_asr_errors(asr):
    from aha_b200 import B200Error, synth
    from oracle.audio import WhisperFeatureExtractor
    cfg, w, m, o = asr
    mel = WhisperFeatureExtractor().call(synth.synth_audio(1.0)[None], 16000)[0]
    ids = synth.asr_prompt_ids(cfg, 5)
    m.clear_cache()
    with pytest.raises(B200Error, match="not equal to audio_feature len"):
        m.forward_initial(ids, 0, [mel])


def _rand_ids(n, vocab, seed):
    return np.random.default_rng(seed).integers(0, min(vocab, 1000), n).astype(np.uint32)


# GQA groups other than 2 (every shipped Qwen3 size has nh / nkv = 2): MHA and a group of 4, fused and per-op decode
@pytest.mark.parametrize("preset", ["tiny-g1", "tiny-g4"])
@pytest.mark.parametrize("impl", [1, 3, 4])
def test_decode_with_other_gqa_groups(preset, impl):
    cfg, w, m = make_model("qwen3", preset, max_ctx=512, decode_impl=impl)
    o = make_oracle("qwen3", cfg, w)
    try:
        ids = _rand_ids(70, cfg["vocab_size"], 11)
        got = m.forward_initial(ids, 0)[0, 0]
        want = o.forward_initial(ids.reshape(1, -1), 0)[0, 0]
        assert np.abs(got - want).max() <= TOL
        tok = int(np.argmax(want))
        for step in range(16):
            lg = m.forward_step(np.array([tok], np.uint32), 70 + step)[0, 0]
            lo = o.forward_step(np.array([[tok]]), 70 + step)[0, 0]
            assert np.abs(lg - lo).max() <= TOL, (step, np.abs(lg - lo).max())
            tok = int(np.argmax(lo))
    finally:
        m.close()


def test_bf16_checkpoint_is_narrowed_exactly_or_refused():
    """Shipped Qwen3 checkpoints are bf16: values inside fp16's normal range convert exactly (logits equal the oracle on the bf16
    values); a value fp16 cannot hold makes create fail loudly instead of loading an inf."""
    from aha_b200 import B200Model, synth
    from aha_b200._lib import to_bf16
    from aha_b200.inference import B200Error
    cfg = synth.get_config("qwen3", "tiny")
    w16 = synth.make_weights("qwen3", cfg, 0)
    wb = {k: to_bf16(v.astype(np.float32)) for k, v in w16.items()}
    as_f32 = {k: (v.view(np.ndarray).astype(np.uint32) << 16).view(np.float32).reshape(w16[k].shape) for k, v in wb.items()}
    for k, v in as_f32.items():   # keep the test inside the exactly-representable range (tiny values would be refused)
        small = (np.abs(v) < 6.2e-5) & (v != 0)
        if small.any():
            v[small] = 0.0
            wb[k] = to_bf16(v)
    m = B200Model("qwen3", cfg, {k: v.reshape(w16[k].shape) for k, v in wb.items()}, max_ctx=256)
    try:
        o = make_oracle("qwen3", cfg, as_f32)
        ids = _rand_ids(40, cfg["vocab_size"], 2)
        got = m.forward_initial(ids, 0)[0, 0]
        want = o.forward_initial(ids.reshape(1, -1), 0)[0, 0]
        assert np.abs(got - want).max() <= TOL
    finally:
        m.close()
    bad = dict(wb)
    big = as_f32["model.norm.weight"].copy()   # norm gains stay fp32 on the device: use a linear weight for the range check
    k = "model.layers.0.mlp.down_proj.weight"
    v = as_f32[k].copy(); v[0, 0] = 1e6
    bad[k] = to_bf16(v).reshape(v.shape)
    with pytest.raises(B200Error, match="fp16 range"):
        B200Model("qwen3", cfg, {kk: vv.reshape(w16[kk].shape) for kk, vv in bad.items()}, max_ctx=256)
