"""The float64 decoder reference (tests/decode_ref.py) against the float32 oracle (oracle/qwen3.py): a prefill and a step-by-step
decode of the oracle give the reference's logits at the same positions, within float32 noise, for 2-way and 4-way GQA and an untied
lm_head."""
import numpy as np
import pytest

import decode_ref


def _setup(preset):
    from aha_b200 import synth
    from oracle.qwen3 import Qwen3Model
    cfg = synth.get_config("qwen3", preset)
    w = synth.make_weights("qwen3", cfg, 0)
    return cfg, w, Qwen3Model(cfg, w)


@pytest.mark.parametrize("preset", ["tiny", "tiny-g4", "tiny-untied"])
def test_reference_matches_the_oracle_decode(preset):
    from aha_b200 import synth
    cfg, w, o = _setup(preset)
    V = cfg["vocab_size"]
    prompt = synth.synth_text_ids(37, V, 1)
    steps = synth.synth_text_ids(12, V, 2)
    ref = decode_ref.logits(cfg, w, [np.concatenate([prompt, steps])])[0]
    assert ref.shape == (len(prompt) + len(steps), V)
    want = [o.forward_initial(prompt.reshape(1, -1), 0)[0, 0]]
    want += [o.forward_step(np.array([[t]]), len(prompt) + i)[0, 0] for i, t in enumerate(steps)]
    got = ref[len(prompt) - 1:]
    scale = max(1.0, np.abs(got).max())
    for i, wl in enumerate(want):   # position len(prompt) - 1 + i
        err = np.abs(got[i] - wl).max()
        assert err <= 2e-5 * scale, (preset, i, err)
    # every position, not only the decoded ones: the oracle's prefill of each prefix ends at that position
    for n in (1, 2, 17, 32, 33):
        o.clear_cache()
        wl = o.forward_initial(prompt[:n].reshape(1, -1), 0)[0, 0]
        assert np.abs(ref[n - 1] - wl).max() <= 2e-5 * scale, (preset, n)


def test_sequences_are_independent_in_one_call():
    from aha_b200 import synth
    cfg, w, _ = _setup("tiny")
    V = cfg["vocab_size"]
    a, b = synth.synth_text_ids(20, V, 3), synth.synth_text_ids(45, V, 4)
    both = decode_ref.logits(cfg, w, [a, b])
    np.testing.assert_allclose(both[0], decode_ref.logits(cfg, w, [a])[0], rtol=0, atol=1e-12)
    np.testing.assert_allclose(both[1], decode_ref.logits(cfg, w, [b])[0], rtol=0, atol=1e-12)


def test_rms_norm_puts_eps_inside_the_root():
    g = np.float16([1.5, 0.5, 2.0, 1.0])
    assert np.array_equal(decode_ref.rms_norm(np.zeros((2, 4)), g, 1e-6), np.zeros((2, 4)))   # 0 / sqrt(0 + eps): exactly zero
    x = np.array([3e-4, -1e-4, 2e-4, 0.0])
    want = x / np.sqrt((x * x).mean() + 1e-6) * g.astype(np.float64)   # eps is comparable to mean(x^2) here
    assert np.abs(decode_ref.rms_norm(x, g, 1e-6) - want).max() <= 1e-15
    assert np.abs(decode_ref.rms_norm(x, g, 1e-6) - x / np.sqrt((x * x).mean()) * g).max() > 0.1


def test_log_softmax_is_float64_and_normalised():
    rng = np.random.default_rng(5)
    l = rng.standard_normal((3, 151936)) * 4
    l[1, 7] = 80.0   # a peaked row
    ls = decode_ref.log_softmax(l)
    assert ls.dtype == np.float64
    np.testing.assert_allclose(np.exp(ls).sum(-1), 1.0, rtol=0, atol=1e-12)
    np.testing.assert_allclose(ls - l, (ls - l)[:, :1].repeat(l.shape[1], 1), rtol=0, atol=1e-12)


def test_rope_angle_is_rounded_to_float32():
    from oracle.rope import RoPE
    cos, sin = decode_ref.rope_tables(5000, 128, 1e6)
    oc, os_ = RoPE(128, 1e6).forward(0, 5000)
    assert np.abs(cos - oc).max() <= 1e-6 and np.abs(sin - os_).max() <= 1e-6   # the same float32 angles
    a = np.float32(4999) * np.float32(1.0)
    assert cos[4999, 0] == np.cos(np.float64(a))
