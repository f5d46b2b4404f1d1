"""Attention end to end where no host-data seam exists: a GQA group of 6 through prefill, the per-op decode step and both batch sessions,
and sharply peaked attention through every decode step, the fused kernel's included, against the oracle."""
import numpy as np
import pytest

from conftest import TOL, make_oracle, top2_gap
from test_batch_wide_gpu import SAMPLERS, _check_oracle_ids, _Session

pytestmark = pytest.mark.gpu


def _weights(nh=None, nkv=None, norm_scale=1.0):
    from aha_b200 import synth
    cfg = synth.get_config("qwen3", "tiny")
    if nh:
        cfg.update(num_attention_heads=nh, num_key_value_heads=nkv)
    w = synth.make_weights("qwen3", cfg, 0)
    for n in w:
        if n.endswith(("q_norm.weight", "k_norm.weight")):
            w[n] = (w[n].astype(np.float32) * norm_scale).astype(w[n].dtype)
    return cfg, w


def _ids(n, cfg, seed):
    from aha_b200 import synth
    return synth.synth_text_ids(n, cfg["vocab_size"] - 8, seed)


# ------------------------------------------------------------------------------------------------------------ GQA group 6

@pytest.fixture(scope="module")
def g6():
    cfg, w = _weights(12, 2)   # G = 6: decode_attn_*<128, 6>, which no preset reaches
    return cfg, w, make_oracle("qwen3", cfg, w)


@pytest.mark.parametrize("attn_impl", [0, 1, 2])
def test_group6_prefill_logits(g6, attn_impl):
    from aha_b200 import B200Model
    cfg, w, o = g6
    m = B200Model("qwen3", cfg, w, eos_ids=[], max_ctx=1024, attn_impl=attn_impl)
    try:
        for n, seed in ((1, 1), (77, 2), (300, 3)):
            ids = _ids(n, cfg, seed)
            got = m.forward_initial(ids, 0)[0, 0]
            want = o.forward_initial(ids.reshape(1, -1), 0)[0, 0]
            assert np.abs(got - want).max() <= TOL, (n, float(np.abs(got - want).max()))
            m.clear_cache()
            o.clear_cache()
    finally:
        m.close()


def test_group6_teacher_forced_decode_across_pages(g6):
    """20 prompt tokens, then 60 forced steps through the per-op step (the fused kernel refuses G > 4), over the page boundaries at 32
    and 64"""
    from aha_b200 import B200Model
    cfg, w, o = g6
    m = B200Model("qwen3", cfg, w, eos_ids=[], max_ctx=1024)
    try:
        ids = _ids(80, cfg, 4)
        o.clear_cache()
        got = m.forward_initial(ids[:20], 0)[0, 0]
        want = o.forward_initial(ids[:20].reshape(1, -1), 0)[0, 0]
        assert np.abs(got - want).max() <= TOL
        for t in range(20, 80):
            got = m.forward_step(ids[t:t + 1], t)[0, 0]
            want = o.forward_step(ids[t:t + 1].reshape(1, 1), t)[0, 0]
            assert np.abs(got - want).max() <= TOL, (t, float(np.abs(got - want).max()))
        assert m.stats()["kernels_per_decode_step"] > 1
    finally:
        m.close()
        o.clear_cache()


class _Narrow(_Session):
    def __init__(self, m):
        self.m, self.out, self.running, self.counts = m, {}, {}, set()
        m.batch_open()


@pytest.mark.parametrize("wide", [False, True])
def test_group6_batch_sessions_give_oracle_ids(g6, wide):
    from aha_b200 import B200Model
    cfg, w, o = g6
    reqs = []
    for i, samp in enumerate(SAMPLERS + [{}, {}]):
        r = dict(input_ids=_ids(5 + 47 * i, cfg, 10 + i), max_tokens=12 + 5 * i, **samp)
        if samp.get("temperature"):
            r["seed"] = 100 + i
        reqs.append(r)
    m = B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"]], max_ctx=4096, max_prefill=512)
    try:
        s = _Session(m, 16) if wide else _Narrow(m)
        s.add_many([(i, r) for i, r in enumerate(reqs[:4])])
        s.step(3)
        for i, r in enumerate(reqs[4:], 4):
            s.add(i, r)
        s.drain()
        s.close()
        _check_oracle_ids(o, reqs, [s.out[i] for i in range(len(reqs))])
    finally:
        m.close()


# ------------------------------------------------------------------------------------------------------------ peaked attention

# q_norm / k_norm weights x 4: on a 1600-token prompt the oracle's last 64 rows of every head put a median 0.94 of their mass on one
# key, and 57 % of them more than 0.9 (x 1: a median 0.01; x 3: 0.75; x 6: 0.999).
PEAK_SCALE = 4.0


@pytest.mark.parametrize("decode_impl", [1, 3, 4])
def test_peaked_attention_decode_steps(decode_impl):
    """1600 prompt tokens: each of the fused kernel's 32 splits walks several half-pages"""
    from aha_b200 import B200Model
    cfg, w = _weights(norm_scale=PEAK_SCALE)
    o = make_oracle("qwen3", cfg, w)
    m = B200Model("qwen3", cfg, w, eos_ids=[], max_ctx=2048, decode_impl=decode_impl)
    try:
        ids = _ids(1600, cfg, 3)
        got = m.forward_initial(ids, 0)[0, 0]
        want = o.forward_initial(ids.reshape(1, -1), 0)[0, 0]
        assert np.abs(got - want).max() <= TOL
        tok = int(np.argmax(want))
        for t in range(1600, 1608):
            got = m.forward_step(np.array([tok], np.uint32), t)[0, 0]
            want = o.forward_step(np.array([[tok]]), t)[0, 0]
            assert np.abs(got - want).max() <= TOL, (t, float(np.abs(got - want).max()))
            if top2_gap(want) > 2 * TOL:
                assert int(np.argmax(got)) == int(np.argmax(want)), t
            tok = int(np.argmax(want))
        assert (m.stats()["kernels_per_decode_step"] == 1) == (decode_impl != 1)
    finally:
        m.close()
