"""The fused decode step hands q / k / v to the attention inside each kv-head group: the (G + 2) * head_dim qkv rows of a group
are shared by the group's attention CTAs (decode_fused.cuh: qkv_slab).  These shapes make the shares uneven and make them
straddle the q / k / v segments of the packed matrix, with tail stages; every fused mode must still decode exactly like the
per-op kernels."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _model(nh, nkv, impl):
    from aha_b200 import B200Model, synth
    cfg = synth.get_config("qwen3", "tiny")
    cfg.update(num_attention_heads=nh, num_key_value_heads=nkv)
    w = synth.make_weights("qwen3", cfg, 0)
    return cfg, B200Model("qwen3", cfg, w, eos_ids=[], max_ctx=1024, decode_impl=impl)


# (12, 6): G = 2 over 6 kv heads -> 22 attention splits per group on a 132-SM H100, 512 rows per group: shares of 23 or 24 rows.
# (12, 3): G = 4 -> 768 rows per group over 32 splits: shares of 24 rows, one of them across the q / k boundary.
@pytest.mark.parametrize("nh,nkv", [(12, 6), (12, 3)])
def test_fused_step_matches_per_op_with_uneven_qkv_shares(nh, nkv):
    from aha_b200 import synth
    cfg, ref = _model(nh, nkv, 1)
    models = [_model(nh, nkv, impl)[1] for impl in (0, 4)]   # grid barriers, hybrid
    try:
        ids = synth.synth_text_ids(300, cfg["vocab_size"] - 8, 5)
        ref.forward_initial(ids, 0)
        want = ref.decode_steps(7, 300, 24)
        want_logits = ref.forward_step(np.array([11], np.uint32), 324)[0, 0]
        for k, m in enumerate(models):
            m.forward_initial(ids, 0)
            assert m.decode_steps(7, 300, 24) == want, k
            assert m.stats()["kernels_per_decode_step"] == 1, k   # the fused kernel is in use
            got = m.forward_step(np.array([11], np.uint32), 324)[0, 0]
            assert np.abs(got - want_logits).max() <= 1e-4, (k, float(np.abs(got - want_logits).max()))
    finally:
        ref.close()
        for m in models:
            m.close()
