"""Log-probability records, host side (no GPU): the float64 reference the GPU tests compare with, the flag packing of the C ABI and the
Python-side argument checks."""
import ctypes as C

import numpy as np
import pytest
from scipy.special import log_softmax

import logprob_ref as R
from aha_b200 import _lib as L


@pytest.mark.parametrize("V,scale", [(1024, 1.0), (4097, 8.0), (151936, 3.0)])
def test_reference_matches_scipy_log_softmax(V, scale):
    rng = np.random.default_rng(V)
    x = (rng.standard_normal(V) * scale).astype(np.float32)
    want = log_softmax(x.astype(np.float64))
    got = R.log_softmax64(x)
    assert np.max(np.abs(got - want)) < 1e-12
    tok = int(rng.integers(0, V))
    lp, ids, tops = R.logprobs(x, tok, 20)
    assert lp == pytest.approx(want[tok], abs=1e-12)
    assert ids == sorted(range(V), key=lambda i: (-float(x[i]), i))[:20]
    assert np.allclose(tops, want[ids], atol=1e-12, rtol=0)


def test_reference_orders_ties_by_ascending_id():
    x = np.array([1.0, 3.0, 3.0, -2.0, 3.0, 1.0, 0.0, -0.0], np.float32)
    assert list(R.top_order(x, 8)) == [1, 2, 4, 0, 5, 6, 7, 3]
    _, ids, tops = R.logprobs(x, 1, 3)
    assert ids == [1, 2, 4] and tops[0] == tops[1] == tops[2]


def test_flag_packing_matches_the_header():
    assert L.GEN_LOGPROBS == 8 and L.MAX_TOP_LOGPROBS == 20
    assert L.gen_top_logprobs(5) == 5 << 8
    assert L.gen_top_logprobs(300) == 300 << 8          # not masked: the library refuses it instead of wrapping it to 44
    assert L.logprob_flags() == 0 and L.logprob_flags(False, 0) == 0
    assert L.logprob_flags(True) == 8
    assert L.logprob_flags(True, 20) == 8 | (20 << 8)
    # the record's layout is the header's (static_assert'ed on the device side too)
    assert C.sizeof(L.Logprobs) == 184
    offs = {name: getattr(L.Logprobs, name).offset for name, _ in L.Logprobs._fields_}
    assert offs == dict(token=0, index=4, logprob=8, n_top=12, top_ids=16, top_logprobs=96, valid=176, reserved=180)


def test_python_side_argument_checks():
    with pytest.raises(ValueError, match="needs logprobs=True"):
        L.logprob_flags(False, 3)
    with pytest.raises(ValueError, match="0 to 20"):
        L.logprob_flags(True, 21)
    with pytest.raises(ValueError, match="0 to 20"):
        L.logprob_flags(True, -1)
    with pytest.raises(ValueError, match="vocabulary"):
        L.logprob_flags(True, 12, vocab_size=10)
    with pytest.raises(TypeError):
        L.logprob_flags(True, 2.5)
    with pytest.raises(TypeError):
        L.logprob_flags(True, True)


def test_record_conversion_keeps_float32_values():
    r = L.Logprobs()
    r.token, r.index, r.logprob, r.n_top, r.valid = 7, 3, -1.25, 2, 1
    r.top_ids[0], r.top_ids[1], r.top_ids[2] = 7, 9, 11
    r.top_logprobs[0], r.top_logprobs[1] = -1.25, -2.5
    d = L.logprobs_record(r)
    assert d == dict(token=7, index=3, logprob=np.float32(-1.25), top_ids=[7, 9], top_logprobs=[np.float32(-1.25), np.float32(-2.5)])
    assert isinstance(d["logprob"], np.float32)


def test_header_declares_the_logprob_entries():
    import os
    from conftest import ROOT
    text = open(os.path.join(ROOT, "include", "aha_b200.h")).read()
    for s in ("#define AHA_GEN_LOGPROBS 8u", "#define AHA_MAX_TOP_LOGPROBS 20", "aha_b200_generate_logprobs(", "aha_b200_generate_stream_logprobs(",
              "aha_b200_batch_logprobs(", "aha_b200_debug_logprobs(", "aha_logprobs_callback", "#define AHA_B200_ABI_VERSION 3"):
        assert s in text, s
