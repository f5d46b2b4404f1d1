"""Logit rules on the host: aha_b200_rules_check accepts well-formed rules and refuses each malformed case with its own message, the
ctypes mirror matches the header, and the oracle restatement (tests/penalty_ref.py) gives hand-computed values."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import penalty_ref as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def _raw_check(r, V):
    from aha_b200 import _lib as L
    lib = L.load()
    if lib.aha_b200_rules_check(C.byref(r), V) != 0:
        return lib.aha_b200_last_error(None).decode()
    return None


@pytest.mark.parametrize("V", [1, 8, 151936])
def test_well_formed_rules_pass(lib_built, V):
    from aha_b200 import rules_check
    rules_check(vocab_size=V)
    rules_check(2.0, -2.0, {0: 100.0}, vocab_size=V)
    rules_check(-2.0, 2.0, {str(V - 1): -100}, vocab_size=V)
    rules_check(0.5, 0.5, {t: (t % 201) - 100.0 for t in range(V)}, vocab_size=V)    # every token listed once


@pytest.mark.parametrize("what,kw", [
    ("presence_penalty", dict(presence_penalty=2.5)),
    ("presence_penalty", dict(presence_penalty=float("nan"))),
    ("frequency_penalty", dict(frequency_penalty=-2.01)),
    ("frequency_penalty", dict(frequency_penalty=float("inf"))),
    ("outside the vocabulary", dict(logit_bias={8: 1.0})),
    ("listed twice", dict(logit_bias=[(3, 1.0), (3, 2.0)])),
    ("not a finite value in \\[-100, 100\\]", dict(logit_bias={2: 100.5})),
    ("not a finite value in \\[-100, 100\\]", dict(logit_bias={2: float("-inf")})),
    ("not a finite value in \\[-100, 100\\]", dict(logit_bias={2: float("nan")})),
])
def test_malformed_rules_are_refused(lib_built, what, kw):
    from aha_b200 import B200Error, rules_check
    with pytest.raises(B200Error, match=what):
        rules_check(vocab_size=8, **kw)


def test_null_pointers_and_reserved_are_refused(lib_built):
    from aha_b200 import _lib as L
    r, _keep = L.logit_rules(logit_bias={1: 1.0})
    assert _raw_check(r, 8) is None
    r2 = L.LogitRules(n_bias=1, bias_ids=r.bias_ids)
    assert "bias_ids and bias_values are required" in _raw_check(r2, 8)
    r3 = L.LogitRules(n_bias=1, bias_values=r.bias_values)
    assert "bias_ids and bias_values are required" in _raw_check(r3, 8)
    r4, _k4 = L.logit_rules()
    r4.reserved[1] = 1
    assert "reserved must be 0" in _raw_check(r4, 8)
    r5, _k5 = L.logit_rules(logit_bias=[(t, 0.0) for t in range(4)])
    assert "exceeds the vocabulary" in _raw_check(r5, 3)
    from aha_b200 import _lib
    assert _lib.load().aha_b200_rules_check(None, 8) != 0


def test_ctypes_layout_matches_the_header():
    from aha_b200 import _lib as L
    R = L.LogitRules
    offs = {name: getattr(R, name).offset for name, _ in R._fields_}
    assert offs == dict(presence_penalty=0, frequency_penalty=4, bias_ids=8, bias_values=16, n_bias=24, fsm=32, reserved=36)
    assert C.sizeof(R) == 48
    hdr = open(os.path.join(ROOT, "include", "aha_b200.h")).read()
    body = re.search(r"typedef struct aha_logit_rules \{(.*?)\} aha_logit_rules;", hdr, re.S).group(1)
    fields = re.findall(r"^\s*[\w\s\*]+?[\s\*](\w+)(?:\[\d+\])?;", body, re.M)
    assert fields == [name for name, _ in R._fields_]


def test_header_declares_the_entries_and_keeps_abi_3():
    hdr = open(os.path.join(ROOT, "include", "aha_b200.h")).read()
    for sym in ("aha_b200_rules_check", "aha_b200_rules_create", "aha_b200_rules_destroy", "aha_b200_debug_sample_rules"):
        assert re.search(r"\bint " + sym + r"\(", hdr), sym
    assert re.search(r"#define AHA_GEN_LOGIT_RULES 32u", hdr)
    assert re.search(r"#define AHA_B200_ABI_VERSION 3\b", hdr)
    from aha_b200 import _lib as L
    assert L.GEN_LOGIT_RULES == 32 and L.GEN_CONSTRAINED == 16


# ---------------------------------------------------------------------------------------------------------- the oracle restatement
def _s(**kw):
    import constrain_ref as cr
    return cr.sampler(**kw)


def test_counts_cover_the_whole_history_and_presence_applies_once():
    x = np.array([1.0, 2.0, 3.0, 4.0], F32)
    gen = [1, 1, 1, 3]
    y = P.transform(_s(repeat_penalty=1.0), x, gen, dict(frequency_penalty=0.5, presence_penalty=0.25))
    assert y.tolist() == [1.0, 2.0 - 1.5 - 0.25, 3.0, 4.0 - 0.5 - 0.25]
    # counts are over the whole output even with repeat_last_n = 1 (which limits only the repeat penalty)
    long = [2] * 100 + [0]
    y = P.transform(_s(repeat_penalty=2.0, repeat_last_n=1), x, long, dict(frequency_penalty=0.01))
    assert y[0] == F32(F32(0.5) - F32(F32(1) * F32(0.01)))
    assert y[2] == F32(3.0 - F32(F32(100) * F32(0.01)))


def test_each_step_rounds_on_its_own():
    # c * f rounded before the subtraction: an FMA would keep the product's low bits
    x = np.array([F32(1.0000001)], F32)
    f = F32(0.1)
    y = P.apply_counts(x, [0] * 3, f, F32(1e-8))
    prod = F32(F32(3) * f)
    assert y[0] == F32(F32(x[0] - prod) - F32(1e-8))


def test_minus_inf_stays_under_mask_bias_and_penalties():
    import constrain_ref as cr
    fsm = cr.from_rows([([1, 2], [0, 0])])
    x = np.array([5.0, -1.0, 2.0, 7.0], F32)
    y = P.transform(_s(repeat_penalty=1.3), x, [0, 3, 3, 1], dict(frequency_penalty=-2.0, presence_penalty=-2.0,
                                                                     logit_bias={0: 100.0, 3: 50.0}), fsm, 0)
    assert y[0] == -np.inf and y[3] == -np.inf
    assert y[1] == F32(F32(F32(-1.0) * F32(1.3)) + F32(2.0)) + F32(2.0)   # penalised, then -(1 * -2) - (-2)
    assert y[2] == 2.0


def test_bias_comes_before_the_repeat_penalty():
    x = np.array([1.0, -1.0], F32)
    y = P.transform(_s(repeat_penalty=2.0), x, [0, 1], dict(logit_bias={0: -3.0, 1: 3.0}))
    # bias first: 1 - 3 = -2 -> * 2 = -4; -1 + 3 = 2 -> / 2 = 1 (the other order would give -2.5 and 2.5)
    assert y.tolist() == [-4.0, 1.0]


def test_zero_rules_change_nothing():
    x = np.random.default_rng(0).normal(size=64).astype(F32)
    y = P.transform(_s(repeat_penalty=1.1), x, [3, 3, 9], dict(frequency_penalty=0.0, presence_penalty=0.0, logit_bias={}))
    z = P.transform(_s(repeat_penalty=1.1), x, [3, 3, 9], None)
    assert np.array_equal(y, z)
