"""Speculative decoding without a GPU: the Python argument checks of generate_speculative and the Python restatement of the draft rule."""
import numpy as np
import pytest

from spec_ref import draft, simulate


def test_spec_params_packs_the_request():
    from aha_b200 import _lib as L
    sp, keep = L.spec_params([5, 6, 7], prompt_lookup=True, max_draft=4, ngram=2, vocab_size=100)
    assert sp.n_prediction == 3 and [sp.prediction[i] for i in range(3)] == [5, 6, 7] and keep.dtype == np.uint32
    assert sp.max_draft == 4 and sp.ngram == 2 and sp.flags == L.SPEC_PROMPT_LOOKUP
    sp, keep = L.spec_params(None)
    assert sp.n_prediction == 0 and not sp.prediction and sp.flags == 0 and sp.max_draft == 7 and sp.ngram == 3
    assert L.spec_params([], ngram=0)[0].n_prediction == 0


@pytest.mark.parametrize("kw,err", [
    (dict(max_draft=0), ValueError), (dict(max_draft=16), ValueError), (dict(max_draft=2.0), TypeError), (dict(max_draft=True), TypeError),
    (dict(ngram=-1), ValueError), (dict(ngram=9), ValueError), (dict(ngram="3"), TypeError),
    (dict(prediction=[1, 100]), ValueError), (dict(prediction=[-1]), ValueError), (dict(prediction=[0.5]), TypeError),
])
def test_spec_params_refusals(kw, err):
    from aha_b200 import _lib as L
    with pytest.raises(err):
        L.spec_params(vocab_size=100, **kw)


def test_spec_structs_match_the_header_layout():
    import ctypes as C
    from aha_b200 import _lib as L
    assert C.sizeof(L.SpecParams) == 40 and L.SpecParams.max_draft.offset == 16 and L.SpecParams.flags.offset == 24
    assert C.sizeof(L.SpecStats) == 16


def test_draft_takes_the_longest_suffix_then_the_most_recent_occurrence():
    pred = [1, 2, 3, 9, 9, 2, 3, 4, 5, 6]
    # suffix (2, 3) occurs at 1 and 5: the most recent one (5) wins
    assert draft([7, 2, 3], pred, None, 3, 3) == [4, 5, 6]
    assert draft([7, 2, 3], pred, None, 2, 3) == [4, 5]
    # (1, 2, 3) occurs at 0 only: longer suffixes win over more recent shorter ones
    assert draft([1, 2, 3], pred, None, 4, 3) == [9, 9, 2, 3]
    assert draft([1, 2, 3], pred, None, 4, 1) == [4, 5, 6]
    # an occurrence must be followed by a token; truncated at the end of the source
    assert draft([5, 6], pred, None, 7, 3) == []
    assert draft([4], pred, None, 7, 3) == [5, 6]
    assert draft([42], pred, None, 7, 3) == []


def test_draft_prefers_the_prediction_and_looks_up_prompt_then_output():
    prompt = [10, 11, 12, 13]
    assert draft([11], [11, 50], prompt, 3, 3) == [50]                     # same n: the prediction first
    assert draft([10, 11], [11, 50], prompt, 3, 3) == [12, 13, 10]         # a longer suffix in the lookup text wins; it runs into the output
    assert draft([10, 11], [11, 50], None, 3, 3) == [50]                   # without lookup
    assert draft([13, 20, 13], [], prompt, 3, 3) == [20, 13]               # the output itself, most recent occurrence first
    assert draft([12], [], prompt, 1, 3) == [13]


def test_simulate_counts_passes():
    out = list(range(100, 120))
    assert simulate(out, None, None, 7, 3) == (19, 0, 0)                   # no source: one token per pass
    p, d, a = simulate(out, out, None, 7, 3)                               # exact prediction: every pass takes all its drafts
    assert (p, d, a) == (3, 17, 17)                                        # 1 + 8 + 8, then the last 3 drafts (the output ends there)
    assert simulate(out, out, None, 15, 3) == (2, 18, 18)
    edited = out[:5] + [7] + out[6:]
    p2, d2, a2 = simulate(out, edited, None, 7, 3)
    assert p2 > p and a2 < d2
