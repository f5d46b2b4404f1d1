"""Token automata on the host: aha_b200_fsm_check accepts what the builders of tests/constrain_ref.py make and refuses every malformed
automaton with a message, and the regex builder's automaton accepts exactly the token sequences whose text the regex matches."""
import itertools

import numpy as np
import pytest

import constrain_ref as R


def _check(fsm, V):
    from aha_b200 import fsm_check
    off, tok, nxt, start = fsm
    fsm_check(off, tok, nxt, start, V)


@pytest.mark.parametrize("V", [1, 2, 257, 4097, 151936])
def test_builders_pass_the_check(lib_built, V):
    _check(R.all_allowed(V), V)
    _check(R.chain([V - 1, 0, V // 2, V - 1], 0), V)
    _check(R.random_fsm(V, 9, V), V)


def test_regex_automaton_passes_the_check(lib_built):
    table = R.token_table(300, 7)
    _check(R.regex_fsm(table, 7), 300)


def _good():
    return [np.array([0, 2, 3], np.uint64), np.array([1, 5, 4], np.uint32), np.array([1, 0, 1], np.uint32), 0]


def _bad_cases():
    def mod(f):
        g = [np.array(x) if isinstance(x, np.ndarray) else x for x in _good()]
        f(g)
        return g
    def put(i, j, v):
        def f(g):
            g[i][j] = v
        return f
    return [
        ("allows no token", mod(put(0, 1, 0))),                      # state 0 empty (offsets 0, 0, 3 -> state 1 has 3)
        ("outside the vocabulary", mod(put(1, 2, 8))),
        ("strictly ascending", mod(put(1, 1, 1))),                   # duplicate in state 0
        ("strictly ascending", mod(put(1, 0, 6))),                   # unsorted in state 0
        ("next\\[1\\] = 2 is not below n_states", mod(put(2, 1, 2))),
        ("start 2 is not below n_states", mod(lambda g: g.__setitem__(3, 2))),
        ("offsets\\[0\\] must be 0", mod(put(0, 0, 1))),
        ("non-decreasing", mod(lambda g: g.__setitem__(0, np.array([0, 2, 1, 3], np.uint64)))),   # offsets[1] > offsets[2]
    ]


@pytest.mark.parametrize("i", range(8))
def test_malformed_automata_are_refused(lib_built, i):
    from aha_b200 import B200Error
    what, fsm = _bad_cases()[i]
    _check(_good(), 8)
    with pytest.raises(B200Error, match=what):
        _check(fsm, 8)


def test_null_pointers_and_no_states_are_refused(lib_built):
    import ctypes as C
    from aha_b200 import _lib as L
    lib = L.load()
    off, tok, nxt, _ = _good()
    f, _keep = L.token_fsm(off, tok, nxt, 0)
    assert lib.aha_b200_fsm_check(C.byref(f), 8) == 0
    assert lib.aha_b200_fsm_check(None, 8) == 1
    assert b"fsm is NULL" in lib.aha_b200_last_error(None)
    for field, msg in (("offsets", b"offsets is NULL"), ("tokens", b"tokens and next are required"), ("next", b"tokens and next are required")):
        g, _k = L.token_fsm(off, tok, nxt, 0)
        setattr(g, field, None)
        assert lib.aha_b200_fsm_check(C.byref(g), 8) == 1
        assert msg in lib.aha_b200_last_error(None), field
    g, _k = L.token_fsm(np.zeros(1, np.uint64), [], [], 0)
    assert lib.aha_b200_fsm_check(C.byref(g), 8) == 1
    assert b"n_states must be at least 1" in lib.aha_b200_last_error(None)


def test_regex_automaton_accepts_exactly_the_regex():
    """every token sequence of up to 3 pieces (and every sequence of up to 9 the automaton itself generates): the automaton walks it
    iff its text is a prefix of a match, and ends in the accepting state (EOS allowed) iff the text matches"""
    V, eos = 300, 7
    table = R.token_table(V, eos)
    fsm = R.regex_fsm(table, eos)
    pieces = [t for t, s in enumerate(table) if s is not None and not s.startswith("<")]
    assert len(pieces) == len(R._PIECES)

    def viable(text):   # a prefix of some match: every such prefix is completed by one of these tails
        return any(R.regex_match(text + tail) for tail in ["", "}", "0}", ":0}", '":0}', 'a":0}', '"a":0}', '{"a":0}'])

    n_match = 0
    seqs = itertools.chain.from_iterable(itertools.product(pieces, repeat=k) for k in range(1, 4))
    for seq in seqs:
        q = 0
        for t in seq:
            q = R.step(fsm, q, t)
            if q is None:
                break
        text = "".join(table[t] for t in seq)
        assert (q is not None) == viable(text), (text, q)
        if q is not None:
            accepts = R.step(fsm, q, eos) is not None
            assert accepts == R.regex_match(text), text
            n_match += accepts
    rng = np.random.default_rng(0)
    for _ in range(300):     # random walks of the automaton: always a viable prefix; a match exactly where EOS is allowed
        q, ids = 0, []
        for _ in range(int(rng.integers(1, 10))):
            a = R.allowed(fsm, q)
            t = int(a[rng.integers(len(a))])
            if t == eos:
                break
            ids.append(t)
            q = R.step(fsm, q, t)
        text = R.decode(table, ids)
        assert viable(text), text
        assert (R.step(fsm, q, eos) is not None) == R.regex_match(text), text
        n_match += R.regex_match(text)
    assert n_match > 10
    assert not R.regex_match('{"a":}') and R.regex_match('{"a":123}')
