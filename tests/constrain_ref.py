"""Constrained decoding restated on the host: token automata in the CSR form of aha_token_fsm, their builders, and generation
with the mask applied before the sampler (the oracle of AHA_GEN_CONSTRAINED).

An automaton is (offsets, tokens, next, start): state s allows tokens[offsets[s]:offsets[s + 1]] (strictly ascending) and next[j]
is the state after tokens[j].  A constrained draw sets every token the current state does not allow to -inf, runs the request's
sampler unchanged (the repeat penalty leaves -inf entries at -inf), and moves the state along the drawn token."""
import re

import numpy as np

F32 = np.float32


# ----------------------------------------------------------------------------------------------------------------- builders
def from_rows(rows, start=0):
    """[(allowed tokens, successor states), ...] per state -> (offsets, tokens, next, start), every row sorted by token"""
    offsets, tokens, nxt = [0], [], []
    for toks, succ in rows:
        order = np.argsort(np.asarray(toks, np.int64), kind="stable")
        tokens += [int(toks[i]) for i in order]
        nxt += [int(succ[i]) for i in order]
        offsets.append(len(tokens))
    return (np.array(offsets, np.uint64), np.array(tokens, np.uint32), np.array(nxt, np.uint32), start)


def chain(seq, end_token):
    """one allowed token per state: state i allows seq[i] and moves to i + 1; the last state loops on end_token"""
    rows = [([t], [i + 1]) for i, t in enumerate(seq)]
    rows.append(([end_token], [len(seq)]))
    return from_rows(rows)


def all_allowed(V):
    """one state that allows every token and loops on itself"""
    return (np.array([0, V], np.uint64), np.arange(V, dtype=np.uint32), np.zeros(V, np.uint32), 0)


def random_fsm(V, n_states, seed):
    """seeded random automaton: per-state allowed-set sizes from 1 to V (log-uniform, with the extremes included), random successors"""
    rng = np.random.default_rng(seed)
    rows = []
    for s in range(n_states):
        k = 1 if s == 0 else V if s == 1 else int(np.clip(np.exp(rng.uniform(0, np.log(V))), 1, V))
        toks = rng.choice(V, size=k, replace=False)
        rows.append((toks, rng.integers(0, n_states, k)))
    return from_rows(rows)


def allowed(fsm, state):
    off, tok = fsm[0], fsm[1]
    return tok[int(off[state]):int(off[state + 1])]


def step(fsm, state, token):
    """the state after `token`, or None when the state does not allow it"""
    off, tok, nxt = fsm[0], fsm[1], fsm[2]
    a, b = int(off[state]), int(off[state + 1])
    j = a + int(np.searchsorted(tok[a:b], token))
    return int(nxt[j]) if j < b and int(tok[j]) == token else None


# ----------------------------------------------------------------------------------------------------------------- regex
REGEX = r'\{"a":[0-9]+\}'
# the character DFA of REGEX: state -> {char: state}; state 7 accepts
_DFA = {0: {"{": 1}, 1: {'"': 2}, 2: {"a": 3}, 3: {'"': 4}, 4: {":": 5}, 5: {d: 6 for d in "0123456789"},
        6: dict({d: 6 for d in "0123456789"}, **{"}": 7}), 7: {}}
_ACCEPT = 7
_PIECES = ["{", '"', "a", ":", "}", '{"', 'a"', '":', '"a":', "0", "1", "2", "3", "4", "5", "6", "7", "8", "9", "12", "345", "0}", "9}",
           "}}", "b", "x", "ab", ",", " ", '"b"', "{}", "[", "a:"]


def token_table(V, eos):
    """synthetic token -> string table of V tokens: the pieces above (multi-character ones included) spread over the ids, junk elsewhere;
    `eos` maps to None"""
    rng = np.random.default_rng(V)
    table = [f"<{i}>" for i in range(V)]
    ids = [i for i in rng.permutation(V) if i != eos][:len(_PIECES)]
    for i, s in zip(ids, _PIECES):
        table[i] = s
    table[eos] = None
    return table


def walk(text, q=0):
    """the DFA state after `text` from q, or None"""
    for ch in text:
        q = _DFA[q].get(ch)
        if q is None:
            return None
    return q


def regex_fsm(table, eos):
    """the token automaton of REGEX over `table`: the DFA's states, token t allowed in q when its string walks through the DFA from q; the
    accepting state allows only eos and loops on it"""
    rows = []
    for q in range(len(_DFA)):
        if q == _ACCEPT:
            rows.append(([eos], [q]))
            continue
        toks, succ = [], []
        for t, s in enumerate(table):
            if s is None:
                continue
            r = walk(s, q)
            if r is not None:
                toks.append(t); succ.append(r)
        rows.append((toks, succ))
    return from_rows(rows)


def decode(table, ids):
    return "".join(table[t] for t in ids if table[t] is not None)


def regex_match(text):
    return re.fullmatch(REGEX, text) is not None


# ----------------------------------------------------------------------------------------------------------------- generation
def mask(logits, fsm, state):
    x = np.full(len(logits), -np.inf, F32)
    a = allowed(fsm, state)
    x[a] = np.asarray(logits, F32)[a]
    return x


def penalise(s, logits, generated):
    """use_repeat_penalty on masked logits: a -inf entry stays -inf"""
    if s.repeat_penalty == 1.0 or s.repeat_last_n == 0:
        return logits
    x = np.array(logits, F32)
    ctx = generated[max(0, len(generated) - s.repeat_last_n):]
    for t in dict.fromkeys(int(t) for t in ctx):
        if t < len(x) and x[t] != -np.inf:
            x[t] = x[t] / F32(s.repeat_penalty) if x[t] >= 0 else x[t] * F32(s.repeat_penalty)
    return x


def sample_and_push(s, logits, generated, fsm, state):
    """oracle.sample.Sampler.sample_and_push of a constrained request -> (token, next state)"""
    from oracle.sample import sample, sampling_mode
    x = penalise(s, mask(np.asarray(logits, F32).reshape(-1), fsm, state), generated)
    if not np.isfinite(x).any():
        raise ValueError("no allowed token has a finite logit")
    tok = sample(x, s.temperature, s.top_p, s.top_k, s.rng, s.draws)
    if sampling_mode(s.temperature, s.top_p, s.top_k) != "argmax":
        s.draws += 1
    nxt = step(fsm, state, tok)
    assert nxt is not None, (state, tok)
    generated.append(tok)
    return tok, nxt


def sampler(**samp):
    from oracle.sample import Sampler
    return Sampler(samp.get("temperature"), samp.get("top_p"), samp.get("top_k"), samp.get("repeat_penalty", 1.0), samp.get("repeat_last_n", 64),
                   seed=samp.get("seed", 299792458))


def generate(o, ids, data, n, fsm, **samp):
    """tests/test_prefix_cache_gpu.py::_oracle_generate with the mask before every draw and the state walk"""
    s = sampler(**samp)
    o.clear_cache()
    toks, eos = [], o.stop_token_ids()
    t, q = sample_and_push(s, o.forward_initial(np.asarray(ids).reshape(1, -1), 0, data), toks, fsm, fsm[3])
    for i in range(1, n):
        t, q = sample_and_push(s, o.forward_step(np.array([[t]]), len(ids) + i - 1), toks, fsm, q)
        if t in eos:
            break
    o.clear_cache()
    return toks
