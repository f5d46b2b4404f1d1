"""Frequency / presence penalties and logit bias restated on the host (the oracle of AHA_GEN_LOGIT_RULES), composed with the masked
generation loop of constrain_ref.

A draw takes the raw fp32 logits x through, in this order:
  1. the automaton's mask (constrain_ref.mask), when the rules name one;
  2. bias: y[t] = x[t] + bias[t], one fp32 add per listed token;
  3. the repeat penalty (constrain_ref.penalise: a -inf entry stays -inf);
  4. frequency and presence: for every t with c[t] > 0 occurrences among the tokens generated before this draw (the whole output),
     y[t] = (y[t] - fl(c[t] * frequency)) - presence, each product and difference rounded to fp32 on its own;
then the request's sampler (temperature, top-k, top-p) unchanged."""
from collections import Counter

import numpy as np

import constrain_ref as cr

F32 = np.float32


def apply_bias(x, logit_bias):
    """step 2: logit_bias = {id: value} (or (id, value) pairs)"""
    y = np.array(x, F32)
    for t, v in (logit_bias.items() if isinstance(logit_bias, dict) else (logit_bias or ())):
        y[int(t)] = F32(y[int(t)] + F32(v))
    return y


def apply_counts(x, generated, frequency, presence):
    """step 4 over the whole of `generated` (the prompt does not count)"""
    y = np.array(x, F32)
    for t, c in Counter(int(t) for t in generated).items():
        if t < len(y):
            y[t] = F32(F32(y[t] - F32(F32(c) * F32(frequency))) - F32(presence))
    return y


def transform(s, logits, generated, rules, fsm=None, state=None):
    """steps 1-4 of one draw: rules = dict(presence_penalty, frequency_penalty, logit_bias) or None"""
    x = np.asarray(logits, F32).reshape(-1)
    if fsm is not None:
        x = cr.mask(x, fsm, state)
    if rules:
        x = apply_bias(x, rules.get("logit_bias"))
    x = cr.penalise(s, x, generated)
    if rules:
        x = apply_counts(x, generated, rules.get("frequency_penalty", 0.0), rules.get("presence_penalty", 0.0))
    return x


def sample_and_push(s, logits, generated, rules, fsm=None, state=None):
    """oracle.sample.Sampler.sample_and_push with the rules -> (token, next automaton state or None)"""
    from oracle.sample import sample, sampling_mode
    x = transform(s, logits, generated, rules, fsm, state)
    tok = sample(x, s.temperature, s.top_p, s.top_k, s.rng, s.draws)
    if sampling_mode(s.temperature, s.top_p, s.top_k) != "argmax":
        s.draws += 1
    nxt = cr.step(fsm, state, tok) if fsm is not None else None
    assert fsm is None or nxt is not None, (state, tok)
    generated.append(tok)
    return tok, nxt


def generate(o, ids, data, n, rules, fsm=None, **samp):
    """constrain_ref.generate with the rules applied before every draw"""
    s = cr.sampler(**samp)
    o.clear_cache()
    toks, eos = [], o.stop_token_ids()
    q = fsm[3] if fsm is not None else None
    t, q = sample_and_push(s, o.forward_initial(np.asarray(ids).reshape(1, -1), 0, data), toks, rules, fsm, q)
    for i in range(1, n):
        t, q = sample_and_push(s, o.forward_step(np.array([[t]]), len(ids) + i - 1), toks, rules, fsm, q)
        if t in eos:
            break
    o.clear_cache()
    return toks
