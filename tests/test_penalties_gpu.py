"""Frequency / presence penalties and logit bias (AHA_GEN_LOGIT_RULES): every draw takes the logits through the automaton's mask, the
bias, the repeat penalty and the penalties over the tokens generated so far.  Checked against tests/penalty_ref.py: the sampler kernels
row by row, then every generation path end to end."""
from collections import Counter

import numpy as np
import pytest

import constrain_ref as R
import penalty_ref as P
from conftest import make_model, make_oracle
from test_constrain_gpu import MODES, SAMPLERS, _ids, _Session, _every_path

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tiny():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=1024)
    yield cfg, w, m
    m.close()


# ---------------------------------------------------------------------------------------------------------------- the kernels
def _rules_cases(V, rng):
    few = rng.choice(V, size=min(V, 40), replace=False)
    return [
        dict(presence_penalty=0.5, frequency_penalty=0.5, logit_bias={int(t): float(rng.uniform(-3, 3)) for t in few}),
        dict(presence_penalty=-2.0, frequency_penalty=2.0, logit_bias={int(few[0]): 100.0}),
        dict(presence_penalty=1.5, frequency_penalty=-0.75, logit_bias={int(t): -100.0 for t in few[:10]}),
        dict(frequency_penalty=0.3),
    ]


@pytest.mark.parametrize("V", [257, 151936])
@pytest.mark.parametrize("with_fsm", [False, True])
def test_kernels_against_the_oracle(tiny, V, with_fsm):
    """both kernels, every mode, with and without repeat penalty and automaton; token, state and automaton state bit for bit, twice"""
    m = tiny[2]
    rng = np.random.default_rng(V + with_fsm)
    logits = (rng.standard_normal(V) * 3).astype(np.float32)
    fsm = None
    if with_fsm:
        big = np.unique(rng.choice(V, size=V // 2, replace=False))
        fsm = R.from_rows([(big, [1] * big.size), (np.arange(V), [0] * V)])
    for ci, rules in enumerate(_rules_cases(V, rng)):
        rows = []
        for k, mode in enumerate(MODES):
            hot = rng.choice(V, size=6, replace=False)
            ctx = rng.choice(hot, size=[0, 1, 40, 300][k % 4]).astype(np.uint32)       # many repeats of a few tokens
            rows.append((dict(mode, seed=11 + k), ctx, [0, 15, 16, 0xFFFFFFFF][(k + ci) % 4], k % 2))
        want = []
        for p, ctx, draw, q in rows:
            s = R.sampler(**p)
            s.draws = draw
            want.append(P.sample_and_push(s, logits, list(int(t) for t in ctx), rules, fsm, q if fsm else None))
        for kernel in (0, 1):
            params = [p for p, _, _, _ in rows] + [dict(temperature=0.9, top_k=7, seed=5)]
            ctxs = [c for _, c, _, _ in rows] + [rows[2][1]]
            draws = [d for _, _, d, _ in rows] + [3]
            states = [q for _, _, _, q in rows] + [0]
            ruled = [True] * len(rows) + [False]          # a row without rules beside them draws what it draws alone
            act = list(reversed(range(len(params)))) if kernel == 1 else None
            kw = dict(kernel=kernel, act=act, rules=rules, ruled=ruled)
            if fsm is not None:
                kw.update(fsm=fsm[:3], constrained=[True] * len(rows) + [False], fsm_states=states)
            got = m.debug_sample_rows(logits, params, ctxs, draws, **kw)
            again = m.debug_sample_rows(logits, params, ctxs, draws, **kw)
            for key in got:
                assert np.array_equal(got[key], again[key]), key
            for r in range(len(rows)):
                tok = int(got["token"][r])
                assert tok == want[r][0], (kernel, ci, r, params[r])
                if fsm is not None:
                    assert int(got["fsm_state"][r]) == want[r][1]
                assert int(got["n_draws"][r]) == (draws[r] + (1 if params[r].get("temperature") else 0)) & 0xFFFFFFFF
            alone = m.debug_sample_rows(logits, params[-1:], ctxs[-1:], draws[-1:])
            assert int(got["token"][-1]) == int(alone["token"][0])


def test_kernel_refusals(tiny):
    from aha_b200 import B200Error
    m = tiny[2]
    lg = np.zeros(16, np.float32)
    with pytest.raises(B200Error, match="listed twice"):
        m.debug_sample_rows(lg, [dict(temperature=1.0)], rules=dict(logit_bias=[(1, 1.0), (1, 2.0)]))
    with pytest.raises(B200Error, match="outside the vocabulary"):
        m.debug_sample_rows(lg, [dict(temperature=1.0)], rules=dict(logit_bias={16: 1.0}))
    with pytest.raises(B200Error, match="passed as fsm"):
        m.debug_sample_rows(lg, [dict(temperature=1.0)], rules=dict(fsm=3))
    assert m.debug_sample_rows(lg, [dict()], rules=dict(logit_bias={9: 1.0}))["token"][0] == 9


# ---------------------------------------------------------------------------------------------------------------- every path
RULES = [dict(presence_penalty=0.8, frequency_penalty=0.6), dict(frequency_penalty=1.5, logit_bias={7: 2.0, 11: -3.5, 13: 0.25}),
         dict(presence_penalty=-0.5, frequency_penalty=0.25, logit_bias={3: 5.0}), dict(presence_penalty=2.0)]


def _want(o, r, rules_by_id):
    kw = {k: v for k, v in r.items() if k not in ("input_ids", "max_tokens", "rules")}
    return P.generate(o, r["input_ids"], None, r["max_tokens"], rules_by_id.get(r.get("rules")), **kw)


def _margin(o, r, rules_by_id, k):
    """distance of the oracle's k-th draw from a decision boundary (test_constrain_gpu._margin with the rules' transform)"""
    from oracle.sample import softmax_blocked
    kw = {key: v for key, v in r.items() if key not in ("input_ids", "max_tokens", "rules")}
    rules = rules_by_id.get(r.get("rules"))
    s = R.sampler(**kw)
    o.clear_cache()
    toks = []
    lg = o.forward_initial(np.asarray(r["input_ids"]).reshape(1, -1), 0)
    for i in range(k):
        t, _ = P.sample_and_push(s, lg, toks, rules)
        lg = o.forward_step(np.array([[t]]), len(r["input_ids"]) + i)
    x = P.transform(s, lg, toks, rules)
    if not kw.get("temperature"):
        a, b = np.sort(x)[-2:]
        return float(b - a)
    p = softmax_blocked(x, s.temperature).astype(np.float64)
    if kw.get("top_p") or kw.get("top_k"):
        return float(np.abs(np.cumsum(np.sort(p)[::-1]) - (kw.get("top_p") or 1.0)).min())
    cum = np.cumsum(p)
    return float(np.abs(cum - s.rng.uniform01(s.draws) * cum[-1]).min() / cum[-1])


def _check_oracle(o, reqs, got, rules_by_id, exact):
    """every request's ids equal the oracle loop's; without `exact` one may part from it at a draw the oracle takes within 5e-5 of a
    decision boundary (the wide step's fp32 sums run in another order than numpy's)"""
    near = 0
    for i, r in enumerate(reqs):
        want = _want(o, r, rules_by_id)
        if got[i] != want:
            k = next(j for j in range(min(len(want), len(got[i]))) if got[i][j] != want[j])
            assert not exact and _margin(o, r, rules_by_id, k) < 5e-5, (i, k, got[i], want)
            near += 1
    assert near <= 1


def _case(cfg, m, seed, n_req, budget):
    V = cfg["vocab_size"]
    rules_by_id = {m.rules_create(**x): x for x in RULES}
    ids = list(rules_by_id)
    reqs = []
    for i in range(n_req):
        r = dict(input_ids=_ids(5 + 11 * i, V, seed * 100 + i), max_tokens=budget, **SAMPLERS[i % len(SAMPLERS)])
        if i % 4 != 3:
            r["rules"] = ids[i % len(ids)]
        reqs.append(r)
    return rules_by_id, reqs


def test_every_path_reproduces_the_oracle(tiny):
    """single requests give the oracle loop's ids (within the tolerance of tests/test_constrain_gpu.py), and the streaming, static-batch,
    n-choice and narrow-session paths give exactly the single request's ids; a wide session gives the oracle's within the same tolerance"""
    cfg, w, m = tiny
    o = make_oracle("qwen3", cfg, w)
    rules_by_id, reqs = _case(cfg, m, 1, 8, 20)
    try:
        single = [m.generate(**r)[0] for r in reqs]
        _check_oracle(o, reqs, single, rules_by_id, exact=False)
        for r, want in zip(reqs, single):
            for path, ids in _every_path(m, r).items():
                if not path.startswith("wide"):
                    assert ids == want, (path, r.get("rules"), ids, want)
                elif ids != want:
                    _check_oracle(o, [r], [ids], rules_by_id, exact=False)
        # mixed samplers, seeds and rules per slot, admission mid-flight
        for wide in (0, 16):
            s = _Session(m, wide)
            s.add(0, reqs[0])
            s.step(3)
            s.add_many([(i, reqs[i]) for i in range(1, 6)])
            s.step(2)
            s.add_n([6, 7], dict(reqs[6], seeds=[reqs[6].get("seed", 299792458), reqs[7].get("seed", 299792458)]))
            out = s.drain()
            got = [out[i] for i in range(8)]
            reqs_n = reqs[:7] + [dict(reqs[6], seed=reqs[7].get("seed", 299792458))]
            if wide:
                _check_oracle(o, reqs_n, got, rules_by_id, exact=False)
            else:
                assert got == single[:7] + [m.generate(**reqs_n[7])[0]]
    finally:
        for i in rules_by_id:
            m.rules_destroy(i)


def test_reuse_prefix_second_turn(tiny):
    cfg, _, m = tiny
    V = cfg["vocab_size"]
    rid = m.rules_create(presence_penalty=0.7, frequency_penalty=0.4, logit_bias={5: 1.0})
    try:
        p1 = _ids(40, V, 1)
        out1 = m.generate(p1, max_tokens=10, temperature=0.8, seed=2, rules=rid, reuse_prefix=True)[0]
        p2 = np.concatenate([p1, out1[:-1], _ids(7, V, 3)])
        warm = m.generate(p2, max_tokens=12, temperature=0.8, seed=4, rules=rid, reuse_prefix=True)[0]
        assert m.last_prefix_hit() > 0
        m.clear_cache()
        assert warm == m.generate(p2, max_tokens=12, temperature=0.8, seed=4, rules=rid)[0]
    finally:
        m.rules_destroy(rid)


# ---------------------------------------------------------------------------------------------------------------- behaviour
def test_bias_forces_and_bans(tiny):
    cfg, _, m = tiny
    V = cfg["vocab_size"]
    r = dict(input_ids=_ids(20, V, 3), max_tokens=16)
    base = m.generate(**r)[0]
    t = next(t for t in range(42, V) if t not in m.stop_token_ids())
    force = m.rules_create(logit_bias={str(t): 100})
    ban = m.rules_create(logit_bias={base[0]: -100})
    try:
        assert m.generate(rules=force, **r)[0] == [t] * 16
        assert base[0] not in m.generate(rules=ban, **r)[0]
    finally:
        m.rules_destroy(force)
        m.rules_destroy(ban)


def test_frequency_penalty_breaks_a_repetition_loop(tiny):
    cfg, _, m = tiny
    V = cfg["vocab_size"]
    r = dict(input_ids=_ids(16, V, 0), max_tokens=64)
    base = m.generate(**r)[0]
    top = max(Counter(base).values())
    assert top >= 4, base                      # the greedy run repeats itself
    rid = m.rules_create(frequency_penalty=2.0, presence_penalty=2.0)
    try:
        pen = m.generate(rules=rid, **r)[0]
    finally:
        m.rules_destroy(rid)
    assert max(Counter(pen).values()) < top and len(set(pen)) > len(set(base))


def test_zero_rules_change_nothing_and_records_stay_raw(tiny):
    cfg, _, m = tiny
    V = cfg["vocab_size"]
    zero = m.rules_create()
    zero_b = m.rules_create(presence_penalty=0.0, frequency_penalty=-0.0)
    try:
        for samp in SAMPLERS:
            r = dict(input_ids=_ids(30, V, 9), max_tokens=24, **samp)
            assert _every_path(m, dict(r, rules=zero)) == _every_path(m, r), samp
            a = m.generate(logprobs=True, top_logprobs=5, rules=zero_b, **r)
            b = m.generate(logprobs=True, top_logprobs=5, **r)
            assert a[0] == b[0] and a[2] == b[2]
            a = m.generate_n(n=2, logprobs=True, top_logprobs=3, rules=zero, **r)
            b = m.generate_n(n=2, logprobs=True, top_logprobs=3, **r)
            assert [(x[0], x[2]) for x in a] == [(x[0], x[2]) for x in b]
    finally:
        m.rules_destroy(zero)
        m.rules_destroy(zero_b)
    # non-zero rules and a chain automaton along the greedy ids: a sampled request carries the greedy request's records bit for bit
    r = dict(input_ids=_ids(25, V, 4), max_tokens=16)
    ids, _, recs = m.generate(logprobs=True, top_logprobs=4, **r)
    f = m.fsm_create(*R.chain(ids, cfg["eos_token_id"]))
    others = [t for t in range(V) if t not in ids][:50]
    rid = m.rules_create(presence_penalty=1.0, frequency_penalty=0.5, logit_bias={t: 3.0 for t in others}, fsm=f)
    try:
        got, _, got_recs = m.generate(logprobs=True, top_logprobs=4, rules=rid, temperature=1.3, seed=8, **r)
        assert got == ids and got_recs == recs
        s = _Session(m, 8)
        s.add("a", dict(r, rules=rid, temperature=1.3, seed=8, logprobs=True, top_logprobs=4))
        assert m.batch_logprobs()[0] == recs[0]
        assert s.drain()["a"] == ids
    finally:
        m.rules_destroy(rid)
        m.fsm_destroy(f)


def test_no_cost_to_requests_without_rules():
    """a request or session without rules launches the same kernels and keeps the same graphs whether or not the handle has served rules"""
    cfg, _, m = make_model("qwen3", "tiny", max_ctx=1024)
    try:
        V = cfg["vocab_size"]
        r = dict(input_ids=_ids(20, V, 5), max_tokens=24)

        def measure():
            k0 = m.stats()["kernel_launches"]
            a = m.generate(**r)[0]
            k1 = m.stats()["kernel_launches"]
            b = m.generate(temperature=0.8, seed=3, **r)[0]
            k2 = m.stats()["kernel_launches"]
            step = m.stats()["kernels_per_decode_step"]
            s = _Session(m, 16)
            s.add_many([(0, r), (1, dict(r, temperature=0.8, seed=3))])
            s.step(5)
            graphs = int(m.debug_read("batch_graphs", 0, 1)[0])
            k3 = m.stats()["kernel_launches"]
            s.drain()
            return (a, b, s.out), (k1 - k0, k2 - k1, step, graphs, k3)

        measure()        # first use: step graphs captured
        before = measure()
        rid = m.rules_create(presence_penalty=0.5, frequency_penalty=0.5, logit_bias={1: 1.0})
        m.generate(rules=rid, **r)
        s = _Session(m, 16)
        s.add("x", dict(r, rules=rid))
        s.drain()
        m.rules_destroy(rid)
        after = measure()
        assert after[0] == before[0]
        assert after[1][:4] == before[1][:4]
    finally:
        m.close()


# ---------------------------------------------------------------------------------------------------------------- speculative decoding
def test_speculative_decoding(tiny):
    """with rules, the ids do not depend on the drafts, and they are the oracle loop's within the wide step's tolerance"""
    from aha_b200 import B200Error
    cfg, w, m = tiny
    o = make_oracle("qwen3", cfg, w)
    V = cfg["vocab_size"]
    spec = dict(presence_penalty=0.6, frequency_penalty=0.9, logit_bias={4: 1.5, 8: -2.0})
    rid = m.rules_create(**spec)
    f = m.fsm_create(*R.all_allowed(V))
    rf = m.rules_create(frequency_penalty=0.5, fsm=f)
    try:
        for samp in (dict(), dict(temperature=0.8, seed=6), dict(temperature=0.9, top_k=20, repeat_penalty=1.2, repeat_last_n=16, seed=4)):
            r = dict(input_ids=_ids(24, V, 2), max_tokens=40, rules=rid, **samp)
            want = m.generate_speculative(max_draft=7, **r)[0]
            _check_oracle(o, [r], [want], {rid: spec}, exact=False)
            assert m.generate_speculative(prediction=want, max_draft=7, **r)[0] == want
            for d in (1, 15):
                assert m.generate_speculative(prediction=want, max_draft=d, **r)[0] == want
                assert m.generate_speculative(prompt_lookup=True, max_draft=d, **r)[0] == want
        with pytest.raises(B200Error, match="name a token automaton are not supported with speculative decoding"):
            m.generate_speculative(prompt_lookup=True, input_ids=_ids(12, V, 5), max_tokens=6, rules=rf)
        r = dict(input_ids=_ids(12, V, 5), max_tokens=6)
        assert m.generate_speculative(prompt_lookup=True, **r)[0] == m.generate_speculative(**r)[0]
    finally:
        m.rules_destroy(rf)
        m.rules_destroy(rid)
        m.fsm_destroy(f)


# ---------------------------------------------------------------------------------------------------------------- refusals
def test_refusals_leave_the_handle_and_session_usable(tiny):
    from aha_b200 import B200Error, B200Model
    from aha_b200 import _lib as L
    cfg, _, m = tiny
    V = cfg["vocab_size"]
    r = dict(input_ids=_ids(12, V, 5), max_tokens=6)
    want = m.generate(**r)[0]
    with pytest.raises(B200Error, match="no logit-rules object has id 999"):
        m.generate(rules=999, **r)
    with pytest.raises(B200Error, match="no token automaton has id 999"):
        m.rules_create(fsm=999)
    with pytest.raises(B200Error, match="listed twice"):
        m.rules_create(logit_bias=[(1, 1.0), (1, 1.0)])
    f = m.fsm_create(*R.all_allowed(V))
    rid = m.rules_create(frequency_penalty=0.5, fsm=f)
    with pytest.raises(B200Error, match="exclude each other"):
        m.generate(rules=rid, flags=L.GEN_CONSTRAINED, **r)
    with pytest.raises(B200Error, match=f"named by logit-rules object {rid}"):
        m.fsm_destroy(f)
    s = _Session(m)
    s.add("a", dict(r, max_tokens=10, rules=rid))
    with pytest.raises(B200Error, match="no logit-rules object has id 999"):
        m.batch_add_many([dict(r), dict(r, rules=999)])
    with pytest.raises(B200Error, match=f"applies to the running request in slot 0"):
        m.rules_destroy(rid)
    s.add("b", dict(r))
    out = s.drain()
    assert out["b"] == want
    m.rules_destroy(rid)
    m.fsm_destroy(f)
    with pytest.raises(B200Error, match=f"no logit-rules object has id {rid}"):
        m.generate(rules=rid, **r)
    with pytest.raises(B200Error, match=f"no logit-rules object has id {rid}"):
        m.rules_destroy(rid)
    with pytest.raises(B200Error, match="no logit-rules object has id 999"):
        m.generate_n(n=2, rules=999, **r)
    assert m.generate(**r)[0] == want
    cfg_a, _, a = make_model("qwen3_asr", "tiny", max_ctx=512)
    try:
        a._gen_params = lambda *args: B200Model._gen_params(*args, rules=1)
        with pytest.raises(B200Error, match="asr_generate: AHA_GEN_LOGIT_RULES"):
            a.asr_generate([(np.array([1, 2, 3], np.uint32), np.zeros((128, 100), np.float32))], max_tokens=4)
    finally:
        a.close()
