"""Constrained decoding (AHA_GEN_CONSTRAINED): every token is drawn from the tokens the request's token automaton allows in its current
state, and the state follows the drawn token.  Checked against the masked oracle of tests/constrain_ref.py: the sampler kernels row by row,
then every generation path end to end."""
import numpy as np
import pytest

import constrain_ref as R
from conftest import make_model, make_oracle

pytestmark = pytest.mark.gpu


def _ids(n, vocab, seed):
    from aha_b200 import synth
    return synth.synth_text_ids(n, vocab - 8, seed)


# ---------------------------------------------------------------------------------------------------------------- the kernels

MODES = [dict(), dict(repeat_penalty=1.3, repeat_last_n=64), dict(temperature=0.8), dict(temperature=0.9, top_k=5),
         dict(temperature=0.7, top_p=0.8, repeat_penalty=0.5, repeat_last_n=4), dict(temperature=1.1, top_k=40, top_p=0.9),
         dict(temperature=0.6, top_k=1000, top_p=1.0, repeat_penalty=3.0, repeat_last_n=64), dict(temperature=1.0, top_p=0.3)]


def _masks(V, logits, rng):
    """one allowed token; a few that exclude the unmasked argmax; sets straddling the 256-entry chunk edges; all but one"""
    am = int(np.argmax(logits))
    others = np.setdiff1d(np.arange(V), [am])
    out = [np.array([int(rng.integers(V))])]
    if V > 1:
        out.append(rng.choice(others, size=min(5, others.size), replace=False))
        out.append(np.setdiff1d(np.arange(V), [am]))
    edge = np.concatenate([np.arange(e - 3, min(e + 3, V)) for e in (256, 512, 4096) if e < V] + [np.zeros(0, int)])
    if edge.size:
        out.append(edge)
    return [np.unique(m) for m in out]


@pytest.fixture(scope="module")
def tiny():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=1024)
    yield cfg, w, m
    m.close()


@pytest.mark.parametrize("V", [1, 257, 4097, 151936])
def test_kernels_against_the_masked_oracle(tiny, V):
    m = tiny[2]
    rng = np.random.default_rng(V)
    logits = (rng.standard_normal(V) * 3).astype(np.float32)
    masks = _masks(V, logits, rng)
    n = len(masks)
    fsm = R.from_rows([(mk, [(i + 1 + j) % n for j in range(mk.size)]) for i, mk in enumerate(masks)])
    rows = []
    for i, mk in enumerate(masks):
        forbidden = np.setdiff1d(np.arange(min(V, 600)), mk)[:3]
        for k, mode in enumerate(MODES):
            ctx = np.concatenate([mk[:2], forbidden, mk[-1:]]).astype(np.uint32) if k not in (0, 2) else np.zeros(0, np.uint32)
            rows.append((i, dict(mode, seed=77 + k), ctx, [0, 15, 16, 17, 0xFFFFFFFF][(i + k) % 5]))
    want = []
    for q, p, ctx, draw in rows:
        s = R.sampler(**p)
        s.draws = draw
        want.append(R.sample_and_push(s, logits, list(ctx), fsm, q))
    for kernel in (0, 1):
        for a in range(0, len(rows), 63):
            chunk = rows[a:a + 63]
            params = [p for _, p, _, _ in chunk]
            ctxs = [c for _, _, c, _ in chunk]
            draws = [d for _, _, _, d in chunk]
            states = [q for q, _, _, _ in chunk]
            if kernel == 1:    # an unconstrained row in the same launch draws what it draws alone
                params.append(dict(temperature=0.9, top_k=7, seed=5))
                ctxs.append(np.zeros(0, np.uint32)); draws.append(3); states.append(0)
            act = list(reversed(range(len(params)))) if kernel == 1 else None
            con = [True] * len(chunk) + [False] * (len(params) - len(chunk))
            got = m.debug_sample_rows(logits, params, ctxs, draws, kernel=kernel, act=act, fsm=fsm[:3], constrained=con, fsm_states=states)
            for r in range(len(chunk)):
                assert (int(got["token"][r]), int(got["fsm_state"][r])) == want[a + r], (kernel, a + r, rows[a + r][:2])
                assert int(got["n_draws"][r]) == draws[r] + (1 if params[r].get("temperature") else 0) & 0xFFFFFFFF
            if kernel == 1:
                alone = m.debug_sample_rows(logits, params[-1:], ctxs[-1:], draws[-1:], kernel=1)
                assert int(got["token"][-1]) == int(alone["token"][0]) and int(got["fsm_state"][-1]) == 0


def test_kernel_refusals(tiny):
    from aha_b200 import B200Error
    m = tiny[2]
    V = 300
    logits = np.zeros(V, np.float32)
    logits[10:] = -np.inf
    fsm = R.from_rows([(np.arange(20, 30), np.zeros(10, int))])
    for mode in (dict(), dict(temperature=0.8), dict(temperature=0.8, top_k=3), dict(temperature=0.8, top_p=0.5)):
        with pytest.raises(B200Error, match="all zero or not finite"):    # no allowed token has a finite logit
            m.debug_sample_rows(logits, [mode], fsm=fsm[:3])
    with pytest.raises(B200Error, match="outside the vocabulary"):
        m.debug_sample_rows(np.zeros(20, np.float32), [{}], fsm=fsm[:3])
    with pytest.raises(B200Error, match="fsm_state_in"):
        m.debug_sample_rows(np.zeros(V, np.float32), [{}], fsm=fsm[:3], fsm_states=[1])
    got = m.debug_sample_rows(np.zeros(V, np.float32), [{}], fsm=fsm[:3])     # the handle is still usable
    assert int(got["token"][0]) == 20 and int(got["fsm_state"][0]) == 0


# ---------------------------------------------------------------------------------------------------------------- end to end

SAMPLERS = [{}, dict(temperature=0.8, seed=3), dict(temperature=0.9, top_k=20, repeat_penalty=1.2, repeat_last_n=16, seed=4),
            dict(temperature=0.7, top_p=0.85, repeat_penalty=1.1, repeat_last_n=8, seed=5)]


class _Session:
    def __init__(self, m, wide=0):
        self.m, self.out, self.running, self.counts = m, {}, {}, set()
        m.batch_open_wide(wide) if wide else m.batch_open()

    def admitted(self, name, slot, tok, fin):
        self.out[name] = [tok]
        if not fin:
            self.running[slot] = name

    def add(self, name, r):
        self.admitted(name, *self.m.batch_add(**r))

    def add_many(self, named):
        for (name, _), res in zip(named, self.m.batch_add_many([r for _, r in named])):
            self.admitted(name, *res)

    def add_n(self, names, r):
        for name, res in zip(names, self.m.batch_add_n(n=len(names), **r)):
            self.admitted(name, *res)

    def step(self, n=1):
        for _ in range(n):
            if self.running:
                self.counts.add(len(self.running))
            for slot, (tok, fin) in self.m.batch_step().items():
                self.out[self.running[slot]].append(tok)
                if fin:
                    del self.running[slot]

    def drain(self):
        while self.running:
            self.step()
        self.m.batch_close()
        return self.out


def _stream(m, r):
    got = []
    m.generate_stream(on_token=lambda t, i: got.append(t) and False, **r)
    return got


def _every_path(m, r, n_choices=2):
    """{path: ids} of request r through every entry that accepts a constraint"""
    out = dict(generate=m.generate(**r)[0], stream=_stream(m, r))
    out["generate_batch"] = m.generate_batch([r, dict(r, seed=r.get("seed", 299792458))])[0][0]
    out["generate_n"] = m.generate_n(n=n_choices, seeds=[r.get("seed", 299792458)] * n_choices, **r)[0][0]
    for wide in (0, 16):
        s = _Session(m, wide)
        s.add("add", r)
        s.add_many([("many0", r), ("many1", dict(r))])
        s.add_n(["n0", "n1"], dict(r, seeds=[r.get("seed", 299792458)] * 2))
        for name, ids in s.drain().items():
            out[f"{'wide' if wide else 'narrow'}_{name}"] = ids
    return out


@pytest.mark.parametrize("k", range(len(SAMPLERS)))
def test_chain_is_reproduced_on_every_path(tiny, k):
    cfg, _, m = tiny
    V = cfg["vocab_size"]
    seq = [int(t) for t in np.random.default_rng(k).choice(V - 1, 12, replace=False)]
    f = m.fsm_create(*R.chain(seq, cfg["eos_token_id"]))
    try:
        for path, ids in _every_path(m, dict(input_ids=_ids(20, V, k), max_tokens=len(seq), fsm=f, **SAMPLERS[k])).items():
            assert ids == seq, path
    finally:
        m.fsm_destroy(f)


def test_all_allowed_changes_nothing(tiny):
    """ids and records identical to the unconstrained run on every path, greedy included"""
    cfg, _, m = tiny
    V = cfg["vocab_size"]
    f = m.fsm_create(*R.all_allowed(V))
    try:
        for samp in SAMPLERS:
            r = dict(input_ids=_ids(30, V, 9), max_tokens=24, **samp)
            assert _every_path(m, dict(r, fsm=f)) == _every_path(m, r), samp
            a = m.generate(logprobs=True, top_logprobs=5, fsm=f, **r)
            b = m.generate(logprobs=True, top_logprobs=5, **r)
            assert a[0] == b[0] and a[2] == b[2]
            a = m.generate_n(n=2, logprobs=True, top_logprobs=3, fsm=f, **r)
            b = m.generate_n(n=2, logprobs=True, top_logprobs=3, **r)
            assert [(x[0], x[2]) for x in a] == [(x[0], x[2]) for x in b]
    finally:
        m.fsm_destroy(f)


def test_records_stay_raw(tiny):
    """a sampled request forced along the greedy ids carries the greedy request's records bit for bit"""
    cfg, _, m = tiny
    V = cfg["vocab_size"]
    r = dict(input_ids=_ids(25, V, 4), max_tokens=16)
    ids, _, recs = m.generate(logprobs=True, top_logprobs=4, **r)
    f = m.fsm_create(*R.chain(ids, cfg["eos_token_id"]))
    try:
        got, _, got_recs = m.generate(logprobs=True, top_logprobs=4, fsm=f, temperature=1.3, seed=8, **r)
        assert got == ids and got_recs == recs
        s = _Session(m, 8)
        s.add("a", dict(r, fsm=f, temperature=1.3, seed=8, logprobs=True, top_logprobs=4))
        assert m.batch_logprobs()[0] == recs[0]
        s.drain()
    finally:
        m.fsm_destroy(f)


def _random_case(cfg, m, seed, n_req, budget):
    V = cfg["vocab_size"]
    fsms = [R.random_fsm(V, 6, seed * 10 + i) for i in range(2)]
    ids = [m.fsm_create(*f) for f in fsms]
    reqs = []
    for i in range(n_req):
        r = dict(input_ids=_ids(5 + 13 * i, V, seed * 100 + i), max_tokens=budget, **SAMPLERS[i % len(SAMPLERS)])
        if i % 3 != 2:
            r["fsm"] = ids[i % 2]
        reqs.append(r)
    return fsms, ids, reqs


def _want(o, fsms, ids, r):
    kw = {k: v for k, v in r.items() if k not in ("input_ids", "max_tokens", "fsm")}
    if "fsm" not in r:
        from test_prefix_cache_gpu import _oracle_generate
        return _oracle_generate(o, r["input_ids"], None, r["max_tokens"], **kw)
    return R.generate(o, r["input_ids"], None, r["max_tokens"], fsms[ids.index(r["fsm"])], **kw)


@pytest.mark.parametrize("preset,n_req,budget", [("tiny", 6, 24), ("mid", 3, 6)])
def test_random_automata_single_and_narrow(preset, n_req, budget):
    """single requests give the oracle's masked ids, and a narrow session (requests joining mid-flight, constrained beside unconstrained)
    gives every request exactly its single-request ids; the session keeps at most one step graph per running count"""
    cfg, w, m = make_model("qwen3", preset, max_ctx=2048)
    o = make_oracle("qwen3", cfg, w)
    try:
        fsms, ids, reqs = _random_case(cfg, m, 1, n_req, budget)
        want = [m.generate(**r)[0] for r in reqs]
        _check_oracle(o, fsms, ids, reqs, want, cfg["vocab_size"])
        s = _Session(m)
        s.add(0, reqs[0])
        s.step(3)
        s.add_many([(i, reqs[i]) for i in range(1, n_req - 1)])
        s.step(2)
        s.add(n_req - 1, reqs[-1])
        while s.running:
            s.step()
            assert int(m.debug_read("batch_graphs", 0, 1)[0]) <= len(s.counts)
        assert [s.drain()[i] for i in range(n_req)] == want
    finally:
        m.close()


@pytest.mark.parametrize("preset,n_req,budget", [("tiny", 12, 24), ("mid", 3, 6)])
def test_random_automata_wide(preset, n_req, budget):
    """a wide session gives the oracle's ids (its own fp32 sums: a departure only at a draw the oracle takes within 5e-5 of a boundary)"""
    cfg, w, m = make_model("qwen3", preset, max_ctx=2048)
    o = make_oracle("qwen3", cfg, w)
    try:
        fsms, ids, reqs = _random_case(cfg, m, 2, n_req, budget)
        s = _Session(m, 16)
        s.add_many([(i, reqs[i]) for i in range(n_req // 2)])
        s.step(2)
        for i in range(n_req // 2, n_req):
            s.add(i, reqs[i])
        out = s.drain()
        _check_oracle(o, fsms, ids, reqs, [out[i] for i in range(n_req)], cfg["vocab_size"])
    finally:
        m.close()


def _check_oracle(o, fsms, ids, reqs, got, V):
    """every request's ids equal the masked oracle's; one may part from it at a draw the oracle takes within 5e-5 of a decision boundary
    (the GPU's fp32 sums run in another order than numpy's, so the logits differ in their last bits)"""
    near = 0
    for i, r in enumerate(reqs):
        want = _want(o, fsms, ids, r)
        if got[i] != want:
            k = next(j for j in range(min(len(want), len(got[i]))) if got[i][j] != want[j])
            assert _margin(o, fsms, ids, r, k, V) < 5e-5, (i, k)
            near += 1
    assert near <= 1


def _margin(o, fsms, ids, r, k, V):
    """distance of the oracle's k-th draw from a decision boundary: the gap between the two largest allowed logits (greedy) or the distance of
    the draw from the nearest cumulative weight over the masked distribution, relative to the total"""
    from oracle.sample import softmax_blocked
    kw = {key: v for key, v in r.items() if key not in ("input_ids", "max_tokens", "fsm")}
    fsm = fsms[ids.index(r["fsm"])] if "fsm" in r else R.all_allowed(V)
    s = R.sampler(**kw)
    o.clear_cache()
    toks, q = [], fsm[3]
    lg = o.forward_initial(np.asarray(r["input_ids"]).reshape(1, -1), 0)
    for i in range(k):
        t, q = R.sample_and_push(s, lg, toks, fsm, q)
        lg = o.forward_step(np.array([[t]]), len(r["input_ids"]) + i)
    x = R.penalise(s, R.mask(lg.reshape(-1), fsm, q), toks)
    if not kw.get("temperature"):
        a, b = np.sort(x)[-2:]
        return float(b - a)
    p = softmax_blocked(x, s.temperature).astype(np.float64)
    if kw.get("top_p") or kw.get("top_k"):
        return float(np.abs(np.cumsum(np.sort(p)[::-1]) - (kw.get("top_p") or 1.0)).min())   # which tokens enter the nucleus / top-k
    cum = np.cumsum(p)
    return float(np.abs(cum - s.rng.uniform01(s.draws) * cum[-1]).min() / cum[-1])


def test_regex_output_matches(tiny):
    cfg, _, m = tiny
    V, eos = cfg["vocab_size"], cfg["eos_token_id"]
    table = R.token_table(V, eos)
    f = m.fsm_create(*R.regex_fsm(table, eos))
    try:
        ended = 0
        for seed in range(12):
            ids = m.generate(_ids(10, V, seed), max_tokens=40, temperature=1.0, seed=seed, fsm=f)[0]
            if ids[-1] == eos:
                ended += 1
                assert R.regex_match(R.decode(table, ids[:-1])), R.decode(table, ids)
        assert ended >= 1
    finally:
        m.fsm_destroy(f)


def test_reuse_prefix_second_turn(tiny):
    cfg, _, m = tiny
    V = cfg["vocab_size"]
    f = m.fsm_create(*R.random_fsm(V, 5, 77))
    try:
        p1 = _ids(40, V, 1)
        out1 = m.generate(p1, max_tokens=10, temperature=0.8, seed=2, fsm=f, reuse_prefix=True)[0]
        p2 = np.concatenate([p1, out1[:-1], _ids(7, V, 3)])
        warm = m.generate(p2, max_tokens=12, temperature=0.8, seed=4, fsm=f, reuse_prefix=True)[0]
        assert m.last_prefix_hit() > 0
        m.clear_cache()
        cold = m.generate(p2, max_tokens=12, temperature=0.8, seed=4, fsm=f)[0]
        assert warm == cold
    finally:
        m.fsm_destroy(f)


def test_refusals_leave_the_handle_usable(tiny):
    from aha_b200 import B200Error, B200Model
    cfg, _, m = tiny
    V = cfg["vocab_size"]
    r = dict(input_ids=_ids(12, V, 5), max_tokens=6)
    f = m.fsm_create(*R.all_allowed(V))
    want = m.generate(**r)[0]
    with pytest.raises(B200Error, match="AHA_GEN_CONSTRAINED is not supported with speculative decoding"):
        m.generate_speculative(prompt_lookup=True, flags=16, **r)
    with pytest.raises(B200Error, match="no token automaton has id 999"):
        m.generate(fsm=999, **r)
    with pytest.raises(B200Error, match="no token automaton has id 999"):
        m.batch_open_wide(4)
        try:
            m.batch_add_many([dict(r), dict(r, fsm=999)])
        finally:
            m.batch_close()
    with pytest.raises(B200Error, match="no token automaton has id 999"):
        m.generate_n(n=2, fsm=999, **r)
    m.fsm_destroy(f)
    with pytest.raises(B200Error, match=f"no token automaton has id {f}"):
        m.generate(fsm=f, **r)
    with pytest.raises(B200Error, match=f"no token automaton has id {f}"):
        m.fsm_destroy(f)
    assert m.generate(**r)[0] == want
    cfg_a, _, a = make_model("qwen3_asr", "tiny", max_ctx=512)
    try:
        a._gen_params = lambda *args: B200Model._gen_params(*args, fsm=1)
        with pytest.raises(B200Error, match="asr_generate: AHA_GEN_CONSTRAINED"):
            a.asr_generate([(np.array([1, 2, 3], np.uint32), np.zeros((128, 100), np.float32))], max_tokens=4)
    finally:
        a.close()


def test_destroy_waits_for_the_running_slot(tiny):
    from aha_b200 import B200Error
    cfg, _, m = tiny
    V = cfg["vocab_size"]
    f = m.fsm_create(*R.random_fsm(V, 4, 3))
    s = _Session(m)
    s.add("a", dict(input_ids=_ids(9, V, 6), max_tokens=8, fsm=f))
    s.add("b", dict(input_ids=_ids(9, V, 7), max_tokens=3))
    with pytest.raises(B200Error, match="constrains the running request in slot 0"):
        m.fsm_destroy(f)
    while s.running:
        s.step()
    m.fsm_destroy(f)
    s.drain()
