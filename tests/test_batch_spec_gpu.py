"""Speculative requests inside wide batch sessions (aha_b200_batch_add_speculative / _batch_step_spec / _batch_logprobs_spec /
_batch_spec_stats).

A speculative request in a session must yield bit for bit the ids, records and stats generate_speculative yields for it alone, whatever
slot it holds, whatever runs beside it and at whatever step it joins; its plain neighbours must yield what they yield without it; a session
without speculative requests stepped by batch_step_spec must launch what batch_step_n launches.  The batched verify attention is checked on
host data through debug_verify_attn_batch."""
import numpy as np
import pytest

from attn_ref import attention
from conftest import make_model, make_oracle
from test_batch_wide_gpu import SAMPLERS, _check_oracle_ids
from test_speculative_gpu import _ids, _key, _requests

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------ batched verify attention

@pytest.fixture(scope="module")
def tiny():
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=2048)
    yield cfg, w, m
    m.close()


@pytest.mark.parametrize("G", [1, 2, 4, 6])
def test_batched_verify_attention(tiny, G):
    m = tiny[2]
    nkv = 2
    rng = np.random.default_rng(7 * G)
    Rs = [1, 2, 8, 16, 8, 2]
    pos0s = [0, 30, 63, 64, 130, 300]            # contexts ending inside, on and across page (32) and chunk (64) boundaries
    n_pages = [-(-(p + R) // 32) for p, R in zip(pos0s, Rs)]
    pool = int(sum(n_pages)) + 5                 # pages no table references stay NaN
    perm = rng.permutation(pool)                 # every request's pages scattered over the pool
    tables, at = [], 0
    for n in n_pages:
        tables.append(perm[at:at + n])
        at += n
    qs = [rng.standard_normal((R, G * nkv, 128)).astype(np.float32) for R in Rs]
    ks = [rng.standard_normal((p + R, nkv, 128)).astype(np.float32) for p, R in zip(pos0s, Rs)]
    vs = [rng.standard_normal((p + R, nkv, 128)).astype(np.float32) for p, R in zip(pos0s, Rs)]
    got = m.debug_verify_attn_batch(qs, ks, vs, pos0s, tables, pool)
    for j in range(len(Rs)):
        assert np.abs(got[j] - attention(qs[j], ks[j], vs[j], causal=True)).max() <= 1e-5, j
        alone = m.debug_verify_attn(qs[j], ks[j], vs[j], pos0s[j])       # the single-request kernel on the same data
        assert np.array_equal(alone, got[j]), j
    # the same requests in another order, on other pages: each request's bits do not move
    order = [3, 0, 5, 1, 4, 2]
    again = m.debug_verify_attn_batch([qs[j] for j in order], [ks[j] for j in order], [vs[j] for j in order], [pos0s[j] for j in order],
                                      [pool - 1 - tables[j] for j in order], pool)
    for i, j in enumerate(order):
        assert np.array_equal(again[i], got[j]), j


# ------------------------------------------------------------------------------------------------------------ session driver

def _run(m, width, plan, steps_max=400):
    """Run a wide session of `width` slots.  plan: {step index: [("plain" | "spec", request dict), ...]} -- admitted before that step.
    -> ({request id: ids}, {request id: records}, {request id: stats}, {request id: slot})"""
    ids, recs, stats, slot_of, req_of = {}, {}, {}, {}, {}
    n_req = 0
    m.batch_open_wide(width)
    try:
        for step in range(steps_max):
            for kind, r in plan.get(step, []):
                rid = n_req
                n_req += 1
                if kind == "spec":
                    s, t, fin = m.batch_add_speculative(**r)
                else:
                    s, t, fin = m.batch_add(**r)
                ids[rid] = [t]
                if r.get("logprobs"):
                    recs[rid] = list(m.batch_logprobs_spec().get(s, []))
                    assert len(recs[rid]) == 1
                slot_of[rid] = s
                if not fin:
                    req_of[s] = rid
                elif kind == "spec":
                    stats[rid] = m.batch_spec_stats().get(s, dict(passes=0, drafted=0, accepted=0))
            if not req_of and step > max(plan):
                break
            out = m.batch_step_spec()
            lp = m.batch_logprobs_spec()
            st = m.batch_spec_stats()
            last = m.batch_logprobs()
            for s, (toks, fin) in out.items():
                rid = req_of[s]
                ids[rid] += toks
                if rid in recs:
                    assert len(lp[s]) == len(toks)
                    recs[rid] += lp[s]
                    assert _key(last[s]) == _key(lp[s][-1])          # batch_logprobs: the slot's last delivered token
                if fin:
                    del req_of[s]
                    stats[rid] = st.get(s, dict(passes=0, drafted=0, accepted=0))
        assert not req_of
    finally:
        m.batch_close()
    return ids, recs, stats, slot_of


def _alone(m, r):
    res = m.generate_speculative(**r)
    return res[0], (res[3] if r.get("logprobs") else None), res[2]


def _plain(r):
    return {k: v for k, v in r.items() if k not in ("prediction", "prompt_lookup", "max_draft", "ngram")}


@pytest.fixture(scope="module")
def pair():
    """two handles on the same weights: CUDA graphs and eager launches"""
    cfg, w, m = make_model("qwen3", "tiny", max_ctx=4096)
    _, _, e = make_model("qwen3", "tiny", max_ctx=4096, use_graph=False)
    yield cfg, m, e
    m.close()
    e.close()


def _edited(ref, V, rng):
    sub = [int(rng.integers(0, V)) if i % 5 == 3 else t for i, t in enumerate(ref)]
    return [t for i, t in enumerate(sub) if i % 11 != 7]


# ------------------------------------------------------------------------------------------------------------ exactness

@pytest.mark.parametrize("samp", SAMPLERS)
def test_spec_in_session_equals_alone(pair, samp):
    """Speculative requests with exact / edited / absent predictions and prompt lookup, of several R, joining at several steps in several
    slots beside plain requests, yield what generate_speculative yields for each alone (top-20 records included)."""
    cfg, m, _ = pair
    V = cfg["vocab_size"]
    rng = np.random.default_rng(11)
    base = [dict(input_ids=_ids(40 + 23 * i, V, 300 + i), max_tokens=30 + 5 * i, logprobs=True, top_logprobs=20, **samp) for i in range(4)]
    for i, r in enumerate(base):
        if r.get("temperature"):
            r["seed"] = 50 + i
    ref = [m.generate_speculative(max_draft=1, **r)[0] for r in base]
    specs = [dict(base[0], prediction=ref[0], max_draft=7),
             dict(base[1], prediction=_edited(ref[1], V, rng), max_draft=4, prompt_lookup=True),
             dict(base[2], max_draft=15, prompt_lookup=True),
             dict(base[3], prediction=ref[3][:12], max_draft=2)]
    want = [_alone(m, r) for r in specs]
    plain = [dict(input_ids=_ids(30 + 9 * i, V, 400 + i), max_tokens=25 + 7 * i, logprobs=i % 2 == 0, **SAMPLERS[i % len(SAMPLERS)])
             for i in range(5)]
    plan = {0: [("plain", plain[0]), ("spec", specs[0]), ("plain", plain[1])],
            2: [("spec", specs[1]), ("plain", plain[2])],
            5: [("plain", plain[3]), ("spec", specs[2])],
            9: [("spec", specs[3]), ("plain", plain[4])]}
    ids, recs, stats, _ = _run(m, 12, plan)
    rids = [1, 3, 6, 7]
    for k, rid in enumerate(rids):
        w_ids, w_rec, w_st = want[k]
        assert ids[rid] == w_ids, k
        assert [_key(x) for x in recs[rid]] == [_key(x) for x in w_rec], k
        assert stats[rid] == w_st, k
    # neighbours: the plain requests yield exactly what a wide session without speculative requests yields for them
    plain_plan = {0: [("plain", plain[0]), ("plain", plain[1])], 2: [("plain", plain[2])], 5: [("plain", plain[3])], 9: [("plain", plain[4])]}
    p_ids, p_recs, _, _ = _run(m, 12, plain_plan)
    for rid, prid in zip([0, 2, 4, 5, 8], range(5)):
        assert ids[rid] == p_ids[prid], prid
        if plain[prid]["logprobs"]:
            assert [_key(x) for x in recs[rid]] == [_key(x) for x in p_recs[prid]], prid


def test_penalties_bias_prefix_cache_and_eager(pair):
    """Frequency / presence penalties and logit bias, a prefix-cache hit, and eager launches give the alone bits."""
    cfg, m, e = pair
    V = cfg["vocab_size"]
    system = _ids(96, V, 77)
    rids = {}
    for h in (m, e):
        rid = h.rules_create(presence_penalty=0.6, frequency_penalty=0.4, logit_bias={5: 3.0, 9: -50.0})
        rids[h] = rid
    r0 = dict(input_ids=np.concatenate([system, _ids(20, V, 78)]), max_tokens=40, temperature=0.8, top_k=40, seed=4, logprobs=True,
              top_logprobs=3)
    r1 = dict(input_ids=np.concatenate([system, _ids(33, V, 79)]), max_tokens=36, logprobs=True)
    ref0 = m.generate_speculative(max_draft=1, rules=rids[m], **r0)[0]
    s0 = dict(r0, prediction=ref0, max_draft=7, prompt_lookup=True)
    s1 = dict(r1, max_draft=5, prompt_lookup=True)
    for h in (m, e):
        want = [_alone(h, dict(s0, rules=rids[h])), _alone(h, s1)]
        h.batch_open_wide(8)
        try:
            h.batch_prefix_cache(4096)
            slot, t, _ = h.batch_add(**dict(_plain(s1), max_tokens=3))    # its prompt's full pages enter the index
            while h.batch_step_spec():
                pass
            a = h.batch_add_speculative(**dict(s0, rules=rids[h]))
            b = h.batch_add_speculative(**s1)
            hits = h.batch_prefix_stats()[1]
            assert hits.get(a[0], 0) == 64 and hits.get(b[0], 0) == 96      # capped at seq_len - 32 (116 and 129 prompt tokens)
            got = {a[0]: [a[1]], b[0]: [b[1]]}
            rec = {s: list(h.batch_logprobs_spec()[s]) for s in got}
            st = {}
            while True:
                out = h.batch_step_spec()
                if not out:
                    break
                lp, ss = h.batch_logprobs_spec(), h.batch_spec_stats()
                for s, (toks, fin) in out.items():
                    got[s] += toks
                    rec[s] += lp[s]
                    if fin:
                        st[s] = ss[s]
        finally:
            h.batch_close()
        for s, w in ((a[0], want[0]), (b[0], want[1])):
            assert got[s] == w[0] and [_key(x) for x in rec[s]] == [_key(x) for x in w[1]] and st[s] == w[2], h is e
    for h in (m, e):
        h.rules_destroy(rids[h])


# ------------------------------------------------------------------------------------------------------------ oracle

@pytest.mark.parametrize("preset,budget", [("tiny", 40), ("tiny-g1", 40), ("tiny-g4", 40), ("mid", 10)])
def test_oracle_ids(preset, budget):
    cfg, w, m = make_model("qwen3", preset, max_ctx=2048)
    o = make_oracle("qwen3", cfg, w)
    try:
        reqs = _requests(cfg["vocab_size"], 7, 20, budget)
        plan = {i: [("spec", dict(r, prompt_lookup=True, max_draft=3 + 2 * (i % 3)))] for i, r in enumerate(reqs)}
        ids, _, _, _ = _run(m, 16, plan)
        _check_oracle_ids(o, reqs, [ids[i] for i in range(len(reqs))])
    finally:
        m.close()


def test_oracle_ids_qwen3vl_image():
    from aha_b200 import synth
    from oracle.qwen3vl import process_image
    cfg, w, m = make_model("qwen3vl", "tiny", max_ctx=2048, max_patches=1024)
    o = make_oracle("qwen3vl", cfg, w)
    try:
        pv, grid = process_image(synth.synth_image(256, 320, 1))
        ids = synth.vl_prompt_ids(cfg, grid, 16)
        data = [pv, grid, None, None, None]
        reqs = [dict(input_ids=ids, data=data, max_tokens=24, **kw) for kw in
                ({}, dict(temperature=0.8, top_k=20, top_p=0.9, repeat_penalty=1.2, repeat_last_n=16, seed=5))]
        plan = {0: [("spec", dict(reqs[0], prompt_lookup=True, max_draft=4))], 1: [("spec", dict(reqs[1], prompt_lookup=True, max_draft=6))]}
        out, _, _, _ = _run(m, 4, plan)
        _check_oracle_ids(o, reqs, [out[0], out[1]])
    finally:
        m.close()


# ------------------------------------------------------------------------------------------------------------ ends of requests

def test_eos_max_tokens_and_slot_reuse():
    from aha_b200 import B200Model, synth
    cfg = synth.get_config("qwen3", "tiny")
    w = synth.make_weights("qwen3", cfg, 0)
    V = cfg["vocab_size"]
    r = dict(input_ids=_ids(60, V, 8), max_tokens=40, temperature=1.0, top_k=50, seed=2)
    m = B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"]], max_ctx=1024)
    try:
        full = m.generate_speculative(**r)[0]
    finally:
        m.close()
    k = next(i for i in range(5, len(full)) if full[i] not in full[1:i])
    m = B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"], full[k]], max_ctx=1024)
    try:
        want = m.generate_speculative(prediction=full, max_draft=15, **r)
        assert want[0] == full[:k + 1]
        m.batch_open_wide(2)
        try:
            s, t, _ = m.batch_add_speculative(prediction=full, max_draft=15, **r)
            got, n_steps = [t], 0
            while True:
                out = m.batch_step_spec()
                n_steps += 1
                toks, fin = out[s]
                got += toks
                if fin:
                    break
            assert got == full[:k + 1] and m.batch_spec_stats()[s] == want[2]
            assert n_steps == want[2]["passes"]                                 # the EOS ended the request in the step that emitted it
            free = m.batch_prefix_stats()[0]["free_pages"]
            assert free == 1024 // 32                                             # its pages went back
            s2, _, _ = m.batch_add_speculative(prediction=full, max_draft=15, **r)
            assert s2 == s and m.batch_spec_stats() == {}                        # the freed slot is taken; its counters start again
        finally:
            m.batch_close()
    finally:
        m.close()
    m = B200Model("qwen3", cfg, w, eos_ids=[cfg["eos_token_id"]], max_ctx=1024)
    try:
        for mt in (1, 2, 5, 9, 13):
            want = m.generate_speculative(prediction=full, max_draft=7, **dict(r, max_tokens=mt))
            ids, _, st, _ = _run(m, 3, {0: [("spec", dict(r, prediction=full, max_draft=7, max_tokens=mt))]})
            assert ids[0] == want[0] == full[:mt], mt
            if mt > 1:
                assert st[0] == want[2], mt
    finally:
        m.close()


# ------------------------------------------------------------------------------------------------------------ off means off, graphs

def test_off_means_off(pair):
    cfg, m, _ = pair
    V = cfg["vocab_size"]
    reqs = [dict(input_ids=_ids(20 + 5 * i, V, 500 + i), max_tokens=12 + i, logprobs=i == 2, **SAMPLERS[i % len(SAMPLERS)]) for i in range(6)]
    runs = []
    for spec_step in (False, True):
        m.batch_open_wide(8)
        try:
            res = m.batch_add_many(reqs)
            ids = {s: [t] for s, t, _ in res}
            m.reset_stats()
            while True:
                if spec_step:
                    got = m.batch_step_spec()
                    assert all(len(toks) == 1 for toks, _ in got.values())
                    out = {s: (toks[0], fin) for s, (toks, fin) in got.items()}
                else:
                    out = m.batch_step()
                if not out:
                    break
                for s, (t, _) in out.items():
                    ids[s].append(t)
            runs.append((ids, m.stats()["kernel_launches"]))
        finally:
            m.batch_close()
    assert runs[0] == runs[1]


def test_graphs_by_key_and_eager(pair):
    """Speculative requests of different R swapped in at the same totals replay the graphs of their step shapes (plain rows, requests,
    verify rows); only new shapes capture.  Eager launches give the same bits."""
    cfg, m, e = pair
    V = cfg["vocab_size"]
    mk = lambda i, md: dict(input_ids=_ids(30 + i, V, 600 + i), max_tokens=20, prompt_lookup=True, max_draft=md)
    plain = dict(input_ids=_ids(25, V, 650), max_tokens=60)
    plans = [[("plain", plain), ("spec", mk(0, 3)), ("spec", mk(1, 7))],      # 1 plain row, 2 requests of 4 + 8 rows
             [("plain", plain), ("spec", mk(0, 7)), ("spec", mk(1, 3))],      # the same totals, R swapped between the requests
             [("plain", plain), ("spec", mk(2, 5)), ("spec", mk(3, 5))]]
    for plan in plans:
        a, b = _run(m, 8, {0: plan}), _run(e, 8, {0: plan})
        assert a[0] == b[0] and a[2] == b[2]
    m.batch_open_wide(8)
    try:
        shapes = set()
        for plan in plans:
            R, running = {}, set()
            for kind, r in plan:
                s, _, fin = (m.batch_add_speculative if kind == "spec" else m.batch_add)(**r)
                if kind == "spec":
                    R[s] = r["max_draft"] + 1
                if not fin:
                    running.add(s)
            while True:
                specs = [R[s] for s in running if s in R]
                shapes.add((len(running) - len(specs), len(specs), sum(specs)) if specs else ("plain", len(running)))
                out = m.batch_step_spec()
                running -= {s for s, (_, fin) in out.items() if fin}
                if not running:
                    break
            assert m.debug_read("batch_graphs", 0, 1)[0] == len(shapes), shapes
    finally:
        m.batch_close()


# ------------------------------------------------------------------------------------------------------------ refusals

def test_refusals(tiny):
    from aha_b200 import B200Error, _lib as L
    cfg, w, m = tiny
    V = cfg["vocab_size"]
    ids = _ids(20, V, 1)
    r = dict(input_ids=ids, max_tokens=200)
    gp = lambda **kw: L.GenParams(**dict(dict(temperature=0.0, repeat_penalty=1.0, repeat_last_n=64, max_tokens=8, seed=1), **kw))
    m.batch_open()
    try:
        with pytest.raises(B200Error, match="wide session"):
            m.batch_add_speculative(**r)
    finally:
        m.batch_close()
    fsm = m.fsm_create([0, 1], [3], [0])
    rules = m.rules_create(presence_penalty=0.5, fsm=fsm)
    m.batch_open_wide(40)
    try:
        m.batch_add(**r)
        m.batch_add_speculative(max_draft=15, **r)
        state = lambda: (m.batch_prefix_stats(), m.batch_spec_stats(), m.debug_read("batch_graphs", 0, 1)[0])
        before = state()
        bad = np.array([V], np.uint32)
        for params, spec, msg in ((gp(), L.SpecParams(max_draft=0), "max_draft must be 1 to 15"),
                                  (gp(), L.SpecParams(max_draft=16), "max_draft must be 1 to 15"),
                                  (gp(), L.SpecParams(max_draft=4, ngram=9), "ngram must be"),
                                  (gp(), L.SpecParams(max_draft=4, flags=2), "unknown spec flags"),
                                  (gp(flags=L.GEN_REUSE_PREFIX), L.SpecParams(max_draft=4), "not supported with speculative decoding"),
                                  (gp(flags=L.GEN_CONTINUE_RNG), L.SpecParams(max_draft=4), "not supported with speculative decoding"),
                                  (gp(flags=L.GEN_EOS_ON_FIRST), L.SpecParams(max_draft=4), "not supported with speculative decoding"),
                                  (gp(flags=L.GEN_CONSTRAINED, reserved=fsm), L.SpecParams(max_draft=4), "CONSTRAINED is not supported"),
                                  (gp(flags=L.GEN_LOGIT_RULES, reserved=rules), L.SpecParams(max_draft=4), "name a token automaton"),
                                  (gp(), L.SpecParams(max_draft=4, prediction=bad.ctypes.data_as(L._U32P), n_prediction=1), "out of range")):
            with pytest.raises(B200Error, match=msg):
                _add_raw(m, ids, params, spec)
        # the row budget from both sides: 1 + 16 rows run, 2 more requests of 16 make 49; a third does not fit, nor 16 plain requests
        for _ in range(2):
            m.batch_add_speculative(max_draft=15, **r)
        before = state()
        with pytest.raises(B200Error, match="exceed 64"):
            m.batch_add_speculative(max_draft=15, **r)
        with pytest.raises(B200Error, match="exceed 64"):
            m.batch_add_many([r] * 16)
        with pytest.raises(B200Error, match="exceed 64"):
            m.batch_add_n(n=16, **r)
        with pytest.raises(B200Error, match="exceeds max_ctx"):
            m.batch_add_speculative(_ids(2000, V, 2), max_tokens=42, max_draft=7)        # 2000 + 42 + 7 > 2048
        assert state() == before                                                          # refused calls changed nothing
        with pytest.raises(B200Error, match="batch_step_spec"):
            m.batch_step()
        with pytest.raises(B200Error, match="batch_step_spec"):
            _step_n(m, 40)
    finally:
        m.batch_close()
        m.rules_destroy(rules)
        m.fsm_destroy(fsm)


def _step_n(m, w):
    import ctypes as C
    toks, status, n = (C.c_uint32 * w)(), (C.c_int32 * w)(), C.c_size_t(0)
    m._check(m._lib.aha_b200_batch_step_n(m._h, toks, status, w, C.byref(n)))


def _add_raw(m, ids, params, spec):
    import ctypes as C
    from aha_b200 import _lib as L
    ids = np.ascontiguousarray(ids, np.uint32)
    req = L.BatchRequest()
    req.ids = ids.ctypes.data_as(C.POINTER(C.c_uint32))
    req.seq_len = ids.size
    req.params = params
    slot, fin, tok = C.c_int32(-1), C.c_int32(0), C.c_uint32(0)
    m._check(m._lib.aha_b200_batch_add_speculative(m._h, C.byref(req), C.byref(spec), C.byref(slot), C.byref(tok), C.byref(fin), None))
