"""LoRA adapters in wide batch sessions (aha_b200_batch_add_lora) at the Qwen3-0.6B text row shape (2 layers, 4096-token vocabulary):
accuracy against the merged float64 decoder (tests/lora_ref.py), bit-identity of base requests beside adapter requests, invariance of an
adapter request to its slot, neighbours, join step and packing, the zero adapter, prefix-cache keying, suspend / resume and refusals."""
import numpy as np
import pytest

import lora_ref
from test_decode_f64_gpu import Shape, _check_session

pytestmark = pytest.mark.gpu

RANKS = [1, 8, 16, 64]


def _cfg():
    from aha_b200 import synth
    cfg = synth.get_config("qwen3", "q0.6")
    cfg.update(num_hidden_layers=2, vocab_size=4096, eos_token_id=4095)
    return cfg


class LoraShape(Shape):
    """the 0.6B rows, with float64 logits under an adapter cached per (adapter key, sequence)"""

    def __init__(self):
        super().__init__("0.6b", _cfg())
        self._ref = {}

    def lora_logits(self, key, adapter, scale, seq, start):
        k = (key, tuple(int(t) for t in seq))
        if k not in self._ref:
            self._ref[k] = lora_ref.logits(self.cfg, self.w, adapter, scale, [np.asarray(seq)])[0]
        return self._ref[k][start:]


@pytest.fixture(scope="module")
def shape():
    return LoraShape()


@pytest.fixture(scope="module")
def model(shape):
    m = shape.model(max_ctx=16384)
    yield m
    m.close()


def _adapter(shape, r, seed, **kw):
    return lora_ref.make_adapter(shape.cfg, seed, r, **kw)


def _run(m, reqs, adapters, width=9, lp=True, steps_before=None):
    """requests [(prompt, max_tokens)] with adapters[i] admitted together (batch_add_lora) into a fresh wide session -> (ids, records)
    per request"""
    m.batch_open_wide(width)
    try:
        rq = [dict(input_ids=p, max_tokens=n, logprobs=lp, top_logprobs=5 if lp else 0) for p, n in reqs]
        res = m.batch_add_lora(rq, adapters)
        return _drain(m, res, lp)
    finally:
        m.batch_close()


def _drain(m, res, lp, toks=None, recs=None):
    toks = toks or [[t] for _, t, _ in res]
    first = m.batch_logprobs() if lp else {}
    recs = recs or [[first.get(s)] for s, _, _ in res]
    running = {s: i for i, (s, _, fin) in enumerate(res) if not fin}
    while running:
        out = m.batch_step()
        rec = m.batch_logprobs() if lp else {}
        for s, (t, fin) in out.items():
            i = running[s]
            toks[i].append(t)
            recs[i].append(rec.get(s))
            if fin:
                del running[s]
    return toks, recs


def _same(a, b):
    assert a[0] == b[0]
    for ra, rb in zip(a[1], b[1]):
        for x, y in zip(ra, rb):
            if x is None or y is None:
                assert x is y
            else:
                assert x["token"] == y["token"] and x["top_ids"] == y["top_ids"]
                assert np.array_equal(np.float32(x["logprob"]), np.float32(y["logprob"]))
                assert np.array_equal(np.array(x["top_logprobs"], np.float32), np.array(y["top_logprobs"], np.float32))


@pytest.mark.parametrize("r", RANKS)
def test_accuracy_against_the_merged_float64_decoder(shape, model, r):
    """three requests under one adapter of rank r beside a base request: every record within the wide path's bound of the float64 decoder
    on the merged weights, greedy ids equal to its argmax where the gap allows, and ids that differ from the base model's"""
    ad = _adapter(shape, r, 100 + r)
    scale = 16.0 / r
    aid = model.lora_create(ad, scale)
    try:
        reqs = [(shape.ids(S, 200 + i), n) for i, (S, n) in enumerate([(70, 12), (33, 10), (5, 14), (40, 8)])]
        toks, recs = _run(model, reqs, [aid, aid, aid, 0])
    finally:
        model.lora_destroy(aid)
    lora_shape = _Under(shape, ("acc", r), ad, scale)
    _check_session(lora_shape, f"lora r={r}", reqs[:3], toks[:3], recs[:3])
    _check_session(shape, f"lora r={r} base row", reqs[3:], toks[3:], recs[3:])
    base = [_check_base_ids(shape, p, n) for p, n in reqs[:3]]
    assert any(b != t for b, t in zip(base, toks[:3])), "the adapter changes no id: it is too weak to test anything"


class _Under:
    """a Shape whose logits are the merged adapter's (what _check_session reads)"""

    def __init__(self, shape, key, adapter, scale):
        self.shape, self.key, self.adapter, self.scale = shape, key, adapter, scale
        self.name = shape.name

    def logits(self, seq, start):
        return self.shape.lora_logits(self.key, self.adapter, self.scale, seq, start)


def _check_base_ids(shape, prompt, n):
    """greedy ids of the base model from the float64 decoder"""
    seq = list(prompt)
    for _ in range(n):
        seq.append(int(np.argmax(shape.logits(np.array(seq, np.uint32), len(seq) - 1)[-1])))
    return seq[len(prompt):]


def test_base_requests_unchanged_beside_adapters(shape, model):
    """base requests give bit-identical ids and records beside adapter neighbours (distinct adapters, mixed ranks), and a session that
    admits no adapter request launches the same kernels and graphs whether adapters are loaded or not"""
    reqs = [(shape.ids(S, 300 + i), n) for i, (S, n) in enumerate([(70, 10), (40, 9), (96, 7)])]

    def base_session():
        model.reset_stats()
        model.batch_open_wide(9)
        try:
            res = model.batch_add_many([dict(input_ids=p, max_tokens=n, logprobs=True, top_logprobs=5) for p, n in reqs])
            out = _drain(model, res, True)
            graphs = int(model.debug_read("batch_graphs", 0, 1)[0])
        finally:
            model.batch_close()
        st = model.stats()
        return out, (st["kernel_launches"], st["graph_launches"], graphs)

    plain, counts = base_session()
    ids = [model.lora_create(_adapter(shape, r, 400 + r), 1.0) for r in (1, 16, 64)]
    try:
        again, counts2 = base_session()
        assert counts2 == counts
        _same(again, plain)
        nb = [(shape.ids(S, 310 + i), 9) for i, S in enumerate([50, 33, 64])]
        mixed = [reqs[0], nb[0], reqs[1], nb[1], nb[2], reqs[2]]
        toks, recs = _run(model, mixed, [0, ids[0], 0, ids[1], ids[2], 0])
    finally:
        for i in ids:
            model.lora_destroy(i)
    _same(([toks[0], toks[2], toks[5]], [recs[0], recs[2], recs[5]]), plain)


def test_adapter_request_invariance(shape, model):
    """one adapter request alone, packed with other adapters' requests at another slot, and joining at a later step: bit-identical"""
    a, b = model.lora_create(_adapter(shape, 16, 500), 1.0), model.lora_create(_adapter(shape, 8, 501), 2.0)
    try:
        p = shape.ids(48, 510)
        alone = _run(model, [(p, 10)], [a])
        others = [(shape.ids(S, 520 + i), 10) for i, S in enumerate([40, 64, 35])]
        packed = _run(model, others + [(p, 10)], [b, 0, b, a])
        _same(([packed[0][3]], [packed[1][3]]), alone)
        # joining a running session at a later step, in another slot
        model.batch_open_wide(9)
        try:
            res0 = model.batch_add_lora([dict(input_ids=q, max_tokens=20, logprobs=True, top_logprobs=5) for q, _ in others], [b, a, 0])
            for _ in range(3):
                model.batch_step()
            res = model.batch_add_lora([dict(input_ids=p, max_tokens=10, logprobs=True, top_logprobs=5)], [a])
            assert res[0][0] == 3
            toks, recs = [[res[0][1]]], [[model.batch_logprobs()[3]]]
            while len(toks[0]) < 10:
                out = model.batch_step()
                toks[0].append(out[3][0])
                recs[0].append(model.batch_logprobs()[3])
        finally:
            model.batch_close()
        _same((toks, recs), alone)
        assert res0
    finally:
        model.lora_destroy(a)
        model.lora_destroy(b)


def test_zero_adapter_is_the_base_model(shape, model):
    z = model.lora_create(_adapter(shape, 16, 600, zero_b=True), 3.0)
    try:
        reqs = [(shape.ids(S, 610 + i), 8) for i, S in enumerate([70, 12])]
        base = _run(model, reqs, [0, 0])
        zero = _run(model, reqs, [z, z])
    finally:
        model.lora_destroy(z)
    _same(zero, base)


def test_prefix_cache_is_keyed_by_adapter(shape, model):
    a, b = model.lora_create(_adapter(shape, 16, 700), 1.0), model.lora_create(_adapter(shape, 16, 701), 1.0)
    p = shape.ids(100, 710)
    try:
        cold = _run(model, [(p, 6)], [a])
        model.batch_open_wide(9)
        try:
            model.batch_prefix_cache(4096)
            first = _drain(model, model.batch_add_lora([dict(input_ids=p, max_tokens=6, logprobs=True, top_logprobs=5)], [a]), True)
            _same(first, cold)
            for ad, want_hit in ((b, False), (0, False), (a, True)):
                res = model.batch_add_lora([dict(input_ids=p, max_tokens=6, logprobs=True, top_logprobs=5)], [ad])
                hits = model.batch_prefix_stats()[1]
                assert (res[0][0] in hits) == want_hit, (ad, hits)
                out = _drain(model, res, True)
                if ad == a:
                    _same(out, cold)
            cached = model.batch_prefix_stats()[0]["cached_pages"]
            model.lora_destroy(a)
            a = None
            assert model.batch_prefix_stats()[0]["cached_pages"] < cached
        finally:
            model.batch_close()
    finally:
        for i in (a, b):
            if i:
                model.lora_destroy(i)


def test_suspend_resume_carries_the_adapter(shape, model):
    a = model.lora_create(_adapter(shape, 16, 800), 1.0)
    p = shape.ids(60, 810)
    try:
        straight = _run(model, [(p, 12)], [a])
        model.batch_swap_space(4096)
        model.batch_open_wide(9)
        try:
            res = model.batch_add_lora([dict(input_ids=p, max_tokens=12, logprobs=True, top_logprobs=5)], [a])
            toks, recs = [[res[0][1]]], [[model.batch_logprobs()[res[0][0]]]]
            for _ in range(4):
                out = model.batch_step()
                toks[0].append(out[res[0][0]][0])
                recs[0].append(model.batch_logprobs()[res[0][0]])
            sid = model.batch_suspend(res[0][0])
            with pytest.raises(Exception, match="suspended request"):
                model.lora_destroy(a)
            slot = model.batch_resume(sid)
            while len(toks[0]) < 12:
                out = model.batch_step()
                toks[0].append(out[slot][0])
                recs[0].append(model.batch_logprobs()[slot])
        finally:
            model.batch_close()
        _same((toks, recs), straight)
    finally:
        model.lora_destroy(a)
        model.batch_swap_space(0)


def test_refusals_change_nothing(shape, model):
    from aha_b200 import B200Error
    cfg = shape.cfg
    good = _adapter(shape, 8, 900, targets=("q", "v"), layers=[0])
    bad = {
        "unknown name": dict(good, **{"model.layers.0.mlp.foo.lora_A.weight": good["model.layers.0.self_attn.q_proj.lora_A.weight"]}),
        "DoRA": dict(good, **{"model.layers.0.self_attn.q_proj.lora_magnitude_vector": np.ones(2048, np.float16)}),
        "A without B": {k: v for k, v in good.items() if "q_proj.lora_B" not in k},
        "shape": dict(good, **{"model.layers.0.self_attn.q_proj.lora_B.weight": np.zeros((1024, 8), np.float16)}),
        "rank": _adapter(shape, 65, 901, targets=("q",), layers=[0]),
        "layer": _adapter(shape, 8, 902, targets=("q",), layers=[cfg["num_hidden_layers"]]),
    }
    for why, ad in bad.items():
        with pytest.raises(B200Error):
            model.lora_create(ad, 1.0)
    with pytest.raises(B200Error, match="finite"):
        model.lora_create(good, float("nan"))
    a = model.lora_create({"base_model.model." + k: v for k, v in good.items()}, 2.0)
    assert a >= 1
    p = shape.ids(40, 910)
    try:
        model.batch_open()
        try:
            with pytest.raises(B200Error, match="wide session"):
                model.batch_add_lora([dict(input_ids=p, max_tokens=4)], [a])
        finally:
            model.batch_close()
        model.batch_open_wide(9)
        try:
            with pytest.raises(B200Error, match="no LoRA adapter"):
                model.batch_add_lora([dict(input_ids=p, max_tokens=4), dict(input_ids=p, max_tokens=4)], [0, a + 1000])
            res = model.batch_add_lora([dict(input_ids=p, max_tokens=4)], [a])
            assert res[0][0] == 0   # the refused call took no slot
            with pytest.raises(B200Error, match="runs the request"):
                model.lora_destroy(a)
            with pytest.raises(B200Error, match="LoRA request is running"):
                model.batch_add_speculative(p, prediction=p[:8], max_tokens=4)
            _drain(model, res, False)
        finally:
            model.batch_close()
    finally:
        model.lora_destroy(a)
    with pytest.raises(B200Error, match="no LoRA adapter"):
        model.lora_destroy(a)


# -------------------------------------------------------------------------------------------- every prefill path that adds the tail
#   short alone : a prompt under 32 tokens admitted alone -> gemm_simt (M < 32) on fp32 rows, its tail as extra K from fp32 t
#   gemm_impl=1 : every prefill GEMM on gemm_simt, shrink from the fp32 rows (xn, attn, hbuf)
#   tile 128    : AHA_GEMM_WIDE=0, the pre-split data flow on 128 x 128 wgmma tiles
#   split       : AHA_PRESPLIT=0, every GEMM splits its own fp32 input (128 x 256 tiles), shrink from the fp32 rows
PREFILL_PATHS = {"short alone": ({}, None), "gemm_impl=1": (dict(gemm_impl=1), None), "tile 128": ({}, ("AHA_GEMM_WIDE", "0")),
                 "split": ({}, ("AHA_PRESPLIT", "0"))}


@pytest.mark.parametrize("path", list(PREFILL_PATHS))
def test_prefill_paths_against_the_merged_float64_decoder(shape, model, path, monkeypatch):
    kw, env = PREFILL_PATHS[path]
    ad, scale = _adapter(shape, 16, 1100), 1.0
    if env:
        monkeypatch.setenv(*env)
    m = model if path == "short alone" else shape.model(max_ctx=4096, **kw)
    try:
        aid = m.lora_create(ad, scale)
        try:
            if path == "short alone":
                reqs = [(shape.ids(S, 1110 + i), 10) for i, S in enumerate([12, 5, 31])]
                toks, recs = [], []
                for q in reqs:
                    t, r = _run(m, [q], [aid])
                    toks += t
                    recs += r
            else:
                reqs = [(shape.ids(S, 1120 + i), n) for i, (S, n) in enumerate([(70, 8), (40, 8), (12, 8)])]
                toks, recs = _run(m, reqs, [aid] * len(reqs))
        finally:
            m.lora_destroy(aid)
    finally:
        if m is not model:
            m.close()
    _check_session(_Under(shape, ("paths", 16), ad, scale), f"lora prefill {path}", reqs, toks, recs)


def _bf16_to_f32(b):
    return (np.asarray(b).view(np.uint16).astype(np.uint32) << 16).view(np.float32)


def test_bf16_and_f32_adapters(shape, model):
    """the same values given as fp16, bf16 and f32 give bit-identical ids and records; a bf16 value below fp16's normal range is refused"""
    from aha_b200 import B200Error, _lib as L
    src = {k: v.astype(np.float32) for k, v in _adapter(shape, 8, 1200).items()}
    for v in src.values():
        v[np.abs(v) < 2.0 ** -14] = 0.0          # what a bf16 checkpoint must hold to narrow to fp16 exactly
    bf = {k: L.to_bf16(v) for k, v in src.items()}
    f32 = {k: _bf16_to_f32(v) for k, v in bf.items()}
    f16 = {k: v.astype(np.float16) for k, v in f32.items()}
    reqs = [(shape.ids(S, 1210 + i), 8) for i, S in enumerate([40, 70])]
    outs = []
    for ad in (f16, bf, f32):
        aid = model.lora_create(ad, 2.0)
        try:
            outs.append(_run(model, reqs, [aid, aid]))
        finally:
            model.lora_destroy(aid)
    _same(outs[1], outs[0])
    _same(outs[2], outs[0])
    tiny = dict(bf)
    name = next(k for k in bf if k.endswith("lora_B.weight"))
    t = np.array(f32[name])
    t[0, 0] = 1e-6
    tiny[name] = L.to_bf16(t)
    with pytest.raises(B200Error, match="below fp16"):
        model.lora_create(tiny, 2.0)


def test_resume_beside_a_speculative_request_is_refused(shape, model):
    """a suspended adapter request does not come back while a speculative request runs (the verify pass has no adapter tail); once the
    speculative request has ended it resumes"""
    from aha_b200 import B200Error
    a = model.lora_create(_adapter(shape, 16, 1300), 1.0)
    p, q = shape.ids(40, 1310), shape.ids(40, 1311)
    model.batch_swap_space(4096)
    try:
        model.batch_open_wide(9)
        try:
            s0, _, _ = model.batch_add_lora([dict(input_ids=p, max_tokens=12)], [a])[0]
            model.batch_step()
            sid = model.batch_suspend(s0)
            s1, _, fin = model.batch_add_speculative(q, prediction=q[:8], max_tokens=12)
            assert not fin
            with pytest.raises(B200Error, match="a speculative request is running"):
                model.batch_resume(sid)
            model.batch_cancel(s1)
            assert model.batch_resume(sid) == 0
            model.batch_step()
        finally:
            model.batch_close()
    finally:
        model.lora_destroy(a)
        model.batch_swap_space(0)


def test_accuracy_at_the_tiny_shape():
    """the tiny text shape (H 256, I 512, 4 / 2 heads): one wgmma k-block of the base weights per 64 columns, tails on every group"""
    from aha_b200 import synth
    sh = Shape("0.6b", synth.get_config("qwen3", "tiny"))
    ad, scale = lora_ref.make_adapter(sh.cfg, 1400, 8, b_std=0.3), 2.0
    m = sh.model(max_ctx=4096)
    try:
        aid = m.lora_create(ad, scale)
        reqs = [(sh.ids(S, 1410 + i), 10) for i, S in enumerate([40, 9, 70])]
        toks, recs = _run(m, reqs, [aid, aid, 0])
    finally:
        m.close()
    ref = {}

    class Tiny:
        name = "0.6b"

        def logits(self, seq, start):
            k = tuple(int(t) for t in seq)
            if k not in ref:
                ref[k] = lora_ref.logits(sh.cfg, sh.w, ad, scale, [np.asarray(seq)])[0]
            return ref[k][start:]

    _check_session(Tiny(), "lora tiny", reqs[:2], toks[:2], recs[:2])
    _check_session(sh, "lora tiny base row", reqs[2:], toks[2:], recs[2:])
