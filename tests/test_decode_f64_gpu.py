"""Every decode path against the float64 decoder (tests/decode_ref.py) at the Qwen3-0.6B, Qwen3-VL-2B and Qwen3-VL-8B text row shapes
(2 layers each), and exact greedy ties at the full 151,936-token vocabulary.

Paths: the per-op kernels (decode_impl=1, under a CUDA graph and eager), the fused step in both modes (decode_impl=3 / 4; the 8B rows
have K = 12288 and are refused by it, so decode_impl=0 runs the per-op step there), narrow batch sessions under each AHA_BATCH_GEMV
projection (0 = weights in registers, 1 = SIMT GEMM, 2 = cp.async ring) and wide batch sessions (gemv_wide.cuh).

Errors are measured relative to the logit scale of the shape, err = max |got - ref| / max(1, max |ref|), and bounded per shape by BOUND,
set from the worst error measured on an H100 with a margin.  A greedy id must equal the float64 argmax wherever the float64 top-2 gap
exceeds twice the bound; a batch request is checked on its own emitted ids (teacher-forced reference), so a flipped near-tie cannot
derail the comparison of its later steps."""
import numpy as np
import pytest

import decode_ref

pytestmark = pytest.mark.gpu

# err <= BOUND[shape] on every path.  Worst error measured on one H100 80GB HBM3 (power limit 700 W) over every path of a shape (logits,
# chosen-token logprob, top-5 values): 0.6B rows 7.4e-6, 2B rows 1.3e-5, 8B rows 2.8e-5.  The bounds leave a margin of 2.2-2.7x.
# Rounding the wide path's activations to fp16 (its lo half dropped) measured 3.1e-4 to 6.9e-4.
BOUND = {"0.6b": 2e-5, "2b": 3e-5, "8b": 6e-5}

PROMPT, STEPS = 70, 24      # the prompt crosses two 32-token page boundaries; the steps cross a third


def _config(shape):
    from aha_b200 import synth
    cfg = synth.get_config("qwen3", "q0.6")
    cfg.update(num_hidden_layers=2)
    if shape == "2b":
        cfg.update(hidden_size=2048, intermediate_size=6144, vocab_size=4096, eos_token_id=4095, rope_theta=5000000.0)
    elif shape == "8b":
        cfg.update(hidden_size=4096, intermediate_size=12288, num_attention_heads=32, num_key_value_heads=8, tie_word_embeddings=False,
                   vocab_size=4096, eos_token_id=4095, rope_theta=5000000.0)
    return cfg


class Shape:
    """one shape's weights and its float64 reference, the final hidden states cached per token sequence"""

    def __init__(self, name, cfg=None):
        from aha_b200 import synth
        self.name = name
        self.cfg = cfg or _config(name)
        self.w = synth.make_weights("qwen3", self.cfg, 0)
        self.head = decode_ref.lm_head(self.cfg, self.w)
        self.head64 = np.asarray(self.head, np.float64)   # widened once: the full vocabulary is 1.2 GB of float64 at H 1024
        self.V = self.cfg["vocab_size"]
        self._hid = {}

    def model(self, **kw):
        from aha_b200 import B200Model
        return B200Model("qwen3", self.cfg, self.w, eos_ids=[], **kw)

    def hidden(self, seqs):
        keys = [tuple(int(t) for t in s) for s in seqs]
        todo = sorted(set(k for k in keys if k not in self._hid))
        if todo:
            for k, h in zip(todo, decode_ref.hidden(self.cfg, self.w, [np.array(k) for k in todo])):
                self._hid[k] = h
        return [self._hid[k] for k in keys]

    def logits(self, seq, start):
        """float64 logits of seq at positions start .. len(seq) - 1"""
        return self.hidden([seq])[0][start:] @ self.head64.T

    def ids(self, n, seed):
        from aha_b200 import synth
        return synth.synth_text_ids(n, self.V, seed)


@pytest.fixture(scope="module", params=["0.6b", "2b", "8b"])
def shape(request):
    return Shape(request.param)


def _scale(ref):
    return max(1.0, float(np.abs(ref).max()))


def _report(shape, path, what, err):
    print(f"\n[decode f64] {shape.name:5s} {path:24s} {what:8s} worst rel err {err:.2e} (bound {BOUND[shape.name]:.0e})")
    assert err <= BOUND[shape.name], (shape.name, path, what, err)


def _gap_ok(shape, row, scale):
    """the float64 argmax of row is unambiguous at the bound: top-2 gap > 2 * bound * scale"""
    a, b = np.partition(row, -2)[-2:]
    return b - a > 2 * BOUND[shape.name] * scale


# ------------------------------------------------------------------------------------------------------- single request, teacher-forced

def _teacher_forced(m, prompt, steps):
    """prefill, then forward_step on the given ids -> (logits [1 + len(steps)][V], last_argmax per row)"""
    out, am = [m.forward_initial(prompt, 0)[0, 0]], [m.last_argmax]
    for i, t in enumerate(steps):
        out.append(m.forward_step(np.array([t], np.uint32), len(prompt) + i)[0, 0])
        am.append(m.last_argmax)
    return np.array(out), am


def _check_teacher_forced(shape, path, got, am, ref):
    scale = _scale(ref)
    _report(shape, path, "logits", float(np.abs(got - ref).max()) / scale)
    checked = 0
    for r in range(len(ref)):
        if _gap_ok(shape, ref[r], scale):
            assert am[r] == int(np.argmax(ref[r])), (shape.name, path, r)
            checked += 1
    assert checked >= len(ref) // 2, (shape.name, path, checked)


def test_single_request_every_decode_impl(shape):
    prompt, steps = shape.ids(PROMPT, 11), shape.ids(STEPS, 12)
    ref = shape.logits(np.concatenate([prompt, steps]), PROMPT - 1)
    runs = [("per-op graph", dict(decode_impl=1)), ("per-op eager", dict(decode_impl=1, use_graph=False))]
    if shape.name == "8b":
        from aha_b200 import B200Error
        for impl in (3, 4):
            with pytest.raises(B200Error, match="K > 8192"):
                shape.model(decode_impl=impl, max_ctx=1024)
        runs.append(("auto (per-op)", dict(decode_impl=0)))
    else:
        runs += [("fused barriers", dict(decode_impl=3)), ("fused packets", dict(decode_impl=4))]
    for path, kw in runs:
        m = shape.model(max_ctx=1024, **kw)
        try:
            got, am = _teacher_forced(m, prompt, steps)
            kps = m.stats()["kernels_per_decode_step"]
            if kw["decode_impl"] >= 3:
                assert kps == 1, (path, kps)
            elif kw.get("use_graph", True):
                assert kps > 1, (path, kps)    # the per-op step: one graph of many kernels
        finally:
            m.close()
        _check_teacher_forced(shape, path, got, am, ref)


# ------------------------------------------------------------------------------------------------------------------- batch sessions

def _run_session(m, reqs, wide=0):
    """greedy requests with logprobs through one session -> per request (ids, records)"""
    m.batch_open_wide(wide) if wide else m.batch_open()
    toks, recs, running = [], [], {}
    try:
        for i, (prompt, n) in enumerate(reqs):
            slot, tok, fin = m.batch_add(prompt, max_tokens=n, logprobs=True, top_logprobs=5)
            toks.append([tok])
            recs.append([m.batch_logprobs()[slot]])
            if not fin:
                running[slot] = i
        while running:
            res = m.batch_step()
            lp = m.batch_logprobs()
            for slot, (tok, fin) in res.items():
                i = running[slot]
                toks[i].append(tok)
                recs[i].append(lp[slot])
                if fin:
                    del running[slot]
    finally:
        m.batch_close()
    return toks, recs


def _check_session(shape, path, reqs, toks, recs):
    """every record against the float64 log-softmax of the request's own trajectory"""
    err_lp = err_top = 0.0
    greedy = 0
    for (prompt, n), ids, rs in zip(reqs, toks, recs):
        assert len(ids) == n and [r["token"] for r in rs] == ids
        ref = shape.logits(np.concatenate([prompt, ids[:-1]]).astype(np.uint32), len(prompt) - 1)
        ls = decode_ref.log_softmax(ref)
        for k, (tok, r) in enumerate(zip(ids, rs)):
            scale = _scale(ref[k])
            err_lp = max(err_lp, abs(float(r["logprob"]) - ls[k, tok]) / scale)
            order = np.argsort(-ls[k], kind="stable")[:6]
            want = ls[k, order]
            err_top = max(err_top, float(np.abs(np.array(r["top_logprobs"], np.float64) - want[:5]).max()) / scale)
            for q in range(5):   # the id at rank q wherever its value stands apart from both neighbours
                gap = 2 * BOUND[shape.name] * scale
                apart = (q == 0 or want[q - 1] - want[q] > gap) and want[q] - want[q + 1] > gap
                if apart:
                    assert r["top_ids"][q] == order[q], (shape.name, path, k, q)
            if _gap_ok(shape, ref[k], scale):
                assert tok == order[0], (shape.name, path, k)
                greedy += 1
    _report(shape, path, "logprob", err_lp)
    _report(shape, path, "top-5", err_top)
    assert greedy >= sum(n for _, n in reqs) // 2, (shape.name, path, greedy)


@pytest.fixture(scope="module")
def batch_model(shape):
    m = shape.model(max_ctx=16384)
    yield m
    m.close()


@pytest.mark.parametrize("gemv", [0, 1, 2])
def test_narrow_batch_session(shape, batch_model, gemv, monkeypatch):
    """5 requests of different prompt lengths (pages crossed at different steps), each projection of the narrow step"""
    monkeypatch.setenv("AHA_BATCH_GEMV", str(gemv))
    reqs = [(shape.ids(S, 40 + i), n) for i, (S, n) in enumerate([(70, 20), (33, 12), (5, 24), (100, 8), (64, 16)])]
    toks, recs = _run_session(batch_model, reqs)
    _check_session(shape, f"narrow AHA_BATCH_GEMV={gemv}", reqs, toks, recs)


@pytest.mark.parametrize("n", [9, 64])
def test_wide_batch_session(shape, batch_model, n):
    """9 requests, and 64 at the 0.6B / 2B rows built from four prompts (column independence is test_kernel_column_invariance's)"""
    if n == 64 and shape.name == "8b":
        pytest.skip("64 requests run at the 0.6B and 2B rows")
    base = [(shape.ids(S, 60 + i), k) for i, (S, k) in enumerate([(70, 16), (31, 10), (96, 6), (3, 20), (64, 12), (40, 9), (17, 14),
                                                                    (120, 5), (50, 11)])]
    reqs = base if n == 9 else [base[i % 4] for i in range(64)]
    toks, recs = _run_session(batch_model, reqs, wide=n)
    _check_session(shape, f"wide {n}", reqs, toks, recs)


# ---------------------------------------------------------------------------------------------------------- exact argmax ties
#
# The 0.6B rows with an untied lm_head and the full vocabulary.  Row t of the lm_head (the float64 argmax at a step) is copied into lower
# rows: its logit there is then the same, and the first maximal index must win on every path.  Where the copy goes covers each level of
# the argmax reductions (gemv_kernel at this vocabulary: 4 rows per warp, 32 rows per CTA, 4748 CTAs, whose candidates argmax_final_dev's
# 32 lanes scan 32 apart before their shuffle tree).  One copy goes above t and must lose.

def _plant_rows(level, t, V):
    if level == "lane":        # in the same warp's 4 rows
        return [t & ~3] if t % 4 else [t - 4, t - 3]
    if level == "warp":        # another warp of the same CTA
        return [t - 4 - t % 4] if t % 32 >= 4 else [t - 32, t - 28]
    if level == "cta":         # a neighbouring CTA (argmax_final_dev's shuffle tree)
        return [t - 40]
    if level == "cta32":       # 32 CTAs lower (the same lane of argmax_final_dev's scan)
        return [t - 1024]
    if level == "row0":
        return [0]
    return [t + 37 if t + 37 < V else t + 1]   # "above": must lose


LEVELS = ["lane", "warp", "cta", "cta32", "row0", "above"]
TIE_MARGIN = 1e-3   # the least float64 gap from the tied top to the runner-up: logits are below 8 here, so far above any kernel error


class Ties:
    """an lm_head with planted ties, and the float64 logits of every checked row under it (a copied row's logit is its source's)"""

    def __init__(self, shape):
        self.shape = shape
        self.head = np.array(shape.head)
        self.copies = []        # (rows, source) in the order applied
        self.logit = {}         # row name -> float64 logits under self.head
        self.want = {}          # row name -> (expected id, the ids tied at the top)

    def _add(self, name, h):
        l = self.shape.head64 @ h
        for pos, t in self.copies:
            l[pos] = l[t]
        self.logit[name] = l
        return l

    def watch(self, name, h):
        """a row whose winner must stay as it is now -> that winner"""
        t = int(np.argmax(self._add(name, h)))
        self.want[name] = (t, (t,))
        assert self._consistent(), name
        return t

    def plant(self, name, h, level):
        """copy this row's argmax row of the lm_head to the rows of `level` -> False when no placement keeps every row's winner"""
        t = int(np.argmax(self._add(name, h)))
        for shift in range(0, 8 * 64, 64):
            pos = [p - shift if level != "above" else p for p in _plant_rows(level, t, self.shape.V)]
            if min(pos) < 0 or (level == "above" and shift):
                break
            saved = {k: l[pos].copy() for k, l in self.logit.items()}
            for l in self.logit.values():
                l[pos] = l[t]
            self.want[name] = (min(pos + [t]), tuple(sorted(set(pos + [t]))))
            if self._consistent():
                self.copies.append((pos, t))
                self.head[pos] = self.head[t]
                return True
            for k, l in self.logit.items():
                l[pos] = saved[k]
        self.want.pop(name, None)
        self.logit.pop(name)
        return False

    def _consistent(self):
        """every row has its expected winner, tied only with its own copies, and a margin over the runner-up far above any kernel error"""
        for name, (want, tied) in self.want.items():
            l = self.logit[name]
            m = l.max()
            top = np.flatnonzero(l == m)
            if int(top[0]) != want or tuple(int(i) for i in top) != tied:
                return False
            if m - l[l < m].max() <= TIE_MARGIN:
                return False
        return True


@pytest.fixture(scope="module")
def ties():
    from aha_b200 import synth
    sh = Shape("0.6b untied", dict(_config("0.6b"), tie_word_embeddings=False))
    prompt, steps = sh.ids(PROMPT, 21), sh.ids(STEPS, 22)
    tf = sh.hidden([np.concatenate([prompt, steps])])[0][PROMPT - 1:]
    T = Ties(sh)
    planted_tf = []
    for r in range(len(tf)):
        if T.plant(("tf", r), tf[r], LEVELS[r % len(LEVELS)]):
            planted_tf.append(r)
    # batch requests: the prefill's first token must stay what it is; the tie goes at the first decode step, whose input is that token
    reqs, planted_b = [], []
    for i in range(9):
        p = sh.ids(20 + 9 * i, 30 + i)
        first = T.watch(("prefill", i), sh.hidden([p])[0][-1])
        if T.plant(("b", i), sh.hidden([np.append(p, np.uint32(first))])[0][-1], LEVELS[i % len(LEVELS)]):
            planted_b.append(i)
        reqs.append(p)
    assert len(planted_tf) >= 20 and len(planted_b) >= 8, (planted_tf, planted_b)
    w = dict(sh.w)
    w["lm_head.weight"] = T.head
    sh.w = w
    return sh, T, prompt, steps, planted_tf, reqs, planted_b


@pytest.mark.parametrize("impl", [1, 3, 4])
def test_argmax_ties_single_request(ties, impl):
    sh, T, prompt, steps, planted, _, _ = ties
    m = sh.model(decode_impl=impl, max_ctx=1024)
    try:
        got, am = _teacher_forced(m, prompt, steps)
    finally:
        m.close()
    for r in planted:
        want, tied = T.want[("tf", r)]
        v = got[r, list(tied)]
        assert np.array_equal(v, np.full_like(v, v[0])), (impl, r, tied, v)   # identical rows give identical bits
        assert am[r] == want, (impl, r, am[r], want, tied)


@pytest.mark.parametrize("path", ["narrow 0", "narrow 1", "narrow 2", "wide"])
def test_argmax_ties_batch_sessions(ties, path, monkeypatch):
    sh, T, _, _, _, prompts, planted = ties
    if path.startswith("narrow"):
        monkeypatch.setenv("AHA_BATCH_GEMV", path[-1])
        prompts, planted = prompts[:8], [i for i in planted if i < 8]
    m = sh.model(max_ctx=8192)
    try:
        toks, recs = _run_session(m, [(p, 2) for p in prompts], wide=9 if path == "wide" else 0)
    finally:
        m.close()
    for i in planted:
        want, tied = T.want[("b", i)]
        assert toks[i][0] == T.want[("prefill", i)][0], (path, i)
        assert toks[i][1] == want, (path, i, toks[i][1], want, tied)
        rec = recs[i][1]
        vals = {tid: v for tid, v in zip(rec["top_ids"], rec["top_logprobs"])}
        assert all(t in vals for t in tied[:5]), (path, i, tied, rec["top_ids"])
        v = np.array([vals[t] for t in tied[:5]], np.float32)
        assert np.array_equal(v, np.full_like(v, v[0])), (path, i, tied, v)
