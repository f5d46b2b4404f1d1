"""Float64 restatement of scoring given text (aha_b200_score; new design: the reference model returns no prompt log-probabilities, so this is
test infrastructure restating the definition in include/aha_b200.h, not a port of reference code).

Record i of a text is the float64 log-softmax of the logits at position i - 1, taken at ids[i].  The oracle's layers give every position's
final hidden state (its per-layer trace keeps all rows; forward() keeps only the last one); the final RMSNorm and the lm_head are restated
here in float64."""
import numpy as np


def head64(hidden, norm, eps, lm_head):
    """pre-norm rows [M, H] -> float64 logits [M, V]"""
    x = np.asarray(hidden, np.float64)
    x = x / np.sqrt((x * x).mean(-1, keepdims=True) + eps) * np.asarray(norm, np.float64)
    return x @ np.asarray(lm_head, np.float64).T


def log_softmax(logits):
    m = logits.max(-1, keepdims=True)
    return logits - (m + np.log(np.exp(logits - m).sum(-1, keepdims=True)))


def oracle_hidden(kind, oracle, ids):
    """-> (pre-norm final hidden state of every position [S, H], final norm gain, eps, lm_head) of a text-only prompt"""
    ids = np.asarray(ids, np.int64).reshape(1, -1)
    oracle.clear_cache()
    if kind == "qwen3":
        oracle.trace = []
        oracle.forward_hidden(ids)
        h, oracle.trace = oracle.trace[-1][0], None
        out = h, oracle.norm, oracle.cfg["rms_norm_eps"], oracle.lm_head
    else:
        t = oracle.text
        t.trace = []
        oracle.forward(ids)
        h, t.trace = t.trace[-1][0], None
        out = h, t.norm, t.tc["rms_norm_eps"], oracle.lm_head
    oracle.clear_cache()
    return out


def score(kind, oracle, ids, start=1):
    """float64 log-softmax rows [S - start, V] at positions start - 1 .. S - 2 and the records' logprobs"""
    h, norm, eps, lm = oracle_hidden(kind, oracle, ids)
    lp = log_softmax(head64(h[start - 1:len(ids) - 1], norm, eps, lm))
    tgt = np.asarray(ids[start:], np.int64)
    return lp, lp[np.arange(len(tgt)), tgt]


def check_top(got_ids, got_lp, ref_rows, tol):
    """every row: the ids of the first k alternatives equal the float64 order wherever the float64 gaps around that rank exceed tol, and
    their logprobs are within tol"""
    k = got_ids.shape[1]
    for r in range(got_ids.shape[0]):
        order = np.argsort(-ref_rows[r], kind="stable")[:k + 1]
        vals = ref_rows[r][order]
        for j in range(k):
            lo_gap = vals[j - 1] - vals[j] if j > 0 else np.inf
            hi_gap = vals[j] - vals[j + 1] if j + 1 < len(vals) else np.inf
            if lo_gap > tol and hi_gap > tol:
                assert got_ids[r, j] == order[j], (r, j, got_ids[r], order)
        assert np.abs(got_lp[r] - ref_rows[r][got_ids[r]]).max(initial=0.0) <= tol, r
