"""Reference for the token log-probability records (new design: the reference model's responses carry no log-probabilities, so this is
test infrastructure restating the definition in include/aha_b200.h, not a port of reference code).

logprobs(logits, token, n): the float64 log-softmax of the fp32 row at `token`, and the n largest entries ordered by
(fp32 logit descending, id ascending) with their float64 log-probabilities."""
import numpy as np


def log_softmax64(logits):
    x = np.asarray(logits, np.float32).reshape(-1).astype(np.float64)
    m = x.max()
    return x - (m + np.log(np.exp(x - m).sum()))


def top_order(logits, n):
    """ids of the n largest fp32 logits, by (logit desc, id asc): a stable sort on the negated row."""
    x = np.asarray(logits, np.float32).reshape(-1)
    return np.argsort(-x, kind="stable")[:n]


def logprobs(logits, token, n):
    """-> (logprob of token, top ids, their logprobs), all from the float64 log-softmax of the fp32 row."""
    lp = log_softmax64(logits)
    ids = top_order(logits, n)
    return float(lp[int(token)]), [int(i) for i in ids], [float(lp[i]) for i in ids]
