"""Minimum word error rate training (DESIGN.md 4.11) restated in float64 -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

For utterance b: the reference r_b is truth[b, 1 : truth_length[b]] (the transcript between BOS and its closing <S/E>).
Its K hypotheses are n-best rows cut at their first <S/E> (rescore_ref.cut); a hypothesis equal to one ranked higher is
dropped.  W_k = Levenshtein distance (unit costs) between y_k and r_b.  l_k = sum over the n_k + 1 positions of
log_softmax(logits)[t, y'_t], y' = y <S/E>.  Over the kept k: P = softmax(l), L_b = sum_k P_k (W_k - mean W), and the
whole loss is mean_b L_b + lambda * L_CE.  dL/dl_k = P_k (W_k - sum_j P_j W_j) / B.
"""
import torch

from tests.rescore_ref import EOS, cut, token_logprobs  # noqa: F401  (re-exported for the tests)


def edit_distance(a, b):
    """The textbook Levenshtein DP over two token lists."""
    a, b = list(a), list(b)
    prev = list(range(len(b) + 1))
    for i in range(1, len(a) + 1):
        cur = [i] + [0] * len(b)
        for j in range(1, len(b) + 1):
            cur[j] = min(prev[j] + 1, cur[j - 1] + 1, prev[j - 1] + (a[i - 1] != b[j - 1]))
        prev = cur
    return prev[-1]


def reference(truth_row, truth_length):
    """truth[b, 1 : truth_length[b]] as a list."""
    return [int(v) for v in truth_row[1:int(truth_length)]]


def kept(hyps):
    """The rescoring rule: hypothesis k is kept unless it equals one of a lower k."""
    return [all(list(hyps[j]) != list(hyps[k]) for j in range(k)) for k in range(len(hyps))]


def utterance_loss(l, W, keep):
    """L_b = sum_k P_k (W_k - mean W) over the kept hypotheses, differentiable in l (float64 [K])."""
    idx = torch.tensor([k for k in range(len(keep)) if keep[k]])
    lk = l[idx]
    Wk = torch.as_tensor(W, dtype=torch.float64)[idx]
    P = torch.softmax(lk, dim=0)
    return (P * (Wk - Wk.mean())).sum()


def coefficients(l, W, keep, scale=1.0):
    """The closed form dL_b/dl_k * scale = P_k (W_k - sum_j P_j W_j) * scale, 0 for a dropped k (float64 [K]), written with
    W centred on its mean over the kept k, as the kernel forms it: exactly 0 when every kept W is the same."""
    l = torch.as_tensor(l, dtype=torch.float64)
    W = torch.as_tensor(W, dtype=torch.float64)
    m = torch.tensor(keep)
    P = torch.zeros_like(l)
    P[m] = torch.softmax(l[m], dim=0)
    dw = torch.where(m, W - W[m].mean(), torch.zeros_like(W))
    return P * (dw - (P * dw).sum()) * scale


def sequence_logprob(tok_lp, n):
    """l = the sum of the n + 1 token log-probs of y <S/E> (float64)."""
    return torch.as_tensor(tok_lp, dtype=torch.float64)[:n + 1].sum()


def batch_loss(tok_lp, hyps, refs):
    """mean_b L_b from float64 token log-probs [B, K, >= max n + 1] (differentiable), the hypotheses (lists [B][K]) and the
    references (lists [B])."""
    B = len(hyps)
    total = torch.zeros((), dtype=torch.float64)
    for b in range(B):
        W = [edit_distance(y, refs[b]) for y in hyps[b]]
        l = torch.stack([tok_lp[b, k, :len(y) + 1].sum() for k, y in enumerate(hyps[b])])
        total = total + utterance_loss(l, W, kept(hyps[b]))
    return total / B


def error_counts(nbest, ref):
    """eval.py's counts for one utterance: (errors of the first hypothesis, fewest errors in the n-best, len(ref))."""
    e = [edit_distance(y, ref) for y in nbest]
    return e[0], min(e), len(ref)
