"""CTC rescoring of the attention n-best (DESIGN.md 4.18) restated in float64 -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The CTC score of a target row is log p_ctc(labels | x) = -F.ctc_loss(reduction='none', zero_infinity=False) on the head's
log-softmax over the utterance's valid frames, one row at a time; it is -inf where no alignment exists, and also for a
label equal to the blank or outside [0, V) and for an utterance without frames.  A hypothesis y is scored on y <S/E>.

The re-ranking is tests/rescore_ref.py's with the CTC score as one more second-pass model whose token log-probs are the
score at position 0: s = s1 + weight * (the other models' sums + the CTC score).  A hypothesis whose CTC score is -inf
scores -inf whatever the weight, so it ranks after every hypothesis with an alignment, in first-pass order.
"""
import torch
import torch.nn.functional as F

from tests import rescore_ref as rr

NEG_INF = rr.NEG_INF


def ctc_score(logp, labels, blank=0):
    """logp [n_frames, V] log-probs of an utterance's valid frames, labels a list of ints -> float64 log p_ctc(labels)."""
    n_frames, V = logp.shape
    if n_frames == 0 or any(l == blank or not 0 <= l < V for l in labels):
        return NEG_INF
    nll = F.ctc_loss(logp.double()[:, None], torch.tensor([labels], dtype=torch.long), [n_frames], [len(labels)], blank=blank,
                     reduction='none', zero_infinity=False)
    return -float(nll[0])


def row_labels(row):
    """A target row as the kernel reads it: the entries before the first negative one."""
    labels = []
    for v in row:
        if int(v) < 0:
            break
        labels.append(int(v))
    return labels


def nbest_scores(logp, B, T, in_len, targets, blank=0):
    """The kernel's contract: logp [B*T, V], in_len [B], targets [B, K, Lp] -> float64 [B, K]."""
    lp = logp.double().view(B, T, -1)
    K = targets.shape[1]
    out = torch.empty(B, K, dtype=torch.float64)
    for b in range(B):
        n = max(0, min(int(in_len[b]), T))
        for k in range(K):
            out[b, k] = ctc_score(lp[b, :n], row_labels(targets[b, k]), blank)
    return out


def rerank(hyps, s1, other_tok_lps, ctc, weight, nbest, dtype=torch.float64):
    """One utterance: hyps K cut hypotheses in first-pass order, s1 their first-pass scores, other_tok_lps[k] the token
    log-prob sequences of the other second-pass models (LM) for hyps[k] <S/E>, ctc[k] its CTC score.  -> rescore_ref.rerank's
    nbest (k, y, s)."""
    s1 = [NEG_INF if c == NEG_INF else s for s, c in zip(s1, ctc)]
    tok = [list(other_tok_lps[k]) + [torch.tensor([0.0 if c == NEG_INF else c], dtype=torch.float64)] for k, c in enumerate(ctc)]
    return rr.rerank(hyps, s1, tok, weight, nbest, dtype)
