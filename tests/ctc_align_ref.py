"""CTC forced alignment on the CPU -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

  - viterbi_align: the recursion of otb_ctc_align (csrc/ctc_align.cu) with its tie-break, in numpy, float32 by default
    (the kernel's arithmetic: each step is one max and one IEEE add, so the results are bit-identical) or float64.
  - best_alignment: every alignment of a tiny problem enumerated, in float64.
  - torchaudio_align: torchaudio.functional.forced_align + merge_tokens for one utterance, in the same output layout.
"""
import itertools

import numpy as np
import torch

NEG_INF = float('-inf')


def viterbi_align(lp, tokens, n_frames=None, blank=0, dtype=np.float32):
    """lp [T, V] log-probs of one utterance (numpy or torch), tokens: the target (a sequence of ints), n_frames: the valid
    frames (default T).  -> (labels int32 [T], frame_scores [T], spans int32 [L, 2], path_score), with the kernel's rules:

      state s of l' = blank (even s) or tokens[s // 2] (odd s); delta_{-1}(0) = 0, every other delta_{-1} = -inf;
      delta_t(s) = max over (stay, one back, two back if l'_s is a token other than l'_{s-2}) + lp_t(l'_s), where a later
      choice wins only when strictly better; the end is state S-1 unless delta(S-2) is strictly better.
    Frames at or past n_frames get label -1 and score -inf.  An utterance without an alignment of finite log-prob (too few
    frames, a blank or out-of-range token, no frames for a non-empty target) gets path_score -inf, labels -1, spans -1;
    an empty target with no frames has path_score 0."""
    lp = np.asarray(lp.cpu() if isinstance(lp, torch.Tensor) else lp, dtype=dtype)
    T, V = lp.shape
    Tb = T if n_frames is None else max(0, min(int(n_frames), T))
    tokens = [int(v) for v in tokens]
    L, S = len(tokens), 2 * len(tokens) + 1
    labels = np.full(T, -1, np.int32)
    scores = np.full(T, NEG_INF, dtype)
    spans = np.full((L, 2), -1, np.int32)
    if any(v < 0 or v >= V or v == blank for v in tokens) or (L > 0 and Tb == 0):
        return labels, scores, spans, dtype(NEG_INF)
    if Tb == 0:
        return labels, scores, spans, dtype(0.0)
    lab = np.full(S, blank, np.int64)
    lab[1::2] = tokens
    skip = np.zeros(S, bool)
    skip[3::2] = lab[3::2] != lab[1:-2:2]
    neg = dtype(NEG_INF)
    d = np.full(S, neg, dtype)
    d[0] = 0
    bp = np.zeros((Tb, S), np.int8)
    for t in range(Tb):
        x1 = np.concatenate(([neg], d[:-1]))
        x2 = np.where(skip, np.concatenate(([neg, neg], d))[:S], neg)
        best, c = d.copy(), np.zeros(S, np.int8)
        m1 = x1 > best
        best[m1], c[m1] = x1[m1], 1
        m2 = x2 > best
        best[m2], c[m2] = x2[m2], 2
        d = (best + lp[t, lab]).astype(dtype)
        bp[t] = c
    e = S - 1 if S == 1 or not d[S - 2] > d[S - 1] else S - 2
    score = d[e]
    if not score > NEG_INF:
        return labels, scores, spans, dtype(NEG_INF)
    states = np.empty(Tb, np.int64)
    s = e
    for t in range(Tb - 1, -1, -1):
        states[t] = s
        s -= int(bp[t, s])
    labels[:Tb] = lab[states]
    scores[:Tb] = lp[np.arange(Tb), lab[states]]
    for i in range(L):
        where = np.nonzero(states == 2 * i + 1)[0]
        spans[i] = (where[0], where[-1] + 1)
    return labels, scores, spans, score


def collapse(path, blank=0):
    out, prev = [], None
    for k in path:
        if k != prev and k != blank:
            out.append(k)
        prev = k
    return out


def best_alignment(lp, tokens, blank=0):
    """max over every frame labelling that collapses to tokens of its summed log-prob, float64 (-inf when none does)."""
    lp = np.asarray(lp, np.float64)
    T, V = lp.shape
    best = NEG_INF
    for path in itertools.product(range(V), repeat=T):
        if collapse(path, blank) == list(tokens):
            best = max(best, float(sum(lp[t, k] for t, k in enumerate(path))))
    return best


def torchaudio_align(lp, tokens, blank=0):
    """torchaudio's forced_align (one utterance, lp [T, V] float32 on any device) -> (labels int32 [T], frame_scores [T],
    spans int32 [L, 2] from merge_tokens), on the CPU.  torchaudio refuses an empty target; its one alignment, all blank,
    is returned for it."""
    import torchaudio.functional as AF
    T = lp.shape[0]
    if not len(tokens):
        return np.full(T, blank, np.int32), lp[:, blank].cpu().numpy(), np.zeros((0, 2), np.int32)
    tg = torch.tensor([list(tokens)], dtype=torch.int32, device=lp.device)
    labels, scores = AF.forced_align(lp[None].contiguous(), tg, torch.tensor([T], device=lp.device),
                                     torch.tensor([len(tokens)], device=lp.device), blank=blank)
    labels, scores = labels[0].cpu(), scores[0].cpu()
    spans = [(sp.start, sp.end) for sp in AF.merge_tokens(labels, scores, blank=blank)]
    return labels.numpy().astype(np.int32), scores.numpy(), np.array(spans, np.int32).reshape(-1, 2)


def tokens_with_repeats(L, V, g, p_repeat=0.3):
    """L tokens in 1..V-1 (never the blank 0), each a repeat of the one before with probability p_repeat."""
    out = []
    for i in range(L):
        if i and float(torch.rand((), generator=g)) < p_repeat:
            out.append(out[-1])
        else:
            out.append(int(torch.randint(1, V, (), generator=g)))
    return out


def min_frames(tokens):
    """The fewest frames an alignment needs: one per token plus a blank between adjacent repeats."""
    return len(tokens) + sum(1 for a, b in zip(tokens, tokens[1:]) if a == b)
