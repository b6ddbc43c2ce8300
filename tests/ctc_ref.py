"""The CTC-only model and CTC decoding on the CPU -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

  - ctc_model_loss / loss_and_grads_train: CTCModel.forward (model/ctc.py:83-96) in train(): the oracle's front end and
    encoder (oracle/speech_model.py; a Conformer through tests/conformer_train_ref.py's training-mode BatchNorm), the
    oracle's ctc_loss on truth[:, 1:-1] with targets_length - 1 labels.  `drop(site, t)` replays the residual dropout.
  - greedy_collapse: recognize_greedy (recognize/ctc.py:38-58), exactly as the reference loops.
  - prefix_beam_search: the CTC prefix beam search of otb_ctc_prefix_beam, in float64, with its tie-break spelled out.
  - prefix_marginals: every alignment enumerated, for tiny T and V.
tests/golden/live_ref_ctc.pt pins the first two to the reference's own modules.
"""
import itertools
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import speech_model as om
from tests import conformer_train_ref as ctr

NEG_INF = float('-inf')


def ctc_model_loss(x, mask, truth, truth_length, sd, params, drop=None, policy=None):
    """-> (loss, new BatchNorm running statistics {} for a Transformer encoder)."""
    new_stats = {}
    if params['encoder_type'] == 'conformer':
        with ctr.train_mode(new_stats, drop):
            memory, mmask = om.encode(x, mask, sd, params, policy)
    else:
        om.set_dropout(drop)
        try:
            memory, mmask = om.encode(x, mask, sd, params, policy)
        finally:
            om.set_dropout(None)
    loss = om.ctc_loss(memory, mmask, truth[:, 1:-1], truth_length - 1, sd, policy=policy)
    return loss, new_stats


def loss_and_grads_train(x, mask, truth, truth_length, sd, params, drop=None):
    """-> (loss, {name: grad or None}, new running statistics); a Conformer's post_ffn.* gets None, as in the reference."""
    leaf = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and 'running_' not in k) for k, v in sd.items()}
    loss, stats = ctc_model_loss(x, mask, truth, truth_length, leaf, params, drop)
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in leaf.items() if v.requires_grad}, stats


def log_probs(x, mask, sd, params, policy=None):
    """CTCModel.inference as the port defines it: front end + encoder (eval) + head -> (log-probs [B, T', V], lengths [B])."""
    memory, mmask = om.encode(x, mask, sd, params, policy)
    logits = om.linear(memory, sd, 'assistor.output_layer', policy)
    return F.log_softmax(logits, dim=-1), mmask.sum(dim=-1)


def greedy_collapse(best, length):
    """recognize_greedy's loop over the best token of each frame (recognize/ctc.py:46-56): PAD / blank (0) and a repeat of
    the previous frame's token are dropped; last_k moves on every frame."""
    pred, last_k = [], 0
    for i in range(int(length)):
        k = int(best[i])
        if k == last_k or k == 0:
            last_k = k
            continue
        last_k = k
        pred.append(k)
    return pred


def log_add(a, b):
    """csrc/ctc.cu's log-add, m + log1p(exp(min - m)), in float64 -- or in float32 for np.float32 operands."""
    if a == NEG_INF:
        return b
    if b == NEG_INF:
        return a
    m = max(a, b)
    if isinstance(m, np.float32):
        return m + np.log1p(np.exp(min(a, b) - m))
    return m + math.log1p(math.exp(min(a, b) - m))


def frame_topk(row, K):
    """The K best (id, log-prob) of one frame, best first, ties to the lower id (otb_ctc_frame_topk)."""
    row = [float(v) for v in row]
    return [(i, row[i]) for i in sorted(range(len(row)), key=lambda i: (-row[i], i))[:K]]


def prefix_beam_search(frames, beam, blank=0, fp32=False):
    """CTC prefix beam search over frames = [[(id, log-prob), ...] per valid frame] (each frame's top-K, best first).
    -> [(tokens tuple, log(p_b + p_nb))] best first, at most `beam` entries.

    The beam starts as the empty prefix with p_b = 0, p_nb = -inf.  Per frame, with slot i = (P_i, p_b, p_nb) and
    tot_i = logaddexp(p_b, p_nb):
      keep P_i:        p_b' = tot_i + lp(blank);  p_nb' = p_nb + lp(last(P_i)), plus, when P_i minus its last token c is
                       slot p, the extension of slot p by c (from p_b of slot p if c repeats last(P_p), else from tot_p);
      extend P_i by c: (c not blank, P_i + c not in the beam) p_nb' = (c == last(P_i) ? p_b : tot_i) + lp(c).
    A missing log-prob (a token outside the frame's top-K) is -inf.  Candidate j = i (K + 1) + r -- r = 0 keeps slot i,
    r = 1 + k extends it by the frame's k-th token -- and the beam keeps the `beam` best candidates by (score descending,
    j ascending), dropping -inf; the slots of the next frame are in that order.
    fp32=True runs the arithmetic in float32, as the kernel does (IEEE sums are then the kernel's; exp / log1p may differ
    by an ulp), so that near-equal candidates are ranked alike."""
    num = np.float32 if fp32 else float
    cur = [((), num(0.0), num(NEG_INF))]
    for cands in frames:
        lp = {}
        for c, v in cands:
            lp.setdefault(int(c), num(v))
        S = len(cands) + 1
        slot = {P: i for i, (P, _, _) in enumerate(cur)}
        scored = []
        blank_lp = lp.get(blank, num(NEG_INF))
        for i, (P, pb, pnb) in enumerate(cur):
            tot = log_add(pb, pnb)
            last = P[-1] if P else -1
            rep = lp.get(last, num(NEG_INF))
            npb = tot + blank_lp if blank_lp != NEG_INF else num(NEG_INF)
            npnb = pnb + rep if (rep != NEG_INF and pnb != NEG_INF) else num(NEG_INF)
            if P and P[:-1] in slot and rep != NEG_INF:
                Pp, ppb, ppnb = cur[slot[P[:-1]]]
                frm = ppb if (Pp[-1] if Pp else -1) == last else log_add(ppb, ppnb)
                if frm != NEG_INF:
                    npnb = log_add(npnb, frm + rep)
            scored.append((log_add(npb, npnb), i * S, P, npb, npnb))
            for r, (c, v) in enumerate(cands):
                c = int(c)
                if c == blank or c < 0 or P + (c,) in slot:
                    continue
                frm = pb if c == last else tot
                sc = frm + num(v) if frm != NEG_INF else num(NEG_INF)
                scored.append((sc, i * S + 1 + r, P + (c,), num(NEG_INF), sc))
        scored = sorted((s for s in scored if s[0] != NEG_INF), key=lambda s: (-s[0], s[1]))
        cur = [(P, pb, pnb) for _, _, P, pb, pnb in scored[:beam]]
    return [(P, float(log_add(pb, pnb))) for P, pb, pnb in cur]


def prefix_marginals(lp, blank=0):
    """{prefix: log of the summed probability of every alignment that collapses to it} for lp [T, V] (float64)."""
    T, V = len(lp), len(lp[0])
    out = {}
    for path in itertools.product(range(V), repeat=T):
        s = sum(float(lp[t][k]) for t, k in enumerate(path))
        pref, prev = [], None
        for k in path:
            if k != prev and k != blank:
                pref.append(k)
            prev = k
        key = tuple(pref)
        out[key] = log_add(out.get(key, NEG_INF), s)
    return out


def synth_log_probs(T, V, seed, scale=3.0):
    """Tie-free log-probs [T, V] (float32) for the search tests."""
    g = torch.Generator().manual_seed(seed)
    return torch.log_softmax(scale * torch.randn(T, V, generator=g), dim=-1)
