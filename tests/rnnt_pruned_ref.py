"""Pruned RNN-T (DESIGN.md 4.22) restated in float64 on top of tests/rnnt_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

simple_logprobs: the simple joint's node log-probs for logits am[t] + lm[u].  prune_ranges: the range rule, in float32
with the window sums in ascending u so that it matches otb_rnnt_prune_ranges integer for integer.  band_nll: the lattice
loss with every node outside its frame's band removed.  model_loss: the whole pruned objective of a TransducerModel,
simple_loss_scale * L_simple + L_pruned, with the bf16 storage policy of the CUDA path; the bands come from the
restatement's own simple loss and carry no gradient.
"""
import numpy as np
import torch

from oracle import speech_model as om
from tests import rnnt_ref


def simple_logprobs(am, lm, labels):
    """am [T, V], lm [U + 1, V], labels [U] -> (lpb [T, U + 1], lpy [T, U]) of logits am[t] + lm[u]."""
    return rnnt_ref.node_logprobs(am[:, None, :] + lm[None, :, :], labels)


def occupancy(lpb, lpy):
    """Node occupancy [T, U + 1] of one utterance: the posterior probability that an alignment passes through each node,
    i.e. minus the gradient of the nll with respect to the node's two outgoing log-probs."""
    a = lpb.detach().double().clone().requires_grad_(True)
    c = lpy.detach().double().clone().requires_grad_(True)
    rnnt_ref.lattice_nll(a, c).backward()
    occ = -a.grad.clone()
    occ[:, :-1] -= c.grad
    return occ


def prune_ranges(occ, T, U, S):
    """s [T] of one utterance from occ [T, U + 1] (float32): the arg-max window, then the rule of DESIGN.md 4.22."""
    occ = np.asarray(occ, dtype=np.float32)
    s_max = max(0, U + 1 - S)
    s = np.zeros(T, dtype=np.int64)
    for t in range(T):
        best, best_s = np.float32(-np.inf), 0
        for s0 in range(s_max + 1):
            w = np.float32(0.0)
            for u in range(s0, min(s0 + S, U + 1)):
                w = np.float32(w + occ[t, u])
            if w > best:
                best, best_s = w, s0
        s[t] = best_s
    if T < 1:
        return s
    s[0] = 0
    for t in range(1, T):
        s[t] = min(max(s[t], s[t - 1]), s[t - 1] + S - 1)
    s = np.minimum(s, s_max)
    lo = U - S + 1
    for t in range(T - 1, -1, -1):
        s[t] = max(s[t], lo)
        lo = s[t] - (S - 1)
    return s


def check_ranges(s, T, U, S):
    """The constraints the rule guarantees when U <= T (S - 1) -> list of the violated ones."""
    bad = []
    if T < 1:
        return bad
    s_max = max(0, U + 1 - S)
    if s[0] != 0:
        bad.append('s_0 = 0')
    if any(s[t + 1] < s[t] for t in range(T - 1)):
        bad.append('non-decreasing')
    if any(s[t + 1] > s[t] + S - 1 for t in range(T - 1)):
        bad.append('overlap')
    if any(x > s_max for x in s):
        bad.append('s_t <= max(0, U + 1 - S)')
    if s[T - 1] < U - S + 1:
        bad.append('the last band holds U')
    return bad


def band_mask(s, T, U1, S):
    """[T, U1] bool: node (t, u) exists when s_t <= u < s_t + S."""
    u = torch.arange(U1)[None, :]
    st = torch.as_tensor(np.asarray(s))[:, None]
    return (u >= st) & (u < st + S)


def band_nll(lpb, lpy, s, S):
    """-log of the sum over the alignments that stay inside the bands (+inf when none does): alpha over the band nodes
    only, node by node (the -inf of a missing node never enters a sum, so autograd stays finite)."""
    T, U1 = lpb.shape
    ninf = torch.tensor(float('-inf'), dtype=lpb.dtype)
    prev = {}
    for t in range(T):
        cur = {}
        for u in range(int(s[t]), min(int(s[t]) + S, U1)):
            terms = []
            if t == 0 and u == 0:
                terms.append(torch.zeros((), dtype=lpb.dtype))
            if u in prev and float(prev[u].detach()) > float('-inf'):
                terms.append(prev[u] + lpb[t - 1, u])
            if u - 1 in cur and float(cur[u - 1].detach()) > float('-inf'):
                terms.append(cur[u - 1] + lpy[t, u - 1])
            cur[u] = torch.logsumexp(torch.stack(terms), 0) if terms else ninf
        prev = cur
    if float(prev.get(U1 - 1, ninf).detach()) == float('-inf'):
        return -ninf
    return -(prev[U1 - 1] + lpb[T - 1, U1 - 1])


def has_complete_path(s, T, U, S):
    """Is there a monotone path (0, 0) -> (T - 1, U) through the band nodes (blank: t + 1, label: u + 1)?"""
    keep = band_mask(s, T, U + 1, S).numpy()
    reach = np.zeros((T, U + 1), dtype=bool)
    for t in range(T):
        for u in range(U + 1):
            if not keep[t, u]:
                continue
            reach[t, u] = (t == 0 and u == 0) or (t > 0 and reach[t - 1, u]) or (u > 0 and reach[t, u - 1])
    return bool(reach[T - 1, U])


# ------------------------------------------------------------------------------------------------ the whole model
def model_loss(x, mask, truth, truth_length, sd, params, drop=None, policy='bf16', bands=None, record=None):
    """The pruned objective simple_loss_scale * L_simple + L_pruned of a TransducerModel with joint prune_range S ->
    (loss, new BatchNorm running statistics).  bands (per utterance, its s over its frames) replaces the restatement's own
    ranges; record (a list) receives the restatement's own ranges."""
    S = params['joint']['prune_range']
    alpha = params['joint'].get('simple_loss_scale', 0.5)
    memory, mmask, stats = rnnt_ref._encode_train(x, mask, sd, params, drop, policy)
    labels = truth[:, 1:-1]
    tokens = torch.cat((torch.zeros(truth.shape[0], 1, dtype=torch.long), labels), dim=1)
    om.set_dropout(drop)
    try:
        g = rnnt_ref.predictor(tokens, sd, params['decoder'].get('num_layers', 1), policy)
    finally:
        om.set_dropout(None)
    am = om.linear(memory, sd, 'joint.simple_am_proj', policy)
    lm = om.linear(g, sd, 'joint.simple_lm_proj', policy)
    logits = rnnt_ref.joint_logits(memory, g, sd, policy)
    t_len, u_len = mmask.sum(-1), truth_length - 1
    simple, pruned = [], []
    for b in range(x.shape[0]):
        T, U = int(t_len[b]), int(u_len[b])
        lb = labels[b, :U].long()
        lpb, lpy = simple_logprobs(am[b, :T], lm[b, :U + 1], lb)
        simple.append(rnnt_ref.lattice_nll(lpb, lpy))
        s = prune_ranges(occupancy(lpb, lpy).float().numpy(), T, U, S)
        if record is not None:
            record.append(s)
        if bands is not None:
            s = bands[b]
        fb, fy = rnnt_ref.node_logprobs(logits[b, :T, :U + 1], lb)
        pruned.append(band_nll(fb, fy, s, S))
    return alpha * torch.stack(simple).mean() + torch.stack(pruned).mean(), stats


def loss_and_grads(x, mask, truth, truth_length, sd, params, drop=None, bands=None, record=None):
    """-> (loss, {name: grad or None}, new running statistics), through autograd."""
    leaf = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and 'running_' not in k) for k, v in sd.items()}
    loss, stats = model_loss(x, mask, truth, truth_length, leaf, params, drop, bands=bands, record=record)
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in leaf.items() if v.requires_grad}, stats
