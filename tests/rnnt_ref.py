"""The transducer (RNN-T) lattice and TransducerModel on top of oracle/speech_model.py -- TEST INFRASTRUCTURE, NOT PRODUCT
CODE.

lattice_nll restates the loss of one utterance in float64 from its definition: alpha over the [T, U + 1] lattice (a blank
moves t on, label y_{u+1} moves u on), nll = -(alpha(T - 1, U) + log p(blank | T - 1, U)); its gradient comes from
autograd.  Each row of alpha is one logcumsumexp, so lattices of 1023 labels stay cheap.  enumerate_nll sums every
alignment explicitly (small lattices).  model_loss is the whole TransducerModel in fp32 with the bf16 storage policy of the
CUDA path (policy='bf16': the encoder's, the prediction network's (tests/rnnlm_ref.py) and the joint's operands rounded
where the kernels store bf16), in training mode with the product's dropout masks replayed.
"""
import itertools

import torch
import torch.nn.functional as F

from oracle import speech_model as om
from tests import conformer_train_ref as ctr
from tests import rnnlm_ref

BLANK = 0


def lattice_alpha(lpb, lpy):
    """lpb [T, U + 1] log p(blank) and lpy [T, U] log p(y_{u+1}) of each node -> alpha [T, U + 1]."""
    T, U1 = lpb.shape
    rows = []
    prev = None
    zero = torch.zeros(1, dtype=lpb.dtype)
    for t in range(T):
        # S[u] = sum_{k < u} lpy[t, k]; alpha[t, u] = S[u] + logsumexp_{u' <= u} (entry[u'] - S[u'])
        S = torch.cat((zero, torch.cumsum(lpy[t], 0)))
        if prev is None:
            entry = torch.cat((zero, torch.full((U1 - 1,), float('-inf'), dtype=lpb.dtype)))
        else:
            entry = prev + lpb[t - 1]
        prev = S + torch.logcumsumexp(entry - S, 0)
        rows.append(prev)
    return torch.stack(rows)


def lattice_nll(lpb, lpy):
    """-log P(y | x) of one utterance: every alignment of its lattice summed, ending in blank at (T - 1, U)."""
    return -(lattice_alpha(lpb, lpy)[-1, -1] + lpb[-1, -1])


def enumerate_nll(lpb, lpy):
    """The same by listing the alignments: the U labels placed among the first T + U - 1 symbols, blanks elsewhere."""
    T, U1 = lpb.shape
    U = U1 - 1
    total = []
    for pos in itertools.combinations(range(T + U - 1), U):
        t = u = 0
        s = 0.0
        for i in range(T + U - 1):
            if i in pos:
                s = s + lpy[t, u]
                u += 1
            else:
                s = s + lpb[t, u]
                t += 1
        total.append(s + lpb[T - 1, U])
    return -torch.logsumexp(torch.stack(total), 0)


def node_logprobs(logits, labels):
    """logits [T, U + 1, V] of one utterance and its labels [U] -> (lpb [T, U + 1], lpy [T, U])."""
    lp = F.log_softmax(logits, dim=-1)
    U = labels.shape[0]
    lpy = lp[:, :U, :].gather(2, labels.view(1, U, 1).expand(lp.shape[0], U, 1)).squeeze(2)
    return lp[..., BLANK], lpy


def batch_loss(logits, labels, t_len, u_len):
    """torchaudio.functional.rnnt_loss(logits [B, T, U + 1, V], labels, t_len, u_len, blank 0, reduction 'mean')."""
    out = []
    for b in range(logits.shape[0]):
        T, U = int(t_len[b]), int(u_len[b])
        lpb, lpy = node_logprobs(logits[b, :T, :U + 1], labels[b, :U].long())
        out.append(lattice_nll(lpb, lpy))
    return torch.stack(out).mean()


# ------------------------------------------------------------------------------------------------ the whole model
def _encode_train(x, mask, sd, params, drop, policy):
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
    return memory, mmask, new_stats


def predictor(tokens, sd, num_layers, policy=None):
    """The prediction network over tokens [B, U + 1] = [BLK, y] -> g [B, U + 1, H] (its dropout at ('decoder.rnn', k))."""
    x = om._r(sd['decoder.embedding.weight'], policy)[tokens]
    B, H = tokens.shape[0], sd['decoder.rnn.weight_hh_l0'].shape[1]
    for k in range(num_layers):
        y, _, _ = rnnlm_ref.lstm_layer(x, torch.zeros(B, H), torch.zeros(B, H),
                                       *(sd[f'decoder.rnn.{n}_l{k}'] for n in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh')),
                                       policy=policy)
        x = om._drop('decoder.rnn', k, om._r(y, policy)) if k + 1 < num_layers else y
    return x


def joint_logits(memory, g, sd, policy=None):
    """memory [B, T', d], g [B, U + 1, H] -> logits [B, T', U + 1, V] of the joint network."""
    ep = om._r(om.linear(memory, sd, 'joint.enc_proj', policy), policy)
    pp = om._r(om.linear(g, sd, 'joint.dec_proj', policy, bias=False), policy)
    hj = torch.tanh(ep[:, :, None, :] + pp[:, None, :, :])
    return om.linear(hj, sd, 'joint.output_layer', policy)


def model_loss(x, mask, truth, truth_length, sd, params, drop=None, policy='bf16'):
    """TransducerModel's training loss -> (loss, new BatchNorm running statistics)."""
    memory, mmask, stats = _encode_train(x, mask, sd, params, drop, policy)
    labels = truth[:, 1:-1]
    tokens = torch.cat((torch.zeros(truth.shape[0], 1, dtype=torch.long), labels), dim=1)
    om.set_dropout(drop)
    try:
        g = predictor(tokens, sd, params['decoder'].get('num_layers', 1), policy)
    finally:
        om.set_dropout(None)
    logits = joint_logits(memory, g, sd, policy)
    return batch_loss(logits, labels, mmask.sum(-1), truth_length - 1), stats


def loss_and_grads(x, mask, truth, truth_length, sd, params, drop=None):
    """-> (loss, {name: grad or None}, new running statistics), through autograd."""
    leaf = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and 'running_' not in k) for k, v in sd.items()}
    loss, stats = model_loss(x, mask, truth, truth_length, leaf, params, drop)
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in leaf.items() if v.requires_grad}, stats


def encode_eval(x, mask, sd, params, policy='bf16'):
    """Front end + encoder in eval mode -> (memory [B, T', d], lengths [B])."""
    memory, mmask = om.encode(x, mask, sd, params, policy)
    return memory, mmask.sum(-1)
