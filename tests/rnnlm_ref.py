"""RecurrentLanguageModel (model/lm.py:31-90) on top of oracle/speech_model.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A functional fp32 restatement of the reference's recurrent LM: embedding -> nn.LSTM (batch_first, gates i, f, g, o) ->
output_project, its label-smoothed loss, and its gradients through autograd.  policy='bf16' rounds where the CUDA path
stores bf16 (x, h, the weights); G_x, the gates and c stay fp32.  Dropout between the layers goes through the oracle's
replay hook (oracle.speech_model.set_dropout) at sites (prefix + 'rnn', layer).  tests/golden/live_ref_rnnlm.pt pins it to
the reference's own module (tests/test_rnnlm_ref.py).
"""
import torch
import torch.nn.functional as F

from oracle import speech_model as om


def lstm_layer(x, h0, c0, w_ih, w_hh, b_ih, b_hh, policy=None):
    """One nn.LSTM layer: x [N, L, I], h0 / c0 [N, H] -> (y [N, L, H], h_n, c_n)."""
    gx = om._r(x, policy) @ om._r(w_ih, policy).t() + b_ih + b_hh
    w = om._r(w_hh, policy)
    h, c, ys = h0, c0, []
    for t in range(x.shape[1]):
        i, f, g, o = (gx[:, t] + om._r(h, policy) @ w.t()).chunk(4, dim=-1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
        h = torch.sigmoid(o) * torch.tanh(c)
        ys.append(h)
    return torch.stack(ys, 1), h, c


def rnn_lm_logits(tokens, sd, prefix, num_layers, hidden=None, policy=None):
    """RecurrentLanguageModel.predict up to the logits: tokens i64 [N, L], hidden (h, c) [layers, N, H] or None
    -> (logits [N, L, V], (h_n, c_n) [layers, N, H]).  The output of every layer but the last passes the dropout hook, as
    nn.LSTM applies `dropout` there in training."""
    x = om._r(sd[prefix + 'embedding.weight'], policy)[tokens]
    N, H = tokens.shape[0], sd[prefix + 'rnn.weight_hh_l0'].shape[1]
    hs, cs = [], []
    for k in range(num_layers):
        h0 = hidden[0][k] if hidden is not None else torch.zeros(N, H)
        c0 = hidden[1][k] if hidden is not None else torch.zeros(N, H)
        y, h, c = lstm_layer(x, h0, c0, *(sd[f'{prefix}rnn.{n}_l{k}'] for n in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh')),
                             policy=policy)
        hs.append(h)
        cs.append(c)
        x = om._drop(prefix + 'rnn', k, om._r(y, policy)) if k + 1 < num_layers else y
    out_w = sd.get(prefix + 'output_project.weight', sd[prefix + 'embedding.weight'])
    logits = om._r(x, policy) @ om._r(out_w, policy).t() + sd[prefix + 'output_project.bias']
    return logits, (torch.stack(hs), torch.stack(cs))


def rnn_lm_predict(tokens, sd, prefix, num_layers, hidden=None, policy=None):
    """RecurrentLanguageModel.predict (model/lm.py:80-86) -> (log-probs [N, L, V], (h_n, c_n))."""
    logits, hidden = rnn_lm_logits(tokens, sd, prefix, num_layers, hidden, policy)
    return F.log_softmax(logits, dim=-1), hidden


def rnn_lm_loss(inputs, targets, sd, prefix, params, policy=None):
    """RecurrentLanguageModel.forward (model/lm.py:62-73): label-smoothed CE of the logits, PAD ignored."""
    logits, _ = rnn_lm_logits(inputs, sd, prefix, params['num_layers'], policy=policy)
    return om.label_smoothing_loss(logits, targets, params['smoothing'])


def rnn_lm_loss_and_grads(inputs, targets, sd, params, policy=None):
    """loss.backward() through autograd -> (loss, {name: grad}) with the reference's names; a tied output_project.weight
    (model/lm.py:54-56) contributes to 'embedding.weight' and has no entry of its own."""
    leaf = {k: v.detach().clone().float().requires_grad_(True) for k, v in sd.items()}
    if params['share_embedding']:
        leaf.pop('output_project.weight', None)
    loss = rnn_lm_loss(inputs, targets, leaf, '', params, policy=policy)
    loss.backward()
    return loss.detach(), {k: v.grad if v.grad is not None else torch.zeros_like(v) for k, v in leaf.items()}
