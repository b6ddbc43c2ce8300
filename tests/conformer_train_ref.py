"""SpeechToText with a Conformer encoder in train(), on top of oracle/speech_model.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The oracle restates the reference's forward in eval mode.  Training differs inside the Conformer block only:
  - nn.BatchNorm1d of the convolution module (module/conformer.py:51) normalises with the batch statistics over all B*T'
    positions (padded frames included) and updates running_mean / running_var (momentum 0.1, unbiased variance);
  - the three residual-dropout sites of each block (encoder/conformer.py:53,58,63) apply a mask.  torch's Philox masks cannot
    be reproduced, so `drop((block prefix, k), t)` replays the product's masks (k = 0 macaron feed-forward, 1 attention,
    2 conv module), as oracle.speech_model.set_dropout does for the Transformer layers.
The block itself is the oracle's own `conformer_block` / `conformer_encoder`: for the duration of the encoder call, the three
sub-layer functions it looks up are wrapped -- the conv module by its training-mode version below, and each sub-layer output
by the dropout replay.  tests/golden/live_ref_conformer_train.pt pins the result to the reference's own modules in train().
"""
import contextlib

import torch.nn.functional as F

from oracle import speech_model as om


def conv_module_train(x, mask, sd, prefix, new_stats, momentum=0.1, eps=1e-5):
    """oracle.conformer_conv_module with BatchNorm in train mode; the updated running statistics go to
    new_stats[prefix + '.batch_norm.running_*']."""
    m = mask.unsqueeze(2)
    y = F.glu(om.linear(x, sd, prefix + '.pointwise_conv1')).masked_fill(~m, 0.0)
    w = sd[prefix + '.depthwise_conv.weight']
    y = F.conv1d(y.transpose(1, 2), w, sd.get(prefix + '.depthwise_conv.bias'), padding=(w.shape[-1] - 1) // 2, groups=w.shape[0])
    bn = prefix + '.batch_norm'
    rm, rv = sd[bn + '.running_mean'].detach().clone(), sd[bn + '.running_var'].detach().clone()
    y = F.batch_norm(y, rm, rv, sd[bn + '.weight'], sd[bn + '.bias'], True, momentum, eps)
    new_stats[bn + '.running_mean'], new_stats[bn + '.running_var'] = rm, rv
    y = y * F.sigmoid(y)
    y = om.linear(y.transpose(1, 2), sd, prefix + '.pointwise_conv2')
    return y.masked_fill(~m, 0.0)


@contextlib.contextmanager
def train_mode(new_stats, drop=None):
    """Run oracle.conformer_block in train(): training-mode BatchNorm and the residual-dropout replay."""
    ffn, mha, conv = om.ffn, om.mha_self_relpos, om.conformer_conv_module
    dr = drop if drop is not None else (lambda site, t: t)

    def block(prefix):
        return prefix.rsplit('.', 1)[0]

    def ffn_train(x, sd, prefix, activation, policy=None):
        y = ffn(x, sd, prefix, activation, policy)
        return dr((block(prefix), 0), y) if prefix.endswith('.pre_ffn') else y

    def mha_train(x, mask, pos, sd, prefix, n_heads, policy=None):
        a, w = mha(x, mask, pos, sd, prefix, n_heads, policy)
        return dr((block(prefix), 1), a), w

    def conv_train(x, mask, sd, prefix, policy=None, bn_eps=1e-5):
        return dr((block(prefix), 2), conv_module_train(x, mask, sd, prefix, new_stats, eps=bn_eps))

    om.ffn, om.mha_self_relpos, om.conformer_conv_module = ffn_train, mha_train, conv_train
    try:
        yield
    finally:
        om.ffn, om.mha_self_relpos, om.conformer_conv_module = ffn, mha, conv


def loss_train(x, mask, truth, sd, params, truth_length=None, drop=None):
    """SpeechToText.forward in train() with a rel-pos Conformer encoder -> (loss, new running statistics).
    drop(site, tensor) -> tensor replays the residual dropout (site = ('encoder.blocks.i', k) or ('decoder.blocks.i', k))."""
    new_stats = {}
    with train_mode(new_stats, drop):
        memory, mmask = om.encode(x, mask, sd, params)
    om.set_dropout(drop)
    try:
        logits = om.transformer_decoder(truth[:, :-1], memory, mmask, sd, 'decoder.', **om.decoder_kwargs(params))
    finally:
        om.set_dropout(None)
    loss = om.label_smoothing_loss(logits, truth[:, 1:], params.get('smoothing', 0.1))
    w = params.get('ctc_weight', 0.0)
    if w > 0:
        loss = (1 - w) * loss + w * om.ctc_loss(memory, mmask, truth[:, 1:], truth_length, sd)
    return loss, new_stats


def loss_and_grads_train(x, mask, truth, sd, params, truth_length=None, drop=None):
    """-> (loss, {name: grad or None}, new running statistics).  A parameter the forward never reads (post_ffn.*) gets
    None, as its .grad stays None in the reference."""
    tied = params['decoder'].get('share_embedding', False)
    leaf = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and 'running_' not in k) for k, v in sd.items()}
    if tied:
        leaf['decoder.output_layer.weight'] = leaf['decoder.embedding.weight']
    loss, stats = loss_train(x, mask, truth, leaf, params, truth_length, drop)
    loss.backward()
    grads = {k: v.grad for k, v in leaf.items() if v.requires_grad and not (tied and k == 'decoder.output_layer.weight')}
    return loss.detach(), grads, stats
