"""The reference's low-frame-rate front ends, `concat` and `concat-with-linear` (otrans/frontend/concat.py:11-56), restated
on top of oracle/speech_model.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

`concat_frontend` stacks frames with Tensor.unfold (the reference uses nn.Unfold over the whole [T, F] plane).
`frontend_of(params)` puts it in the place of the oracle's conv front end for the duration of a call, so every oracle
entry that runs `om.encode` (the model losses of oracle/speech_model.py, tests/ctc_ref.py and tests/conformer_train_ref.py,
the recognizer restatements) runs the model's own front end."""
import contextlib

import torch

from oracle import speech_model as om


def geometry(T, left, right, frame_rate):
    """-> (n, s, pad, T_p, T') as concat.py:26-39 computes them."""
    n, s = left + right + 1, int(frame_rate / 10)
    pad = (s - (T - n) % s) % s
    return n, s, pad, T + pad, (T + pad - n) // s + 1


def concat_frontend(x, mask, sd, prefix, fe, with_linear, policy=None):
    """ConcatFeatureFrontEnd.forward (+ the Linear of ConcatWithLinearFrontEnd, dropout 0): x [B, T, F], mask bool [B, T]
    -> (y [B, T', n F] or [B, T', D], mask [B, T'])."""
    B, T, F = x.shape
    n, s, pad, Tp, T2 = geometry(T, fe['left_frames'], fe['right_frames'], fe.get('frame_rate', 30))
    x = torch.cat([x, x.new_zeros(B, pad, F)], dim=1)
    mask = torch.cat([mask, mask.new_zeros(B, pad)], dim=1)
    y = x.unfold(1, n, s)                                   # [B, T', F, n]
    y = y.transpose(2, 3).reshape(B, T2, n * F)             # frame-major: j F + f
    if with_linear:
        y = om.linear(y, sd, prefix + 'linear', policy)
    return y, mask[:, fe['left_frames']::s]


@contextlib.contextmanager
def frontend_of(params):
    """Within the block, om.encode runs params' front end (a conv front end leaves the oracle as it is)."""
    kind = params['frontend_type']
    if kind == 'conv':
        yield
        return
    fe, with_linear, conv = params['frontend'], kind == 'concat-with-linear', om.conv_frontend

    def stacked(x, mask, sd, prefix='', policy=None, layer_norm_out=False):
        return concat_frontend(x, mask, sd, prefix, fe, with_linear, policy)
    om.conv_frontend = stacked
    try:
        yield
    finally:
        om.conv_frontend = conv


def speech2text_loss_and_grads(x, mask, truth, truth_length, sd, params):
    """SpeechToText.forward in train() (residual dropout 0, a Transformer encoder) and autograd -> (loss, {name: grad})."""
    leaf = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
    with frontend_of(params):
        loss, _ = om.model_forward_loss(x, mask, truth, leaf, params, truth_length=truth_length)
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in leaf.items() if v.requires_grad}
