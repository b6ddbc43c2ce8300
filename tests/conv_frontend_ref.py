"""The reference's conv front end (otrans/frontend/conv.py:15-153) at any kernel size and stride, restated on top of
oracle/speech_model.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The oracle's `conv_frontend` runs its `conv2d_layer` at the default 3x3 / stride 2, and that layer slices the mask by
one int stride.  `conv_frontend_of(params)` puts a front end that takes each layer's kernel and [time, freq] stride in its
place for the duration of a call, so every oracle entry that runs `om.encode` (the model losses of
oracle/speech_model.py, tests/ctc_ref.py, the recognizer restatements) runs the model's own geometry."""
import contextlib

import torch.nn.functional as F

from oracle import speech_model as om


def pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def layers(fe):
    """frontend kwargs -> ((kt1, kf1), (st1, sf1)), ((kt2, kf2), (st2, sf2))."""
    ks, ss = fe.get('kernel_size', [[3, 3], [3, 3]]), fe.get('stride', [2, 2])
    return tuple((pair(k), pair(s)) for k, s in zip(ks, ss))


def conv2d_layer(x, mask, sd, prefix, kernel, stride, policy=None):
    """Conv2dLayer.forward + return_output_mask (conv.py:50-83): relu(conv2d(x)) with padding (0, kf // 2), and
    mask[:, kt // 2 :: st][:, :t] from the time entries."""
    (kt, kf), (st, sf) = kernel, stride
    y = F.conv2d(om._r(x, policy), om._r(sd[prefix + '.conv_layer.weight'], policy), sd[prefix + '.conv_layer.bias'],
                 stride=(st, sf), padding=(0, kf // 2))
    y = y.relu()
    return y, mask[:, kt // 2::st][:, :y.shape[2]]


def conv_frontend(x, mask, sd, prefix, fe, policy=None, layer_norm_out=False):
    """ConvFrontEnd.forward at fe's geometry: x [B, T, F], mask bool [B, T] -> (y [B, T', D], mask [B, T'])."""
    (k1, s1), (k2, s2) = layers(fe)
    y = x.unsqueeze(1)
    y, mask = conv2d_layer(y, mask, sd, prefix + 'conv1', k1, s1, policy)
    y = om._r(y, policy)
    y, mask = conv2d_layer(y, mask, sd, prefix + 'conv2', k2, s2, policy)
    b, c, t, f = y.shape
    y = y.transpose(1, 2).reshape(b, t, c * f)
    y = om.linear(y, sd, prefix + 'output_layer', policy)
    if layer_norm_out:
        y = om.layer_norm(y, sd, prefix + 'layer_norm')
    return y, mask


@contextlib.contextmanager
def conv_frontend_of(params):
    """Within the block, om.encode runs params' conv front end at its kernel sizes and strides."""
    fe, conv = params['frontend'], om.conv_frontend

    def geometric(x, mask, sd, prefix='', policy=None, layer_norm_out=False):
        return conv_frontend(x, mask, sd, prefix, fe, policy, layer_norm_out)
    om.conv_frontend = geometric
    try:
        yield
    finally:
        om.conv_frontend = conv
