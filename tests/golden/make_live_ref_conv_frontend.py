"""Regenerate tests/golden/live_ref_conv_frontend.pt from the reference's OWN modules (byte-compiled into oracle/_ref by
oracle/build_ref.py), on the CPU:

  frontend    ConvFrontEnd (frontend/conv.py:86-153) at several kernel sizes and strides (GEOMETRIES) on a ragged batch,
              with and without front_end_layer_norm.  Stored: weights, outputs and masks.
  geometry    for every kernel size k in 1..7 and stride s in 1..4, both layers (k, s), and T = 1..64: the reference
              module's T' and its output mask's length, or -1, -1 where its conv2d raises.
  speech2text End2EndModel['speech2text'] with a conv front end at stride [2, 3] (6x) and front_end_layer_norm, a one-block
              Transformer encoder and decoder (d_model 64) and joint CTC 0.3, in train() with residual_dropout 0: the
              loss and every gradient.
  ctc         End2EndModel['ctc'] with a conv front end of kernels [[5, 5], [3, 3]] at stride [3, 2] (6x) and a
              one-block Transformer encoder (d_model 64): the loss and every gradient.

Weights are stored as key shapes + seed (tests/test_head_dim_96.synth_state_dict); gradients as
tests/test_transformer_lm_ref.sample keeps them (a fixed quarter of each tensor larger than 4096 elements).

    python oracle/build_ref.py && python tests/golden/make_live_ref_conv_frontend.py     # needs the reference tree
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import build_ref  # noqa: E402
from tests.test_head_dim_96 import synth_state_dict  # noqa: E402
from tests.test_transformer_lm_ref import sample  # noqa: E402

SEED = 2048
V = 30
# (kernel_size, stride) as the reference's YAML writes them
GEOMETRIES = [([[3, 3], [3, 3]], [2, 2]), ([[3, 3], [3, 3]], [2, 3]), ([[5, 5], [3, 3]], [3, 2]), ([[3, 3], [3, 3]], [1, 2]),
              ([[3, 5], [5, 3]], [[2, 1], [2, 2]]), ([7, 2], [4, [1, 3]]), ([[1, 4], [6, 1]], [[3, 4], 2])]


def frontend_kwargs(kernel_size, stride, layer_norm=False, F=23):
    return dict(input_size=F, output_size=32, in_channel=1, mid_channel=8, out_channel=16, kernel_size=kernel_size,
                stride=stride, dropout=0.0, act_func_type='relu', front_end_layer_norm=layer_norm)


def speech2text_params():
    return {'type': 'speech2text', 'frontend_type': 'conv', 'encoder_type': 'transformer', 'decoder_type': 'transformer',
            'frontend': dict(input_size=20, output_size=64, in_channel=1, mid_channel=8, out_channel=16,
                             kernel_size=[[3, 3], [3, 3]], stride=[2, 3], dropout=0.0, act_func_type='relu',
                             front_end_layer_norm=True),
            'encoder': dict(d_model=64, n_heads=1, d_ff=64, n_blocks=1, pos_dropout=0.0, slf_attn_dropout=0.0, ffn_dropout=0.0,
                            residual_dropout=0.0, normalize_before=False, concat_after=False, activation='glu',
                            relative_positional=False),
            'decoder': dict(vocab_size=V, d_model=64, n_heads=1, d_ff=64, memory_dim=64, n_blocks=1, pos_dropout=0.0,
                            slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0, residual_dropout=0.0,
                            activation='glu', normalize_before=False, concat_after=False, share_embedding=False),
            'encoder_output_size': 64, 'ctc_weight': 0.3, 'smoothing': 0.1}


def ctc_params():
    return {'type': 'ctc', 'frontend_type': 'conv', 'encoder_type': 'transformer',
            'frontend': dict(input_size=16, output_size=64, in_channel=1, mid_channel=8, out_channel=8,
                             kernel_size=[[5, 5], [3, 3]], stride=[3, 2], dropout=0.0, act_func_type='relu',
                             front_end_layer_norm=False),
            'encoder': dict(d_model=64, n_heads=1, d_ff=64, n_blocks=1, pos_dropout=0.0, slf_attn_dropout=0.0, ffn_dropout=0.0,
                            residual_dropout=0.0, normalize_before=False, concat_after=False, activation='glu',
                            relative_positional=False),
            'encoder_output_size': 64, 'vocab_size': V}


def batch(F, seed):
    """Ragged inputs of 120 frames (20 after 6x subsampling); truth = BOS, labels, EOS, PAD* with 6, 3 and 4 labels."""
    g = torch.Generator().manual_seed(seed)
    B, T, L = 3, 120, 8
    lens = torch.tensor([120, 97, 71])
    mask = torch.arange(T)[None] < lens[:, None]
    x = torch.randn(B, T, F, generator=g) * mask.unsqueeze(2)
    tgt = torch.randint(2, V, (B, L), generator=g)
    tgt[:, 0] = 1
    tgt[0, 7] = 1
    tgt[1, 4:] = torch.tensor([1, 0, 0, 0])
    tgt[2, 5:] = torch.tensor([1, 0, 0])
    return x, mask, tgt, (tgt[:, 1:] != 0).sum(1)


def shapes_of(module):
    return {k: (tuple(v.shape), str(v.dtype).replace('torch.', '')) for k, v in module.state_dict().items()}


def frontend_cases():
    from otrans.frontend.conv import ConvFrontEnd
    out = []
    g = torch.Generator().manual_seed(31)
    for i, (ks, st) in enumerate(GEOMETRIES):
        for ln in (False, True):
            kw = frontend_kwargs(ks, st, ln)
            fe = ConvFrontEnd(**kw)
            shapes = shapes_of(fe)
            fe.load_state_dict(synth_state_dict(shapes, SEED + 2 * i + ln), strict=True)
            T = 61
            x = torch.randn(3, T, kw['input_size'], generator=g)
            mask = torch.arange(T)[None] < torch.tensor([T, 50, 37])[:, None]
            with torch.no_grad():
                y, m = fe(x, mask)
            out.append({'kwargs': kw, 'x': x, 'mask': mask, 'y': y, 'mask_out': m, 'sd_shapes': shapes,
                        'sd_seed': SEED + 2 * i + ln, 'output_size': (fe.conv1.output_size, fe.conv2.output_size)})
    return out


def geometry_table():
    """-> i16 [rows, 5]: k, s, T, T' and the output mask's length (-1, -1 where the reference raises)."""
    from otrans.frontend.conv import ConvFrontEnd
    table = []
    for k in range(1, 8):
        for s in range(1, 5):
            fe = ConvFrontEnd(**frontend_kwargs([k, k], [s, s], F=9))
            for T in range(1, 65):
                mask = torch.arange(T)[None] < T - T // 3
                try:
                    with torch.no_grad():
                        y, m = fe(torch.zeros(1, T, 9), mask)
                    table.append((k, s, T, y.shape[1], m.shape[1]))
                except RuntimeError:
                    table.append((k, s, T, -1, -1))
    return torch.tensor(table, dtype=torch.int16)


def train_case(kind):
    from otrans.model import End2EndModel
    p = speech2text_params() if kind == 'speech2text' else ctc_params()
    ref = End2EndModel[kind](p)
    shapes = shapes_of(ref)
    ref.load_state_dict(synth_state_dict(shapes, SEED), strict=True)
    ref.train()
    x, mask, tgt, tlen = batch(p['frontend']['input_size'], 41 if kind == 'speech2text' else 43)
    loss, _ = ref({'inputs': x, 'mask': mask}, {'targets': tgt, 'targets_length': tlen})
    loss.backward()
    grads = {n: (sample(q.grad) if q.grad is not None else None) for n, q in ref.named_parameters()}
    return {'params': p, 'sd_shapes': shapes, 'sd_seed': SEED, 'x': x, 'mask': mask, 'tgt': tgt, 'tlen': tlen,
            'loss_ref': loss.detach(), 'g_ref': grads}


if __name__ == '__main__':
    if build_ref.load() is None:
        raise SystemExit('oracle/_ref is missing: run oracle/build_ref.py where the reference tree exists')
    torch.save({'frontend': frontend_cases(), 'geometry': geometry_table(), 'speech2text': train_case('speech2text'),
                'ctc': train_case('ctc')}, os.path.join(HERE, 'live_ref_conv_frontend.pt'))
