"""Regenerate tests/golden/live_ref_layer_options.pt from the reference's OWN modules (byte-compiled into oracle/_ref by
oracle/build_ref.py): End2EndModel['speech2text'] in train() with the feed-forward activations and the attention dropout
that training takes beside GLU / ReLU and residual_dropout.  Each case runs `loss, _ = model(inputs, targets);
loss.backward()` once and stores the loss and every parameter gradient:

  - a post-norm and a pre-norm Transformer encoder / decoder with gelu, tanh and swish feed-forwards, every dropout 0;
  - a Conformer encoder (macaron, rel-pos attention, training-mode BatchNorm) with a swish feed-forward, dropout 0;
  - a post-norm Transformer with residual_dropout, slf_attn_dropout and src_attn_dropout 0.1 each.  The masks torch drew
    are recorded by forward hooks on every nn.Dropout (keep = output != 0) and stored per (block, sub-layer), so that the
    restatement can replay them: the attention's dropout on its projected output (attention.py:46) and the layer's
    residual dropout on top of it, two masks on one tensor.

The weights are not stored: the fixture keeps the key shapes and a seed (tests/test_head_dim_96.synth_state_dict, which
draws every key independently -- hence an untied output layer).  The models are small (d_model 16, 2 heads, one block per
stack) and each case's gradients are one flat fp32 tensor beside their names and shapes, so the fixture stays at a few
hundred kB; the batch is stored once.

    python oracle/build_ref.py && python tests/golden/make_live_ref_layer_options.py     # needs the reference tree
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import build_ref  # noqa: E402
from tests.test_head_dim_96 import synth_state_dict  # noqa: E402

SEED = 512
D = 16
FRONTEND = dict(input_size=20, output_size=D, in_channel=1, mid_channel=4, out_channel=4, kernel_size=[[3, 3], [3, 3]],
                stride=[2, 2], dropout=0.0, act_func_type='relu', front_end_layer_norm=False)


def decoder(activation, pre, slf=0.0, src=0.0, res=0.0):
    return dict(vocab_size=20, d_model=D, n_heads=2, d_ff=24, memory_dim=D, n_blocks=1, pos_dropout=0.0, slf_attn_dropout=slf,
                src_attn_dropout=src, ffn_dropout=0.0, residual_dropout=res, activation=activation, normalize_before=pre,
                concat_after=False, share_embedding=False)


def transformer_params(activation, pre, slf=0.0, src=0.0, res=0.0):
    return {'type': 'speech2text', 'frontend_type': 'conv', 'encoder_type': 'transformer', 'decoder_type': 'transformer',
            'frontend': dict(FRONTEND),
            'encoder': dict(d_model=D, n_heads=2, d_ff=24, n_blocks=1, pos_dropout=0.0, slf_attn_dropout=slf, ffn_dropout=0.0,
                            residual_dropout=res, normalize_before=pre, concat_after=False, activation=activation,
                            relative_positional=False),
            'decoder': decoder(activation, pre, slf, src, res), 'ctc_weight': 0.0, 'smoothing': 0.1}


def conformer_params(activation):
    return {'type': 'speech2text', 'frontend_type': 'conv', 'encoder_type': 'conformer', 'decoder_type': 'transformer',
            'frontend': dict(FRONTEND),
            'encoder': dict(d_model=D, d_ff=24, cov_kernel_size=5, n_heads=2, nblocks=1, pos_dropout=0.0, slf_attn_dropout=0.0,
                            ffn_dropout=0.0, residual_dropout=0.0, conv_dropout=0.0, macaron_style=True, ffn_scale=0.5,
                            conv_bias=True, activation=activation, positional_encoding=True, relative_positional=True),
            'decoder': decoder(activation, False), 'encoder_output_size': D, 'ctc_weight': 0.3, 'smoothing': 0.1}


CASES = {f'{"prenorm" if pre else "postnorm"}-{act}': transformer_params(act, pre)
         for pre in (False, True) for act in ('gelu', 'tanh', 'swish')}
CASES['conformer-swish'] = conformer_params('swish')
CASES['attn-dropout'] = transformer_params('gelu', False, slf=0.1, src=0.1, res=0.1)

# (block prefix, sub-layer) of every nn.Dropout the layers apply: the residual ones and the attention's own
_SUBLAYER = {'dropout1': 0, 'dropout2': 1, 'dropout3': 2, 'slf_attn.dropout': 0, 'src_attn.dropout': 1}


def batch():
    g = torch.Generator().manual_seed(23)
    B, T, L = 3, 70, 8
    lens = torch.tensor([70, 55, 41])
    mask = torch.arange(T)[None] < lens[:, None]
    x = torch.randn(B, T, 20, generator=g) * mask.unsqueeze(2)
    tgt = torch.randint(3, 20, (B, L), generator=g)
    tgt[:, 0] = 1
    tgt[0, L - 2:] = torch.tensor([1, 0])
    tgt[1, L - 1] = 1
    tgt[2, 4:] = torch.tensor([1, 0, 0, 0])
    return x, mask, tgt, (tgt[:, 1:] != 0).sum(1)


def case(p, seed, batch):
    from otrans.model import End2EndModel
    ref = End2EndModel['speech2text'](p)
    shapes = {k: (tuple(v.shape), str(v.dtype).replace('torch.', '')) for k, v in ref.state_dict().items()}
    ref.load_state_dict(synth_state_dict(shapes, seed), strict=True)
    ref.train()
    masks, hooks = {}, []
    for name, mod in ref.named_modules():
        if isinstance(mod, torch.nn.Dropout) and mod.p > 0.0:
            block, _, tail = name.partition('.blocks.')
            i, _, sub = tail.partition('.')
            key = (f'{block}.blocks.{i}', _SUBLAYER[sub], 'attn' if sub.endswith('attn.dropout') else 'res')

            def hook(m, inp, out, key=key):
                masks[key] = (out != 0).detach().clone()
            hooks.append(mod.register_forward_hook(hook))
    torch.manual_seed(seed)
    x, mask, tgt, tlen = batch
    loss, _ = ref({'inputs': x, 'mask': mask}, {'targets': tgt, 'targets_length': tlen})
    loss.backward()
    for h in hooks:
        h.remove()
    named = [(n, q.grad) for n, q in ref.named_parameters()]
    with_grad = [(n, g) for n, g in named if g is not None]
    return {'params': p, 'sd_shapes': shapes, 'sd_seed': seed, 'loss_ref': loss.detach(), 'masks': masks,
            'g_names': [n for n, _ in with_grad], 'g_shapes': [tuple(g.shape) for _, g in with_grad],
            'g_flat': torch.cat([g.reshape(-1) for _, g in with_grad]).clone(), 'g_none': [n for n, g in named if g is None]}


if __name__ == '__main__':
    if build_ref.load() is None:
        raise SystemExit('oracle/_ref is missing: run oracle/build_ref.py where the reference tree exists')
    b = batch()
    torch.save({'batch': dict(zip(('x', 'mask', 'tgt', 'tlen'), b)),
                'cases': {name: case(p, SEED + k, b) for k, (name, p) in enumerate(CASES.items())}},
               os.path.join(HERE, 'live_ref_layer_options.pt'))
