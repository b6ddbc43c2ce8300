"""Regenerate tests/golden/live_ref_conformer_train.pt from the reference's OWN modules (byte-compiled into oracle/_ref by
oracle/build_ref.py): End2EndModel['speech2text'] with a rel-pos Conformer encoder (macaron, conv after attention, the
shipped block) and a Transformer decoder, in train(), with residual_dropout 0 (the reference's F.dropout masks cannot be
replayed) and joint CTC 0.3.  It runs `loss, _ = model(inputs, targets); loss.backward()` once and stores the loss, every
parameter gradient (None where .grad stayed None: post_ffn.*), and the BatchNorm running statistics after the forward.
The weights are not stored: the fixture keeps the key shapes and a seed (tests/test_head_dim_96.synth_state_dict, which
draws every key independently -- hence an untied output layer).

    python oracle/build_ref.py && python tests/golden/make_live_ref_conformer_train.py     # needs the reference tree
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import build_ref  # noqa: E402
from tests.test_head_dim_96 import synth_state_dict  # noqa: E402

SEED = 256


def params():
    return {'type': 'speech2text', 'frontend_type': 'conv', 'encoder_type': 'conformer', 'decoder_type': 'transformer',
            'frontend': dict(input_size=20, output_size=32, in_channel=1, mid_channel=4, out_channel=8,
                             kernel_size=[[3, 3], [3, 3]], stride=[2, 2], dropout=0.0, act_func_type='relu',
                             front_end_layer_norm=False),
            'encoder': dict(d_model=32, d_ff=24, cov_kernel_size=5, n_heads=4, nblocks=2, pos_dropout=0.0, slf_attn_dropout=0.0,
                            ffn_dropout=0.0, residual_dropout=0.0, conv_dropout=0.0, macaron_style=True, ffn_scale=0.5,
                            conv_bias=True, activation='glu', positional_encoding=True, relative_positional=True),
            'decoder': dict(vocab_size=40, d_model=32, n_heads=4, d_ff=48, memory_dim=32, n_blocks=2, pos_dropout=0.0,
                            slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0, residual_dropout=0.0,
                            activation='glu', normalize_before=False, concat_after=False, share_embedding=False),
            'encoder_output_size': 32, 'ctc_weight': 0.3, 'smoothing': 0.1}


def batch():
    g = torch.Generator().manual_seed(17)
    B, T, L = 3, 70, 8
    lens = torch.tensor([70, 55, 41])
    mask = torch.arange(T)[None] < lens[:, None]
    x = torch.randn(B, T, 20, generator=g) * mask.unsqueeze(2)
    tgt = torch.randint(3, 40, (B, L), generator=g)
    tgt[:, 0] = 1
    tgt[0, L - 2:] = torch.tensor([1, 0])
    tgt[1, L - 1] = 1
    tgt[2, 4:] = torch.tensor([1, 0, 0, 0])
    return x, mask, tgt, (tgt[:, 1:] != 0).sum(1)


def case():
    from otrans.model import End2EndModel
    p = params()
    ref = End2EndModel['speech2text'](p)
    shapes = {k: (tuple(v.shape), str(v.dtype).replace('torch.', '')) for k, v in ref.state_dict().items()}
    ref.load_state_dict(synth_state_dict(shapes, SEED), strict=True)
    ref.train()
    x, mask, tgt, tlen = batch()
    loss, _ = ref({'inputs': x, 'mask': mask}, {'targets': tgt, 'targets_length': tlen})
    loss.backward()
    grads = {n: (q.grad.clone() if q.grad is not None else None) for n, q in ref.named_parameters()}
    stats = {n: b.detach().clone() for n, b in ref.named_buffers() if 'running_' in n or 'num_batches' in n}
    return {'params': p, 'sd_shapes': shapes, 'sd_seed': SEED, 'x': x, 'mask': mask, 'tgt': tgt, 'tlen': tlen,
            'loss_ref': loss.detach(), 'g_ref': grads, 'stats_ref': stats}


if __name__ == '__main__':
    if build_ref.load() is None:
        raise SystemExit('oracle/_ref is missing: run oracle/build_ref.py where the reference tree exists')
    torch.save(case(), os.path.join(HERE, 'live_ref_conformer_train.pt'))
