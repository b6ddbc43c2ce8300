"""Regenerate tests/golden/live_ref_concat_frontend.pt from the reference's OWN modules (byte-compiled into oracle/_ref by
oracle/build_ref.py), on the CPU:

  frontend    ConcatFeatureFrontEnd and ConcatWithLinearFrontEnd (frontend/concat.py) on ragged batches of F = 5 features
              (n F never a multiple of 8) for several (left, right, frame_rate, T): T - n a multiple of the stride and not,
              T < n with T_p >= n, n = 1.  Stored: outputs and masks.
  geometry    for every (left 0..4, right < s, s = 1..4, frame_rate 10 s) and T = 1..64: the reference module's T' and the
              length of its output mask for an utterance of T - T // 3 valid frames, or -1 where nn.Unfold raises.
  speech2text End2EndModel['speech2text'] with a concat-with-linear front end (n 3, s 3: n F = 60, K padded to 64 on the
              GPU), a one-block Transformer encoder and decoder (d_model 64) and joint CTC 0.3, in train() with
              residual_dropout 0: the loss and every gradient.
  ctc         End2EndModel['ctc'] with a concat front end (n 4, s 2: overlapping stacks) and a one-block rel-pos Conformer
              (d_model 64): the loss, every gradient (None where .grad stayed None) and the BatchNorm running statistics.

The models are small so that the fixture stays small (about 0.4 MB).

Weights are stored as key shapes + seed (tests/test_head_dim_96.synth_state_dict); gradients as
tests/test_transformer_lm_ref.sample keeps them (a fixed quarter of each tensor larger than 4096 elements).

    python oracle/build_ref.py && python tests/golden/make_live_ref_concat_frontend.py     # needs the reference tree
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

SEED = 1024
V = 30
FRONTEND_CASES = [(3, 0, 40, 16), (3, 0, 40, 18), (2, 1, 20, 9), (1, 1, 30, 2), (5, 0, 60, 1), (0, 0, 10, 5), (4, 2, 30, 23)]


def speech2text_params():
    return {'type': 'speech2text', 'frontend_type': 'concat-with-linear', 'encoder_type': 'transformer',
            'decoder_type': 'transformer',
            'frontend': dict(input_size=20, output_size=64, left_frames=1, right_frames=1, frame_rate=30, dropout=0.0),
            'encoder': dict(d_model=64, n_heads=1, d_ff=64, n_blocks=1, pos_dropout=0.0, slf_attn_dropout=0.0, ffn_dropout=0.0,
                            residual_dropout=0.0, normalize_before=False, concat_after=False, activation='glu',
                            relative_positional=False),
            'decoder': dict(vocab_size=V, d_model=64, n_heads=1, d_ff=64, memory_dim=64, n_blocks=1, pos_dropout=0.0,
                            slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0, residual_dropout=0.0,
                            activation='glu', normalize_before=False, concat_after=False, share_embedding=False),
            'encoder_output_size': 64, 'ctc_weight': 0.3, 'smoothing': 0.1}


def ctc_params():
    return {'type': 'ctc', 'frontend_type': 'concat', 'encoder_type': 'conformer',
            'frontend': dict(input_size=16, left_frames=2, right_frames=1, frame_rate=20),
            'encoder': dict(d_model=64, d_ff=64, cov_kernel_size=5, n_heads=1, nblocks=1, pos_dropout=0.0, slf_attn_dropout=0.0,
                            ffn_dropout=0.0, residual_dropout=0.0, conv_dropout=0.0, macaron_style=True, ffn_scale=0.5,
                            conv_bias=True, activation='glu', positional_encoding=True, relative_positional=True),
            'encoder_output_size': 64, 'vocab_size': V}


def batch(F, seed):
    """Ragged inputs; truth = BOS, labels, EOS, PAD* with 6, 3 and 4 labels."""
    g = torch.Generator().manual_seed(seed)
    B, T, L = 3, 70, 8
    lens = torch.tensor([70, 55, 41])
    mask = torch.arange(T)[None] < lens[:, None]
    x = torch.randn(B, T, F, generator=g) * mask.unsqueeze(2)
    tgt = torch.randint(2, V, (B, L), generator=g)
    tgt[:, 0] = 1
    tgt[0, 7] = 1
    tgt[1, 4:] = torch.tensor([1, 0, 0, 0])
    tgt[2, 5:] = torch.tensor([1, 0, 0])
    return x, mask, tgt, (tgt[:, 1:] != 0).sum(1)


def frontend_cases():
    from otrans.frontend import ConcatFeatureFrontEnd, ConcatWithLinearFrontEnd
    out = []
    g = torch.Generator().manual_seed(31)
    for left, right, rate, T in FRONTEND_CASES:
        x = torch.randn(2, T, 5, generator=g)
        mask = torch.arange(T)[None] < torch.tensor([T, max(1, T - T // 3)])[:, None]
        y, m = ConcatFeatureFrontEnd(5, left, right, rate)(x, mask)
        lin = ConcatWithLinearFrontEnd(5, 16, left, right, rate)
        shapes = {k: (tuple(v.shape), str(v.dtype).replace('torch.', '')) for k, v in lin.state_dict().items()}
        lin.load_state_dict(synth_state_dict(shapes, SEED + T), strict=True)
        with torch.no_grad():
            yl, ml = lin(x, mask)
        assert torch.equal(m, ml)
        out.append({'left': left, 'right': right, 'frame_rate': rate, 'x': x, 'mask': mask, 'y': y, 'mask_out': m,
                    'sd_shapes': shapes, 'sd_seed': SEED + T, 'y_linear': yl})
    return out


def geometry_table():
    """-> i16 [rows, 6]: left, right, frame_rate, T, T' and the output mask's length (-1, -1 where nn.Unfold raises)."""
    from otrans.frontend import ConcatFeatureFrontEnd
    table = []
    for s in range(1, 5):
        for right in range(s):
            for left in range(5):
                fe = ConcatFeatureFrontEnd(1, left, right, 10 * s)
                for T in range(1, 65):
                    mask = torch.arange(T)[None] < T - T // 3
                    try:
                        y, m = fe(torch.zeros(1, T, 1), mask)
                        table.append((left, right, 10 * s, T, y.shape[1], int(m.sum())))
                    except RuntimeError:
                        table.append((left, right, 10 * s, T, -1, -1))
    return torch.tensor(table, dtype=torch.int16)


def train_case(kind):
    from otrans.model import End2EndModel
    p = speech2text_params() if kind == 'speech2text' else ctc_params()
    ref = End2EndModel[kind](p)
    shapes = {k: (tuple(v.shape), str(v.dtype).replace('torch.', '')) for k, v in ref.state_dict().items()}
    ref.load_state_dict(synth_state_dict(shapes, SEED), strict=True)
    ref.train()
    x, mask, tgt, tlen = batch(p['frontend']['input_size'], 41 if kind == 'speech2text' else 43)
    loss, _ = ref({'inputs': x, 'mask': mask}, {'targets': tgt, 'targets_length': tlen})
    loss.backward()
    grads = {n: (sample(q.grad) if q.grad is not None else None) for n, q in ref.named_parameters()}
    stats = {n: b.detach().clone() for n, b in ref.named_buffers() if 'running_' in n or 'num_batches' in n}
    return {'params': p, 'sd_shapes': shapes, 'sd_seed': SEED, 'x': x, 'mask': mask, 'tgt': tgt, 'tlen': tlen,
            'loss_ref': loss.detach(), 'g_ref': grads, 'stats_ref': stats}


if __name__ == '__main__':
    if build_ref.load() is None:
        raise SystemExit('oracle/_ref is missing: run oracle/build_ref.py where the reference tree exists')
    torch.save({'frontend': frontend_cases(), 'geometry': geometry_table(), 'speech2text': train_case('speech2text'),
                'ctc': train_case('ctc')}, os.path.join(HERE, 'live_ref_concat_frontend.pt'))
