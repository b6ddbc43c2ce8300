"""Low-frame-rate front ends against the conv front end, at 32 utterances x 1000 frames x 80 fbank bins:

  - otb_frame_stack alone (n 4, s 4: 250 rows of 320 columns per utterance), with the bytes it must move (f32 features
    in, bf16 rows out) computed from the shapes and the achieved bandwidth;
  - the front end alone into d_model 256: conv (transformer_baseline.yaml) against concat-with-linear (left 3, right 0,
    frame_rate 40), each with the encoder's x*sqrt(d)+PE fused as encode_bf16 runs it;
  - front end + the transformer_baseline encoder (12 blocks) for both, through SpeechToText.encode_bf16.

CUDA events after warm-up; each figure is the mean over --iters calls.  The card, its power limit and its maximum SM
clock are read in the same run.  Needs a GPU.

    python tools/lfr_frontend.py [--iters 50]
"""
import argparse
import copy
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench  # noqa: E402
from ctc_model import card, timed  # noqa: E402
from opentransformer_b200 import ops  # noqa: E402
from opentransformer_b200.model import SpeechToText  # noqa: E402

DEV = torch.device('cuda:0')
B, T, F = 32, 1000, 80


def models():
    conv = bench.model_params()
    lfr = copy.deepcopy(conv)
    lfr['frontend_type'] = 'concat-with-linear'
    lfr['frontend'] = dict(input_size=F, output_size=256, left_frames=3, right_frames=0, frame_rate=40, dropout=0.0)
    out = {}
    for name, p in (('conv', conv), ('concat-with-linear', lfr)):
        torch.manual_seed(1234)
        out[name] = SpeechToText(p).eval().to(DEV)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    args = ap.parse_args()
    print(f'card: {card()}')
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, T, F, generator=g).to(DEV)
    mask = torch.ones(B, T, dtype=torch.bool, device=DEV)
    n, s = 4, 4
    T2 = (T - n) // s + 1
    out = torch.empty(B * T2, n * F, dtype=ops.BF16, device=DEV)
    ms = timed(lambda: ops.frame_stack(x, n, s, T2, out=out), args.iters * 4)
    nbytes = B * T * F * 4 + B * T2 * n * F * 2
    print(f'otb_frame_stack {B}x{T}x{F} -> [{B * T2}, {n * F}] bf16: {ms * 1e3:.1f} us, {nbytes / 1e6:.1f} MB moved, '
          f'{nbytes / (ms * 1e-3) / 1e12:.2f} TB/s')
    with torch.no_grad():
        for name, m in models().items():
            fe, enc = m.frontend, m.encoder
            T2m = fe.output_length(T)
            scale, table = enc.pos_emb.scale_and_table(T2m, DEV)
            t_fe = timed(lambda: fe.forward_bf16(x, scale, table), args.iters)
            t_all = timed(lambda: m.encode_bf16(x, mask), args.iters)
            print(f'{name}: T\' {T2m}; front end {t_fe:.3f} ms; front end + encoder {t_all:.3f} ms')


if __name__ == '__main__':
    main()
