"""Conv front end geometries at 32 utterances x 1000 frames x 80 fbank bins, on the config-5 model (bench.train_params:
the shipped Speech-Transformer, d_model 256, 12 encoder / 6 decoder blocks, conv front end 64 -> 128 channels):

  - the front end alone (conv1, the conv2 implicit GEMM, the Linear with the encoder's x*sqrt(d)+PE fused);
  - conv2 alone, with its achieved TFLOP/s from the shapes (2 B T2 F2 C2 kt2 kf2 C1 over its time);
  - front end + the 12-block encoder, through SpeechToText.encode_bf16;
  - one FusedTrainer step (forward, hand-written backward, clip + Adam; no SpecAugment).

CUDA events after warm-up; each figure is the mean over --iters calls (--train-iters steps).  The card, its power limit
and its maximum SM clock are read in the same run.  Needs a GPU.

    python tools/conv_frontend.py [--iters 50] [--train-iters 10]
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
from opentransformer_b200.model import SpeechToText  # noqa: E402
from opentransformer_b200 import ops  # noqa: E402
from opentransformer_b200.train import FusedTrainer  # noqa: E402

DEV = torch.device('cuda:0')
B, T, F = 32, 1000, 80
GEOMETRIES = [('3x3 s2 (shipped)', [[3, 3], [3, 3]], [2, 2]), ('3x3 s[2,3] (6x)', [[3, 3], [3, 3]], [2, 3]),
              ('[5,5],[3,3] s[3,2] (6x)', [[5, 5], [3, 3]], [3, 2]), ('3x3 s[1,2] (2x)', [[3, 3], [3, 3]], [1, 2]),
              ('[3,5],[5,3] s[[2,1],[2,2]] (4x)', [[3, 5], [5, 3]], [[2, 1], [2, 2]])]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--train-iters', type=int, default=10)
    args = ap.parse_args()
    print(f'card: {card()}')
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, T, F, generator=g).to(DEV)
    mask = torch.ones(B, T, dtype=torch.bool, device=DEV)
    tgt = bench.synthetic_targets(B, 7).to(DEV)
    for name, ks, st in GEOMETRIES:
        p = copy.deepcopy(bench.train_params())
        p['frontend'].update(kernel_size=ks, stride=st)
        torch.manual_seed(1234)
        m = SpeechToText(p).to(DEV).eval()
        fe, enc = m.frontend, m.encoder
        (T1, F1), (T2, F2) = fe.sizes(T)
        pk = fe._pack.get()
        C2 = pk['w2'].shape[0]
        with torch.no_grad():
            scale, table = enc.pos_emb.scale_and_table(T2, DEV)
            t_fe = timed(lambda: fe.forward_bf16(x, scale, table), args.iters)
            h1 = ops.conv1_relu(x, pk['w1'], pk['b1'], geom=fe.geom)
            t_c2 = timed(lambda: ops.conv2_relu(h1, pk['w2'], pk['b2'], B, T, F, geom=fe.geom), args.iters)
            t_all = timed(lambda: m.encode_bf16(x, mask), args.iters)
        flop = 2.0 * B * T2 * F2 * C2 * pk['w2'].shape[1]
        m.train()
        tr = FusedTrainer(m, clip_grad=5.0, accum_steps=1)
        t_step = timed(lambda: tr.step(x, mask, tgt), args.train_iters, warmup=3)
        print(f'{name}: T\' {T2} (T1 {T1}, F1 {F1}, F2 {F2}); front end {t_fe:.3f} ms; conv2 {t_c2 * 1e3:.1f} us '
              f'({flop / (t_c2 * 1e-3) / 1e12:.0f} TFLOP/s, K {pk["w2"].shape[1]}); front end + encoder {t_all:.3f} ms; '
              f'training step {t_step:.1f} ms')
        del tr, m
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
