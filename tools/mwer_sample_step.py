"""Sampling-based minimum word error rate training at the benchmark's training geometry (bench.py config 5: the
transformer_baseline.yaml model with every dropout rate 0, 32 utterances x 1000 frames, 32-token targets, accumulation 1,
CUDA graph), next to the n-best estimator:

  - the optimizer step without MWER, with FusedTrainer(mwer_nbest=4) and with FusedTrainer(mwer_samples=4) (max_len 60),
    alternating;
  - the decode of each MWER step alone: the n-best (recognize_ids, persistent kernel) and the K samples (sample_ids on the
    per-step graph path), both in eval mode with second_pass_rows and its host synchronisation;
  - the length Lp of the rows each decode hands to the training pass;
  - the sampled step and its decode again with <S/E> ruled out (output bias -1e4), so that every sample runs to max_len:
    random weights make <S/E> the near-certain first draw.

CUDA events around --iters calls after 3 warm-up calls; each figure is measured --reps times in one run.  It prints the card,
its power limit and its maximum SM clock, read in the same run.  Needs a GPU.

    python tools/mwer_sample_step.py [--iters 10] [--reps 3]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench  # noqa: E402
from ctc_model import card, timed  # noqa: E402
from mwer_step import trainer  # noqa: E402
from opentransformer_b200 import modules  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/mwer_sample_step.py needs a GPU')
    dev = torch.device('cuda:0')
    B, K = bench.B_PER_GPU, 4
    x, mask = bench.synthetic_batch(B, 0)
    tgt = bench.synthetic_targets(B, 0)
    x, mask, tgt = x.to(dev), mask.to(dev), tgt.to(dev)
    out = {'card': card(), 'batch': B, 'frames': bench.T_FRAMES, 'K': K, 'mwer_max_len': 60, 'iters': args.iters}

    trainers = {'plain': trainer(dev), 'nbest': trainer(dev, mwer_nbest=K, mwer_max_len=60),
                'sample': trainer(dev, mwer_samples=K, mwer_max_len=60)}
    steps = {name: [] for name in trainers}
    for _ in range(args.reps):
        for name, tr in trainers.items():
            steps[name].append(timed(lambda: tr.step(x, mask, tgt), args.iters))
    out['step_ms'] = steps

    for name in ('nbest', 'sample'):
        tr = trainers[name]
        batch = tr.model.train_batch(x, mask, tgt)
        with torch.no_grad():
            out[f'{name}_decode_ms'] = [timed(lambda: tr._with_nbest(batch), args.iters) for _ in range(args.reps)]
            out[f'{name}_Lp'] = int(tr._with_nbest(batch)[-1].shape[1])
        out[f'{name}_graphs_cached'] = len(tr._graphs)
    # random weights with the tied embedding make <S/E> the near-certain first draw, so the samples above end at once; with
    # <S/E> ruled out (output bias -1e4) every sample runs to max_len, the decode's worst case and the n-best's Lp
    tr = trainers['sample']
    with torch.no_grad():
        tr.model.decoder.output_layer.bias[1] = -1e4
    modules.bump_param_generation()
    out['sample_full_length_step_ms'] = [timed(lambda: tr.step(x, mask, tgt), args.iters) for _ in range(args.reps)]
    batch = tr.model.train_batch(x, mask, tgt)
    with torch.no_grad():
        out['sample_full_length_decode_ms'] = [timed(lambda: tr._with_nbest(batch), args.iters) for _ in range(args.reps)]
        out['sample_full_length_Lp'] = int(tr._with_nbest(batch)[-1].shape[1])
    bd = next(iter(trainers['sample']._recognizer._decoders.values()))
    out['sample_decoder'] = {'persistent': bd.persistent, 'captured_step': bd.step.graph is not None,
                             'launches_per_step': bd.step.launches}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
