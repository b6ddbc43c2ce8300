"""Minimum word error rate training at the benchmark's training geometry (bench.py config 5: the transformer_baseline.yaml
model with every dropout rate 0, 32 utterances x 1000 frames, 32-token targets, accumulation 1, CUDA graph):

  - the optimizer step without MWER against FusedTrainer(mwer_nbest=4) (max_len 60, eval.py's -ml), alternating;
  - the MWER step split into the n-best decode (recognize_ids in eval mode + second_pass_rows, with its host
    synchronisation) and the rest of the step (the training pass on the n-best, replayed from its CUDA graph once the
    n-best's length has recurred, and the optimizer update).  The decode is timed alone with weights that do not change
    between calls, so the inference pack rebuild that a real step's decode pays after the update is counted in the rest;
  - the n-best's length Lp, which random weights drive to max_len + 1.

CUDA events around --iters calls after 3 warm-up calls; each figure is measured --reps times in one run.  It prints the card,
its power limit and its maximum SM clock, read in the same run.  Needs a GPU.

    python tools/mwer_step.py [--iters 10] [--reps 3]
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
from opentransformer_b200.model import SpeechToText  # noqa: E402
from opentransformer_b200.train import FusedTrainer  # noqa: E402


def trainer(dev, **kw):
    torch.manual_seed(1234)
    model = SpeechToText(bench.train_params()).to(dev).train()
    return FusedTrainer(model, lr=1e-3, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6, clip_grad=5.0, model_size=256,
                        warmup_steps=12000, accum_steps=1, **kw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/mwer_step.py needs a GPU')
    dev = torch.device('cuda:0')
    B, K = bench.B_PER_GPU, 4
    x, mask = bench.synthetic_batch(B, 0)
    tgt = bench.synthetic_targets(B, 0)
    x, mask, tgt = x.to(dev), mask.to(dev), tgt.to(dev)
    out = {'card': card(), 'batch': B, 'frames': bench.T_FRAMES, 'mwer_nbest': K, 'mwer_max_len': 60, 'iters': args.iters}

    trainers = {'plain': trainer(dev), 'mwer': trainer(dev, mwer_nbest=K, mwer_max_len=60)}
    steps = {name: [] for name in trainers}
    for _ in range(args.reps):
        for name, tr in trainers.items():
            steps[name].append(timed(lambda: tr.step(x, mask, tgt), args.iters))
    out['step_ms'] = steps

    tr = trainers['mwer']
    batch = tr.model.train_batch(x, mask, tgt)
    with torch.no_grad():
        decode = [timed(lambda: tr._with_nbest(batch), args.iters) for _ in range(args.reps)]
        out['nbest_Lp'] = int(tr._with_nbest(batch)[-1].shape[1])
    out['decode_ms'] = decode
    out['training_pass_and_update_ms'] = [s - d for s, d in zip(steps['mwer'], decode)]
    out['graphs_cached'] = len(tr._graphs)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
