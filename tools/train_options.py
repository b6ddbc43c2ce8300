"""FusedTrainer's training options at the benchmark's training geometry (bench.py config 5: the transformer_baseline.yaml
model with every dropout rate 0, 32 utterances x 1000 frames, 32-token targets, accumulation 1, CUDA graph):

  - the optimizer step plain against MixSpeech at the same B (MixSpeech: the mix, then two passes over B/2 rows);
  - the fused Adam launch (otb_sumsq + otb_adam_step_sched) with grad_noise 0 against grad_noise > 0, over the model's
    flat parameter buffer;
  - FusedTrainer.state_dict() + torch.save, and torch.load + load_state_dict, to a temporary file.

CUDA events around --iters calls after 3 warm-up calls; each figure is measured --reps times in one run, the variants
alternating.  It prints the card, its power limit and its maximum SM clock, read in the same run.  Needs a GPU.

    python tools/train_options.py [--iters 20] [--reps 3]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench  # noqa: E402
from ctc_model import card, timed  # noqa: E402
from opentransformer_b200 import ops  # noqa: E402
from opentransformer_b200.model import SpeechToText  # noqa: E402
from opentransformer_b200.train import FusedTrainer  # noqa: E402


def trainer(dev, **kw):
    torch.manual_seed(1234)
    model = SpeechToText(bench.train_params()).to(dev).train()
    return model, FusedTrainer(model, lr=1e-3, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6, clip_grad=5.0, model_size=256,
                               warmup_steps=12000, accum_steps=1, **kw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/train_options.py needs a GPU')
    dev = torch.device('cuda:0')
    B = bench.B_PER_GPU
    x, mask = bench.synthetic_batch(B, 0)
    tgt = bench.synthetic_targets(B, 0)
    x, mask, tgt = x.to(dev), mask.to(dev), tgt.to(dev)
    out = {'card': card(), 'batch': B, 'frames': bench.T_FRAMES, 'iters': args.iters}

    # ---- optimizer step: plain against MixSpeech, alternating
    steps = {'plain': [], 'mixspeech': []}
    trainers = {'plain': trainer(dev)[1], 'mixspeech': trainer(dev, mixspeech=True)[1]}
    for _ in range(args.reps):
        for name, tr in trainers.items():
            steps[name].append(timed(lambda: tr.step(x, mask, tgt), args.iters))
    out['step_ms'] = steps
    n_params = trainers['plain'].flat_p.numel()
    del trainers
    torch.cuda.empty_cache()

    # ---- the fused Adam launch over the flat buffer, sigma 0 against sigma > 0
    _, tr = trainer(dev, grad_noise=0.01)
    tr.flat_g.normal_(0.0, 1e-3)
    seed = tr.noise_seed
    adam = {'sigma_0': [], 'sigma_0.01': []}

    def launch(sigma):
        ops.sumsq(tr.flat_g, tr.sumsq)
        ops.adam_step_sched(tr.flat_p, tr.flat_g, tr.m, tr.v, tr.sumsq, 5.0, 1e-3, 256, 12000, 1.0, (0.9, 0.98), 1e-9, 1e-6,
                            tr.counters, tr.hyper, noise_std=sigma, noise_seed=seed, noise_mask=tr.noise_mask)
    for _ in range(args.reps):
        adam['sigma_0'].append(timed(lambda: launch(0.0), 10 * args.iters))
        adam['sigma_0.01'].append(timed(lambda: launch(0.01), 10 * args.iters))
    out['adam_ms'] = adam
    out['adam_elements'] = n_params
    # bytes the step moves: p, m, v read and written, g read (the noise mask adds n / 8)
    out['adam_hbm_bytes'] = {'sigma_0': 28 * n_params, 'sigma_0.01': 28 * n_params + n_params // 8}

    # ---- checkpoint: state_dict + torch.save, torch.load + load_state_dict
    save, load = [], []
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'latest_optimizer.pt')
        for _ in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            torch.save(tr.state_dict(), path)
            t1 = time.perf_counter()
            tr.load_state_dict(torch.load(path, weights_only=False))
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            save.append(1e3 * (t1 - t0))
            load.append(1e3 * (t2 - t1))
        out['checkpoint_bytes'] = os.path.getsize(path)
    out['save_ms'], out['load_ms'] = save, load
    print(json.dumps(out))


if __name__ == '__main__':
    main()
