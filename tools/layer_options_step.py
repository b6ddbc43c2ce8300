"""Time one FusedTrainer optimizer step at bench.py's training geometry (Speech-Transformer d_model 256, 12 encoder / 6
decoder blocks, B 32 x 1000 frames, 32-token targets, CUDA graph, accumulation 1) with the feed-forward activation glu,
gelu and swish, each with the attention's output dropout off and on (slf_attn_dropout = src_attn_dropout = 0.1; every
other rate 0 as in bench.py's config 5).  gelu and swish add one elementwise pass over the [B T', d_ff] hidden activation
forward (otb_act_fwd) and backward (otb_act_bwd) where glu runs otb_glu_fwd / otb_glu_bwd over twice as wide a w_1
output; the attention dropout adds a mask to the residual GEMM epilogues and to their backward replay.  The variants are
timed in alternation, `--reps` rounds of `--steps` steps each.

    python tools/layer_options_step.py [--steps 20] [--reps 3]

Prints the card, its power limit and maximum SM clock, then one JSON line per variant."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
from opentransformer_b200.model import SpeechToText  # noqa: E402
from opentransformer_b200.train import FusedTrainer  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def params(act, attn):
    p = bench.train_params()
    for part in ('encoder', 'decoder'):
        p[part]['activation'] = act
        p[part]['slf_attn_dropout'] = attn
    p['decoder']['src_attn_dropout'] = attn
    return p


def make(act, attn, dev):
    torch.manual_seed(1234)
    model = SpeechToText(params(act, attn)).to(dev).train()
    tr = FusedTrainer(model, lr=1e-3, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6, clip_grad=5.0, model_size=256,
                      warmup_steps=12000, accum_steps=1, use_graph=True)
    for _ in range(4):                       # the graph is captured on the 2nd step
        tr.step(*BATCH)
    torch.cuda.synchronize()
    return tr


def time_steps(tr, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        tr.step(*BATCH)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('layer_options_step.py times the GPU: no CUDA device')
    dev = torch.device('cuda:0')
    print('card (name, power limit, max SM clock):', card())
    x, m = bench.synthetic_batch(bench.B_PER_GPU, 0)
    BATCH = (x.to(dev), m.to(dev), bench.synthetic_targets(bench.B_PER_GPU, 1).to(dev))
    variants = [(act, attn) for act in ('glu', 'gelu', 'swish') for attn in (0.0, 0.1)]
    trainers = {v: make(*v, dev) for v in variants}
    times = {v: [] for v in variants}
    for _ in range(args.reps):
        for v in variants:
            times[v].append(time_steps(trainers[v], args.steps))
    base = min(times[('glu', 0.0)])
    for (act, attn), ts in times.items():
        print(json.dumps({'activation': act, 'attn_dropout': attn, 'ms_per_step': [round(t, 3) for t in ts],
                          'best_vs_glu_no_attn_dropout': round(min(ts) / base, 4), 'B': bench.B_PER_GPU, 'steps': args.steps}))
