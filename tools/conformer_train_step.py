"""Time one optimizer step of the BASELINE config-4 Conformer (d_model 256, 12 blocks, 6 decoder blocks, residual_dropout
0.1 as shipped) with FusedTrainer (CUDA graph, accumulation 1) on 32 x 1000 frames and 32-token targets, next to the
config-5 Transformer step; then a separate torch.profiler run gives the share of device time in the Conformer's training
kernels.

    python tools/conformer_train_step.py [--steps 20] [--reps 3] [--out DIR]

Prints the card, its power limit and maximum SM clock, and one JSON line per model."""
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


def conformer_train_params():
    p = bench.conformer_params()
    p['encoder']['residual_dropout'] = 0.1
    p['decoder']['residual_dropout'] = 0.1
    return p


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def make(params, dev):
    torch.manual_seed(1234)
    model = SpeechToText(params).to(dev).train()
    tr = FusedTrainer(model, lr=1e-3, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6, clip_grad=5.0, model_size=256,
                      warmup_steps=12000, accum_steps=1, use_graph=True)
    x, m = bench.synthetic_batch(bench.B_PER_GPU, 0)
    t = bench.synthetic_targets(bench.B_PER_GPU, 1)
    return tr, (x.to(dev), m.to(dev), t.to(dev))


def time_steps(tr, batch, steps, reps, warmup=4):
    for _ in range(warmup):                 # the graph is captured on the 2nd step
        tr.step(*batch)
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            tr.step(*batch)
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1) / steps)
    return out


NEW_KERNELS = ('attn_bwd_dq_kernel<true>', 'attn_bwd_dkv_kernel<true>', 'dwconv_sum', 'bn_var', 'bn_finalize', 'bn_swish',
               'bn_bwd_reduce', 'bn_bwd_dx', 'dwconv_bwd_dx', 'dwconv_wgrad', 'dropout_add')


def profile(tr, batch, steps, out_dir):
    from torch.profiler import ProfilerActivity, profile as tprofile
    for _ in range(4):
        tr.step(*batch)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            tr.step(*batch)
        torch.cuda.synchronize()
    rows = [(e.key, e.device_time_total) for e in prof.key_averages()]
    total = sum(t for _, t in rows if t > 0)
    share = {}
    for key, t in rows:
        for k in NEW_KERNELS:
            if k in key:
                share[k] = share.get(k, 0.0) + t
    res = {'device_ms_per_step': total / 1e3 / steps,
           'share': {k: round(v / total, 4) for k, v in sorted(share.items(), key=lambda kv: -kv[1])},
           'new_kernels_share': round(sum(share.values()) / total, 4),
           'top': [(k, round(t / total, 4)) for k, t in sorted(rows, key=lambda kv: -kv[1])[:15]]}
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, 'conformer_train_profile.json'), 'w') as f:
            json.dump(res, f, indent=1)
    return res


def band_cost(dev, B=32, T=249, H=4, iters=50):
    """The attention backward alone at the config-4 encoder shape, without and with the rel-pos band (band reads in both
    kernels + the dBD stores of the dQ kernel): ms per call, CUDA events."""
    from opentransformer_b200 import ops
    d = 64 * H
    g = torch.Generator(device=dev).manual_seed(0)
    ext = torch.randn(B * T, 4 * d, device=dev, generator=g).to(torch.bfloat16)
    dout = torch.randn(B * T, d, device=dev, generator=g).to(torch.bfloat16)
    ld = (2 * T - 1 + 3) // 4 * 4
    bd = torch.randn(H, B * T, ld, device=dev, generator=g)
    lens = torch.full((B,), T, dtype=torch.int32, device=dev)
    dbd = torch.zeros(H, B * T, ops.rel_band_ld(T), dtype=torch.bfloat16, device=dev)
    de = torch.empty_like(ext)
    out = {}
    for name, band in (('plain', None), ('band', bd)):
        ctx, lse = ops.attention_train(ext, ext, ext, B, H, T, T, kv_len=lens, q_col0=0, k_col0=2 * d, v_col0=3 * d, bd=band)

        def call():
            ops.attention_bwd(ext, ext, ext, ctx, dout, lse, B, H, T, T, de, de, de, kv_len=lens, q_col0=0, k_col0=2 * d,
                              v_col0=3 * d, dq_col0=0, dk_col0=2 * d, dv_col0=3 * d, bd=band, dbd=dbd if band is not None else None)
        for _ in range(5):
            call()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            call()
        e1.record()
        e1.synchronize()
        out[name] = round(e0.elapsed_time(e1) / iters, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA GPU')
    dev = torch.device('cuda:0')
    print('card (name, power limit, max SM clock):', card())
    for name, params in (('conformer_cfg4_train', conformer_train_params()), ('transformer_cfg5_train', bench.train_params())):
        tr, batch = make(params, dev)
        ms = time_steps(tr, batch, a.steps, a.reps)
        print(json.dumps({'model': name, 'batch': f'{bench.B_PER_GPU} x {bench.T_FRAMES} frames, 32-token targets',
                          'ms_per_step': [round(v, 2) for v in ms], 'steps_per_rep': a.steps}))
        if name.startswith('conformer'):
            res = profile(tr, batch, 5, a.out)
            print(json.dumps({'model': name, 'profile': res}))
        del tr, batch
        torch.cuda.empty_cache()
    print(json.dumps({'attention_bwd_ms_B32_T249': band_cost(dev)}))


if __name__ == '__main__':
    main()
