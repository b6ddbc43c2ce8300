"""The CTC-only model at the transformer_baseline.yaml front end and encoder (12 blocks, d_model 256, 4 heads, d_ff 2048 GLU,
residual_dropout 0.1) with a 4234-token CTC head, at 32 utterances x 1000 frames:

  - one FusedTrainer optimizer step (forward + hand-written backward + clip + Adam, CUDA graph), in ms;
  - CTCRecognizer.recognize in utterances per second, greedy and beam 10, next to the encoder + head alone (its share)
    and the decode kernels alone (otb_ctc_frame_topk + otb_ctc_greedy / otb_ctc_prefix_beam on the same logits).

It prints the card, its power limit and its maximum SM clock, read in the same run.  Needs a GPU.

    python tools/ctc_model.py [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from opentransformer_b200 import ops, train  # noqa: E402
from opentransformer_b200.model import CTCModel  # noqa: E402
from opentransformer_b200.recognize import CTC_CUTOFF_TOP_N, CTCRecognizer  # noqa: E402


def params():
    return {'type': 'ctc', 'frontend_type': 'conv', 'encoder_type': 'transformer',
            'frontend': dict(input_size=80, output_size=256, in_channel=1, mid_channel=64, out_channel=128,
                             kernel_size=[[3, 3], [3, 3]], stride=[2, 2], dropout=0.0, act_func_type='relu',
                             front_end_layer_norm=False),
            'encoder': dict(d_model=256, n_heads=4, d_ff=2048, n_blocks=12, pos_dropout=0.0, slf_attn_dropout=0.0,
                            ffn_dropout=0.0, residual_dropout=0.1, normalize_before=False, concat_after=False,
                            activation='glu', relative_positional=False),
            'encoder_output_size': 256, 'vocab_size': 4234}


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else 'unknown'


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--frames', type=int, default=1000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/ctc_model.py measures on the GPU; none is visible')
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    model = CTCModel(params()).to(dev)
    B, T = a.batch, a.frames
    g = torch.Generator().manual_seed(1)
    lens = torch.randint(int(0.8 * T), T + 1, (B,), generator=g)
    lens[0] = T
    mask = (torch.arange(T)[None] < lens[:, None]).to(dev)
    x = (torch.randn(B, T, 80, generator=g).to(dev) * mask.unsqueeze(2))
    L = 30
    tgt = torch.randint(2, 4234, (B, L), generator=g)
    tgt[:, 0] = 1
    tgt[:, -1] = 1
    tlen = torch.full((B,), L - 1)
    tgt, tlen = tgt.to(dev), tlen.to(dev)

    res = {'card': card(), 'batch': B, 'frames': T}
    model.train()
    tr = train.FusedTrainer(model, accum_steps=1, use_graph=True)
    res['train_step_ms'] = timed(lambda: tr.step(x, mask, tgt, tlen), a.iters)

    model.eval()
    with torch.no_grad():
        logits, n, _, T2 = model.logits_bf16(x, mask)
        enc_ms = timed(lambda: model.logits_bf16(x, mask), a.iters)
        for mode, beam in (('greedy', 1), ('beam', 10)):
            rec = CTCRecognizer(model, beam_width=beam, mode=mode)
            ms = timed(lambda: rec.recognize(x, mask), a.iters)
            if mode == 'greedy':
                def dec():
                    lp, tok = ops.ctc_frame_topk(logits, B, T2, 4234, n, 1)
                    ops.ctc_greedy(lp, tok, B, T2, n)
            else:
                def dec():
                    lp, tok = ops.ctc_frame_topk(logits, B, T2, 4234, n, CTC_CUTOFF_TOP_N)
                    ops.ctc_prefix_beam(lp, tok, B, T2, n, beam)
            dec_ms = timed(dec, a.iters)
            lp, tok = ops.ctc_frame_topk(logits, B, T2, 4234, n, CTC_CUTOFF_TOP_N if mode == 'beam' else 1)
            topk_ms = timed(lambda: ops.ctc_frame_topk(logits, B, T2, 4234, n, tok.shape[1]), a.iters)
            res[mode] = {'beam': beam, 'recognize_ms': ms, 'utt_per_s': B / ms * 1e3, 'encoder_and_head_ms': enc_ms,
                         'encoder_share': enc_ms / ms, 'decode_kernels_ms': dec_ms, 'frame_topk_ms': topk_ms,
                         'frame_topk_GBps': B * T2 * 4234 * 4 / topk_ms / 1e6}
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
