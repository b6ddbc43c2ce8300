"""Cost of the attention maps (return_attn_weights, otb_attention_probs) at the shipped model sizes:

  - transformer_baseline.yaml (bench.model_params(): d_model 256, 4 heads of 64, abs-pos) and conformer_baseline.yaml
    (d_model 384, 4 heads of 96, rel-pos band), each at 32 x 1000 frames (T' 249) and 8 x 4000 frames (T' 999);
  - the encoder forward (encode_bf16, eager) without and with the maps, alternating, --reps times;
  - otb_attention_probs alone on one block's shape: time, bytes written (B H T' T' 4), bytes read (Q and K, and for the
    Conformer the band rows, read once per sweep), and the achieved bandwidth against the H100 SXM's 3.35 TB/s.

CUDA events around --iters calls after 3 warm-up calls.  It prints the card, its power limit and its maximum SM clock, read in
the same run.  Needs a GPU.

    python tools/attn_weights.py [--iters 20] [--reps 3]
"""
import argparse
import copy
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench  # noqa: E402
from ctc_model import card, timed  # noqa: E402
from opentransformer_b200 import ops  # noqa: E402
from opentransformer_b200.model import SpeechToText  # noqa: E402
from opentransformer_b200.modules import rel_pos_band  # noqa: E402
from tests.test_head_dim_96 import CONFORMER_BASELINE  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def probs_alone(enc, B, T2, dev, iters):
    """One block's otb_attention_probs on random operands of the encoder's layout."""
    blk = enc.blocks[0]
    conformer = hasattr(blk, 'mha')
    attn = blk.mha if conformer else blk.slf_attn
    H = attn.nheads if conformer else blk.n_heads
    d = enc.d_model
    dk = d // H
    g = torch.Generator().manual_seed(0)
    lens = torch.full((B,), T2, dtype=torch.int32, device=dev)
    out = torch.empty(B, H, T2, T2, dtype=torch.float32, device=dev)
    if conformer:
        m = torch.randn(B * T2, 4 * d, generator=g).to(torch.bfloat16).to(dev)
        bd = rel_pos_band(m, torch.randn(2 * T2 - 1, d, generator=g).to(torch.bfloat16).to(dev), H, B, T2)
        call = lambda: ops.attention_probs(m, m, B, H, T2, T2, kv_len=lens, q_col0=0, k_col0=2 * d, bd=bd, d_k=dk, out=out)  # noqa: E731
        band_read = 2 * B * H * T2 * T2 * 4
    else:
        m = torch.randn(B * T2, 3 * d, generator=g).to(torch.bfloat16).to(dev)
        call = lambda: ops.attention_probs(m, m, B, H, T2, T2, kv_len=lens, q_col0=0, k_col0=d, d_k=dk, out=out)  # noqa: E731
        band_read = 0
    ms = timed(call, iters)
    written = B * H * T2 * T2 * 4
    read = 2 * B * T2 * d * 2 + band_read
    return {'ms': ms, 'bytes_written': written, 'bytes_read': read,
            'write_TBps': written / (ms * 1e-3) / 1e12, 'total_TBps': (written + read) / (ms * 1e-3) / 1e12,
            'share_of_3.35TBps': (written + read) / (ms * 1e-3) / HBM_BYTES_PER_S}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/attn_weights.py needs a GPU')
    dev = torch.device('cuda:0')
    res = {'card': card(), 'iters': args.iters, 'configs': []}
    for name, params in (('transformer_baseline', bench.model_params()), ('conformer_baseline', copy.deepcopy(CONFORMER_BASELINE))):
        torch.manual_seed(1234)
        model = SpeechToText(params).eval().to(dev)
        for B, T in ((32, 1000), (8, 4000)):
            g = torch.Generator().manual_seed(B)
            x = torch.randn(B, T, 80, generator=g).to(dev)
            mask = torch.ones(B, T, dtype=torch.bool, device=dev)
            _, _, T2, _ = ops.conv_geometry(T, 80)
            off, on = [], []
            with torch.no_grad():
                for _ in range(args.reps):
                    off.append(timed(lambda: model.encode_bf16(x, mask), args.iters))
                    on.append(timed(lambda: model.encode_bf16(x, mask, attn_sink=[]), args.iters))
                alone = probs_alone(model.encoder, B, T2, dev, args.iters)
            n_blocks = len(model.encoder.blocks)
            H = alone['bytes_written'] // (B * T2 * T2 * 4)
            res['configs'].append({'model': name, 'batch': B, 'frames': T, 'T2': T2, 'blocks': n_blocks,
                                   'maps_MB': n_blocks * B * H * T2 * T2 * 4 / 1e6, 'encoder_ms_off': off,
                                   'encoder_ms_on': on, 'probs_one_block': alone})
            print(json.dumps(res['configs'][-1]), flush=True)
        del model
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
