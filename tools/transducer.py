"""The transducer model at the transformer_baseline.yaml front end and encoder (12 blocks, d_model 256, 4 heads, d_ff 2048
GLU, residual_dropout 0.1), a 1 x 320 LSTM prediction network and a 512-wide joint over 4234 tokens, at 32 utterances x
1000 frames with 30-token transcripts:

  - one FusedTrainer optimizer step (forward + hand-written backward + clip + Adam, CUDA graph), in ms, and its peak memory;
  - TransducerRecognizer.recognize (greedy) on the same batch;
  - the transducer kernels alone on the step's lattice (CUDA events over repeated launches), and the output layer's GEMMs.

With --prune-range S it also times the FusedTrainer step of the full and of the pruned loss (joint prune_range S,
DESIGN.md 4.22) in the same run, with their peak memory, at 30-label transcripts and at 200-label ones.

It prints the card, its power limit and its maximum SM clock, read in the same run.  Needs a GPU.

    python tools/transducer.py [--iters 10] [--prune-range 5]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from opentransformer_b200 import ops, train  # noqa: E402
from opentransformer_b200.model import TransducerModel  # noqa: E402
from opentransformer_b200.recognize import TransducerRecognizer  # noqa: E402
from tools.ctc_model import card, params as ctc_params, timed  # noqa: E402


def params():
    p = ctc_params()
    return {'type': 'transducer', 'frontend_type': 'conv', 'encoder_type': 'transformer', 'frontend': p['frontend'],
            'encoder': p['encoder'], 'decoder_type': 'rnn',
            'decoder': dict(vocab_size=4234, hidden_size=320, num_layers=1, dropout=0.0), 'joint': {'inner_size': 512}}


def _batch(B, T, L, V, dev, seed=1):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(int(0.8 * T), T + 1, (B,), generator=g)
    lens[0] = T
    mask = (torch.arange(T)[None] < lens[:, None]).to(dev)
    x = (torch.randn(B, T, 80, generator=g).to(dev) * mask.unsqueeze(2))
    tgt = torch.randint(2, V, (B, L), generator=g)
    tgt[:, 0] = 1
    tgt[:, -1] = 1
    return x, mask, tgt.to(dev), torch.full((B,), L - 1).to(dev)


def full_vs_pruned(S, B, T, iters, dev):
    """FusedTrainer step time (CUDA graph, CUDA events after warm-up) and peak memory of the full and the pruned loss,
    alternated in one run, at 30- and 200-label transcripts."""
    out = []
    for labels in (30, 200):
        x, mask, tgt, tlen = _batch(B, T, labels + 2, 4234, dev)
        row = {'labels': labels}
        for name, prune in (('full', None), ('pruned', S)):
            p = params()
            p['joint'] = dict(p['joint'], prune_range=prune)
            torch.manual_seed(0)
            model = TransducerModel(p).to(dev).train()
            tr = train.FusedTrainer(model, accum_steps=1, use_graph=True)
            tr.step(x, mask, tgt, tlen)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            row[f'{name}_step_ms'] = timed(lambda: tr.step(x, mask, tgt, tlen), iters)
            row[f'{name}_peak_GB'] = torch.cuda.max_memory_allocated() / 1e9
            row[f'{name}_loss'] = float(tr.step(x, mask, tgt, tlen))
            del tr, model
            torch.cuda.empty_cache()
        out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--frames', type=int, default=1000)
    ap.add_argument('--prune-range', type=int, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/transducer.py measures on the GPU; none is visible')
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    model = TransducerModel(params()).to(dev)
    B, T, L, V = a.batch, a.frames, 32, 4234
    g = torch.Generator().manual_seed(1)
    lens = torch.randint(int(0.8 * T), T + 1, (B,), generator=g)
    lens[0] = T
    mask = (torch.arange(T)[None] < lens[:, None]).to(dev)
    x = (torch.randn(B, T, 80, generator=g).to(dev) * mask.unsqueeze(2))
    tgt = torch.randint(2, V, (B, L), generator=g)
    tgt[:, 0] = 1
    tgt[:, -1] = 1
    tlen = torch.full((B,), L - 1)                      # 30 labels: U + 1 = 31 lattice columns
    tgt, tlen = tgt.to(dev), tlen.to(dev)

    res = {'card': card(), 'batch': B, 'frames': T, 'labels': L - 2}
    model.train()
    tr = train.FusedTrainer(model, accum_steps=1, use_graph=True)
    tr.step(x, mask, tgt, tlen)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    res['train_step_ms'] = timed(lambda: tr.step(x, mask, tgt, tlen), a.iters)
    res['train_peak_GB'] = torch.cuda.max_memory_allocated() / 1e9

    model.eval()
    rec = TransducerRecognizer(model, max_len=100)
    with torch.no_grad():
        res['recognize_ms'] = timed(lambda: rec.recognize(x, mask), max(1, a.iters // 2), warmup=1)
        res['encoder_ms'] = timed(lambda: model.encode_bf16(x, mask), a.iters)
        ids, n, _ = rec.recognize_ids(x, mask)
        res['recognized_tokens_mean'] = float(n.float().mean())

        # the kernels on the step's lattice
        mem, lengths, B, T2 = model.encode_bf16(x, mask)
        op = model._pack.get()
        U1 = L - 1
        u_len = (tlen - 1).to(torch.int32)
        labels = tgt[:, 1:-1].to(torch.int32).contiguous()
        ep = ops.linear(mem, op['enc'].w, op['enc'].b, ops.EPI_BIAS)
        pp = torch.randn(B * U1, 512, device=dev).to(ops.BF16)
        hj = ops.rnnt_joint(ep, pp, B, T2, U1, lengths, u_len)
        rows, ld = B * T2 * U1, model.joint.ld_logits
        k = {'lattice_rows': rows}
        k['joint_ms'] = timed(lambda: ops.rnnt_joint(ep, pp, B, T2, U1, lengths, u_len, out=hj), a.iters)
        k['joint_bwd_ms'] = timed(lambda: ops.rnnt_joint_bwd(hj, hj, B, T2, U1, lengths, u_len), a.iters)
        chunk = train.RNNT_WORKSPACE_BYTES // (4 * ld) // 8 * 8
        ws = torch.empty(chunk, ld, device=dev)
        logits = ops.linear(hj[:chunk], op['out_w'], op['out_b'], ops.EPI_BIAS, out=ws)
        k['chunk_rows'] = chunk
        k['output_gemm_chunk_ms'] = timed(lambda: ops.linear(hj[:chunk], op['out_w'], op['out_b'], ops.EPI_BIAS, out=ws), a.iters)
        k['output_gemm_TFLOPs'] = 2.0 * chunk * 512 * ld / k['output_gemm_chunk_ms'] / 1e9
        lp = torch.zeros(rows, 3, device=dev)
        k['logprob_chunk_ms'] = timed(lambda: ops.rnnt_logprob(logits, 0, V, B, T2, U1, lengths, u_len, labels, lp), a.iters)
        k['logprob_GBps'] = chunk * ld * 4 / k['logprob_chunk_ms'] / 1e6
        for r0 in range(0, rows, chunk):
            n_r = min(chunk, rows - r0)
            ops.rnnt_logprob(ops.linear(hj[r0:r0 + n_r], op['out_w'], op['out_b'], ops.EPI_BIAS, out=ws[:n_r]), r0, V, B, T2, U1,
                             lengths, u_len, labels, lp)
        k['loss_ms'] = timed(lambda: ops.rnnt_loss(lp, B, T2, U1, lengths, u_len), a.iters)
        _, _, grad = ops.rnnt_loss(lp, B, T2, U1, lengths, u_len)
        logits = ops.linear(hj[:chunk], op['out_w'], op['out_b'], ops.EPI_BIAS, out=ws)
        k['dlogits_chunk_ms'] = timed(lambda: ops.rnnt_dlogits(logits, 0, V, B, T2, U1, lengths, u_len, labels, lp, grad), a.iters)
        res['kernels'] = k
    if a.prune_range is not None:
        del tr, rec, hj, ws, logits, lp, grad
        torch.cuda.empty_cache()
        res['prune_range'] = a.prune_range
        res['full_vs_pruned'] = full_vs_pruned(a.prune_range, a.batch, a.frames, a.iters, dev)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
