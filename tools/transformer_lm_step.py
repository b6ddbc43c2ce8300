"""Time training the transformer_lm.yaml language model (vocab 4233, 6 blocks of d_model 256 / 4 heads / GLU d_ff 1024,
residual_dropout 0.1, tied) on the CUDA path next to the reference's own TransformerLanguageModel (oracle/_ref, built by
oracle/build_ref.py) on the same GPU, at 16 x 48 and 64 x 48 tokens, with CUDA events after warm-up, each figure the median
of `--reps` repetitions:

  * forward + backward through the autograd seam (lm.train(); loss, _ = lm(...); loss.backward());
  * one optimizer step of FusedTrainer: accum_steps 4 micro-batches, clip 5, TransformerScheduler + Adam, CUDA graph;
  * the reference, fp32 eager autograd: its forward + loss.backward(), and the same optimizer step (4 x forward + backward,
    clip_grad_norm_(5), torch.optim.Adam with the scheduler's learning rate set by hand).

    python tools/transformer_lm_step.py [--iters 20] [--reps 3] [--out DIR]

Prints the card and its power limit, then one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from opentransformer_b200 import ops  # noqa: E402
from opentransformer_b200.lm import TransformerLanguageModel  # noqa: E402
from opentransformer_b200.train import FusedTrainer, transformer_lr  # noqa: E402
from oracle import build_ref  # noqa: E402

TLM = dict(type='transformer_lm', vocab_size=4233, num_blocks=6, d_model=256, n_heads=4, d_ff=1024, residual_dropout=0.1,
           smoothing=0.1, share_embedding=True)
ACCUM, L = 4, 48


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def timed(fn, iters, reps):
    """Mean ms per call of `iters` back-to-back calls (after 3 warm-up calls), each of `reps` repetitions."""
    for _ in range(3):
        fn()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / iters)
    return out


def put(res, key, times):
    res[key] = statistics.median(times)
    res[key + '_reps'] = [round(t, 3) for t in times]


def batches(N, g, dev):
    """ACCUM micro-batches of N rows: BOS + tokens / tokens + EOS, PAD after ragged lengths (row 0 full)."""
    out = []
    for _ in range(ACCUM):
        toks = torch.randint(2, TLM['vocab_size'], (N, L), generator=g)
        lens = torch.randint(L // 4, L + 1, (N,), generator=g)
        lens[0] = L
        inputs = torch.cat([torch.ones(N, 1, dtype=torch.long), toks[:, :-1]], 1)
        targets = toks.clone()
        for b, n in enumerate(lens.tolist()):
            targets[b, n - 1] = 1
            targets[b, n:] = 0
            inputs[b, n:] = 0
        out.append((inputs.to(dev), targets.to(dev)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    if build_ref.load() is None:
        raise SystemExit('oracle/_ref is missing: run oracle/build_ref.py (or __graft_entry__.build()) first')
    from otrans.model.lm import TransformerLanguageModel as RefLM
    torch.manual_seed(0)
    lm = TransformerLanguageModel(TLM).to(dev).train()
    ref = RefLM(TLM).to(dev).train()
    ref.load_state_dict(lm.state_dict())
    res = {'card': card(), 'V': TLM['vocab_size'], 'blocks': TLM['num_blocks'], 'd_model': TLM['d_model'], 'L': L,
           'accum_steps': ACCUM, 'params': sum(p.numel() for p in lm.parameters())}
    g = torch.Generator().manual_seed(1)
    for N in (16, 64):
        bs = batches(N, g, dev)
        x, y = bs[0]

        def seam():
            loss, _ = lm({'inputs': x}, {'targets': y})
            loss.backward()
        put(res, f'seam_fwd_bwd_ms_N{N}', timed(seam, a.iters, a.reps))
        n0 = ops.COUNTERS['launches']
        seam()
        res[f'seam_launches_N{N}'] = ops.COUNTERS['launches'] - n0

        def ref_fwd_bwd():
            loss, _ = ref({'inputs': x}, {'targets': y})
            loss.backward()
        put(res, f'ref_fwd_bwd_ms_N{N}', timed(ref_fwd_bwd, a.iters, a.reps))

        # a fresh copy of the weights for each trainer: FusedTrainer turns the parameters into views of its flat buffer
        tlm = TransformerLanguageModel(TLM).to(dev).train()
        tlm.load_state_dict(lm.state_dict())
        tr = FusedTrainer(tlm, lr=1e-3, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6, clip_grad=5.0, model_size=256,
                          warmup_steps=12000, accum_steps=ACCUM, use_graph=True)

        def fused_step():
            for xb, yb in bs:
                tr.step(xb, yb)
        put(res, f'fused_opt_step_ms_N{N}', timed(fused_step, a.iters, a.reps))
        res[f'fused_graphs_N{N}'] = len(tr._graphs)

        rlm = RefLM(TLM).to(dev).train()
        rlm.load_state_dict(lm.state_dict())
        opt = torch.optim.Adam(rlm.parameters(), lr=1e-3, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6)
        step = [2]

        def ref_step():
            for xb, yb in bs:
                loss, _ = rlm({'inputs': xb}, {'targets': yb})
                (loss / ACCUM).backward()
            torch.nn.utils.clip_grad_norm_(rlm.parameters(), 5.0)
            step[0] += 1
            for grp in opt.param_groups:
                grp['lr'] = transformer_lr(step[0], 256, 12000)
            opt.step()
            opt.zero_grad()
        put(res, f'ref_opt_step_ms_N{N}', timed(ref_step, a.iters, a.reps))
        res[f'tokens_per_opt_step_N{N}'] = int(sum(int((yb != 0).sum()) for _, yb in bs))
    print(res['card'])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'transformer_lm_step.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
