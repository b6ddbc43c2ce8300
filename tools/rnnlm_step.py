"""Time the rnnlm.yaml recurrent LM (vocab 4233, 2 LSTM layers of 1024, dropout 0.1, tied) on the CUDA path next to
torch.nn.LSTM (cuDNN) on the same shapes, with CUDA events after warm-up, each figure the median of `--reps` repetitions:

  * forward + backward of the whole LM (lm.train(); loss, _ = lm(...); loss.backward()) at B = 16 and 64, L = 48;
  * the recurrence kernels alone (otb_lstm_fwd with the training tape, otb_lstm_bwd), per time step, with the bytes each
    step reads from L2 and its FLOPs computed from the shapes;
  * predict() of one token for N = 320 hypotheses (32 utterances x beam 10, zero state);
  * cuDNN: nn.LSTM(1024, 1024, 2, dropout 0.1) in bf16, forward + backward of the same [L, B, 1024] inputs, and the
    one-step forward at N = 320.

    python tools/rnnlm_step.py [--iters 20] [--reps 3] [--out DIR]

Prints the card and its power limit, then one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from opentransformer_b200 import ops  # noqa: E402
from opentransformer_b200.lm import RecurrentLanguageModel  # noqa: E402

RNNLM = dict(type='rnn_lm', vocab_size=4233, num_layers=2, hidden_size=1024, residual_dropout=0.1, smoothing=0.1, dropout=0.1,
             share_embedding=True)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def timed(fn, iters, reps):
    """Median over reps of the mean ms per call of `iters` back-to-back calls (after 3 warm-up calls)."""
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
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    lm = RecurrentLanguageModel(RNNLM).to(dev)
    H, V, L = 1024, 4233, 48
    cudnn = torch.nn.LSTM(H, H, 2, dropout=0.1).to(dev, torch.bfloat16).train()
    cudnn.flatten_parameters()
    res = {'card': card(), 'H': H, 'V': V, 'L': L, 'layers': 2}
    g = torch.Generator().manual_seed(1)
    for B in (16, 64):
        inputs = torch.randint(2, V, (B, L), generator=g).to(dev)
        targets = torch.randint(2, V, (B, L), generator=g).to(dev)
        lm.train()

        def lm_step():
            loss, _ = lm({'inputs': inputs}, {'targets': targets})
            loss.backward()
        res[f'lm_fwd_bwd_ms_B{B}'] = timed(lm_step, a.iters, a.reps)

        # the recurrence kernels alone, one layer
        pk = lm._pack.get()
        w = pk['layers'][0]['w_hh']
        gx = torch.randn(L * B, 4 * H, device=dev) * 0.1
        fwd = lambda: ops.lstm_fwd(gx.clone(), w, L, B, train=True)
        _, _, _, gates, c_all = fwd()
        dy = (torch.randn(L * B, H, device=dev) * 0.1).to(torch.bfloat16)
        t_f = timed(fwd, a.iters, a.reps)
        t_c = timed(lambda: gx.clone(), a.iters, a.reps)              # the clone inside fwd, subtracted
        t_b = timed(lambda: ops.lstm_bwd(dy, w, gates, c_all, L, B), a.iters, a.reps)
        res[f'lstm_fwd_us_per_step_B{B}'] = 1e3 * (t_f - t_c) / L
        res[f'lstm_bwd_us_per_step_B{B}'] = 1e3 * t_b / L
        grid = H // ops.lstm_config(H, torch.cuda.get_device_properties(dev).multi_processor_count,
                                    torch.cuda.get_device_properties(dev).shared_memory_per_block_optin)[0]
        res[f'lstm_fwd_l2_bytes_per_step_B{B}'] = grid * B * H * 2                 # every CTA stages all of h_{t-1} (bf16)
        res[f'lstm_bwd_l2_bytes_per_step_B{B}'] = grid * B * 4 * H * 2             # ... and all of dG_{t+1} (bf16)
        res[f'lstm_flops_per_step_B{B}'] = 2 * B * H * 4 * H                        # h W_hh^T (forward) or dG W_hh (backward)

        xs = torch.randn(L, B, H, device=dev, dtype=torch.bfloat16, requires_grad=True)

        def cudnn_step():
            y, _ = cudnn(xs)
            y.float().sum().backward()
        res[f'cudnn_lstm_fwd_bwd_ms_B{B}'] = timed(cudnn_step, a.iters, a.reps)
        with torch.no_grad():
            res[f'cudnn_lstm_fwd_ms_B{B}'] = timed(lambda: cudnn(xs), a.iters, a.reps)
            res[f'lstm_fwd_2layers_ms_B{B}'] = timed(lambda: lm._run(inputs.t().contiguous(), pk), a.iters, a.reps)

    lm.eval()
    cudnn.eval()
    N = 320
    tok = torch.randint(2, V, (N, 1), generator=g).to(dev)
    x1 = torch.randn(1, N, H, device=dev, dtype=torch.bfloat16)
    with torch.no_grad():
        res['predict_ms_N320'] = timed(lambda: lm.predict(tok), a.iters, a.reps)
        res['cudnn_lstm_fwd_ms_N320_L1'] = timed(lambda: cudnn(x1), a.iters, a.reps)
    print(res['card'])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'rnnlm_step.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
