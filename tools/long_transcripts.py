"""Long transcripts: the CTC loss past 64 labels and the KV-cached decoder self-attention past 128 cached positions.

  - otb_ctc_loss at B 32, V 4234, L in {64, 65, 256, 1023} labels, with T' = max(250, 2 L + 50) frames so that every
    utterance is feasible (64 takes the short kernels, 65 and up the long ones): the loss alone (alpha/beta + mean), the
    gradient kernel (the difference with dlogits), and ops.ctc_loss as the trainers call it (with the log-softmax);
  - decode_self_attn per call at bench.py's decode geometry (32 utterances x beam 10 = 320 hypotheses, 4 heads of 64)
    at prefix lengths 128, 256, 512 and 1023 (a cache of 1023 positions: the chunked kernel), and at 128 in a cache of
    128 positions (the one-chunk kernel);
  - SpeechToTextRecognizer.recognize_ids on bench.py's model and batch (random weights, EOS biased down, so every
    hypothesis runs to max_len) at max_len 128 (persistent kernel) and 129 (per-step graph path);
  - the KV-cache and CTC-workspace bytes, computed from shapes.

CUDA events after warm-up; each figure is the mean over --iters calls.  The card, its power limit and its maximum SM
clock are read in the same run.  Needs a GPU.

    python tools/long_transcripts.py [--iters 20]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench  # noqa: E402
from ctc_model import card, timed  # noqa: E402
from opentransformer_b200 import ops  # noqa: E402
from opentransformer_b200.recognize import SpeechToTextRecognizer  # noqa: E402

DEV = torch.device('cuda:0')
V = 4234


def ctc_rows(iters):
    """otb_ctc_loss alone on preallocated buffers (the log-softmax done once outside the timed calls): without dlogits it
    runs the alpha/beta kernel and the mean, with dlogits the gradient kernel too; the gradient kernel's time is the
    difference.  ops.ctc_loss, as the trainers call it, adds otb_log_softmax over V and the allocations."""
    from opentransformer_b200 import _lib
    rows = []
    B = 32
    for L in (64, 65, 256, 1023):
        T = max(250, 2 * L + 50)
        g = torch.Generator().manual_seed(L)
        logits = (torch.randn(B * T, 4240, generator=g) * 2).to(DEV)
        tgt = torch.randint(1, V, (B, L), generator=g).to(DEV)
        tlen = torch.full((B,), L, dtype=torch.int32, device=DEV)
        in_len = torch.full((B,), T, dtype=torch.int32, device=DEV)
        logp = ops.log_softmax(logits, V)
        ld = logp.stride(0)
        nll = torch.empty(B, dtype=torch.float32, device=DEV)
        loss = torch.empty(1, dtype=torch.float32, device=DEV)
        ws = torch.empty(B, T, 2 * L + 1, dtype=torch.float32, device=DEV)
        dl = torch.empty(B * T, ld, dtype=ops.BF16, device=DEV)

        def run(grad):
            ops.check(_lib.lib().otb_ctc_loss(ops._p(logp), ld, B, T, V, ops._p(in_len), ops._p(tgt), tgt.stride(0), ops._p(tlen),
                                              L, 0, ops._p(nll), ops._p(loss), ops._p(ws), ops._p(dl) if grad else None,
                                              ld if grad else 0, 1.0, None, ops._stream()), 'otb_ctc_loss')
        fwd = timed(lambda: run(False), iters)
        both = timed(lambda: run(True), iters)
        whole = timed(lambda: ops.ctc_loss(logits, B, T, V, in_len, tgt, tlen, 0, want_grad=True), iters)
        kind = 'short' if L <= 64 else 'long'
        rows.append((f'otb_ctc_loss loss only (alpha/beta + mean, {kind}), B {B}, T\' {T}, L {L}', f'{fwd:.3f} ms',
                     f'workspace {B * T * (2 * L + 1) * 4 / 1e6:.0f} MB'))
        rows.append((f'ctc_grad_kernel ({kind}; difference), B {B}, T\' {T}, L {L}', f'{both - fwd:.3f} ms', ''))
        rows.append((f'ops.ctc_loss with gradient (+ log-softmax over V {V}, allocations), L {L}', f'{whole:.3f} ms', ''))
        del logits, logp, ws, dl
        torch.cuda.empty_cache()
    return rows


def attn_rows(iters):
    rows = []
    N, H, d = 320, 4, 256
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(N, 3 * d, generator=g).to(ops.BF16).to(DEV)
    for Lmax, prefixes in ((128, (128,)), (1023, (128, 256, 512, 1023))):
        kc = torch.randn(Lmax, N, d, generator=g).to(ops.BF16).to(DEV)
        vc = torch.randn(Lmax, N, d, generator=g).to(ops.BF16).to(DEV)
        anc = torch.randint(0, N, (2, N, Lmax), generator=g).to(torch.int32).to(DEV)
        for p in prefixes:
            ctrl = torch.tensor([p - 1, 0, 0, 0], dtype=torch.int32, device=DEV)
            ms = timed(lambda: ops.decode_self_attn(qkv, kc, vc, anc, ctrl, N, H, Lmax), iters * 10)
            rows.append((f'decode_self_attn, N {N}, cache {Lmax}, prefix {p}', f'{ms * 1e3:.1f} us',
                         'chunked' if Lmax > 128 else 'one chunk'))
    return rows


def recognizer_rows(iters):
    rows = []
    model = bench.build_model().to(DEV)
    x, mask = bench.synthetic_batch(bench.B_PER_GPU, 0)
    x, mask = x.to(DEV), mask.to(DEV)
    for max_len in (128, 129):
        rec = SpeechToTextRecognizer(model, beam_width=bench.BEAM, nbest=1, max_len=max_len)
        ms = timed(lambda: rec.recognize_ids(x, mask), max(2, iters // 4), warmup=2)
        steps = int(rec.recognize_ids(x, mask)[2])
        path = 'persistent kernel' if max_len <= 128 else 'per-step graph'
        rows.append((f'recognize_ids, B {bench.B_PER_GPU}, beam {bench.BEAM}, max_len {max_len} ({path})', f'{ms:.1f} ms',
                     f'{steps} steps, {bench.B_PER_GPU * 1e3 / ms:.1f} utt/s'))
    return rows


def memory_rows():
    n_layers, N, d = 6, 320, 256
    rows = []
    for Lmax in (128, 1023):
        kv = n_layers * Lmax * N * d * 2 * 2
        rows.append((f'KV cache, {n_layers} layers x Lmax {Lmax} x N {N} x d {d} x (K, V) bf16', f'{kv / 1e9:.3f} GB',
                     'computed'))
    for B, T, L in ((32, 1000, 64), (32, 1000, 1023)):
        rows.append((f'CTC workspace, B {B} x T\' {T} x (2 L + 1) f32, L {L}', f'{B * T * (2 * L + 1) * 4 / 1e6:.0f} MB',
                     'computed'))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('long_transcripts.py measures on the GPU: no CUDA device')
    print(f'card: {card()}')
    rows = ctc_rows(a.iters) + attn_rows(a.iters) + recognizer_rows(a.iters) + memory_rows()
    w = max(len(r[0]) for r in rows)
    print(f'| {"what".ljust(w)} | time / size | note |')
    print(f'|{"-" * (w + 2)}|---|---|')
    for r in rows:
        print(f'| {r[0].ljust(w)} | {r[1]} | {r[2]} |')


if __name__ == '__main__':
    main()
