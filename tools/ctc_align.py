"""CTC forced alignment at the CTC model's measuring shapes (tools/ctc_model.py): the transformer_baseline.yaml front end and
encoder with a 4234-token head, 32 utterances x 1000 frames (T' = 249), synthetic targets of 30 and 240 tokens (300 do
not fit in 249 frames; 240 distinct-neighbour tokens nearly fill them):

  - otb_ctc_align alone on the head's log-probs, [B, T', 4234] fp32;
  - CTCModel.align end to end (front end, encoder, head, log-softmax, alignment);
  - CTCRecognizer.recognize_spans next to recognize_ids, greedy and beam 10;
  - the baseline: torchaudio.functional.forced_align on CUDA on the same log-probs, one utterance per call (it takes a
    batch of one), with its labels checked against the kernel's.

CUDA events after warm-up; every figure is measured three times in one run.  It prints the card, its power limit and its
maximum SM clock, read in the same run.  Needs a GPU.

    python tools/ctc_align.py [--iters 20]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from ctc_model import card, params, timed  # noqa: E402
from opentransformer_b200 import ops  # noqa: E402
from opentransformer_b200.model import CTCModel  # noqa: E402
from opentransformer_b200.recognize import CTCRecognizer  # noqa: E402

V = 4234


def targets(B, L, T2, g):
    """L tokens per utterance with no adjacent repeats (so L <= T' fits), in the collate's layout <S/E> tokens <S/E>."""
    tok = torch.empty(B, L, dtype=torch.int64)
    tok[:, 0] = torch.randint(2, V, (B,), generator=g)
    for i in range(1, L):
        tok[:, i] = (tok[:, i - 1] - 2 + torch.randint(1, V - 2, (B,), generator=g)) % (V - 2) + 2
    assert L <= T2 and not bool((tok[:, 1:] == tok[:, :-1]).any())
    truth = torch.ones(B, L + 2, dtype=torch.int64)
    truth[:, 1:-1] = tok
    return tok, truth, torch.full((B,), L + 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--frames', type=int, default=1000)
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/ctc_align.py measures on the GPU; none is visible')
    import torchaudio.functional as AF
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    model = CTCModel(params()).to(dev).eval()
    B, T = a.batch, a.frames
    g = torch.Generator().manual_seed(1)
    mask = torch.ones(B, T, dtype=torch.bool, device=dev)          # full-length utterances: every row is the same work
    x = torch.randn(B, T, 80, generator=g).to(dev)
    with torch.no_grad():
        lp, n = model.inference(x, mask)
    T2 = lp.shape[1]
    res = {'card': card(), 'batch': B, 'frames': T, 'encoder_frames': T2, 'reps': a.reps, 'ms': {}}
    ms = res['ms']

    def add(key, v):
        ms.setdefault(key, []).append(round(v, 4))

    cases = {L: targets(B, L, T2, g) for L in (30, 240)}
    dcases = {L: (tok.to(dev), truth.to(dev), tlen.to(dev), torch.full((B,), L, dtype=torch.int32, device=dev))
              for L, (tok, truth, tlen) in cases.items()}
    for L, (tok, truth, tlen, n_tok) in dcases.items():            # the kernel and torchaudio agree on what is timed
        labels, _, _, path = ops.ctc_align(lp, n, tok, n_tok)
        for b in (0, B - 1):
            ta, _ = AF.forced_align(lp[b:b + 1], tok[b:b + 1].int(), n[b:b + 1], n_tok[b:b + 1], blank=0)
            assert torch.equal(ta[0].int(), labels[b]), (L, b)
        assert bool(torch.isfinite(path).all())
    recs = {mode: CTCRecognizer(model, beam_width=beam, mode=mode) for mode, beam in (('greedy', 1), ('beam', 10))}

    for _ in range(a.reps):
        with torch.no_grad():
            for L, (tok, truth, tlen, n_tok) in dcases.items():
                add(f'kernel_L{L}', timed(lambda: ops.ctc_align(lp, n, tok, n_tok), a.iters))
                add(f'align_end_to_end_L{L}', timed(lambda: model.align(x, mask, truth, tlen), a.iters))

                def ta_batch():
                    for b in range(B):
                        AF.forced_align(lp[b:b + 1], tok[b:b + 1].int(), n[b:b + 1], n_tok[b:b + 1], blank=0)
                add(f'torchaudio_cuda_L{L}', timed(ta_batch, max(2, a.iters // 4), warmup=1))
            for mode, rec in recs.items():
                add(f'recognize_ids_{mode}', timed(lambda: rec.recognize_ids(x, mask), a.iters))
                add(f'recognize_spans_{mode}', timed(lambda: rec.recognize_spans(x, mask), a.iters))
    res['kernel_over_torchaudio'] = {L: round(min(ms[f'torchaudio_cuda_L{L}']) / min(ms[f'kernel_L{L}']), 1) for L in cases}
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
