"""LM shallow fusion in the CTC prefix beam search (DESIGN.md 4.19) at the CTC model's geometry of tools/ctc_model.py:
the transformer_baseline.yaml front end and encoder under a 4234-token CTC head, random weights, 32 utterances x 1000
frames (T' 249), beam 10, per batch:

  - the unfused prefix beam search (otb_ctc_frame_topk + otb_ctc_prefix_beam) on the head's logits;
  - the fused search on the same logits, captured graph and eager, for the transformer_lm.yaml LM (6 blocks, d_model 256,
    GLU d_ff 1024) and the rnnlm.yaml LM (2 x 1024), both at vocab 4234;
  - where the time of a fused frame goes: the search step alone, and the LM step alone (eager, per frame);
  - recognize_ids end to end, unfused and fused (graph).

CUDA events after warm-up, the variants alternating over --reps repetitions (all listed).  It prints the card, its power
limit and its maximum SM clock, read in the same run.  Needs a GPU.

    python tools/ctc_lm_fusion.py [--iters 5] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from opentransformer_b200 import ops  # noqa: E402
from opentransformer_b200.ctc_fusion import CTCFusedSearch  # noqa: E402
from opentransformer_b200.lm import RecurrentLanguageModel, TransformerLanguageModel  # noqa: E402
from opentransformer_b200.model import CTCModel  # noqa: E402
from opentransformer_b200.recognize import CTC_CUTOFF_TOP_N, CTCRecognizer  # noqa: E402
from tools.ctc_model import card, params, timed  # noqa: E402

LMW, BETA = 0.3, 0.5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--frames', type=int, default=1000)
    ap.add_argument('--beam', type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/ctc_lm_fusion.py measures on the GPU; none is visible')
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    model = CTCModel(params()).to(dev).eval()
    V, B, T, W = 4234, a.batch, a.frames, a.beam
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, T, 80, generator=g).to(dev)
    mask = torch.ones(B, T, dtype=torch.bool, device=dev)
    lms = {'transformer_lm': lambda: TransformerLanguageModel(dict(
               type='transformer_lm', vocab_size=V, num_blocks=6, d_model=256, n_heads=4, d_ff=1024, residual_dropout=0.1,
               smoothing=0.1, share_embedding=True)),
           'rnnlm': lambda: RecurrentLanguageModel(dict(
               type='rnn_lm', vocab_size=V, num_layers=2, hidden_size=1024, residual_dropout=0.1, smoothing=0.1, dropout=0.1,
               share_embedding=True))}
    res = {'card': card(), 'batch': B, 'frames': T, 'beam': W, 'lm_weight': LMW, 'beta': BETA, 'iters': a.iters,
           'reps': a.reps, 'ms_per_batch': {}, 'ms_per_frame': {}, 'notes': {}}
    with torch.no_grad():
        logits, lengths, _, T2 = model.logits_bf16(x, mask)
        K = min(CTC_CUTOFF_TOP_N, V)
        lp, tok = ops.ctc_frame_topk(logits, B, T2, V, lengths, K)
        res['T_prime'] = T2
        unfused = lambda: ops.ctc_prefix_beam(*ops.ctc_frame_topk(logits, B, T2, V, lengths, K), B, T2, lengths, W)
        rec0 = CTCRecognizer(model, beam_width=W, mode='beam')
        for name, make in lms.items():
            torch.manual_seed(7)
            lm = make().eval().to(dev)
            sg = CTCFusedSearch(lm, B, W, T2, K, dev, LMW, BETA, use_graph=True)
            se = CTCFusedSearch(lm, B, W, T2, K, dev, LMW, BETA, use_graph=False)
            try:
                rg = sg.run(lp, tok, lengths)
            except NotImplementedError as e:           # the recurrence kernel's CTAs do not fit this card
                res['notes'][name] = f'skipped: {e}'
                continue
            re_ = se.run(lp, tok, lengths)
            rec = CTCRecognizer(model, lm=lm, lm_weight=LMW, beta=BETA, beam_width=W, mode='beam', lm_fusion=True)
            res['notes'][name] = {'eager_equals_graph': all(bool(torch.equal(p, q)) for p, q in zip(rg, re_)),
                                  'launches_per_frame': sg.frame.launches,
                                  'mean_1best_len': float(rg[1][:, 0].float().mean())}
            variants = {'unfused_search': unfused,
                        'fused_graph': lambda: sg.run(lp, tok, lengths),
                        'fused_eager': lambda: se.run(lp, tok, lengths),
                        'recognize_ids_unfused': lambda: rec0.recognize_ids(x, mask),
                        'recognize_ids_fused': lambda: rec.recognize_ids(x, mask)}
            # one frame at the last frame index, which rewrites the same slots from the same input every call (plus the
            # fill of the frame counter)
            last = lambda: sg.ctl[0].fill_(T2 - 1)
            per_frame = {'search_step': lambda: (last(), ops.ctc_prefix_beam_step(
                             sg.top_lp, sg.top_id, B, T2, sg.in_len, W, 0, sg.lm_rows, LMW, BETA, sg.slots, sg.ctl, sg.nodes,
                             sg.src, sg.tok, sg.ext, sg.ids, sg.lengths, sg.scores, sg.anc, sg.anc_tmp, sg.pos)),
                         'lm_step': lambda: se._lm_step(),
                         'frame_graph_replay': lambda: (last(), sg.frame.graph.replay())}
            ms = res['ms_per_batch'].setdefault(name, {})
            fr = res['ms_per_frame'].setdefault(name, {})
            for _ in range(a.reps):
                for k, fn in variants.items():
                    ms.setdefault(k, []).append(round(timed(fn, a.iters), 3))
                for k, fn in per_frame.items():
                    fr.setdefault(k, []).append(round(timed(fn, 20 * a.iters), 4))
            sg.run(lp, tok, lengths)
            del sg, se, rec
            torch.cuda.empty_cache()
    res['card_after'] = card()
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
