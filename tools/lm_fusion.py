"""LM shallow fusion at the benchmark geometry: the transformer_baseline.yaml model, random weights, the decoder's <S/E> bias
at -1e4 so that the search runs all 60 steps, 32 utterances x 1000 frames (T' = 249), beam 10.  Per batch (encoder pass +
search + finalize, recognize_ids' work), for the transformer_lm.yaml LM (6 blocks, d_model 256, GLU d_ff 1024) and the
rnnlm.yaml LM (2 x 1024), both at the model's 4234-token vocabulary:

  (a) the search as it ran before the LM entered the captured step: lm_log_probs over the reconstructed prefixes, then the
      eager step of an LM-less BeamDecoder, polling the end after every step;
  (b) the fused step, eager (use_graph=False);
  (c) the fused step on the per-step CUDA graph (the default);
  (d) the per-step graph without an LM, and the persistent kernel without an LM.

It asserts that the recurrent LM's ids and scores are identical between (a) and (c), and reports how many 1-bests of (a)
and (c) agree for the Transformer LM (the cached and the full-prefix LM round differently).  The rnnlm.yaml LM needs 128
co-resident CTAs for its recurrence kernel; a card with fewer SMs refuses it, and the script says so and skips it.

CUDA events, 3 warm-up + --iters timed calls; the variants alternate, --reps times in one run.  It prints the card, its
power limit and its maximum SM clock, read in the same run.  Needs a GPU.

    python tools/lm_fusion.py [--iters 5]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from ctc_model import card, timed  # noqa: E402
from joint_decode import params  # noqa: E402
from opentransformer_b200.lm import RecurrentLanguageModel, TransformerLanguageModel  # noqa: E402
from opentransformer_b200.model import SpeechToText  # noqa: E402
from opentransformer_b200.recognize import BeamDecoder, SpeechToTextRecognizer, lm_log_probs  # noqa: E402

LMW = 0.3


def old_fused_search(model, lm, x, mask, beam, max_len):
    """(a): what recognize_ids did with an LM before: the host loop over lm_log_probs + the eager LM-less step."""
    mem, lens, B, T2 = model.encode_bf16(x, mask)
    bd = BeamDecoder(model.decoder, B, beam, T2, max_len, x.device, use_graph=False, keep_logp=False)
    bd.setup(mem, lens)
    bd.lm_weight = LMW
    for i in range(max_len):
        bd.lm_logp = lm_log_probs(lm, bd.state.reconstruct(i))
        bd._step_kernels()
        if int(bd._read_ctrl()[1]):
            break
    steps = int(bd._read_ctrl()[0])
    preds, scores = bd.state.finalize(0.6, 5, 1)
    return preds[:, :, :steps], scores, steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--frames', type=int, default=1000)
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/lm_fusion.py measures on the GPU; none is visible')
    dev = torch.device('cuda:0')
    torch.manual_seed(1234)
    model = SpeechToText(params()).eval()
    with torch.no_grad():
        model.decoder.output_layer.bias[1] = -1e4
    model = model.to(dev)
    V = model.decoder.vocab_size
    B, T, K, max_len = a.batch, a.frames, 10, 60
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, T, 80, generator=g).to(dev)
    mask = torch.ones(B, T, dtype=torch.bool, device=dev)
    kw = dict(beam_width=K, nbest=1, max_len=max_len, penalty=0.6, lamda=5, ngpu=1)
    lms = {'transformer_lm': lambda: TransformerLanguageModel(dict(
               type='transformer_lm', vocab_size=V, num_blocks=6, d_model=256, n_heads=4, d_ff=1024, residual_dropout=0.1,
               smoothing=0.1, share_embedding=True)),
           'rnnlm': lambda: RecurrentLanguageModel(dict(
               type='rnn_lm', vocab_size=V, num_layers=2, hidden_size=1024, residual_dropout=0.1, smoothing=0.1, dropout=0.1,
               share_embedding=True))}
    res = {'card': card(), 'batch': B, 'frames': T, 'beam': K, 'max_len': max_len, 'lm_weight': LMW, 'iters': a.iters,
           'reps': a.reps, 'ms_per_batch': {}, 'notes': {}}
    rec_none_graph = SpeechToTextRecognizer(model, persistent=False, **kw)
    rec_none_pers = SpeechToTextRecognizer(model, **kw)
    with torch.no_grad():
        for name, make in lms.items():
            torch.manual_seed(7)
            lm = make().eval().to(dev)
            rec_e = SpeechToTextRecognizer(model, lm=lm, lm_weight=LMW, use_graph=False, **kw)
            rec_g = SpeechToTextRecognizer(model, lm=lm, lm_weight=LMW, **kw)
            try:
                pc, sc, nc = rec_g.recognize_ids(x, mask)
            except NotImplementedError as e:           # the recurrence kernel's CTAs do not fit this card
                res['notes'][name] = f'skipped: {e}'
                continue
            pa, sa, na = old_fused_search(model, lm, x, mask, K, max_len)
            pb, sb, nb = rec_e.recognize_ids(x, mask)
            res['notes'][name] = {'steps': [na, nb, nc],
                                  'eager_equals_graph': bool(torch.equal(pb, pc) and torch.equal(sb, sc) and nb == nc),
                                  'one_best_shared_old_vs_graph': f'{int((pa[:, 0] == pc[:, 0]).all(dim=1).sum())}/{B}'}
            if name == 'rnnlm':
                assert na == nc and torch.equal(pa, pc) and torch.equal(sa, sc), 'recurrent LM: (a) and (c) differ'
            ms = res['ms_per_batch'].setdefault(name, {})
            variants = {'a_old_host_loop': lambda: old_fused_search(model, lm, x, mask, K, max_len),
                        'b_fused_eager': lambda: rec_e.recognize_ids(x, mask),
                        'c_fused_graph': lambda: rec_g.recognize_ids(x, mask),
                        'd_no_lm_graph': lambda: rec_none_graph.recognize_ids(x, mask),
                        'd_no_lm_persistent': lambda: rec_none_pers.recognize_ids(x, mask)}
            for _ in range(a.reps):
                for key, fn in variants.items():
                    ms.setdefault(key, []).append(round(timed(fn, a.iters), 3))
            del rec_e, rec_g, lm
            torch.cuda.empty_cache()
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
