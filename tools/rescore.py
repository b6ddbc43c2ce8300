"""N-best rescoring at the benchmark geometry: the transformer_baseline.yaml model with a joint-CTC head, random weights, the
decoder's <S/E> bias at -1e4 so that the attention search runs all 60 steps, 32 utterances x 1000 frames (T' = 249), beam 10:

  - the attention beam search, persistent kernel and per-step CUDA-graph path (recognize_ids, nbest 1);
  - apply_rescoring end to end (CTC prefix beam search over the joint-CTC head, then the attention decoder teacher-forced over
    the 10 hypotheses) and each of its stages on the same encoder output: the CTC first pass (head GEMM + frame top-40 +
    otb_ctc_prefix_beam), the decoder scoring (score_bf16), otb_token_logprob, and the rerank (second_pass_rows +
    otb_nbest_rescore);
  - the second pass on fixed synthetic n-bests of 32 and 64 tokens (random weights give the CTC pass arbitrary lengths);
  - an LM: shallow fusion (the per-step graph path) against apply_lm_rescoring (persistent first pass,
    the LM over the 10 hypotheses), with the transformer_lm.yaml LM (6 blocks, d_model 256, GLU d_ff 1024) at the model's
    4234-token vocabulary;
  - otb_token_logprob's achieved bandwidth: the bytes of the logits rows it reads (rows with a target) over its time.

CUDA events, 3 warm-up + --iters timed calls; every figure is measured --reps times in one run.  It prints the card, its
power limit and its maximum SM clock, read in the same run.  Needs a GPU.

    python tools/rescore.py [--iters 10]
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
from opentransformer_b200 import ops  # noqa: E402
from opentransformer_b200.lm import TransformerLanguageModel  # noqa: E402
from opentransformer_b200.model import SpeechToText  # noqa: E402
from opentransformer_b200.recognize import SpeechToTextRecognizer, ctc_decode, second_pass_rows  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--frames', type=int, default=1000)
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/rescore.py measures on the GPU; none is visible')
    dev = torch.device('cuda:0')
    torch.manual_seed(1234)
    model = SpeechToText(params()).eval()
    with torch.no_grad():
        model.decoder.output_layer.bias[1] = -1e4
    model = model.to(dev)
    V = model.decoder.vocab_size
    lm = TransformerLanguageModel(dict(type='transformer_lm', vocab_size=V, num_blocks=6, d_model=256, n_heads=4, d_ff=1024,
                                       residual_dropout=0.1, smoothing=0.1, share_embedding=True)).to(dev)
    B, T, K, max_len = a.batch, a.frames, 10, 60
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, T, 80, generator=g).to(dev)
    mask = torch.ones(B, T, dtype=torch.bool, device=dev)
    kw = dict(beam_width=K, nbest=1, max_len=max_len, penalty=0.6, lamda=5, ngpu=1)
    rec_pers = SpeechToTextRecognizer(model, **kw)
    rec_graph = SpeechToTextRecognizer(model, persistent=False, **kw)
    rec_resc = SpeechToTextRecognizer(model, apply_rescoring=True, **kw)
    rec_fused = SpeechToTextRecognizer(model, lm=lm, lm_weight=0.3, **kw)
    rec_lm_resc = SpeechToTextRecognizer(model, lm=lm, apply_lm_rescoring=True, rescore_weight=0.3, **kw)
    res = {'card': card(), 'batch': B, 'frames': T, 'beam': K, 'max_len': max_len, 'reps': a.reps, 'ms': {}}
    ms = res['ms']

    def add(key, v):
        ms.setdefault(key, []).append(round(v, 4))

    with torch.no_grad():
        _, _, steps = rec_pers.recognize_ids(x, mask)
        rec_lm_resc.recognize_ids(x, mask)
        res['attention_steps'] = steps
        res['persistent'] = {'attention': next(iter(rec_pers._decoders.values())).persistent,
                             'lm_rescoring_first_pass': next(iter(rec_lm_resc._decoders.values())).persistent}
        mem, mem_len, _, T2 = model.encode_bf16(x, mask)
        res['encoder_frames'] = T2
        blank = model.assistor.blank
        ids, n, sc = ctc_decode(model.assistor.logits_bf16(mem), mem_len, B, T2, V, blank, 'beam', K)
        inputs, tgt, nn, Lp = second_pass_rows(ids, n)
        res['ctc_nbest_Lp'] = Lp
        res['ctc_nbest_mean_len'] = round(float(nn.float().mean()), 2)

        def second_pass(inputs, tgt, nn, Lp):
            logits = model.decoder.score_bf16(inputs, mem, mem_len, B, K, Lp, T2)
            tok = ops.token_logprob(logits, V, tgt.view(-1))
            return ops.nbest_rescore(tgt, nn, sc, tok.view(1, B, K, Lp), 1.0, 1, Lp, 1)

        logits = model.decoder.score_bf16(inputs, mem, mem_len, B, K, Lp, T2)
        tok = ops.token_logprob(logits, V, tgt.view(-1))
        synth = {}
        for L in (32, 64):
            syn = torch.randint(2, V, (B, K, L), generator=g).to(dev)
            synth[L] = second_pass_rows(syn)
        live_rows = int((tgt >= 0).sum())
        for _ in range(a.reps):
            add('attention_persistent', timed(lambda: rec_pers.recognize_ids(x, mask), a.iters))
            add('attention_graph', timed(lambda: rec_graph.recognize_ids(x, mask), a.iters))
            add('apply_rescoring_end_to_end', timed(lambda: rec_resc.recognize_ids(x, mask), a.iters))
            add('stage_encoder', timed(lambda: model.encode_bf16(x, mask), a.iters))
            add('stage_ctc_beam', timed(lambda: ctc_decode(model.assistor.logits_bf16(mem), mem_len, B, T2, V, blank, 'beam', K),
                                        a.iters))
            add('stage_decoder_scoring', timed(lambda: model.decoder.score_bf16(inputs, mem, mem_len, B, K, Lp, T2), a.iters))
            t_tlp = timed(lambda: ops.token_logprob(logits, V, tgt.view(-1)), 10 * a.iters)
            add('stage_token_logprob', t_tlp)
            add('stage_rerank', timed(lambda: (second_pass_rows(ids, n),
                                               ops.nbest_rescore(tgt, nn, sc, tok.view(1, B, K, Lp), 1.0, 1, Lp, 1)), a.iters))
            for L, rows in synth.items():
                add(f'second_pass_synthetic_{L}_tokens', timed(lambda: second_pass(*rows[:3], rows[3]), a.iters))
                lg = model.decoder.score_bf16(rows[0], mem, mem_len, B, K, rows[3], T2)
                add(f'token_logprob_synthetic_{L}_tokens', timed(lambda: ops.token_logprob(lg, V, rows[1].view(-1)), 10 * a.iters))
            add('lm_shallow_fusion', timed(lambda: rec_fused.recognize_ids(x, mask), max(1, a.iters // 5), warmup=1))
            add('apply_lm_rescoring', timed(lambda: rec_lm_resc.recognize_ids(x, mask), a.iters))
        res['token_logprob_bandwidth'] = {}
        for name, rows, rows_live in (('ctc_nbest', B * K * Lp, live_rows),
                                      ('synthetic_32', B * K * 33, B * K * 33), ('synthetic_64', B * K * 65, B * K * 65)):
            key = 'stage_token_logprob' if name == 'ctc_nbest' else f'token_logprob_{name}_tokens'
            t = min(ms[key]) / 1e3
            byts = rows_live * V * 4 + rows * 8
            res['token_logprob_bandwidth'][name] = {'rows': rows, 'rows_read': rows_live, 'bytes': byts,
                                                    'TB_per_s': round(byts / t / 1e12, 3),
                                                    'share_of_3.35_TB_per_s': round(byts / t / HBM_BYTES_PER_S, 3)}
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
