"""CTC rescoring of the attention n-best at the benchmark geometry: the transformer_baseline.yaml model with a joint-CTC head,
random weights, the decoder's <S/E> bias at -1e4 so that the attention search runs all 60 steps, 32 utterances x 1000
frames (T' = 249), beam 10:

  - the attention beam search alone (persistent kernel, recognize_ids, nbest 1);
  - the same search plus apply_ctc_rescoring end to end, and its CTC stages on the same encoder output: the head's
    GEMM + log-softmax, and otb_ctc_nbest_score alone on the search's 10 hypotheses per utterance (and on synthetic rows of
    129 labels, max_len 128's widest);
  - joint CTC/attention decoding at ctc_weight 0.3 (the per-step graph path);
  - otb_ctc_nbest_score's bytes from shapes: the distinct (frame, label) cells of each utterance's log-probs its rows read
    (4 B each, and the 32 B sectors holding them), the targets and the output, over its time and against the data sheet's
    3.35 TB/s.

CUDA events, 3 warm-up + --iters timed calls; every figure is measured --reps times in one run, the configurations in
alternation.  It prints the card, its power limit and its maximum SM clock, read in the same run.  Needs a GPU.

    python tools/ctc_rescore.py [--iters 10]
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
from opentransformer_b200.model import SpeechToText  # noqa: E402
from opentransformer_b200.recognize import SpeechToTextRecognizer, second_pass_rows  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


def cells_read(tgt, mem_len, blank):
    """(distinct (frame, column) cells, distinct (frame, 32-byte sector) pairs) of the log-prob rows the kernel reads: every
    valid frame of utterance b reads the blank and each label of its K rows."""
    cells = sectors = 0
    for b in range(tgt.shape[0]):
        cols = torch.unique(torch.cat((tgt[b][tgt[b] >= 0].long().cpu(), torch.tensor([blank]))))
        cells += int(mem_len[b]) * cols.numel()
        sectors += int(mem_len[b]) * torch.unique(cols // 8).numel()
    return cells, sectors


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--frames', type=int, default=1000)
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/ctc_rescore.py measures on the GPU; none is visible')
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
    rec_att = SpeechToTextRecognizer(model, **kw)
    rec_ctc_resc = SpeechToTextRecognizer(model, apply_ctc_rescoring=True, **kw)
    rec_joint = SpeechToTextRecognizer(model, ctc_weight=0.3, **kw)
    res = {'card': card(), 'batch': B, 'frames': T, 'beam': K, 'max_len': max_len, 'reps': a.reps, 'ms': {}}
    ms = res['ms']

    def add(key, v):
        ms.setdefault(key, []).append(round(v, 4))

    with torch.no_grad():
        _, _, steps = rec_att.recognize_ids(x, mask)
        rec_ctc_resc.recognize_ids(x, mask)
        res['attention_steps'] = steps
        res['persistent'] = {'attention': next(iter(rec_att._decoders.values())).persistent,
                             'ctc_rescoring_first_pass': next(iter(rec_ctc_resc._decoders.values())).persistent,
                             'joint_decoding': False}
        rec_joint.recognize_ids(x, mask)
        res['persistent']['joint_decoding'] = next(iter(rec_joint._decoders.values())).persistent
        bd = next(iter(rec_ctc_resc._decoders.values()))
        first, _ = bd.state.finalize(0.6, 5, K)
        mem, mem_len, _, T2 = model.encode_bf16(x, mask)
        res['encoder_frames'] = T2
        head = model.assistor
        _, tgt, _, Lp = second_pass_rows(first[:, :, :steps])
        logp = ops.log_softmax(head.logits_bf16(mem), V)
        syn = torch.randint(2, V, (B, K, 129), generator=g, dtype=torch.int32).to(dev)
        syn[:, :, -1] = 1
        shapes = {'nbest': tgt, 'synthetic_129': syn}
        res['Lp'] = {k: t.shape[2] for k, t in shapes.items()}
        for _ in range(a.reps):
            add('attention_search', timed(lambda: rec_att.recognize_ids(x, mask), a.iters))
            add('attention_search_plus_ctc_rescoring', timed(lambda: rec_ctc_resc.recognize_ids(x, mask), a.iters))
            add('joint_decoding_ctc_weight_0.3', timed(lambda: rec_joint.recognize_ids(x, mask), max(1, a.iters // 2)))
            add('stage_head_logits_log_softmax', timed(lambda: ops.log_softmax(head.logits_bf16(mem), V), a.iters))
            for name, t in shapes.items():
                add(f'kernel_ctc_nbest_score_{name}',
                    timed(lambda: ops.ctc_nbest_score(logp, B, T2, mem_len, t, head.blank), 10 * a.iters))
        res['kernel_bytes'] = {}
        for name, t in shapes.items():
            sec = min(ms[f'kernel_ctc_nbest_score_{name}']) / 1e3
            cells, sectors = cells_read(t, mem_len, head.blank)
            other = t.numel() * 4 + B * K * 4 + B * 4
            byts, byts_sec = cells * 4 + other, sectors * 32 + other
            res['kernel_bytes'][name] = {
                'cells': cells, 'bytes': byts, 'sector_bytes': byts_sec,
                'TB_per_s': round(byts / sec / 1e12, 4), 'sector_TB_per_s': round(byts_sec / sec / 1e12, 4),
                'share_of_3.35_TB_per_s': round(byts_sec / sec / HBM_BYTES_PER_S, 4),
                'logp_matrix_bytes': logp.numel() * 4}
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
