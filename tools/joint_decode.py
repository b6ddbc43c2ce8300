"""Joint CTC/attention decoding at the benchmark geometry: the transformer_baseline.yaml model with a joint-CTC head, random
weights, the decoder's <S/E> bias at -1e4 so that all 60 steps run, 32 utterances x 1000 frames (T' = 249), beam 10, 16
candidates per hypothesis, the per-step CUDA-graph path:

  - recognize_ids at ctc_weight 0 (graph path, persistent=False) next to ctc_weight 0.3, alternating;
  - one step's otb_ctc_prefix_score + otb_ctc_prefix_advance alone, on the search state the run left behind;
  - the once-per-batch work: the head GEMM + log-softmax + otb_ctc_prefix_init;
  - recognize_spans next to recognize_ids.

CUDA events, 3 warm-up + --iters timed calls; every figure is measured --reps times in one run.  It prints the card, its
power limit and its maximum SM clock, read in the same run.  Needs a GPU.

    python tools/joint_decode.py [--iters 20]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from ctc_model import card, timed  # noqa: E402
from opentransformer_b200 import ops  # noqa: E402
from opentransformer_b200.model import SpeechToText  # noqa: E402
from opentransformer_b200.recognize import SpeechToTextRecognizer  # noqa: E402


def params():
    """egs/aishell/conf/transformer_baseline.yaml `model:` with input_size 80 and the joint-CTC head."""
    return {'type': 'speech2text', 'frontend_type': 'conv', 'encoder_type': 'transformer', 'decoder_type': 'transformer',
            'frontend': dict(input_size=80, output_size=256, in_channel=1, mid_channel=64, out_channel=128,
                             kernel_size=[[3, 3], [3, 3]], stride=[2, 2], dropout=0.0, act_func_type='relu',
                             front_end_layer_norm=False),
            'encoder': dict(d_model=256, n_heads=4, d_ff=2048, n_blocks=12, pos_dropout=0.0, slf_attn_dropout=0.0,
                            ffn_dropout=0.0, residual_dropout=0.1, normalize_before=False, concat_after=False,
                            activation='glu', relative_positional=False),
            'decoder': dict(vocab_size=4234, d_model=256, n_heads=4, d_ff=2048, memory_dim=256, n_blocks=6, pos_dropout=0.0,
                            slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0, residual_dropout=0.1,
                            activation='glu', normalize_before=False, concat_after=False, share_embedding=True),
            'ctc_weight': 0.3, 'encoder_output_size': 256, 'smoothing': 0.1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--frames', type=int, default=1000)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--weight', type=float, default=0.3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/joint_decode.py measures on the GPU; none is visible')
    dev = torch.device('cuda:0')
    torch.manual_seed(1234)
    model = SpeechToText(params()).eval()
    with torch.no_grad():
        model.decoder.output_layer.bias[1] = -1e4
    model = model.to(dev)
    B, T, beam, max_len = a.batch, a.frames, 10, 60
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, T, 80, generator=g).to(dev)
    mask = torch.ones(B, T, dtype=torch.bool, device=dev)
    kw = dict(beam_width=beam, nbest=1, max_len=max_len, penalty=0.6, lamda=5, ngpu=1, persistent=False)
    rec0 = SpeechToTextRecognizer(model, ctc_weight=0.0, **kw)
    rec = SpeechToTextRecognizer(model, ctc_weight=a.weight, **kw)
    _, _, steps0 = rec0.recognize_ids(x, mask)
    _, _, steps = rec.recognize_ids(x, mask)
    bd = next(iter(rec._decoders.values()))
    assert steps0 == steps == max_len and bd.step.graph is not None and not bd.persistent
    ctc, st = bd.ctc, bd.state
    res = {'card': card(), 'batch': B, 'frames': T, 'encoder_frames': ctc.T, 'beam': beam, 'candidates': ctc.P, 'steps': steps,
           'ctc_weight': a.weight, 'launches_per_step': bd.step.launches, 'reps': a.reps,
           'ctc_buffers_mb': round(sum(t.numel() * t.element_size() for t in (ctc.lp, ctc.gamma, ctc.psi, ctc.gamma_cand,
                                                                               ctc.psi_cand, ctc.cand_val, ctc.cand_id)) / 1e6, 1),
           'ms': {}}
    ms = res['ms']

    def add(key, v):
        ms.setdefault(key, []).append(round(v, 4))

    with torch.no_grad():
        mem, mem_len, _, _ = model.encode_bf16(x, mask)

        def score_advance():
            # the state after the run's last step, put back to the step before its end: the same work as any full step
            st.ctrl[0] = max_len - 1
            ctc.score(st, bd.mem_len, bd.ctc_weight, bd.topk_val, bd.topk_idx)
            st.ctrl[0] = max_len
            ctc.advance(st, bd.mem_len)

        def ctrl_only():
            st.ctrl[0] = max_len - 1
            st.ctrl[0] = max_len

        def per_batch():
            ops.log_softmax(model.assistor.logits_bf16(mem), ctc.V, out=ctc.lp)
            ctc.init(bd.mem_len)

        for _ in range(a.reps):
            add('recognize_ids_w0_graph', timed(lambda: rec0.recognize_ids(x, mask), a.iters))
            add('recognize_ids_joint_graph', timed(lambda: rec.recognize_ids(x, mask), a.iters))
            add('recognize_spans_joint', timed(lambda: rec.recognize_spans(x, mask), a.iters))
            add('score_plus_advance_one_step', timed(score_advance, 10 * a.iters) - timed(ctrl_only, 10 * a.iters))
            add('head_logsoftmax_init_per_batch', timed(per_batch, a.iters))
    res['joint_minus_w0_per_step_ms'] = round((min(ms['recognize_ids_joint_graph']) - min(ms['recognize_ids_w0_graph'])) / steps, 4)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
