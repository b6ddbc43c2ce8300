"""LM shallow fusion in the transducer's searches at tools/transducer_beam.py's geometry (transformer_baseline encoder, 1 x 320
LSTM prediction network, 512-wide joint, V 4234, 32 utterances x 1000 frames, max_len 100), blank-biased model (about one
label per 5 encoder frames): TransducerRecognizer.recognize (graph) in greedy mode and ALSD with beam_width 4 and 8, with no
LM, with transformer_lm.yaml's Transformer LM (6 blocks, d 256) and with rnnlm.yaml's recurrent LM (random weights,
lm_weight 0.3, beta 0.5); and each phase of one fused ALSD step timed alone with CUDA events over the steps of a real
search (eager launches).  It prints the card, its power limit and its maximum SM clock, read in the same run.  Needs a GPU.

    python tools/transducer_lm_fusion.py [--iters 5]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from opentransformer_b200.lm import RecurrentLanguageModel, TransformerLanguageModel  # noqa: E402
from opentransformer_b200.model import TransducerModel  # noqa: E402
from opentransformer_b200.recognize import TransducerRecognizer, _TransducerALSD  # noqa: E402
from tools.ctc_model import card, timed  # noqa: E402
from tools.transducer import params  # noqa: E402

MAX_LEN = 100
LMW, BETA = 0.3, 0.5


def lms(V, dev):
    torch.manual_seed(3)
    t = TransformerLanguageModel(dict(type='transformer_lm', vocab_size=V, num_blocks=6, d_model=256, n_heads=4, d_ff=1024,
                                      residual_dropout=0.0, smoothing=0.1, share_embedding=False))
    r = RecurrentLanguageModel(dict(vocab_size=V, share_embedding=False, smoothing=0.1, num_layers=2, hidden_size=1024,
                                    dropout=0.0))
    return {'transformer_lm': t.to(dev).eval(), 'rnnlm': r.to(dev).eval()}


def phase_times(model, lm, x, mask, K, steps):
    """Mean device ms of each phase of a fused ALSD step over the first `steps` steps of a search (eager)."""
    with torch.no_grad():
        mem, lengths, B, T2 = model.encode_bf16(x, mask)
        s = _TransducerALSD(model, B, T2, K, 1, MAX_LEN, x.device, False, lm=lm, lm_weight=LMW, beta=BETA)
        s.start(mem, lengths)
        names = ['joint', 'output_layer', 'logsoftmax_topk', 'beam_step', 'gather', 'predictor', 'commit', 'lm']
        ev = []
        for _ in range(steps):
            row = []
            for phase in s.step_phases():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                phase()
                e1.record()
                row.append((e0, e1))
            ev.append(row)
        torch.cuda.synchronize()
    return {n: sum(r[i][0].elapsed_time(r[i][1]) for r in ev) / steps for i, n in enumerate(names)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--frames', type=int, default=1000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/transducer_lm_fusion.py measures on the GPU; none is visible')
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    model = TransducerModel(params()).to(dev).eval()
    B, T = a.batch, a.frames
    g = torch.Generator().manual_seed(1)
    lens = torch.randint(int(0.8 * T), T + 1, (B,), generator=g)
    lens[0] = T
    mask = (torch.arange(T)[None] < lens[:, None]).to(dev)
    x = (torch.randn(B, T, 80, generator=g).to(dev) * mask.unsqueeze(2))
    T2 = model.frontend.output_length(T)
    res = {'card': card(), 'batch': B, 'frames': T, 'encoder_frames': T2, 'max_len': MAX_LEN, 'lm_weight': LMW, 'beta': BETA}
    bias = model.joint.output_layer.bias
    b0 = bias[0].item()
    lo, hi = 0.0, 8.0
    with torch.no_grad():
        for _ in range(14):             # raise the blank bias until greedy search takes about one label per 5 frames
            bias[0] = b0 + (lo + hi) / 2
            _, n, _ = TransducerRecognizer(model, max_len=MAX_LEN).recognize_ids(x, mask)
            lo, hi = ((lo + hi) / 2, hi) if float(n.float().mean()) > T2 / 5 else (lo, (lo + hi) / 2)
    res['blank_bias_added'] = float(bias[0]) - b0
    all_lms = lms(model.vocab_size, dev)
    with torch.no_grad():
        for name, lm in [('no_lm', None)] + list(all_lms.items()):
            kw = {} if lm is None else dict(lm=lm, lm_weight=LMW, beta=BETA)
            rec = TransducerRecognizer(model, max_len=MAX_LEN, **kw)
            r = {'greedy_ms': timed(lambda: rec.recognize(x, mask), a.iters, warmup=1)}
            _, n, _ = rec.recognize_ids(x, mask)
            r['greedy_tokens_mean'] = float(n.float().mean())
            for K in (4, 8):
                rec = TransducerRecognizer(model, mode='alsd', beam_width=K, nbest=1, max_len=MAX_LEN, **kw)
                r[f'alsd_K{K}_ms'] = timed(lambda: rec.recognize(x, mask), a.iters, warmup=1)
                _, n, _ = rec.recognize_ids(x, mask)
                r[f'alsd_K{K}_steps'] = rec._search.steps
                r[f'alsd_K{K}_tokens_mean'] = float(n.float().mean())
                if lm is not None:
                    r[f'alsd_K{K}_step_phase_ms'] = phase_times(model, lm, x, mask, K, 32)
                del rec
                torch.cuda.empty_cache()
            res[name] = r
    res['peak_gb'] = torch.cuda.max_memory_allocated() / 1e9
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
