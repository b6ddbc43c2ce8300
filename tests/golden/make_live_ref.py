"""Regenerate tests/golden/live_ref_<case>.pt: the reference's OWN modules (byte-compiled into oracle/_ref by oracle/build_ref.py)
run on small random models; the stored state dicts, inputs and reference outputs are what tests/test_oracle_ref.py compares
the oracle port against.

    python oracle/build_ref.py && python tests/golden/make_live_ref.py     # needs the reference tree
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import build_ref  # noqa: E402
from tests.test_oracle_ref import _params  # noqa: E402


def _sd(ref):
    return {k: v.detach().clone().float() for k, v in ref.state_dict().items() if k.split('.')[0] in ('frontend', 'encoder', 'decoder')}


def recognize_case(normalize_before, activation):
    from otrans.model import End2EndModel
    from otrans.recognize.speech2text import SpeechToTextRecognizer
    params = _params(normalize_before, activation)
    torch.manual_seed(4321)
    ref = End2EndModel['speech2text'](params).eval()
    with torch.no_grad():
        ref.decoder.embedding.weight.mul_(0.15)
        ref.decoder.output_layer.bias[1] = 1.5          # hypotheses end at different steps
    g = torch.Generator().manual_seed(5)
    B, T, beam, max_len = 3, 64, 3, 9
    lens = torch.tensor([64, 50, 37])
    mask = torch.arange(T)[None] < lens[:, None]
    x = torch.randn(B, T, 20, generator=g) * mask.unsqueeze(2)
    with torch.no_grad():
        fx, fm = ref.frontend(x, mask)
        mem_ref, mm_ref, _ = ref.encoder(fx, fm)
        rec = SpeechToTextRecognizer(ref, beam_width=beam, nbest=beam, max_len=max_len, idx2unit={i: str(i) for i in range(40)},
                                     penalty=0.6, lamda=5, ngpu=0)
        hyps, scores_ref = rec.recognize(x, mask)
    return {'params': params, 'sd': _sd(ref), 'x': x, 'mask': mask, 'beam': beam, 'max_len': max_len,
            'mem_ref': mem_ref, 'mm_ref': mm_ref, 'hyps': hyps, 'scores_ref': scores_ref.float()}


def gradient_case(normalize_before, activation):
    from otrans.model import End2EndModel
    params = _params(normalize_before, activation)
    torch.manual_seed(99)
    ref = End2EndModel['speech2text'](params)
    ref.train()
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for n, p in ref.named_parameters():
            if 'norm' in n:
                p.add_(0.2 * torch.randn(p.shape, generator=g))
            elif n.endswith('.bias'):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
        ref.decoder.embedding.weight.mul_(0.12)
    sd = _sd(ref)
    B, T, L = 3, 70, 8
    lens = torch.tensor([70, 55, 41])
    mask = torch.arange(T)[None] < lens[:, None]
    x = torch.randn(B, T, 20, generator=g) * mask.unsqueeze(2)
    tgt = torch.randint(3, 40, (B, L), generator=g)
    tgt[:, 0] = 1
    tgt[0, L - 2:] = torch.tensor([1, 0])
    tgt[1, L - 1] = 1
    tgt[2, 4:] = torch.tensor([1, 0, 0, 0])
    loss_ref, _ = ref({'inputs': x, 'mask': mask}, {'targets': tgt, 'targets_length': None})
    loss_ref.backward()
    g_ref = {n: p.grad.clone() for n, p in ref.named_parameters() if p.grad is not None}
    return {'params': params, 'sd': sd, 'x': x, 'mask': mask, 'tgt': tgt, 'loss_ref': loss_ref.detach(), 'g_ref': g_ref}


def relpos_case(kind):
    from otrans.model import End2EndModel
    from otrans.recognize.speech2text import SpeechToTextRecognizer
    params = _params(False, 'glu')
    if kind == 'conformer':
        params['encoder_type'] = 'conformer'
        params['encoder'] = dict(d_model=32, d_ff=24, cov_kernel_size=5, n_heads=4, nblocks=2, pos_dropout=0.0, slf_attn_dropout=0.0,
                                 ffn_dropout=0.0, residual_dropout=0.0, conv_dropout=0.0, macaron_style=True, ffn_scale=0.5,
                                 conv_bias=True, activation='glu', positional_encoding=True, relative_positional=True)
    else:
        params['encoder']['relative_positional'] = True
    torch.manual_seed(77)
    ref = End2EndModel['speech2text'](params).eval()
    g = torch.Generator().manual_seed(11)
    with torch.no_grad():
        for n, buf in ref.named_buffers():
            if n.endswith('running_mean'):
                buf.add_(0.3 * torch.randn(buf.shape, generator=g))
            if n.endswith('running_var'):
                buf.mul_(1.0 + 0.5 * torch.rand(buf.shape, generator=g))
        ref.decoder.embedding.weight.mul_(0.15)
        ref.decoder.output_layer.bias[1] = 1.5
    B, T, beam, max_len = 3, 72, 3, 7
    lens = torch.tensor([72, 60, 33])
    mask = torch.arange(T)[None] < lens[:, None]
    x = torch.randn(B, T, 20, generator=g) * mask.unsqueeze(2)
    with torch.no_grad():
        fx, fm = ref.frontend(x, mask)
        mem_ref, mm_ref, _ = ref.encoder(fx, fm)
        rec = SpeechToTextRecognizer(ref, beam_width=beam, nbest=1, max_len=max_len, idx2unit={i: str(i) for i in range(40)},
                                     penalty=0.6, lamda=5, ngpu=0)
        hyps, _ = rec.recognize(x, mask)
    return {'params': params, 'sd': _sd(ref), 'x': x, 'mask': mask, 'beam': beam, 'max_len': max_len,
            'mem_ref': mem_ref, 'mm_ref': mm_ref, 'hyps': hyps}


if __name__ == '__main__':
    if build_ref.load() is None:
        raise SystemExit('oracle/_ref is missing: run oracle/build_ref.py where the reference tree exists')
    cases = {}
    for nb, act in [(False, 'glu'), (True, 'relu')]:
        cases[f'recognize-{nb}-{act}'] = recognize_case(nb, act)
    for nb, act in [(False, 'glu'), (True, 'glu'), (False, 'relu'), (True, 'relu')]:
        cases[f'gradients-{nb}-{act}'] = gradient_case(nb, act)
    for kind in ('conformer', 'relpos_transformer'):
        cases[f'relpos-{kind}'] = relpos_case(kind)
    for name, case in cases.items():      # one file per case keeps every fixture small
        torch.save(case, os.path.join(HERE, f'live_ref_{name}.pt'))
    print('wrote', len(cases), 'cases to', HERE)
