"""Regenerate the 96-wide-head fixtures from the reference's OWN modules (byte-compiled into oracle/_ref by oracle/build_ref.py):

  live_ref_dk96.pt                      the reference's End2EndModel['speech2text'] with 96-wide heads (Conformer rel-pos encoder
                                        + Transformer decoder, d_model 192, 2 heads, 2 blocks each) on deterministic weights
                                        (tests/test_head_dim_96.synth_state_dict: only the key shapes and the seed are stored),
                                        its input, encoder states, mask, and the hypotheses and scores of
                                        SpeechToTextRecognizer.recognize
  live_ref_conformer_baseline_keys.pt   {state_dict key: shape} of the full conformer_baseline model (no weights)

    python oracle/build_ref.py && python tests/golden/make_live_ref_dk96.py     # needs the reference tree
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import build_ref  # noqa: E402
from tests.test_head_dim_96 import CONFORMER_BASELINE, dk96_params, synth_state_dict  # noqa: E402

SEED = 96


def dk96_case():
    from otrans.model import End2EndModel
    from otrans.recognize.speech2text import SpeechToTextRecognizer
    params = dk96_params()
    ref = End2EndModel['speech2text'](params).eval()
    shapes = {k: (tuple(v.shape), str(v.dtype).replace('torch.', '')) for k, v in ref.state_dict().items()
              if k.split('.')[0] in ('frontend', 'encoder', 'decoder')}
    ref.load_state_dict(synth_state_dict(shapes, SEED), strict=True)
    g = torch.Generator().manual_seed(13)
    B, T, beam, max_len = 3, 120, 3, 8
    lens = torch.tensor([120, 97, 41])
    mask = torch.arange(T)[None] < lens[:, None]
    x = torch.randn(B, T, 80, generator=g) * mask.unsqueeze(2)
    with torch.no_grad():
        fx, fm = ref.frontend(x, mask)
        mem_ref, mm_ref, _ = ref.encoder(fx, fm)
        rec = SpeechToTextRecognizer(ref, beam_width=beam, nbest=beam, max_len=max_len, idx2unit={i: str(i) for i in range(40)},
                                     penalty=0.6, lamda=5, ngpu=0)
        hyps, scores_ref = rec.recognize(x, mask)
    return {'params': params, 'sd_shapes': shapes, 'sd_seed': SEED, 'x': x, 'mask': mask, 'beam': beam, 'max_len': max_len,
            'mem_ref': mem_ref, 'mm_ref': mm_ref, 'hyps': hyps, 'scores_ref': scores_ref.float()}


def conformer_baseline_keys_case():
    from otrans.model import End2EndModel
    ref = End2EndModel['speech2text'](CONFORMER_BASELINE)
    return {k: tuple(v.shape) for k, v in ref.state_dict().items()}


if __name__ == '__main__':
    if build_ref.load() is None:
        raise SystemExit('oracle/_ref is missing: run oracle/build_ref.py where the reference tree exists')
    torch.save(dk96_case(), os.path.join(HERE, 'live_ref_dk96.pt'))
    torch.save(conformer_baseline_keys_case(), os.path.join(HERE, 'live_ref_conformer_baseline_keys.pt'))
    print('wrote live_ref_dk96.pt and live_ref_conformer_baseline_keys.pt to', HERE)
