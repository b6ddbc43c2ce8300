"""Regenerate live_ref_attn_weights.pt from the reference's OWN modules (byte-compiled into oracle/_ref by oracle/build_ref.py):
for each model of tests/attn_weights_ref.CASES (post-norm GLU Transformer, rel-pos Transformer encoder, Conformer with 64-wide
heads, the d_k 96 model) on deterministic weights (synth_state_dict: only the key shapes and the seed are stored):

  enc_ref   encoder.forward's attn_weights, one [B, h, T', T'] map per block
  dec_ref   decoder.forward's (slf_attn_weights, src_attn_weights) per block on a teacher-forced target batch tgt with
            ragged lengths (PAD-filled tails), against the reference's own encoder states mem_ref / mm_ref
  rec_ref   SpeechToTextRecognizer.recognize's attn_weights['encoder'], one map per block

    python oracle/build_ref.py && python tests/golden/make_live_ref_attn_weights.py     # needs the reference tree
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import build_ref  # noqa: E402
from tests.attn_weights_ref import CASES, FIXTURE, case_params  # noqa: E402
from tests.test_head_dim_96 import synth_state_dict  # noqa: E402


def case(name, seed):
    from otrans.model import End2EndModel
    from otrans.recognize.speech2text import SpeechToTextRecognizer
    params = case_params(name)
    ref = End2EndModel['speech2text'](params).eval()
    shapes = {k: (tuple(v.shape), str(v.dtype).replace('torch.', '')) for k, v in ref.state_dict().items()
              if k.split('.')[0] in ('frontend', 'encoder', 'decoder')}
    ref.load_state_dict(synth_state_dict(shapes, seed), strict=True)
    g = torch.Generator().manual_seed(seed + 1)
    B, T, L = 3, 110, 9
    lens = torch.tensor([110, 83, 40])
    mask = torch.arange(T)[None] < lens[:, None]
    x = torch.randn(B, T, 80, generator=g) * mask.unsqueeze(2)
    tgt = torch.randint(3, 40, (B, L), generator=g)
    tgt[:, 0] = 1
    tgt[1, 6:] = torch.tensor([1, 0, 0])
    tgt[2, 3:] = torch.tensor([1, 0, 0, 0, 0, 0])
    with torch.no_grad():
        fx, fm = ref.frontend(x, mask)
        mem_ref, mm_ref, enc_w = ref.encoder(fx, fm)
        _, dec_w = ref.decoder(tgt, mem_ref, mm_ref)
        rec = SpeechToTextRecognizer(ref, beam_width=2, nbest=1, max_len=4, idx2unit={i: str(i) for i in range(40)}, ngpu=0)
        rec.recognize(x, mask)
    n_enc, n_dec = len(enc_w), len(dec_w)
    return {'params': params, 'sd_shapes': shapes, 'sd_seed': seed, 'x': x, 'mask': mask, 'tgt': tgt,
            'mem_ref': mem_ref, 'mm_ref': mm_ref,
            'enc_ref': [enc_w['enc_block_%d' % i]['slf_attn_weights'] for i in range(n_enc)],
            'dec_ref': [(dec_w['dec_block_%d' % i]['slf_attn_weights'], dec_w['dec_block_%d' % i]['src_attn_weights'])
                        for i in range(n_dec)],
            'rec_ref': [rec.attn_weights['encoder']['enc_block_%d' % i]['slf_attn_weights'] for i in range(n_enc)]}


if __name__ == '__main__':
    if build_ref.load() is None:
        raise SystemExit('oracle/_ref is missing: run oracle/build_ref.py where the reference tree exists')
    torch.save({name: case(name, 700 + i) for i, name in enumerate(CASES)}, FIXTURE)
    print('wrote', FIXTURE, os.path.getsize(FIXTURE), 'bytes')
