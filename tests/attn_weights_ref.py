"""Attention maps of the oracle port, and the models of the attention-weights fixture (tests/golden/live_ref_attn_weights.pt,
written by tests/golden/make_live_ref_attn_weights.py from the reference's own modules).

The oracle's attention functions (mha_self, mha_cross, mha_self_relpos) already return the softmax weights next to their
output, and its encoders and decoder drop them.  record_attn_weights() collects them while an oracle forward runs, in call
order: one map per encoder block, and (self, cross) per decoder block."""
import contextlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import speech_model as om          # noqa: E402
from tests.test_head_dim_96 import dk96_params, synth_state_dict   # noqa: E402

FIXTURE = os.path.join(ROOT, 'tests', 'golden', 'live_ref_attn_weights.pt')
CASES = ('postnorm_glu', 'relpos_transformer', 'conformer', 'dk96')


@contextlib.contextmanager
def record_attn_weights():
    """Within the block, every oracle attention call appends its weights [B, h, Tq, Tk] to the yielded list."""
    sink = []
    saved = {n: getattr(om, n) for n in ('mha_self', 'mha_cross', 'mha_self_relpos')}

    def wrap(fn):
        def call(*args, **kw):
            out, w = fn(*args, **kw)
            sink.append(w)
            return out, w
        return call

    for n, fn in saved.items():
        setattr(om, n, wrap(fn))
    try:
        yield sink
    finally:
        for n, fn in saved.items():
            setattr(om, n, fn)


def case_params(name):
    """Small models with 64-wide heads (d_model 128, 2 heads, 2 blocks) and the d_k 96 model of test_head_dim_96."""
    if name == 'dk96':
        return dk96_params()
    p = dk96_params()
    p['frontend'] = dict(p['frontend'], output_size=128)
    p['decoder'] = dict(p['decoder'], d_model=128, memory_dim=128, d_ff=64)
    if name == 'conformer':
        p['encoder'] = dict(p['encoder'], d_model=128, d_ff=64)
        return p
    p['encoder_type'] = 'transformer'
    p['encoder'] = dict(d_model=128, n_heads=2, d_ff=64, n_blocks=2, pos_dropout=0.0, slf_attn_dropout=0.0, ffn_dropout=0.0,
                        residual_dropout=0.0, normalize_before=False, concat_after=False, activation='glu',
                        relative_positional=name == 'relpos_transformer')
    return p


def oracle_maps(c, policy=None, memory=None):
    """-> (encoder maps [n_blocks], decoder maps [(self, cross)] on c['tgt'] against `memory` (default: the reference's
    encoder states c['mem_ref'])) of the oracle, fp32 or with policy='bf16'."""
    params, sd = c['params'], c['sd']
    with torch.no_grad(), record_attn_weights() as enc:
        om.encode(c['x'], c['mask'], sd, params, policy)
    mem = c['mem_ref'] if memory is None else memory
    with torch.no_grad(), record_attn_weights() as dec:
        om.transformer_decoder(c['tgt'], mem, c['mm_ref'], sd, 'decoder.', policy=policy, **om.decoder_kwargs(params))
    return enc, [(dec[2 * i], dec[2 * i + 1]) for i in range(len(dec) // 2)]


def load_cases():
    """{case name: dict} of the fixture, each with its state dict rebuilt from (key shapes, seed)."""
    cases = torch.load(FIXTURE, weights_only=False)
    for c in cases.values():
        c['sd'] = synth_state_dict(c['sd_shapes'], c['sd_seed'])
    return cases
