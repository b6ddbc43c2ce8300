"""The oracle port against the REFERENCE ITSELF: tests/golden/live_ref_<case>.pt hold small random models (state dicts),
their inputs and what the reference's own modules computed from them -- encoder states, recognize() hypotheses and scores,
training loss and every parameter gradient (written by tests/golden/make_live_ref.py from the reference's byte-compiled
modules).  Complements tests/test_oracle_golden.py, which pins the shipped configurations."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import beam_search as obs      # noqa: E402
from oracle import speech_model as om      # noqa: E402

def _case(name):
    return torch.load(os.path.join(ROOT, 'tests', 'golden', f'live_ref_{name}.pt'), weights_only=False)


def _params(normalize_before, activation):
    return {'type': 'speech2text', 'frontend_type': 'conv', 'encoder_type': 'transformer', 'decoder_type': 'transformer',
            'frontend': dict(input_size=20, output_size=32, in_channel=1, mid_channel=4, out_channel=8,
                             kernel_size=[[3, 3], [3, 3]], stride=[2, 2], dropout=0.0, act_func_type='relu',
                             front_end_layer_norm=False),
            'encoder': dict(d_model=32, n_heads=4, d_ff=48, n_blocks=2, pos_dropout=0.0, slf_attn_dropout=0.0,
                            ffn_dropout=0.0, residual_dropout=0.0, normalize_before=normalize_before, concat_after=False,
                            activation=activation, relative_positional=False),
            'decoder': dict(vocab_size=40, d_model=32, n_heads=4, d_ff=48, memory_dim=32, n_blocks=2, pos_dropout=0.0,
                            slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0, residual_dropout=0.0,
                            activation=activation, normalize_before=normalize_before, concat_after=False,
                            share_embedding=True),
            'ctc_weight': 0.0, 'smoothing': 0.1}


@pytest.mark.parametrize('normalize_before,activation', [(False, 'glu'), (True, 'relu')])
def test_port_equals_live_reference(normalize_before, activation):
    c = _case(f'recognize-{normalize_before}-{activation}')
    params, sd, x, mask, beam, max_len = c['params'], c['sd'], c['x'], c['mask'], c['beam'], c['max_len']
    B = x.shape[0]
    with torch.no_grad():
        # encoder states: reference modules vs the port
        mem, mm = om.encode(x, mask, sd, params)
        assert torch.equal(mm, c['mm_ref'])
        torch.testing.assert_close(mem[mm], c['mem_ref'][c['mm_ref']], rtol=1e-4, atol=2e-5)
        # the whole recognize(): ids bit-exact, scores to fp32 tolerance
        nb, ns, _, _ = obs.recognize(x, mask, sd, params, beam=beam, nbest=beam, max_len=max_len, penalty=0.6, lamda=5)
    hyps = c['hyps']
    for b in range(B):
        for r in range(beam):
            port = [int(t) for t in nb[b, r].tolist()]
            port = port[:port.index(1)] if 1 in port else port
            want = [int(t) for t in hyps[b][r].split()] if hyps[b][r] else []
            assert port == want, (b, r, port, want)
    torch.testing.assert_close(ns, c['scores_ref'], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize('normalize_before,activation', [(False, 'glu'), (True, 'glu'), (False, 'relu'), (True, 'relu')])
def test_port_gradients_equal_live_reference_autograd(normalize_before, activation):
    """model.train(); loss, _ = model(inputs, targets); loss.backward() through the REFERENCE's own modules (trainer.py:206-217)
    vs oracle/train_step.loss_and_grads: the loss and every parameter gradient -- in particular for the pre-norm and ReLU
    stacks whose hand-written CUDA backward is tested against this port (tests/test_gpu_train.py)."""
    from oracle import train_step as ot
    c = _case(f'gradients-{normalize_before}-{activation}')
    loss, grads = ot.loss_and_grads(c['x'], c['mask'], c['tgt'], c['sd'], c['params'])
    torch.testing.assert_close(loss, c['loss_ref'], rtol=1e-5, atol=1e-5)
    g_ref = c['g_ref']
    assert set(grads) == set(g_ref), set(grads) ^ set(g_ref)
    for n in grads:
        torch.testing.assert_close(grads[n], g_ref[n], rtol=2e-4, atol=2e-6, msg=lambda m, n=n: f'{n}: {m}')


@pytest.mark.parametrize('kind', ['conformer', 'relpos_transformer'])
def test_port_encoder_states_equal_live_reference_for_relpos_encoders(kind):
    """Conformer (macaron FFN, rel-pos attention without output projection, conv module with BatchNorm running statistics,
    only post_ffn_norm applied: SURVEY.md 8a quirks) and the rel-pos Transformer encoder: valid-frame states of the port vs
    the reference modules, recognize() ids bit-exact."""
    c = _case(f'relpos-{kind}')
    params, sd, x, mask, beam, max_len = c['params'], c['sd'], c['x'], c['mask'], c['beam'], c['max_len']
    with torch.no_grad():
        mem, mm = om.encode(x, mask, sd, params)
        assert torch.equal(mm, c['mm_ref'])
        torch.testing.assert_close(mem[mm], c['mem_ref'][c['mm_ref']], rtol=1e-4, atol=2e-5)
        nb, _, _, _ = obs.recognize(x, mask, sd, params, beam=beam, nbest=1, max_len=max_len, penalty=0.6, lamda=5)
    hyps = c['hyps']
    for b in range(x.shape[0]):
        port = [int(t) for t in nb[b, 0].tolist()]
        port = port[:port.index(1)] if 1 in port else port
        want = [int(t) for t in hyps[b][0].split()] if hyps[b][0] else []
        assert port == want, (b, port, want)
