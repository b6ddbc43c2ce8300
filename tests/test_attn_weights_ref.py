"""Attention weights without a GPU:
  * the oracle port's attention maps reproduce what the reference's own modules returned (tests/golden/live_ref_attn_weights.pt)
    for every encoder and decoder block, valid and padded query rows alike;
  * return_attn_weights defaults to False, and with it off the modules' dicts keep their None entries;
  * ops.attention_probs refuses bad arguments before any device work."""
import pytest
import torch

from tests.attn_weights_ref import CASES, case_params, load_cases, oracle_maps


@pytest.fixture(scope='module')
def cases():
    return load_cases()


@pytest.mark.parametrize('name', CASES)
def test_oracle_maps_equal_live_reference(cases, name):
    c = cases[name]
    enc, dec = oracle_maps(c)
    assert len(enc) == len(c['enc_ref']) == len(c['rec_ref']) and len(dec) == len(c['dec_ref'])
    B, T2 = c['mm_ref'].shape
    for got, want, rec in zip(enc, c['enc_ref'], c['rec_ref']):
        assert got.shape == want.shape == (B, c['params']['encoder']['n_heads'], T2, T2)
        torch.testing.assert_close(got, want, rtol=0, atol=1e-5)
        assert torch.equal(rec, want)           # recognize() stores the encoder pass's own maps
    L = c['tgt'].shape[1]
    for (s, x), (s_ref, x_ref) in zip(dec, c['dec_ref']):
        assert s.shape == (B, c['params']['decoder']['n_heads'], L, L) and x.shape[-2:] == (L, T2)
        torch.testing.assert_close(s, s_ref, rtol=0, atol=1e-5)
        torch.testing.assert_close(x, x_ref, rtol=0, atol=1e-5)
    # the fixture does exercise masking: padded keys and the causal upper triangle are exact zeros
    lens = c['mm_ref'].sum(1)
    assert (lens < T2).any()
    for b in range(B):
        assert torch.all(c['enc_ref'][0][b, :, :, lens[b]:] == 0)
        assert torch.all(c['dec_ref'][0][1][b, :, :, lens[b]:] == 0)
    assert torch.all(c['dec_ref'][0][0].triu(1) == 0)


@pytest.mark.parametrize('name', CASES)
def test_switch_defaults_off_and_dicts_keep_none(name):
    from opentransformer_b200.model import SpeechToText
    m = SpeechToText(case_params(name)).eval()
    assert m.encoder.return_attn_weights is False and m.decoder.return_attn_weights is False
    from opentransformer_b200.modules import encoder_attn_weights
    assert encoder_attn_weights(2, None) == {'enc_block_0': {'slf_attn_weights': None}, 'enc_block_1': {'slf_attn_weights': None}}
    # return_attn_weights is an attribute, not a constructor kwarg and not a parameter or buffer: state_dict is unchanged
    assert not any('attn_weights' in k for k in m.state_dict())


def test_recognizer_attn_weights_start_empty():
    from opentransformer_b200.model import SpeechToText
    from opentransformer_b200.recognize import SpeechToTextRecognizer
    rec = SpeechToTextRecognizer(SpeechToText(case_params('dk96')).eval(), beam_width=2, ngpu=0)
    assert rec.attn_weights == {}


def _cpu_args(**over):
    kw = dict(q=torch.zeros(8, 384, dtype=torch.bfloat16), k=torch.zeros(8, 384, dtype=torch.bfloat16), B=1, H=2, Tq=8, Tk=8)
    kw.update(over)
    return kw


def test_attention_probs_refuses_before_device_work(monkeypatch):
    from opentransformer_b200 import _lib, ops

    def no_library():
        raise AssertionError('the library was reached')
    monkeypatch.setattr(_lib, 'lib', no_library)
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        ops.attention_probs(**_cpu_args())
    # device checks come first; the remaining ones are reached with tensors that claim to be CUDA tensors
    class Fake:
        def __init__(self, t):
            self.t = t
            self.is_cuda, self.dtype, self.shape = True, t.dtype, t.shape

        def is_contiguous(self):
            return self.t.is_contiguous()

    q = Fake(torch.zeros(8, 384, dtype=torch.bfloat16))
    with pytest.raises(TypeError, match='bfloat16'):
        ops.attention_probs(Fake(torch.zeros(8, 384)), q, 1, 2, 8, 8)
    with pytest.raises(NotImplementedError, match=r'\(64, 96\)'):
        ops.attention_probs(q, q, 1, 2, 8, 8, d_k=80)
    with pytest.raises(TypeError, match='int32'):
        ops.attention_probs(q, q, 1, 2, 8, 8, kv_len=Fake(torch.zeros(1, dtype=torch.int64)))
    bd = Fake(torch.zeros(2, 8, 16))
    with pytest.raises(ValueError, match='rel-pos band'):
        ops.attention_probs(q, q, 1, 2, 8, 7, bd=bd)
    with pytest.raises(ValueError, match='rel-pos band'):
        ops.attention_probs(q, q, 1, 2, 8, 8, bd=bd, causal=True)
    with pytest.raises(ValueError, match=r'out must be \[1, 2, 8, 8\]'):
        ops.attention_probs(q, q, 1, 2, 8, 8, out=Fake(torch.zeros(1, 2, 8, 9)))
