"""Shallow fusion on the captured decode step: what is checked before any device work.  A fused LM must share the decoder's
vocabulary, the Transformer LM's KV cache refuses geometries the cached step does not take, and predict keeps the
reference's two-argument signature (model/lm.py:143)."""
import inspect

import pytest
import torch

from tests.test_rescore_ref import _speech, _tlm


def _rnnlm(V):
    from opentransformer_b200.lm import RecurrentLanguageModel
    return RecurrentLanguageModel(dict(type='rnn_lm', vocab_size=V, num_layers=1, hidden_size=64, residual_dropout=0.0,
                                       smoothing=0.1, dropout=0.0, share_embedding=False))


@pytest.mark.parametrize('make_lm', [_tlm, _rnnlm])
def test_fusion_refuses_a_different_vocabulary(make_lm):
    """The reference cannot add [N, 31] LM log-probs to [N, 30] decoder log-probs either; the fused kernel would read the
    LM rows with the wrong length."""
    from opentransformer_b200.recognize import BeamDecoder, SpeechToTextRecognizer
    model = _speech(0.0)
    with pytest.raises(ValueError, match='one vocabulary'):
        SpeechToTextRecognizer(model, lm=make_lm(31), ngpu=0)
    with pytest.raises(ValueError, match='one vocabulary'):
        BeamDecoder(model.decoder, 2, 3, 10, 8, 'cpu', lm=(make_lm(31), 0.3))
    rec = SpeechToTextRecognizer(model, lm=make_lm(30), ngpu=0)               # one vocabulary: accepted
    assert rec._lm_fused()


def test_fusion_refuses_an_unknown_lm():
    from opentransformer_b200.recognize import SpeechToTextRecognizer

    class NGram:
        model_type = 'ngram'
        vocab_size = 30

    with pytest.raises(NotImplementedError, match='shallow fusion is implemented for'):
        SpeechToTextRecognizer(_speech(0.0), lm=NGram(), ngpu=0)


def test_lm_cache_refusals_before_device_work():
    from opentransformer_b200 import ops
    from opentransformer_b200.lm import LMCache
    lm = _tlm().eval()
    with pytest.raises(ValueError, match=r'max_len must be in \[1, 1023\]'):
        lm.init_cache(4, ops.DECODE_MAX_LEN + 1)
    with pytest.raises(ValueError, match='max_len'):
        lm.init_cache(4, 0)
    with pytest.raises(ValueError, match='n_rows'):
        lm.init_cache(0, 8)
    tok = torch.ones(4, 1, dtype=torch.long)
    with pytest.raises(TypeError, match='LMCache'):
        lm.predict(tok, True, {'lm': None})
    cache = object.__new__(LMCache)                                            # the checks come before any field is read
    with pytest.raises(ValueError, match='last_frame must be True'):
        lm.predict(tok, False, cache)


def test_predict_keeps_the_reference_signature():
    """The reference calls predict(targets, last_frame=True) (recognize/base.py:26-37); the cache is an optional third
    argument."""
    from opentransformer_b200.lm import TransformerLanguageModel
    params = list(inspect.signature(TransformerLanguageModel.predict).parameters.values())
    assert [p.name for p in params] == ['self', 'targets', 'last_frame', 'cache']
    assert params[2].default is True and params[3].default is None
