"""The 1023-token bounds of the CTC loss and the KV-cached beam search are refused before any device work."""
import pytest
import torch

from tests.test_transformer_lm_ref import _cuda_calls_fail


def test_ctc_loss_refuses_targets_wider_than_1023(monkeypatch):
    from opentransformer_b200 import ops
    B, T, V = 2, 3000, 50
    logits = torch.zeros(B * T, V)
    in_len = torch.full((B,), T, dtype=torch.int32)
    tgt_len = torch.full((B,), 1024, dtype=torch.int32)
    _cuda_calls_fail(monkeypatch)
    with pytest.raises(ValueError, match='at most 1023'):
        ops.ctc_loss(logits, B, T, V, in_len, torch.ones(B, 1024, dtype=torch.long), tgt_len, want_grad=True)


def test_recognizer_refuses_max_len_1024(monkeypatch):
    from opentransformer_b200.model import SpeechToText
    from opentransformer_b200.recognize import BeamDecoder, SpeechToTextRecognizer
    from tests.test_gpu_model import _params
    model = SpeechToText(_params(n_enc=1, n_dec=1))
    _cuda_calls_fail(monkeypatch)
    with pytest.raises(ValueError, match='at most 1023'):
        SpeechToTextRecognizer(model, max_len=1024)
    with pytest.raises(ValueError, match='at most 1023'):
        BeamDecoder(model.decoder, 2, 3, 50, 1024, torch.device('cpu'))
