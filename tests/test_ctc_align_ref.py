"""CPU checks of the forced-alignment restatement (tests/ctc_align_ref.py) that the GPU tests compare otb_ctc_align with:
against torchaudio's forced_align / merge_tokens and against enumerating every alignment; and the refusals that need no
GPU."""
import itertools

import numpy as np
import pytest
import torch

from tests import ctc_align_ref as car

from opentransformer_b200 import ops
from opentransformer_b200.model import SpeechToText, encoder_frames_to_input


def _lp(T, V, seed, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    return torch.log_softmax(scale * torch.randn(T, V, generator=g), dim=-1)


@pytest.mark.parametrize('T,L,V', [(1, 1, 5), (7, 3, 6), (40, 12, 30), (120, 60, 50), (300, 150, 4234)])
def test_restatement_matches_torchaudio(T, L, V):
    g = torch.Generator().manual_seed(T * 31 + L)
    for trial in range(3):
        tokens = car.tokens_with_repeats(L, V, g)
        Tb = T if trial else max(car.min_frames(tokens), 1)          # the first trial is a tight fit
        lp = _lp(Tb, V, seed=T + 7 * trial)
        labels, scores, spans, path = car.viterbi_align(lp, tokens)
        ta_labels, ta_scores, ta_spans = car.torchaudio_align(lp, tokens)
        assert np.array_equal(labels, ta_labels), trial
        assert np.array_equal(scores.view(np.int32), ta_scores.view(np.int32)), trial       # bit-identical
        assert np.array_equal(spans, ta_spans), trial
        assert path == np.add.accumulate(ta_scores, dtype=np.float32)[-1]


def test_path_score_is_the_best_alignment():
    """For T <= 6 and V <= 4, the float64 restatement's path score is the best of every alignment; its frame labels are
    an alignment of the tokens with that score."""
    cases = 0
    for T in range(1, 7):
        for L in range(0, 4):
            for tokens in itertools.product(range(1, 4), repeat=L):
                if car.min_frames(tokens) > T:
                    continue
                lp = _lp(T, 4, seed=100 * T + 10 * L + sum(tokens)).numpy().astype(np.float64)
                labels, scores, spans, path = car.viterbi_align(lp, tokens, dtype=np.float64)
                want = car.best_alignment(lp, tokens)
                assert abs(path - want) <= 1e-12 * max(1.0, abs(want)), (T, tokens)
                assert car.collapse(labels.tolist()) == list(tokens)
                assert abs(float(scores.sum()) - want) <= 1e-12 * max(1.0, abs(want))
                cases += 1
    assert cases > 100


def test_infeasible_and_empty():
    lp = _lp(4, 6, seed=1)
    for tokens, n in (([2, 2, 3], 3), ([2, 0, 3], 4), ([2, 9], 4), ([2], 0)):
        labels, scores, spans, path = car.viterbi_align(lp, tokens, n_frames=n)
        assert path == float('-inf') and (labels == -1).all() and (spans == -1).all() and np.isneginf(scores).all()
    labels, scores, spans, path = car.viterbi_align(lp, [], n_frames=3)
    assert labels.tolist() == [0, 0, 0, -1] and spans.shape == (0, 2) and path == np.add.accumulate(lp[:3, 0].numpy())[-1]
    assert car.viterbi_align(lp, [], n_frames=0)[3] == 0.0


def test_tie_break():
    """Uniform log-probs: every alignment ties.  Staying wins over moving on, so the token takes the first frame only and
    the path ends in the final blank."""
    lp = np.full((4, 3), np.log(1 / 3), np.float32)
    labels, _, spans, _ = car.viterbi_align(lp, [2])
    assert labels.tolist() == [2, 0, 0, 0] and spans.tolist() == [[0, 1]]
    labels, _, spans, _ = car.viterbi_align(lp, [1, 1])
    assert labels.tolist() == [1, 0, 1, 0] and spans.tolist() == [[0, 1], [2, 3]]
    labels, _, spans, _ = car.viterbi_align(lp[:2], [1, 2])           # the end may not stay in a blank it never reached
    assert labels.tolist() == [1, 2] and spans.tolist() == [[0, 1], [1, 2]]


def test_refusals_need_no_gpu():
    """L above 1023 tokens and a model without a CTC head are refused before any device work."""
    B, T, V = 1, 2000, 10
    rows = torch.zeros(B, T, V)
    with pytest.raises(ValueError, match='1023'):
        ops.ctc_align(rows, torch.tensor([T], dtype=torch.int32), torch.ones(B, 1024, dtype=torch.int64),
                      torch.tensor([1024], dtype=torch.int32))
    fe = dict(input_size=80, output_size=256, in_channel=1, mid_channel=64, out_channel=128, kernel_size=[[3, 3], [3, 3]],
              stride=[2, 2], dropout=0.0, act_func_type='relu', front_end_layer_norm=False)
    enc = dict(d_model=256, n_heads=4, d_ff=1024, n_blocks=1, pos_dropout=0.0, slf_attn_dropout=0.0, ffn_dropout=0.0,
               residual_dropout=0.0, normalize_before=False, concat_after=False, activation='glu', relative_positional=False)
    dec = dict(vocab_size=V, d_model=256, n_heads=4, d_ff=1024, memory_dim=256, n_blocks=1, pos_dropout=0.0,
               slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0, residual_dropout=0.0, activation='glu',
               normalize_before=False, concat_after=False, share_embedding=True)
    model = SpeechToText({'type': 'speech2text', 'frontend_type': 'conv', 'encoder_type': 'transformer',
                          'decoder_type': 'transformer', 'frontend': fe, 'encoder': enc, 'decoder': dec, 'ctc_weight': 0.0})
    x = torch.zeros(1, 40, 80)
    with pytest.raises(ValueError, match='ctc_weight'):
        model.align(x, torch.ones(1, 40, dtype=torch.bool), torch.ones(1, 4, dtype=torch.int64), torch.tensor([3]))


def test_encoder_frames_to_input():
    """Encoder frame t sees input frames [4t, 4t + 7): check it against the convolutions' receptive field."""
    spans = torch.tensor([[[0, 1], [1, 3], [-1, -1]]], dtype=torch.int32)
    assert encoder_frames_to_input(spans).tolist() == [[[0, 7], [4, 15], [-1, -1]]]
    sec = encoder_frames_to_input(spans, frame_shift=0.01)
    assert sec.dtype == torch.float64 and torch.allclose(sec[0, :2], torch.tensor([[0.0, 0.07], [0.04, 0.15]], dtype=torch.float64))
    assert sec[0, 2].tolist() == [-1.0, -1.0]
    conv = torch.nn.Sequential(torch.nn.Conv2d(1, 1, 3, 2), torch.nn.Conv2d(1, 1, 3, 2))
    with torch.no_grad():
        for m in conv:
            m.weight.fill_(1.0)
    x = torch.zeros(1, 1, 40, 9, requires_grad=True)
    conv(x)[0, 0, 3, :].sum().backward()                 # encoder frame 3
    seen = torch.nonzero(x.grad[0, 0].abs().sum(1)).flatten().tolist()
    assert seen == list(range(12, 19))
