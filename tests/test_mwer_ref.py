"""CPU checks of the MWER restatement (tests/mwer_ref.py) that the GPU tests compare the kernels and the training pass with:
the edit distance against an enumeration of edit scripts, the closed-form coefficients against autograd, the cases with
zero gradient, FusedTrainer's refusals before any device work, and the MWER branch's dropout sites."""
import itertools
import random

import pytest
import torch

from tests import mwer_ref as mr
from tests.test_ctc_model_ref import _small_ctc_params
from tests.test_transformer_lm_ref import _cuda_calls_fail, small_params as tlm_params


def _brute_edit_distance(a, b):
    """Breadth-first search over sequences: one insertion, deletion or substitution per step, over the tokens of a and b."""
    a, b = tuple(a), tuple(b)
    alphabet = sorted(set(a) | set(b))
    seen, frontier, depth = {a}, [a], 0
    while b not in seen:
        nxt = []
        for s in frontier:
            cands = [s[:i] + s[i + 1:] for i in range(len(s))]
            cands += [s[:i] + (c,) + s[i:] for i in range(len(s) + 1) for c in alphabet]
            cands += [s[:i] + (c,) + s[i + 1:] for i in range(len(s)) for c in alphabet]
            for c in cands:
                if c not in seen and len(c) <= len(a) + len(b):
                    seen.add(c)
                    nxt.append(c)
        frontier, depth = nxt, depth + 1
    return depth


def test_edit_distance_equals_enumeration():
    for n, m in itertools.product(range(5), range(5)):
        for a in itertools.product((2, 3, 4), repeat=n):
            for b in itertools.product((2, 3), repeat=m):
                if (sum(a) + 7 * sum(b)) % 5:           # a fixed fifth of the pairs keeps this under a few seconds
                    continue
                assert mr.edit_distance(a, b) == _brute_edit_distance(a, b), (a, b)


def test_edit_distance_known_values():
    assert mr.edit_distance([], []) == 0
    assert mr.edit_distance([5, 6, 7], []) == 3 and mr.edit_distance([], [5, 6]) == 2
    assert mr.edit_distance([1, 2, 3], [1, 2, 3]) == 0
    assert mr.edit_distance([1, 2, 3], [4, 5]) == 3
    assert mr.edit_distance([9] * 7, [9] * 4) == 3


@pytest.mark.parametrize('seed', range(6))
def test_closed_form_coefficients_equal_autograd(seed):
    rng = random.Random(seed)
    K = rng.randint(2, 8)
    l = torch.randn(K, dtype=torch.float64, generator=torch.Generator().manual_seed(seed)) * 3
    W = [rng.randint(0, 6) for _ in range(K)]
    keep = [True] + [rng.random() > 0.3 for _ in range(K - 1)]
    lg = l.clone().requires_grad_()
    mr.utterance_loss(lg, W, keep).backward()
    want = lg.grad
    got = mr.coefficients(l, W, keep)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-14), (got, want)
    assert all(float(got[k]) == 0.0 for k in range(K) if not keep[k])


def test_batch_loss_gradient_is_the_coefficients_over_b():
    """dL/dtok_lp[b, k, t] = c_k / B on the n_k + 1 scored positions and 0 after them."""
    g = torch.Generator().manual_seed(3)
    hyps = [[[4, 5], [4], [4, 5], [6, 7, 8]], [[3], [3, 3], [2], []]]
    refs = [[4, 5, 6], [3, 2]]
    tok = (torch.randn(2, 4, 5, dtype=torch.float64, generator=g) - 2).requires_grad_()
    mr.batch_loss(tok, hyps, refs).backward()
    for b in range(2):
        W = [mr.edit_distance(y, refs[b]) for y in hyps[b]]
        l = torch.stack([tok[b, k, :len(y) + 1].sum() for k, y in enumerate(hyps[b])]).detach()
        c = mr.coefficients(l, W, mr.kept(hyps[b])) / 2
        for k, y in enumerate(hyps[b]):
            assert torch.allclose(tok.grad[b, k, :len(y) + 1], c[k].expand(len(y) + 1), rtol=1e-12, atol=1e-15)
            assert float(tok.grad[b, k, len(y) + 1:].abs().sum()) == 0.0


def test_zero_gradient_for_one_kept_hypothesis_and_for_equal_errors():
    l = torch.tensor([-3.0, -1.0, -2.0], dtype=torch.float64)
    one = mr.coefficients(l, [1, 4, 2], [True, False, False])
    assert float(one.abs().max()) == 0.0
    assert float(mr.utterance_loss(l, [1, 4, 2], [True, False, False])) == 0.0
    assert float(mr.coefficients(l, [2, 2, 2], [True, True, True]).abs().max()) == 0.0
    assert float(mr.utterance_loss(l, [2, 2, 2], [True, True, True])) == 0.0


def test_cut_and_duplicates_follow_second_pass_rows():
    rows = [[5, 6, 1, 7], [5, 6, 1, 1], [5, 6, 7, 8], [1, 0, 0, 0]]
    hyps = [mr.cut(r) for r in rows]
    assert hyps == [[5, 6], [5, 6], [5, 6, 7, 8], []]
    assert mr.kept(hyps) == [True, False, True, True]
    assert mr.cut([5, 6, 7, 0], length=2) == [5, 6]
    assert mr.reference([1, 8, 9, 1, 0], 3) == [8, 9]
    assert mr.error_counts([[8], [8, 9], [7, 7, 7]], [8, 9]) == (1, 0, 2)


def _speech_params(ctc=0.0):
    p = {'type': 'speech2text', 'frontend_type': 'conv', 'encoder_type': 'transformer', 'decoder_type': 'transformer',
         'frontend': dict(input_size=80, output_size=256, in_channel=1, mid_channel=64, out_channel=128,
                          kernel_size=[[3, 3], [3, 3]], stride=[2, 2], dropout=0.0, act_func_type='relu',
                          front_end_layer_norm=False),
         'encoder': dict(d_model=256, n_heads=4, d_ff=512, n_blocks=1, pos_dropout=0.0, slf_attn_dropout=0.0,
                         ffn_dropout=0.0, residual_dropout=0.0, normalize_before=False, concat_after=False,
                         activation='glu', relative_positional=False),
         'decoder': dict(vocab_size=40, d_model=256, n_heads=4, d_ff=512, memory_dim=256, n_blocks=1,
                         pos_dropout=0.0, slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0,
                         residual_dropout=0.0, activation='glu', normalize_before=False, concat_after=False,
                         share_embedding=True),
         'ctc_weight': ctc, 'smoothing': 0.1}
    if ctc:
        p['encoder_output_size'] = 256
    return p


def test_fused_trainer_refusals_come_before_device_work(monkeypatch):
    from opentransformer_b200.lm import RecurrentLanguageModel, TransformerLanguageModel
    from opentransformer_b200.model import CTCModel, SpeechToText
    from opentransformer_b200.train import FusedTrainer
    from tests.test_rnnlm_ref import small_params as rnn_params
    speech = SpeechToText(_speech_params())
    others = [CTCModel(_small_ctc_params()), TransformerLanguageModel(tlm_params(True)), RecurrentLanguageModel(rnn_params(True))]
    _cuda_calls_fail(monkeypatch)
    for m in others:
        with pytest.raises(NotImplementedError, match='attention decoder'):
            FusedTrainer(m, mwer_nbest=4)
    for k in (1, 17, -2):
        with pytest.raises(ValueError, match='mwer_nbest'):
            FusedTrainer(speech, mwer_nbest=k)
    with pytest.raises(ValueError, match='mwer_ce_weight'):
        FusedTrainer(speech, mwer_nbest=4, mwer_ce_weight=-0.01)
    with pytest.raises(ValueError, match='mwer_max_len'):
        FusedTrainer(speech, mwer_nbest=4, mwer_max_len=0)
    with pytest.raises(NotImplementedError, match='MixSpeech'):
        FusedTrainer(speech, mwer_nbest=4, mixspeech=True)


def test_mwer_dropout_sites_are_disjoint_from_every_other_range():
    from opentransformer_b200 import lm, train
    mwer = {train.MWER_SITE + 3 * i + k for i in range(64) for k in range(3)}
    others = ({train.ENC_SITE + 3 * i + k for i in range(64) for k in range(3)}
              | {train.DEC_SITE + 3 * i + k for i in range(64) for k in range(3)}
              | {lm.TLM_SITE + 2 * i + k for i in range(64) for k in range(2)} | {lm.RNNLM_SITE + k for k in range(64)})
    assert not (mwer & others)
    # dropout_sites lists what one training pass over the transcript draws; the MWER branch's sites are not in it
    from opentransformer_b200.model import SpeechToText
    sites = {s for s, _, _ in train.dropout_sites(SpeechToText(_speech_params()))}
    assert sites and not (sites & mwer)


def test_recognizer_refuses_an_empty_decoder_cache():
    from opentransformer_b200.model import SpeechToText
    from opentransformer_b200.recognize import SpeechToTextRecognizer
    with pytest.raises(ValueError, match='max_decoders'):
        SpeechToTextRecognizer(SpeechToText(_speech_params()), ngpu=0, max_decoders=0)
