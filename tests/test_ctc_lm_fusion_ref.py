"""CPU checks of the LM-fused CTC prefix beam search (DESIGN.md 4.19): the float64 restatement against the unfused one and
against enumerated alignments, CTCRecognizer's refusals before any device work, and build_recognizer's plumbing."""
import math
from types import SimpleNamespace

import pytest
import torch

from tests import ctc_ref
from tests import ctc_lm_fusion_ref as fr
from tests.test_rescore_ref import _ctc_model, _tlm
from tests.test_transformer_lm_ref import _cuda_calls_fail


def _frames(T, V, K, seed, scale=2.0):
    lp = torch.log_softmax(ctc_ref.synth_log_probs(T, V, seed, scale).double(), dim=-1)
    return lp, [ctc_ref.frame_topk(lp[t].tolist(), K) for t in range(T)]


def _rnnlm(V=30):
    from opentransformer_b200.lm import RecurrentLanguageModel
    return RecurrentLanguageModel(dict(vocab_size=V, share_embedding=True, smoothing=0.1, num_layers=1, hidden_size=64,
                                       dropout=0.0))


@pytest.mark.parametrize('seed', range(6))
@pytest.mark.parametrize('beam', [1, 4, 16])
def test_weight_zero_is_the_unfused_search(seed, beam):
    _, frames = _frames(12, 9, 6, seed)
    ctx = lambda P: [(-1.0 - 0.1 * ((len(P) + c) % 7)) for c in range(9)]
    assert fr.fused_prefix_beam_search(frames, beam, ctx, 0.0, 0.0) == ctc_ref.prefix_beam_search(frames, beam)
    assert fr.fused_prefix_beam_search(frames, beam, ctx, 0.0, 0.0, fp32=True) == \
        ctc_ref.prefix_beam_search(frames, beam, fp32=True)


@pytest.mark.parametrize('T,V,seed', [(3, 3, 0), (4, 3, 1), (3, 4, 2), (5, 3, 3)])
@pytest.mark.parametrize('lm_weight,beta', [(0.5, 0.0), (0.7, 1.3), (0.0, -0.4)])
def test_no_pruning_gives_marginal_plus_lm_terms(T, V, seed, lm_weight, beta):
    """K >= V and a beam above the number of prefixes, context-free LM: every prefix scores its exact CTC marginal plus
    lm_weight * sum log p_lm + beta * length (each alignment of y passes len(y) extensions or merges)."""
    lp, frames = _frames(T, V, V, seed)
    g = torch.Generator().manual_seed(100 + seed)
    row = torch.log_softmax(torch.randn(V, generator=g, dtype=torch.float64), 0).tolist()
    want = ctc_ref.prefix_marginals(lp.tolist())
    got = fr.fused_prefix_beam_search(frames, 10 ** 6, lambda P: row, lm_weight, beta)
    assert {p for p, _ in got} == set(want)
    for p, s in got:
        exp = want[p] + sum(lm_weight * row[c] + beta for c in p)
        assert abs(s - exp) < 1e-9, (p, s, exp)
    assert [s for _, s in got] == sorted((s for _, s in got), reverse=True)


def test_a_context_lm_scores_the_true_prefix():
    """The LM row of an extension is the one of the extended prefix, not of a zero state or another slot."""
    _, frames = _frames(6, 5, 5, 7)
    seen = set()

    def lm(P):
        seen.add(P)
        return [-0.5 * ((sum(P) + c) % 3) - 1.0 for c in range(5)]
    out = fr.fused_prefix_beam_search(frames, 4, lm, 1.0, 0.0)
    assert () in seen and any(len(P) >= 2 for P in seen)
    assert len(out) == 4


def test_the_lm_moves_the_best_prefix():
    """A token the LM gives -30 leaves the n-best under a large weight."""
    lp = torch.full((3, 4), -10.0, dtype=torch.float64)
    lp[0, 2] = lp[1, 0] = lp[2, 2] = math.log(0.9)
    lp = torch.log_softmax(lp, dim=-1)
    frames = [ctc_ref.frame_topk(lp[t].tolist(), 4) for t in range(3)]
    assert 2 in ctc_ref.prefix_beam_search(frames, 4)[0][0]
    row = [-1.0, -1.0, -30.0, -1.0]
    out = fr.fused_prefix_beam_search(frames, 4, lambda P: row, 5.0, 0.0)
    assert all(2 not in P for P, _ in out)


def test_refusals_before_any_device_work(monkeypatch):
    from opentransformer_b200.lm import TransformerLanguageModel
    from opentransformer_b200.recognize import CTCRecognizer
    model, lm = _ctc_model(), _tlm()
    _cuda_calls_fail(monkeypatch)
    with pytest.raises(ValueError, match='lm_fusion needs an lm'):
        CTCRecognizer(model, lm_fusion=True, mode='beam', ngpu=0)
    with pytest.raises(ValueError, match="mode='beam'"):
        CTCRecognizer(model, lm=lm, lm_fusion=True, mode='greedy', ngpu=0)
    with pytest.raises(ValueError, match='twice'):
        CTCRecognizer(model, lm=lm, lm_fusion=True, mode='beam', apply_lm_rescoring=True, ngpu=0)
    with pytest.raises(ValueError, match='one vocabulary'):
        CTCRecognizer(model, lm=_tlm(31), lm_fusion=True, mode='beam', ngpu=0)
    with pytest.raises(NotImplementedError, match='shallow fusion is implemented'):
        CTCRecognizer(model, lm=SimpleNamespace(model_type='ngram', vocab_size=30), lm_fusion=True, mode='beam', ngpu=0)
    rec = CTCRecognizer(model, lm=lm, lm_fusion=True, mode='beam', ngpu=0)
    T = 4 * (1023 + 2) + 3                                        # the conv front end's T' = (T - 3) // 4 = 1025
    assert model.frontend.output_length(T) > 1023
    with pytest.raises(ValueError, match='at most 1023 encoder frames'):
        rec.recognize_ids(torch.zeros(1, T, 80), torch.ones(1, T, dtype=torch.bool))
    with pytest.raises(ValueError, match='at most 1023 encoder frames'):
        rec.recognize_spans(torch.zeros(1, T, 80), torch.ones(1, T, dtype=torch.bool))
    assert isinstance(lm, TransformerLanguageModel)


def test_default_is_off_and_the_rnn_lm_has_no_frame_limit(monkeypatch):
    from opentransformer_b200.recognize import CTCRecognizer
    model = _ctc_model()
    _cuda_calls_fail(monkeypatch)
    rec = CTCRecognizer(model, lm=_tlm(), mode='beam', ngpu=0)
    assert not rec.lm_fusion and not rec.apply_lm_rescoring
    CTCRecognizer(model, lm=_rnnlm(), lm_fusion=True, mode='beam', ngpu=0)._check_frames(torch.zeros(1, 8000, 80))


def test_build_recognizer_plumbing():
    from opentransformer_b200.recognize import build_recognizer
    args = SimpleNamespace(lm_weight=0.3, ngram_lm=None, beam_width=4, ngpu=0, mode='beam', alpha=0.1, beta=0.5)
    rec = build_recognizer('ctc', _ctc_model(), _tlm(), args, None)
    assert not rec.lm_fusion
    args.lm_fusion = True
    rec = build_recognizer('ctc', _ctc_model(), _tlm(), args, None)
    assert rec.lm_fusion and rec.lm_weight == 0.3 and rec.beta == 0.5 and rec.beam_width == 4
    args.mode = 'greedy'
    with pytest.raises(ValueError, match="mode='beam'"):
        build_recognizer('ctc', _ctc_model(), _tlm(), args, None)
