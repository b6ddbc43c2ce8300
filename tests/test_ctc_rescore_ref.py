"""CPU checks of CTC rescoring of the attention n-best (DESIGN.md 4.18): the float64 restatement (tests/ctc_rescore_ref.py)
against every alignment path and its edges, the re-ranking with infeasible hypotheses, the recognizer's refusals before any
device work, build_recognizer's plumbing and ops.ctc_nbest_score's argument checks.  No GPU: models stay on the CPU."""
import itertools
import math
from types import SimpleNamespace

import pytest
import torch

from tests import ctc_rescore_ref as cr
from tests.test_rescore_ref import _ctc_model, _speech, _tlm
from tests.test_transformer_lm_ref import _cuda_calls_fail

NEG_INF = cr.NEG_INF


def _brute_force(logp, labels, blank=0):
    """log sum over every frame labelling that collapses to `labels` (merge repeats, drop blanks)."""
    T, V = logp.shape
    total = NEG_INF
    for path in itertools.product(range(V), repeat=T):
        out, prev = [], None
        for c in path:
            if c != blank and c != prev:
                out.append(c)
            prev = c
        if out == list(labels):
            total = float(torch.logaddexp(torch.tensor(total, dtype=torch.float64),
                                          logp[torch.arange(T), torch.tensor(path)].sum()))
    return total


@pytest.mark.parametrize('labels', [[1], [2, 3], [2, 2], [3, 1, 3], [1, 1, 1]])
def test_score_matches_every_path(labels):
    g = torch.Generator().manual_seed(len(labels) * 7 + labels[0])
    T, V = 5, 4
    logp = torch.log_softmax(torch.randn(T, V, generator=g, dtype=torch.float64), -1)
    want = _brute_force(logp, labels)
    got = cr.ctc_score(logp, labels)
    assert (want == NEG_INF) == (got == NEG_INF)
    if want != NEG_INF:
        assert math.isclose(got, want, rel_tol=1e-12)


def test_score_edges():
    logp = torch.log_softmax(torch.randn(6, 5, dtype=torch.float64), -1)
    assert cr.ctc_score(logp, [2, 0, 3]) == NEG_INF                 # the blank as a label
    assert cr.ctc_score(logp, [2, 5]) == NEG_INF                    # out of range
    assert cr.ctc_score(logp[:0], [2]) == NEG_INF                   # no frames
    assert cr.ctc_score(logp[:3], [2, 2]) != NEG_INF                # a repeat needs a blank between: 3 frames do
    assert cr.ctc_score(logp[:2], [2, 2]) == NEG_INF                # ... 2 do not
    assert cr.ctc_score(logp[:3], [1, 2, 3]) != NEG_INF
    assert cr.ctc_score(logp[:2], [1, 2, 3]) == NEG_INF
    assert math.isclose(cr.ctc_score(logp, []), float(logp[:, 0].sum()), rel_tol=1e-12)   # empty: blanks throughout


def test_row_labels_and_nbest_scores():
    assert cr.row_labels([4, 5, 1, -1, -1]) == [4, 5, 1]
    assert cr.row_labels([4, 5, 1]) == [4, 5, 1]
    B, T, V = 2, 4, 6
    logp = torch.log_softmax(torch.randn(B * T, V, dtype=torch.float64), -1)
    targets = torch.tensor([[[2, 1, -1], [3, 3, 1]], [[2, 1, -1], [4, 1, -1]]], dtype=torch.int32)
    got = cr.nbest_scores(logp, B, T, torch.tensor([4, 0]), targets)
    assert got[0, 0] == cr.ctc_score(logp[:4], [2, 1]) and got[0, 1] == cr.ctc_score(logp[:4], [3, 3, 1])
    assert got[1].tolist() == [NEG_INF, NEG_INF]                    # in_len 0


def _tl(*vals):
    return [torch.tensor(vals, dtype=torch.float64)]


@pytest.mark.parametrize('weight', [1.0, 0.5, 0.0, -1.0])
def test_infeasible_hypotheses_rank_last_in_first_pass_order(weight):
    hyps = [[5, 6], [5], [7], [8], [9, 9]]
    s1 = [-1.0, -2.0, -3.0, -4.0, -5.0]
    ctc = [NEG_INF, -3.0, NEG_INF, -1.0, NEG_INF]
    got = cr.rerank(hyps, s1, [[]] * 5, ctc, weight, 5)
    feasible = sorted((1, 3), key=lambda k: (-(s1[k] + weight * ctc[k]), k))
    assert [k for k, _, _ in got] == feasible + [0, 2, 4]
    assert [s for _, _, s in got[2:]] == [NEG_INF] * 3
    assert [s for _, _, s in got[:2]] == [s1[k] + weight * ctc[k] for k in feasible]


def test_all_infeasible_is_the_first_pass_order_and_duplicates_stay_last():
    hyps = [[5, 6], [5], [7], [5]]
    got = cr.rerank(hyps, [-1.0, -2.0, -3.0, -4.0], [[]] * 4, [NEG_INF] * 4, 1.0, 4)
    assert [k for k, _, _ in got] == [0, 1, 2, None]
    # with an LM term too: the LM cannot lift an infeasible hypothesis
    got = cr.rerank([[5], [6]], [-1.0, -9.0], [_tl(-5.0, -5.0), _tl(0.0, 0.0)], [NEG_INF, -20.0], 1.0, 2)
    assert [k for k, _, _ in got] == [1, 0]


def test_ctc_term_adds_to_the_other_models_before_the_weight():
    got = cr.rerank([[5]], [-2.0], [_tl(-1.0, -0.5)], [-3.0], 0.5, 1)
    assert got[0][2] == -2.0 + 0.5 * (-1.5 - 3.0)


# ------------------------------------------------------------------------------------------------ recognizer arguments
def test_refusals_before_any_device_work(monkeypatch):
    from opentransformer_b200.recognize import SpeechToTextRecognizer
    joint, plain = _speech(0.3), _speech(0.0)
    _cuda_calls_fail(monkeypatch)
    with pytest.raises(ValueError, match='apply_ctc_rescoring needs the joint-CTC head'):
        SpeechToTextRecognizer(plain, apply_ctc_rescoring=True)
    with pytest.raises(ValueError, match='two uses of the joint-CTC head'):
        SpeechToTextRecognizer(joint, ctc_weight=0.3, apply_ctc_rescoring=True)
    with pytest.raises(ValueError, match='apply_ctc_rescoring re-ranks the attention'):
        SpeechToTextRecognizer(joint, apply_rescoring=True, apply_ctc_rescoring=True)


def test_accepted_with_lm_rescoring_and_the_decoder_key_has_no_ctc_term():
    from opentransformer_b200.recognize import SpeechToTextRecognizer
    joint, lm = _speech(0.3), _tlm()
    rec = SpeechToTextRecognizer(joint, lm=lm, apply_ctc_rescoring=True, apply_lm_rescoring=True, rescore_weight=0.5, ngpu=0)
    assert rec.apply_ctc_rescoring and rec.apply_lm_rescoring and not rec._lm_fused()
    assert rec.ctc_weight == 0.0 and rec.persistent                  # the search keeps the persistent kernel's options
    assert not SpeechToTextRecognizer(joint, ngpu=0).apply_ctc_rescoring


def test_build_recognizer_plumbing():
    from opentransformer_b200.recognize import build_recognizer
    joint, lm = _speech(0.3), _tlm()
    args = SimpleNamespace(lm_weight=0.1, ctc_weight=0.0, beam_width=5, nbest=1, max_len=20, penalty=0.6, lamda=5, ngpu=0)
    assert not build_recognizer('speech2text', joint, None, args, None).apply_ctc_rescoring    # absent: the default
    args.apply_ctc_rescoring, args.apply_lm_rescoring = True, True
    rec = build_recognizer('speech2text', joint, lm, args, None)
    assert rec.apply_ctc_rescoring and rec.apply_lm_rescoring
    cargs = SimpleNamespace(lm_weight=0.1, ngram_lm=None, beam_width=5, ngpu=0, mode='beam', alpha=0.1, beta=0.0,
                            apply_ctc_rescoring=True)
    with pytest.raises(ValueError, match='a CTC model has none'):
        build_recognizer('ctc', _ctc_model(), lm, cargs, None)
    cargs.apply_ctc_rescoring = False
    assert build_recognizer('ctc', _ctc_model(), lm, cargs, None).mode == 'beam'


# ------------------------------------------------------------------------------------------------ ops.ctc_nbest_score
def test_ctc_nbest_score_argument_checks():
    from opentransformer_b200 import ops
    B, T, V = 2, 10, 8
    logp = torch.zeros(B * T, V)
    in_len = torch.full((B,), T, dtype=torch.int32)
    tg = torch.ones(B, 3, 4, dtype=torch.int32)
    with pytest.raises(ValueError, match='logp must be'):
        ops.ctc_nbest_score(logp[:-1], B, T, in_len, tg)
    with pytest.raises(ValueError, match='logp must be'):
        ops.ctc_nbest_score(logp.t(), B * T, 1, in_len, tg)
    with pytest.raises(ValueError, match='targets must be'):
        ops.ctc_nbest_score(logp, B, T, in_len, tg[0])
    with pytest.raises(ValueError, match='targets must be'):
        ops.ctc_nbest_score(logp, B, T, in_len, tg[:1])
    with pytest.raises(ValueError, match='1..1024 labels'):
        ops.ctc_nbest_score(logp, B, T, in_len, torch.ones(B, 3, 1025, dtype=torch.int32))
    with pytest.raises(ValueError, match='1..1024 labels'):
        ops.ctc_nbest_score(logp, B, T, in_len, torch.ones(B, 3, 0, dtype=torch.int32))
    with pytest.raises(ValueError, match='in_len must be'):
        ops.ctc_nbest_score(logp, B, T, in_len[:1], tg)
    with pytest.raises(TypeError, match='logp must be torch.float32'):
        ops.ctc_nbest_score(logp.double(), B, T, in_len, tg)
    with pytest.raises(TypeError, match='targets must be torch.int32'):
        ops.ctc_nbest_score(logp, B, T, in_len, tg.long())
    with pytest.raises(TypeError, match='in_len must be torch.int32'):
        ops.ctc_nbest_score(logp, B, T, in_len.long(), tg)
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        ops.ctc_nbest_score(logp, B, T, in_len, tg)
    # the widest row a recognizer can produce (max_len 1023 and the closing <S/E>) passes the checks
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        ops.ctc_nbest_score(logp, B, T, in_len, torch.ones(B, 3, ops.DECODE_MAX_LEN + 1, dtype=torch.int32))
