"""CPU checks of the fused transducer searches' restatement (tests/rnnt_lm_fusion_ref.py) and of TransducerRecognizer's LM
options: at lm_weight = beta = 0 the fused searches are the unfused ones, an unpruned fused ALSD final is the lattice's
alignment sum plus the LM terms, the early end never changes the n-best (beta > 0 included), and every refusal fires
before the library is reached."""
import argparse
import itertools
import math

import pytest

from opentransformer_b200 import lm as LM
from opentransformer_b200 import model as M
from opentransformer_b200 import recognize
from tests import rnnt_beam_ref as beam_ref
from tests import rnnt_lm_fusion_ref as ref
from tests.test_rnnt_beam_ref import _lattice_score
from tests.test_rnnt_ref import params


def test_zero_weight_fusion_is_the_unfused_search():
    for seed in range(20):
        V, K = 3 + seed % 4, 1 + seed % 5
        W, max_len = 1 + seed % K, (2, 6, 30)[seed % 3]
        t_len = [1 + (seed + b) % 7 for b in range(3)] + [0]
        lp = beam_ref.synthetic_lp(seed, V, blank_bias=(seed % 3) - 1.0)
        lm = ref.synthetic_lm(seed, V)
        fused = ref.alsd_search(lp, lm, t_len, K, W, max_len, 0.0, 0.0)
        plain = beam_ref.search(lp, t_len, K, W, max_len)
        for a, b in zip(fused, plain):
            assert a.nbest(W) == b.nbest(W) and a.steps == b.steps
        g = ref.greedy_search(lp, lm, t_len, max_len, 2, 0.0, 0.0)
        g0 = ref.greedy_search(lp, lambda b, y: [float('-inf')] * V, t_len, max_len, 2, 0.0, 0.0)   # the LM is not read
        assert g == g0


@pytest.mark.parametrize('V,max_len,T,lm_weight,beta', [(3, 2, 1, 0.5, 0.0), (3, 2, 4, 0.3, 0.7), (2, 3, 3, 1.0, -0.4),
                                                        (4, 1, 5, 0.0, 1.2)])
def test_unpruned_fused_search_is_the_alignment_sum_plus_lm_terms(V, max_len, T, lm_weight, beta):
    seqs = [s for n in range(max_len + 1) for s in itertools.product(range(1, V), repeat=n)]
    K = W = len(seqs)
    lp = beam_ref.synthetic_lp(V * 100 + T, V)
    lm = ref.synthetic_lm(V + T, V, context_free=True)
    utt = ref.alsd_search(lp, lm, [T], K, W, max_len, lm_weight, beta)[0]
    got = {y: s for y, s in utt.nbest(W)}
    assert sorted(got) == sorted(seqs)
    for y, s in got.items():
        want = _lattice_score(lp, 0, T, y) + sum(lm_weight * lm(0, ())[k] + beta for k in y)
        assert abs(s - want) <= 1e-12 * max(1.0, abs(s)), y


def test_unpruned_fused_search_with_a_context_lm():
    """A context LM gives every alignment of y the same LM term: sum_u lm(y[:u])[y[u]]."""
    V, max_len, T, lw, beta = 3, 3, 4, 0.4, 0.3
    seqs = [s for n in range(max_len + 1) for s in itertools.product(range(1, V), repeat=n)]
    lp = beam_ref.synthetic_lp(11, V)
    lm = ref.synthetic_lm(12, V)
    utt = ref.alsd_search(lp, lm, [T], len(seqs), len(seqs), max_len, lw, beta)[0]
    for y, s in utt.nbest(len(seqs)):
        want = _lattice_score(lp, 0, T, y) + sum(lw * lm(0, y[:u])[y[u]] + beta for u in range(len(y)))
        assert abs(s - want) <= 1e-12 * max(1.0, abs(s)), y


def test_early_end_never_changes_the_fused_nbest():
    ended_early = ended_early_beta = 0
    for seed in range(80):
        V, K = 3 + seed % 5, 1 + seed % 6
        W, max_len = 1 + seed % K, (2, 5, 12)[seed % 3]
        beta = (0.0, 0.8, -0.5, 2.0)[seed % 4]
        lw = (0.0, 0.3, 1.0)[seed % 3]
        t_len = [1 + (seed * 7 + b) % 9 for b in range(3)] + [0]
        lp = beam_ref.synthetic_lp(seed, V, blank_bias=(seed % 4) - 1.0)
        lm = ref.synthetic_lm(seed, V)
        early = ref.alsd_search(lp, lm, t_len, K, W, max_len, lw, beta, early=True)
        full = ref.alsd_search(lp, lm, t_len, K, W, max_len, lw, beta, early=False)
        for a, b in zip(early, full):
            assert a.nbest(W) == b.nbest(W)
            ended_early += a.steps < b.steps
            ended_early_beta += a.steps < b.steps and beta > 0
    assert ended_early > 20 and ended_early_beta > 5


def test_greedy_restatement_scores_the_fused_values():
    V = 5
    lp = beam_ref.synthetic_lp(3, V, blank_bias=0.5)
    lm = ref.synthetic_lm(4, V)
    for (y, s), T in zip(ref.greedy_search(lp, lm, [6, 3], 4, 2, 0.5, 0.25), [6, 3]):
        # replay: the score is the sum of the chosen fused values, blank plain
        total, frame, u = 0.0, 0, 0
        while frame < T:
            row = ref.fused_row(lp(0 if T == 6 else 1, frame, y[:u]), lm(0 if T == 6 else 1, y[:u]), 0.5, 0.25)
            if u < len(y) and int(row.argmax()) == y[u]:
                total += row[y[u]]
                u += 1
            else:
                total += row[0]
                frame += 1
        assert u == len(y) and math.isclose(total, s, rel_tol=1e-12, abs_tol=1e-12)


def _lms(V=40):
    t = LM.TransformerLanguageModel(dict(type='transformer_lm', vocab_size=V, num_blocks=1, d_model=256, n_heads=4, d_ff=256,
                                         residual_dropout=0.0, smoothing=0.1, share_embedding=False))
    r = LM.RecurrentLanguageModel(dict(vocab_size=V, share_embedding=False, smoothing=0.1, num_layers=1, hidden_size=64,
                                       dropout=0.0))
    return t, r


def test_refusals_fire_before_the_library():
    model = M.TransducerModel(params())
    tlm, rlm = _lms()
    other = _lms(41)[1]
    cases = [({'lm': object()}, NotImplementedError), ({'mode': 'alsd', 'lm': object()}, NotImplementedError),
             ({'lm': other}, ValueError), ({'lm': rlm, 'lm_weight': -0.1}, ValueError),
             ({'mode': 'alsd', 'lm': rlm, 'lm_weight': float('nan')}, ValueError),
             ({'mode': 'alsd', 'apply_lm_rescoring': True}, ValueError),
             ({'lm': rlm, 'apply_lm_rescoring': True}, ValueError),
             ({'mode': 'alsd', 'lm': object(), 'apply_lm_rescoring': True}, NotImplementedError),
             ({'mode': 'alsd', 'lm': tlm, 'max_len': 1023}, ValueError),
             ({'lm': tlm, 'max_len': 1023}, ValueError),
             ({'lm': rlm, 'ngram_lm': object()}, NotImplementedError),
             ({'lm': rlm, 'mode': 'beam'}, NotImplementedError), ({'lm': rlm, 'mode': 'modified_beam'}, NotImplementedError)]
    for kw, err in cases:
        with pytest.raises(err):
            recognize.TransducerRecognizer(model, ngpu=0, **kw)
    # accepted at the edges: max_len 1022 with the Transformer LM, any lm_weight >= 0 and beta, rescoring with either LM
    for kw in ({'lm': tlm, 'max_len': 1022}, {'lm': rlm, 'max_len': 1023, 'lm_weight': 0.0, 'beta': -1.0},
               {'mode': 'alsd', 'lm': tlm, 'apply_lm_rescoring': True, 'max_len': 1023},
               {'mode': 'alsd', 'lm': rlm, 'apply_lm_rescoring': True, 'beam_width': 4, 'nbest': 2}):
        recognize.TransducerRecognizer(model, ngpu=0, **kw)


def test_build_recognizer_forwards_the_lm_options():
    model = M.TransducerModel(params())
    _, rlm = _lms()
    old = argparse.Namespace(ngpu=0, max_len=50, mode='alsd', ngram_lm=None, beam_width=8, nbest=3)
    rec = recognize.build_recognizer('transducer', model, None, old, None)
    assert (rec.lm, rec.lm_weight, rec.beta, rec.apply_lm_rescoring, rec.rescore_weight) == (None, 0.1, 0.0, False, 1.0)
    rec = recognize.build_recognizer('transducer', model, rlm, old, None)
    assert rec.lm is rlm and not rec.apply_lm_rescoring
    new = argparse.Namespace(ngpu=0, max_len=50, mode='alsd', ngram_lm=None, beam_width=8, nbest=3, lm_weight=0.3, beta=0.5,
                             apply_lm_rescoring=True, rescore_weight=0.7)
    rec = recognize.build_recognizer('transducer', model, rlm, new, None)
    assert (rec.lm_weight, rec.beta, rec.apply_lm_rescoring, rec.rescore_weight) == (0.3, 0.5, True, 0.7)
    with pytest.raises(ValueError):
        recognize.build_recognizer('transducer', model, None, new, None)
    with pytest.raises(ValueError):
        recognize.build_recognizer('transducer', model, rlm, argparse.Namespace(ngpu=0, lm_weight=-1.0), None)
