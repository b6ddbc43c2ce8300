"""CPU checks of the ALSD restatement (tests/rnnt_beam_ref.py) and of TransducerRecognizer's ALSD refusals and wiring:
with a beam that prunes nothing each final's score is the lattice's sum over its alignments, the early end never changes
the n-best, and merges of re-formed prefixes occur in the sweep."""
import argparse
import itertools

import pytest
import torch

from opentransformer_b200 import model as M
from opentransformer_b200 import recognize
from tests import rnnt_beam_ref as ref
from tests import rnnt_ref
from tests.test_rnnt_ref import params


def _lattice_score(lp, b, T, y):
    """-lattice_nll of labels y under the callback: every alignment of y over T frames."""
    U = len(y)
    lpb = torch.tensor([[lp(b, t, y[:u])[0] for u in range(U + 1)] for t in range(T)], dtype=torch.float64)
    lpy = torch.tensor([[lp(b, t, y[:u])[y[u]] for u in range(U)] for t in range(T)], dtype=torch.float64).view(T, U)
    return -float(rnnt_ref.lattice_nll(lpb, lpy))


@pytest.mark.parametrize('V,max_len,T', [(3, 2, 1), (3, 2, 4), (2, 3, 3), (4, 1, 5)])
def test_unpruned_search_sums_every_alignment(V, max_len, T):
    seqs = [s for n in range(max_len + 1) for s in itertools.product(range(1, V), repeat=n)]
    K = W = len(seqs)                                   # no fewer slots than distinct prefixes: nothing is pruned
    lp = ref.synthetic_lp(V * 100 + T, V)
    utt = ref.search(lp, [T], K, W, max_len)[0]
    got = {y: s for y, s in utt.nbest(W)}
    assert sorted(got) == sorted(seqs)
    for y, s in got.items():
        assert abs(s - _lattice_score(lp, 0, T, y)) <= 1e-12 * max(1.0, abs(s)), y
    if T > 1 and max_len > 0:
        assert utt.merges > 0


def test_early_end_never_changes_the_nbest():
    ended_early = 0
    for seed in range(60):
        V = 3 + seed % 5
        K = 1 + seed % 6
        W = 1 + seed % K
        max_len = (2, 5, 40)[seed % 3]
        t_len = [1 + (seed * 7 + b) % 9 for b in range(3)] + [0]
        lp = ref.synthetic_lp(seed, V, blank_bias=(seed % 4) - 1.0)
        early = ref.search(lp, t_len, K, W, max_len, early=True)
        full = ref.search(lp, t_len, K, W, max_len, early=False)
        for a, b in zip(early, full):
            assert a.nbest(W) == b.nbest(W)
            ended_early += a.steps < b.steps
    assert ended_early > 20


def test_merges_and_reformed_prefixes_occur():
    merges = string_merges = recreated = 0
    for seed in range(40):
        lp = ref.synthetic_lp(1000 + seed, 4, scale=1.0)
        for utt in ref.search(lp, [6, 9], 3, 2, 6):
            merges += utt.merges
            string_merges += utt.string_merges
            recreated += utt.recreated
    print('merges', merges, 'of re-formed prefixes', string_merges, 'prefixes re-formed', recreated)
    assert merges > 100 and string_merges > 0 and recreated > 0


def test_empty_and_one_frame_utterances():
    lp = ref.synthetic_lp(5, 4)
    none, one = ref.search(lp, [0, 1], 4, 3, 3)
    assert none.nbest(3) == [((), ref.NEG)] * 3 and none.steps == 1
    # one frame: the finals are the sequences that end with blank at frame 0, best first
    best = one.nbest(3)
    assert best[0][1] >= best[1][1] >= best[2][1] > ref.NEG


def test_alsd_refusals_and_build():
    model = M.TransducerModel(params())
    for kw, err in (({'mode': 'alsd', 'beam_width': 0}, ValueError), ({'mode': 'alsd', 'beam_width': 16}, ValueError),
                    ({'mode': 'alsd', 'beam_width': 4, 'nbest': 5}, ValueError),
                    ({'mode': 'alsd', 'nbest': 0}, ValueError), ({'nbest': 2}, ValueError),
                    ({'mode': 'alsd', 'lm': object()}, NotImplementedError),
                    ({'mode': 'alsd', 'ngram_lm': object()}, NotImplementedError),
                    ({'mode': 'beam'}, NotImplementedError), ({'mode': 'modified_beam'}, NotImplementedError)):
        with pytest.raises(err):
            recognize.TransducerRecognizer(model, ngpu=0, **kw)
    with pytest.raises(NotImplementedError, match="'alsd'"):
        recognize.TransducerRecognizer(model, ngpu=0, mode='beam')
    rec = recognize.TransducerRecognizer(model, ngpu=0, beam_width=99)         # greedy ignores beam_width
    assert rec.mode == 'greedy'
    args = argparse.Namespace(ngpu=0, max_len=50, mode='alsd', ngram_lm=None, beam_width=8, nbest=3)
    rec = recognize.build_recognizer('transducer', model, None, args, None)
    assert (rec.mode, rec.beam_width, rec.nbest, rec.max_len) == ('alsd', 8, 3, 50)
    rec = recognize.build_recognizer('transducer', model, None, argparse.Namespace(ngpu=0, mode='alsd'), None)
    assert (rec.beam_width, rec.nbest) == (5, 1)
    with pytest.raises(NotImplementedError):
        recognize.build_recognizer('transducer', model, None, argparse.Namespace(ngpu=0, max_len=50, mode='beam'), None)
