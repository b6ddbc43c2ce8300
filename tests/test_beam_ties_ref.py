"""Without a GPU: the tie-exact beam step of tests/beam_ties_ref.py.  On inputs without ties it must equal the oracle's
beam_step bit for bit; on hand-built ties it must rank by (value descending, index ascending) in both selections, which is
the order the CUDA decode paths promise and the one the oracle (torch.topk) leaves undefined."""
import pytest
import torch

from oracle import beam_search as obs
from tests import beam_ties_ref as btr

NEG = float('-inf')


def _init(b, beam):
    preds = torch.full((b * beam, 1), 1, dtype=torch.long)
    scores = torch.tensor([0.0] + [NEG] * (beam - 1)).repeat(b).unsqueeze(1)
    return preds, scores, torch.zeros_like(scores, dtype=torch.bool)


def _same(a, b):
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and torch.equal(x, y)


@pytest.mark.parametrize('b,beam,v,lm', [(3, 4, 50, False), (2, 1, 17, False), (4, 10, 4234, False), (3, 16, 300, True),
                                         (5, 3, 23, True)])
def test_equals_oracle_without_ties(b, beam, v, lm):
    """Random fp32 log-probs, random prefixes, scores and finished flags: tokens, parents, scores and flags bit-exact."""
    g = torch.Generator().manual_seed(b * 1000 + beam * 10 + v)
    n = b * beam
    for trial in range(4):
        lp = torch.log_softmax(torch.randn(n, v, generator=g) * 3, -1)
        lm_lp = torch.log_softmax(torch.randn(n, v, generator=g), -1) if lm else None
        preds = torch.randint(2, v, (n, 5), generator=g)
        scores = -torch.rand(n, 1, generator=g) * 9
        flag = torch.rand(n, 1, generator=g) < 0.3
        tr_o, tr_t = [], []
        ref = obs.beam_step(lp, preds, scores, flag, beam, lm_lp, 0.3, trace=tr_o)
        got = btr.beam_step(lp, preds, scores, flag, beam, lm_lp, 0.3, trace=tr_t)
        _same(got, ref)
        for key in ('k_tok', 'offs', 'parent', 'tok', 'scores'):
            assert torch.equal(tr_t[0][key], tr_o[0][key]), key


def test_equals_oracle_over_a_search_without_ties():
    """Several steps from the initial state (step 0: only hypothesis 0 alive), EOS made likely so hypotheses finish."""
    b, beam, v = 3, 5, 40
    g = torch.Generator().manual_seed(11)
    p_o, s_o, f_o = _init(b, beam)
    p_t, s_t, f_t = _init(b, beam)
    for _ in range(9):
        lp = torch.randn(b * beam, v, generator=g) * 2
        lp[:, 1] += 1.5
        lp = torch.log_softmax(lp, -1)
        p_o, s_o, f_o = obs.beam_step(lp, p_o, s_o, f_o, beam)
        p_t, s_t, f_t = btr.beam_step(lp, p_t, s_t, f_t, beam)
        _same((p_t, s_t, f_t), (p_o, s_o, f_o))
    _same(btr.beam_finalize(p_t, s_t, beam, 2, 0.6, 5), obs.beam_finalize(p_o, s_o, beam, 2, 0.6, 5))


def test_topk_low_index_order():
    x = torch.tensor([[0.5, 2.0, NEG, 2.0, 1.0, 2.0, NEG, 0.5]])
    v, i = btr.topk_low_index(x, 8)
    assert i.tolist() == [[1, 3, 5, 4, 0, 7, 2, 6]]
    assert v.tolist() == [[2.0, 2.0, 2.0, 1.0, 0.5, 0.5, NEG, NEG]]


def test_ties_inside_a_row():
    """One utterance at step 0: hypothesis 0's row has four equal maxima; the three lowest token ids win, in order."""
    beam, v = 3, 12
    preds, scores, flag = _init(1, beam)
    lp = torch.full((beam, v), -9.0)
    lp[:, [10, 4, 7, 2]] = -0.5
    tr = []
    p, s, f = btr.beam_step(lp, preds, scores, flag, beam, trace=tr)
    assert tr[0]['k_tok'][0].tolist() == [2, 4, 7]
    assert p[:, 1].tolist() == [2, 4, 7] and tr[0]['parent'].tolist() == [0, 0, 0]
    assert s.view(-1).tolist() == [-0.5, -0.5, -0.5] and not f.any()


def test_ties_across_hypotheses():
    """Two alive hypotheses with equal scores and identical rows: every beam^2 candidate of hypothesis 0 ties with one of
    hypothesis 1, so the lower flat offset (hypothesis 0) wins each tie."""
    beam, v = 2, 9
    preds = torch.tensor([[1, 5], [1, 6]])
    scores = torch.tensor([[-1.0], [-1.0]])
    flag = torch.zeros(2, 1, dtype=torch.bool)
    lp = torch.full((beam, v), -7.0)
    lp[:, 3] = -0.25
    lp[:, 8] = -0.75
    tr = []
    p, s, f = btr.beam_step(lp, preds, scores, flag, beam, trace=tr)
    assert tr[0]['offs'].tolist() == [[0, 2]]          # (hyp 0, tok 3) then (hyp 1, tok 3), not (hyp 0, tok 8)
    assert p.tolist() == [[1, 5, 3], [1, 6, 3]] and s.view(-1).tolist() == [-1.25, -1.25]
    # three hypotheses, two of them equal: the tie between hypotheses 1 and 2 goes to hypothesis 1
    beam = 3
    preds = torch.tensor([[1, 4], [1, 5], [1, 6]])
    scores = torch.tensor([[-3.0], [-1.0], [-1.0]])
    lp = torch.full((beam, v), -7.0)
    lp[:, 2] = -0.5
    tr = []
    p, s, f = btr.beam_step(lp, preds, scores, torch.zeros(3, 1, dtype=torch.bool), beam, trace=tr)
    assert tr[0]['parent'].tolist() == [1, 2, 0] and p[:, 2].tolist() == [2, 2, 2]
    assert s.view(-1).tolist() == [-1.5, -1.5, -3.5]


def test_tie_at_the_kth_place():
    """The k-th and (k+1)-th largest values are equal, the higher index first in the row: the lower index is kept."""
    beam, v = 4, 16
    preds, scores, flag = _init(1, beam)
    lp = torch.linspace(-20.0, -10.0, v).view(1, v).repeat(beam, 1)
    lp[:, 15], lp[:, 14], lp[:, 13] = -1.0, -2.0, -3.0
    lp[:, 12] = -4.0
    lp[:, 5] = -4.0                                     # ties with token 12 for the 4th place
    tr = []
    btr.beam_step(lp, preds, scores, flag, beam, trace=tr)
    assert tr[0]['k_tok'][0].tolist() == [15, 14, 13, 5]
    assert tr[0]['tok'].tolist() == [15, 14, 13, 5]


def test_step_zero_only_hypothesis_zero_alive():
    """Initial state: every row identical, scores [0, -inf, ...]; all survivors descend from hypothesis 0 even though the
    -inf rows offer the same tokens, and the tokens come out lower index first."""
    b, beam, v = 2, 4, 10
    preds, scores, flag = _init(b, beam)
    lp = torch.full((b * beam, v), -3.0)
    lp[:, 6] = lp[:, 8] = lp[:, 9] = -1.0
    tr = []
    p, s, f = btr.beam_step(lp, preds, scores, flag, beam, trace=tr)
    assert tr[0]['parent'].tolist() == [0, 0, 0, 0, 4, 4, 4, 4]
    assert p[:, 1].tolist() == [6, 8, 9, 0] * 2
    assert s.view(-1).tolist() == [-1.0, -1.0, -1.0, -3.0] * 2


def test_rows_with_fewer_than_beam_finite_values():
    """A row with two finite log-probs and beam 4 (an LM that rules tokens out): the -inf tokens are ranked by index like
    any other value, so the step returns real token ids, and the beam^2 stage orders its -inf candidates by offset."""
    beam, v = 4, 9
    preds, scores, flag = _init(1, beam)
    lp = torch.full((beam, v), -2.0)
    lm = torch.full((beam, v), NEG)
    lm[:, 7] = -0.5
    lm[:, 3] = -0.5
    tr = []
    p, s, f = btr.beam_step(lp, preds, scores, flag, beam, lm, 0.5, trace=tr)
    assert tr[0]['k_tok'].tolist() == [[3, 7, 0, 1]] * beam
    assert p[:, 1].tolist() == [3, 7, 0, 1] and tr[0]['parent'].tolist() == [0, 0, 0, 0]
    assert s.view(-1).tolist() == [-2.25, -2.25, NEG, NEG]
    assert f.view(-1).tolist() == [False, False, False, True]     # token 1 (EOS) reached through a -inf candidate


def test_finished_hypotheses_and_final_sort_ties():
    """A finished hypothesis offers only (score + 0, EOS): three candidates tie across hypotheses in the beam^2 stage and
    come out in hypothesis order; the final sort keeps equal scores in hypothesis order too."""
    beam, v = 3, 8
    preds = torch.tensor([[1, 4, 1], [1, 5, 2], [1, 6, 3]])
    scores = torch.tensor([[-2.0], [-1.5], [-1.5]])
    flag = torch.tensor([[True], [False], [False]])
    lp = torch.full((beam, v), -9.0)
    lp[:, 1] = -0.5
    tr = []
    p, s, f = btr.beam_step(lp, preds, scores, flag, beam, trace=tr)
    assert tr[0]['k_tok'][0].tolist() == [1, 1, 1] and tr[0]['offs'].tolist() == [[0, 3, 6]]
    assert tr[0]['parent'].tolist() == [0, 1, 2] and p[:, 3].tolist() == [1, 1, 1]
    assert s.view(-1).tolist() == [-2.0, -2.0, -2.0] and f.all()
    nb, ns = btr.beam_finalize(p, torch.tensor([[-3.0], [-2.0], [-2.0]]), beam, 3, 0.0, 5)
    assert ns.tolist() == [[-2.0, -2.0, -3.0]]
    assert nb[0, :, 0].tolist() == [5, 6, 4]
