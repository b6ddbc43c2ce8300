"""Ties and non-finite rows on the per-step graph path: the fused log-softmax + top-k (otb_logsoftmax_topk) and both beam
steps (otb_beam_step on log-probs, which ranks with warp_topk, and on the fused top-k) against the tie-exact
restatement of tests/beam_ties_ref.py.  Rows with 127, 128, 129 and V equal maxima, a tie at the k-th place, V = 17 with
k = 16 (every warp's slice of the fused kernel is shorter than k) and rows with fewer than k finite values (an LM that
rules tokens out with lm_logp = -inf).  Both top-k kernels must return the same real token ids, lower index first,
including among -inf entries."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops
    DEV = torch.device('cuda:0')

from tests import beam_ties_ref as btr

NEG = float('-inf')
LM_W = 0.5          # a power of two: lp + w * lm rounds the same in every kernel and on the host


def _rows(kind, n, V, k, seed):
    """f32 [n, V] logits (cpu) and lm_logp (cpu or None) of one kind of row."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, V, generator=g) * 2.0).clamp(-8.0, 8.0)
    lm = None
    if kind.startswith('max'):                         # m equal maxima at random token ids above every other logit
        m = V if kind == 'max_all' else int(kind[3:])
        for r in range(n):
            ids = torch.randperm(V, generator=g)[:m]
            if m == V:
                x[r] = 0.0
            else:
                x[r, ids] = 9.0
    elif kind == 'kth_tie':                            # the k-th and (k+1)-th largest equal: only the lower id is kept
        for r in range(n):
            ids = torch.randperm(V, generator=g)[:k + 1]
            x[r, ids[:k - 1]] = 10.0 + torch.arange(k - 1, dtype=torch.float32)
            lo, hi = int(ids[k - 1:].min()), int(ids[k - 1:].max())
            x[r, hi] = x[r, lo] = 9.0
    elif kind == 'lm_ninf':                            # the LM allows 3 tokens per row; one row it allows none
        lm = torch.full((n, V), NEG)
        for r in range(1, n):
            lm[r, torch.randperm(V, generator=g)[:3]] = torch.log_softmax(torch.randn(3, generator=g), -1)
    elif kind != 'random':
        raise ValueError(kind)
    return x, lm


def _fused(x, V, k, lm):
    """otb_logsoftmax_topk on x (padded to a row pitch of V rounded up to 8) -> (vals, ids i64, materialised log-probs)."""
    ld = (V + 7) // 8 * 8
    xd = torch.full((x.shape[0], ld), 123.0, device=DEV)      # pad columns must never be read
    xd[:, :V] = x.to(DEV)
    lmd = lm.to(DEV) if lm is not None else None
    lp = torch.empty(x.shape[0], V, device=DEV)
    val, idx = ops.logsoftmax_topk(xd, V, k, lmd, LM_W, out_logp=lp)
    val2, idx2 = ops.logsoftmax_topk(xd, V, k, lmd, LM_W)
    assert torch.equal(val2, val) and torch.equal(idx2, idx), 'the top-k must not depend on materialising the log-probs'
    return val.cpu(), idx.long().cpu(), lp.cpu(), xd


CASES = [('max127', 4234, 10), ('max128', 4234, 10), ('max129', 4234, 10), ('max_all', 4234, 10), ('max129', 4234, 16),
         ('max_all', 17, 16), ('kth_tie', 4234, 10), ('kth_tie', 300, 16), ('kth_tie', 17, 16), ('random', 17, 16),
         ('lm_ninf', 4234, 10), ('lm_ninf', 17, 16), ('lm_ninf', 300, 4)]


@pytest.mark.parametrize('kind,V,k', CASES)
def test_fused_logsoftmax_topk_tie_order(kind, V, k):
    x, lm = _rows(kind, 12, V, k, seed=V + k)
    val, idx, lp, _ = _fused(x, V, k, lm)
    ref_v, ref_i = btr.topk_low_index(lp, k)
    bad = (idx != ref_i).any(dim=1).nonzero().view(-1).tolist()
    print(f'{kind} V={V} k={k}: {12 - len(bad)}/12 rows with the tie-exact ids; finite per row '
          f'{torch.isfinite(lp).sum(1).min().item()}..{torch.isfinite(lp).sum(1).max().item()}')
    assert not bad, f'rows {bad}: kernel ids {idx[bad[0]].tolist()} vs tie-exact {ref_i[bad[0]].tolist()}'
    assert torch.equal(val, ref_v)
    assert int(idx.max()) < V


def _state(B, beam, scores, flag):
    st = ops.BeamState(B, beam, 1, DEV)
    st.init()
    st.scores.copy_(scores.view(-1))
    st.flag.copy_(flag.view(-1).to(torch.uint8))
    return st


@pytest.mark.parametrize('start', ['init', 'mid'])
@pytest.mark.parametrize('kind,V,k', CASES)
def test_graph_path_beam_steps_agree_on_ties(kind, V, k, start):
    """One beam step from the initial state (only hypothesis 0 alive) or from a state with equal scores across hypotheses
    and finished hypotheses: otb_beam_step on log-probs + lm (BeamState.step) and on the fused top-k (BeamState.step_topk)
    against the tie-exact step on the same log-probs; tokens, parents, scores and flags bit-exact, and equal to each other."""
    B, beam = 2, k
    n = B * beam
    x, lm = _rows(kind, n, V, k, seed=3 * V + k)
    if start == 'init':
        scores = torch.tensor([0.0] + [NEG] * (beam - 1)).repeat(B).unsqueeze(1)
        flag = torch.zeros(n, 1, dtype=torch.bool)
    else:
        g = torch.Generator().manual_seed(V)
        scores = -torch.randint(1, 4, (n, 1), generator=g).float()          # many equal scores: ties across hypotheses
        flag = torch.rand(n, 1, generator=g) < 0.25
        flag[1::beam] = False
    val, idx, lp_fused, xd = _fused(x, V, k, lm)
    lp_plain = ops.log_softmax(xd, V)
    lmd = lm.to(DEV) if lm is not None else None
    st_a = _state(B, beam, scores, flag)
    st_a.step(lp_plain, V, lmd, LM_W)
    st_b = _state(B, beam, scores, flag)
    st_b.step_topk(val.to(DEV).contiguous(), idx.int().to(DEV).contiguous())
    preds = torch.ones(n, 1, dtype=torch.long)
    lp_a = lp_plain.cpu() + (LM_W * lm if lm is not None else 0.0)
    for name, st, lp in (('step', st_a, lp_a), ('step_topk', st_b, lp_fused)):
        tr = []
        _, r_scores, r_flag = btr.beam_step(lp, preds, scores, flag, beam, trace=tr)
        assert torch.equal(st.tok_hist[0].long().cpu(), tr[0]['tok']), f'{name}: tokens differ'
        assert torch.equal(st.par_hist[0].long().cpu(), tr[0]['parent']), f'{name}: parents differ'
        assert torch.equal(st.scores.cpu(), r_scores.view(-1)), f'{name}: scores differ'
        assert torch.equal(st.flag.bool().cpu(), r_flag.view(-1)), f'{name}: flags differ'
    assert torch.equal(st_a.tok_hist, st_b.tok_hist) and torch.equal(st_a.par_hist, st_b.par_hist)
    assert int(st_a.tok_hist.max()) < V
