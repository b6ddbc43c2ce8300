"""LM shallow fusion in the transducer's greedy and ALSD searches on the GPU (DESIGN.md 4.22), with the Transformer and the
recurrent LM: weight 0 bit-identical to the unfused search, the whole search in lockstep with the float64 restatement
(tests/rnnt_lm_fusion_ref.py) over the GPU's own joint log-probs and LM rows, graph against eager, recapture on a new LM
pack, LM rescoring of the ALSD n-best, and otb_logsoftmax_topk's transducer mode against float64."""
import pytest
import torch

from opentransformer_b200 import ops
from opentransformer_b200.recognize import TransducerRecognizer, lm_token_logprob, second_pass_rows
from tests import rnnt_lm_fusion_ref as ref
from tests.test_gpu_transducer import _batch, _tie_free_model
from tests.test_gpu_transducer_beam import _GpuLattice

pytestmark = pytest.mark.gpu
DEV = 'cuda'
V = 24


def _lm(kind, seed, context_free=False):
    from opentransformer_b200.lm import RecurrentLanguageModel, TransformerLanguageModel
    torch.manual_seed(seed)
    if kind == 'transformer':
        lm = TransformerLanguageModel(dict(type='transformer_lm', vocab_size=V, num_blocks=2, d_model=256, n_heads=4, d_ff=256,
                                           residual_dropout=0.0, smoothing=0.1, share_embedding=False))
    else:
        lm = RecurrentLanguageModel(dict(vocab_size=V, share_embedding=False, smoothing=0.1, num_layers=2, hidden_size=64,
                                         dropout=0.0))
    with torch.no_grad():
        if context_free:
            lm.output_project.weight.zero_()
        lm.output_project.bias.copy_(2.0 * torch.randn(V))
    return lm.to(DEV).eval()


class _LMRows:
    """lm(b, y): float64 log p_lm(. | <S/E>, y), the LM teacher-forced over the whole sequence <S/E> y."""

    def __init__(self, lm):
        self.lm, self.rows = lm, {}

    def __call__(self, b, y):
        y = tuple(y)
        if y not in self.rows:
            inp = torch.tensor([[1] + list(y)] * V, dtype=torch.long, device=DEV)
            tgt = torch.zeros(V, len(y) + 1, dtype=torch.int32, device=DEV)
            tgt[:, -1] = torch.arange(V, device=DEV)
            with torch.no_grad():
                self.rows[y] = lm_token_logprob(self.lm, inp, tgt)[:, -1].double().cpu().numpy()
        return self.rows[y]


def _setup():
    x, mask, _, _ = _batch(lens=(120, 60, 97), seed=5)
    return _tie_free_model(11, x, mask), x.to(DEV), mask.to(DEV)


def _run(model, x, mask, **kw):
    with torch.no_grad():
        return [t.clone() for t in TransducerRecognizer(model, **kw).recognize_ids(x, mask)]


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
@pytest.mark.parametrize('mode,K,W', [('greedy', 1, 1), ('alsd', 1, 1), ('alsd', 4, 1), ('alsd', 4, 4), ('alsd', 15, 4)])
def test_zero_weight_is_bit_identical_to_no_lm(kind, mode, K, W):
    model, x, mask = _setup()
    lm = _lm(kind, 3)
    kw = dict(mode=mode, beam_width=K, nbest=W, max_len=40)
    plain = _run(model, x, mask, **kw)
    fused = _run(model, x, mask, lm=lm, lm_weight=0.0, beta=0.0, **kw)
    for a, b in zip(plain, fused):
        assert torch.equal(a, b)


def _check_against_restatement(model, x, mask, lm, mode, K, W, max_len, lw, beta, tol):
    with torch.no_grad():
        mem, lengths, B, T2 = model.encode_bf16(x, mask)
        lat = _GpuLattice(model, mem, B)
    lmr = _LMRows(lm)
    t_len = lengths.cpu().tolist()
    res = {}
    for use_graph in (False, True):
        res[use_graph] = _run(model, x, mask, lm=lm, lm_weight=lw, beta=beta, mode=mode, beam_width=K, nbest=W,
                              max_len=max_len, use_graph=use_graph)
    for a, b in zip(res[False], res[True]):
        assert torch.equal(a, b)
    ids, n, sc = res[True]
    if mode == 'greedy':
        want = ref.greedy_search(lat, lmr, t_len, max_len, 5, lw, beta)
        for b, (y, s) in enumerate(want):
            assert int(n[b]) == len(y) and ids[b, :len(y)].tolist() == list(y), b
            assert abs(float(sc[b]) - s) <= tol * max(1.0, abs(s)), (b, float(sc[b]), s)
        return want
    want = ref.alsd_search(lat, lmr, t_len, K, W, max_len, lw, beta)
    for b, utt in enumerate(want):
        for w, (y, s) in enumerate(utt.nbest(W)):
            assert int(n[b, w]) == len(y) and ids[b, w, :len(y)].tolist() == list(y), (b, w)
            if s == float('-inf'):
                assert float(sc[b, w]) == s
            else:
                assert abs(float(sc[b, w]) - s) <= tol * max(1.0, abs(s)), (b, w, float(sc[b, w]), s)
    return want


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
@pytest.mark.parametrize('mode,K,W', [('greedy', 1, 1), ('alsd', 1, 1), ('alsd', 4, 4), ('alsd', 15, 1), ('alsd', 15, 4)])
def test_context_free_lm_in_lockstep_with_restatement(kind, mode, K, W):
    """A context-free LM gives the same rows on every path, so the search must follow the restatement exactly."""
    model, x, mask = _setup()
    _check_against_restatement(model, x, mask, _lm(kind, 5, context_free=True), mode, K, W, 30, 0.6, 0.4, 1e-5)


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
@pytest.mark.parametrize('mode,K,W', [('greedy', 1, 1), ('alsd', 4, 4), ('alsd', 15, 4)])
def test_context_lm_carries_each_hypothesis_prefix(kind, mode, K, W):
    """A random LM whose rows depend on the prefix: the search follows the restatement fed the LM teacher-forced on each
    hypothesis' own labels (<S/E> y, the whole sequence at once), so every slot's carried LM state was its own prefix's,
    and each fused score is its alignments' acoustic sum plus lm_weight * the teacher-forced terms + beta |y|."""
    model, x, mask = _setup()
    _check_against_restatement(model, x, mask, _lm(kind, 7), mode, K, W, 30, 0.5, 0.3, 2e-4)


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
def test_new_lm_pack_recaptures_in_place(kind):
    model, x, mask = _setup()
    lm = _lm(kind, 9)
    rec = TransducerRecognizer(model, lm=lm, lm_weight=0.5, beta=0.2, mode='alsd', beam_width=4, nbest=2, max_len=30)
    with torch.no_grad():
        a = [t.clone() for t in rec.recognize_ids(x, mask)]
        s0, g0 = rec._search, rec._search.block.graph
        lm.load_state_dict(_lm(kind, 10).state_dict())
        b = [t.clone() for t in rec.recognize_ids(x, mask)]
        assert rec._search is s0 and g0 is not None and s0.block.graph is not None and s0.block.graph is not g0
        fresh = TransducerRecognizer(model, lm=lm, lm_weight=0.5, beta=0.2, mode='alsd', beam_width=4, nbest=2,
                                     max_len=30).recognize_ids(x, mask)
    for u, v in zip(b, fresh):
        assert torch.equal(u, v)
    assert not all(torch.equal(u, v) for u, v in zip(a, b))


def test_unfused_search_launches_unchanged():
    """Without an LM a step launches exactly the kernels of the unfused search: 7 phases, no LM carry."""
    model, x, mask = _setup()
    for mode in ('greedy', 'alsd'):
        rec = TransducerRecognizer(model, mode=mode, beam_width=4, max_len=30, use_graph=False)
        with torch.no_grad():
            rec.recognize_ids(x, mask)
        s = rec._search
        assert s.lm is None
        if mode == 'alsd':
            assert len(s.step_phases()) == 7
        n0 = ops.COUNTERS['launches']
        with torch.no_grad():
            s._steps()
            n1 = ops.COUNTERS['launches']
            s._predict((s.h, s.c))
        per_step, predictor = (n1 - n0) / s.STEPS, ops.COUNTERS['launches'] - n1
        # joint, output layer, top-k, the predictor, and the greedy step / the beam step, gather and commit
        assert per_step == 3 + predictor + (3 if mode == 'alsd' else 1), (mode, per_step, predictor)


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
def test_lm_rescoring_matches_the_formula(kind):
    model, x, mask = _setup()
    lm = _lm(kind, 12)
    K, W, rw = 6, 3, 0.7
    ids, n, sc = _run(model, x, mask, mode='alsd', beam_width=K, nbest=K, max_len=30)
    rids, rn, rsc = _run(model, x, mask, lm=lm, mode='alsd', beam_width=K, nbest=W, max_len=30, apply_lm_rescoring=True,
                         rescore_weight=rw)
    inputs, targets, nn, Lp = second_pass_rows(ids, n)
    with torch.no_grad():
        tok = lm_token_logprob(lm, inputs, targets.view(-1, Lp))
    tok = torch.where(targets.view(-1, Lp) >= 0, tok, 0.0).view(3, K, Lp).sum(2)
    total = sc.double() + rw * tok.double()
    for b in range(3):
        order = sorted(range(K), key=lambda k: (-float(total[b, k]), k))[:W]
        for w, k in enumerate(order):
            if float(sc[b, k]) == float('-inf'):
                continue
            assert int(rn[b, w]) == int(n[b, k]) and rids[b, w, :int(n[b, k])].tolist() == ids[b, k, :int(n[b, k])].tolist()
            assert abs(float(rsc[b, w]) - float(total[b, k])) <= 1e-4 * max(1.0, abs(float(total[b, k])))


def test_topk_transducer_mode_against_float64():
    g = torch.Generator().manual_seed(3)
    rows, Vx, k = 37, 301, 5
    ld = 304
    x = torch.full((rows, ld), float('nan'))
    x[:, :Vx] = 3.0 * torch.randn(rows, Vx, generator=g)
    lm = torch.log_softmax(2.0 * torch.randn(rows, Vx, generator=g), 1)
    lm[3, 7] = float('-inf')
    xd, lmd = x.to(DEV), lm.to(DEV).contiguous()
    for lw, beta, use_lm in ((0.4, 0.3, True), (0.0, -0.5, False), (1.0, 0.0, True)):
        val = torch.full((rows, k), float('nan'), device=DEV)
        idx = torch.full((rows, k), -7, dtype=torch.int32, device=DEV)
        lp = torch.full((rows, ld), float('nan'), device=DEV)
        ops.logsoftmax_topk(xd, Vx, k, lmd if use_lm else None, lw, out_val=val, out_idx=idx, out_logp=lp, lm_beta=beta,
                            lm_exempt=0)
        plain = torch.log_softmax(x[:, :Vx].double(), 1)
        fused = plain + ((lw * lm.double() if use_lm else 0.0) + beta)
        fused[:, 0] = plain[:, 0]
        assert torch.allclose(lp[:, :Vx].cpu().double(), plain, atol=1e-5)
        assert torch.isnan(lp[:, Vx:]).all()
        for r in range(rows):
            want = sorted(range(Vx), key=lambda i: (-float(fused[r, i]), i))[:k]
            assert idx[r].tolist() == want, r
            assert torch.allclose(val[r].cpu().double(), fused[r, want], atol=1e-5)
    # the attention decoder's mode is unchanged: explicit defaults give the same bits
    a = ops.logsoftmax_topk(xd, Vx, k, lmd, 0.3)
    b = ops.logsoftmax_topk(xd, Vx, k, lmd, 0.3, lm_beta=0.0, lm_exempt=-1)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    with pytest.raises(RuntimeError, match='lm_beta needs'):
        ops.logsoftmax_topk(xd, Vx, k, lmd, 0.3, lm_beta=0.5)
    with pytest.raises(RuntimeError, match='below V'):
        ops.logsoftmax_topk(xd, Vx, k, lmd, 0.3, lm_exempt=Vx)
