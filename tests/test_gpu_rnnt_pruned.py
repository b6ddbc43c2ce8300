"""Pruned RNN-T on the GPU: the simple joint's normalizer and backward, the prune ranges, the banded joint, recursion and
joint backward against float64 (tests/rnnt_pruned_ref.py), the whole pruned training pass against the restatement, the
training entry points, and recognition from a checkpoint that carries the simple projections."""
import numpy as np
import pytest
import torch

from opentransformer_b200 import ops, train
from opentransformer_b200.model import TransducerModel
from opentransformer_b200.recognize import TransducerRecognizer
from oracle import train_step as ot
from tests import rnnt_pruned_ref as prr
from tests import rnnt_ref
from tests.test_gpu_transducer import REL_L2_GRAD, _batch, _bf, _build, _lens, _rel, _replay, _ulp_bf16
from tests.test_rnnt_ref import params

pytestmark = pytest.mark.gpu
DEV = 'cuda'
# The whole pass adds the simple and the pruned objectives' gradients, each with the bf16 rounding of its own gradient
# rows (dlogits, d am, d lm), so the noise floor against the restatement sits a little above the full loss's: on an
# H100 the worst parameter (the first conv layer's weight, Transformer encoder, no dropout) was at 4.1e-2 with every band
# equal to the restatement's, the other cases at 3.1e-2 .. 3.7e-2.
REL_L2_GRAD_PRUNED = 5e-2


def _pparams(S=3, alpha=0.5, **kw):
    p = params(**kw)
    p['joint'] = dict(p['joint'], prune_range=S, simple_loss_scale=alpha)
    return p


def _simple_operands(B, T, U1, V, t_len, u_len, seed):
    g = torch.Generator().manual_seed(seed)
    ld = (V + 7) // 8 * 8
    am = torch.full((B * T, ld), float('nan'))
    lm = torch.full((B * U1, ld), float('nan'))
    am[:, :V] = 2 * torch.randn(B * T, V, generator=g)
    lm[:, :V] = 2 * torch.randn(B * U1, V, generator=g)
    labels = torch.randint(1, V, (B, max(U1 - 1, 1)), generator=g, dtype=torch.int32)
    return am, lm, labels, _lens(t_len, u_len)


CASES = [(3, 37, 5, 50, [37, 1, 20], [4, 0, 2]), (2, 70, 40, 4234, [70, 33], [39, 12])]


# ------------------------------------------------------------------------------------------------ the simple joint
@pytest.mark.parametrize('B,T,U1,V,t_len,u_len', CASES)
def test_simple_lse_matches_float64(B, T, U1, V, t_len, u_len):
    am, lm, labels, (tl, ul) = _simple_operands(B, T, U1, V, t_len, u_len, V)
    lp, m_am, m_lm = ops.rnnt_simple_lse(am.to(DEV), lm.to(DEV), V, B, T, U1, tl, ul, labels.to(DEV))
    lp = lp.cpu().double().view(B, T, U1, 3)
    a64, l64 = am[:, :V].double().view(B, T, V), lm[:, :V].double().view(B, U1, V)
    for b in range(B):
        Tb, Ub = t_len[b], u_len[b]
        z = torch.logsumexp(a64[b, :Tb, None] + l64[b, None, :Ub + 1], -1)
        lpb, lpy = prr.simple_logprobs(a64[b, :Tb], l64[b, :Ub + 1], labels[b, :Ub].long())
        assert float((lp[b, :Tb, :Ub + 1, 0] - z).abs().max()) < 2e-5 * max(1.0, float(z.abs().max()))
        assert float((lp[b, :Tb, :Ub + 1, 1] - lpb).abs().max()) < 1e-4
        if Ub:
            assert float((lp[b, :Tb, :Ub, 2] - lpy).abs().max()) < 1e-4
        assert bool(torch.isinf(lp[b, :Tb, Ub, 2]).all())
        assert float(lp[b, Tb:].abs().sum()) == 0 and float(lp[b, :, Ub + 1:].abs().sum()) == 0


@pytest.mark.parametrize('B,T,U1,V,t_len,u_len', CASES)
def test_simple_bwd_matches_float64(B, T, U1, V, t_len, u_len):
    am, lm, labels, (tl, ul) = _simple_operands(B, T, U1, V, t_len, u_len, V + 1)
    lp, m_am, m_lm = ops.rnnt_simple_lse(am.to(DEV), lm.to(DEV), V, B, T, U1, tl, ul, labels.to(DEV))
    _, _, grad = ops.rnnt_loss(lp, B, T, U1, tl, ul)
    d_am, d_lm = ops.rnnt_simple_bwd(am.to(DEV), lm.to(DEV), V, B, T, U1, tl, ul, labels.to(DEV), lp, m_am, m_lm, grad, 0.5,
                                     torch.tensor([3.0], device=DEV))
    a64 = am[:, :V].double().view(B, T, V).requires_grad_(True)
    l64 = lm[:, :V].double().view(B, U1, V).requires_grad_(True)
    total = 0
    for b in range(B):
        Tb, Ub = t_len[b], u_len[b]
        lpb, lpy = prr.simple_logprobs(a64[b, :Tb], l64[b, :Ub + 1], labels[b, :Ub].long())
        total = total + rnnt_ref.lattice_nll(lpb, lpy)
    (1.5 * total / B).backward()
    ld = d_am.shape[1]
    want_am = torch.zeros(B * T, ld, dtype=torch.float64)
    want_am[:, :V] = a64.grad.reshape(B * T, V)
    want_lm = torch.zeros(B * U1, ld, dtype=torch.float64)
    want_lm[:, :V] = l64.grad.reshape(B * U1, V)
    assert _rel(d_am, _bf(want_am)) < 2e-3
    assert _rel(d_lm, _bf(want_lm)) < 2e-3
    assert float(d_am[:, V:].float().abs().sum()) == 0 and float(d_lm[:, V:].float().abs().sum()) == 0
    again = ops.rnnt_simple_bwd(am.to(DEV), lm.to(DEV), V, B, T, U1, tl, ul, labels.to(DEV), lp, m_am, m_lm, grad, 1.5)
    assert torch.equal(again[0], d_am) and torch.equal(again[1], d_lm)


# ------------------------------------------------------------------------------------------------ prune ranges
@pytest.mark.parametrize('S', [2, 3, 5])
def test_prune_ranges_match_restatement(S):
    rng = np.random.default_rng(S)
    B, T, U1 = 6, 40, 60
    t_len = [40, 1, 17, 30, 25, 0]
    u_len = [min(59, 40 * (S - 1)), 0, 3, 59, S - 1, 4]
    occ = (rng.random((B, T, U1)) * (rng.random((B, T, U1)) < 0.7)).astype(np.float32)
    grad = torch.zeros(B * T * U1, 2)
    grad[:, 0] = -torch.from_numpy(occ).reshape(-1)
    tl, ul = _lens(t_len, u_len)
    s = ops.rnnt_prune_ranges(grad.to(DEV), B, T, U1, tl, ul, S).cpu()
    for b in range(B):
        Tb, Ub = t_len[b], u_len[b]
        want = prr.prune_ranges(occ[b, :Tb, :Ub + 1], Tb, Ub, S)
        assert s[b, :Tb].tolist() == want.tolist(), b
        assert s[b, Tb:].abs().sum() == 0
        if Ub <= Tb * (S - 1) and Tb > 0:
            assert prr.check_ranges(want, Tb, Ub, S) == []


# ------------------------------------------------------------------------------------------------ the banded lattice
def _band(B, T, U1, S, t_len, u_len, seed):
    """s_begin from the rule over random occupancies (a band the kernels accept), as i32 [B, T]."""
    rng = np.random.default_rng(seed)
    s = torch.zeros(B, T, dtype=torch.int32)
    for b in range(B):
        occ = rng.random((t_len[b], u_len[b] + 1)).astype(np.float32)
        s[b, :t_len[b]] = torch.from_numpy(prr.prune_ranges(occ, t_len[b], u_len[b], S).astype(np.int32))
    return s


def test_banded_joint_and_joint_bwd_match_float64():
    B, T, U1, S, D = 3, 9, 8, 3, 64
    t_len, u_len = [9, 4, 6], [7, 2, 0]
    s = _band(B, T, U1, S, t_len, u_len, 1)
    g = torch.Generator().manual_seed(4)
    ep = torch.randn(B * T, D, generator=g).to(ops.BF16)
    pp = torch.randn(B * U1, D, generator=g).to(ops.BF16)
    tl, ul = _lens(t_len, u_len)
    hj = ops.rnnt_joint(ep.to(DEV), pp.to(DEV), B, T, U1, tl, ul, s_begin=s.to(DEV), S=S).cpu().double().view(B, T, S, D)
    want = torch.zeros(B, T, S, D, dtype=torch.float64)
    live = torch.zeros(B, T, S, dtype=torch.bool)
    for b in range(B):
        for t in range(t_len[b]):
            for k in range(S):
                u = int(s[b, t]) + k
                if u <= u_len[b]:
                    live[b, t, k] = True
                    want[b, t, k] = torch.tanh(ep[b * T + t].double() + pp[b * U1 + u].double())
    assert bool(((hj - want).abs() <= _ulp_bf16(want)).all())
    dh = torch.randn(B * T * S, D, generator=g).to(ops.BF16)
    h = hj.reshape(B * T * S, D).to(ops.BF16)
    dep, dpp = ops.rnnt_joint_bwd(dh.to(DEV), h.to(DEV), B, T, U1, tl, ul, s_begin=s.to(DEV), S=S)
    dz = (dh.double() * (1 - h.double() ** 2)).view(B, T, S, D) * live[..., None]
    want_pp = torch.zeros(B, U1, D, dtype=torch.float64)
    for b in range(B):
        for t in range(T):
            for k in range(S):
                if live[b, t, k]:
                    want_pp[b, int(s[b, t]) + k] += dz[b, t, k]
    assert _rel(dep, _bf(dz.sum(2).reshape(B * T, D))) < 1e-3
    assert _rel(dpp, _bf(want_pp.reshape(B * U1, D))) < 1e-3


@pytest.mark.parametrize('case', ['ragged', 'long', 'no_path'])
def test_banded_loss_and_node_grads_match_float64(case):
    if case == 'ragged':
        B, T, U1, S, t_len, u_len = 3, 10, 9, 3, [10, 1, 6], [8, 0, 5]
    elif case == 'long':                    # a band that ends at U_b = 1023
        B, T, U1, S, t_len, u_len = 2, 260, 1024, 5, [260, 30], [1023, 20]
    else:                                   # utterance 1: U_b > T_b (S - 1), no alignment inside any band
        B, T, U1, S, t_len, u_len = 2, 6, 10, 2, [6, 4], [5, 9]
    V = 13
    s = _band(B, T, U1, S, t_len, u_len, 2)
    g = torch.Generator().manual_seed(U1)
    ld = 16
    logits = torch.zeros(B * T * S, ld)
    logits[:, :V] = 2 * torch.randn(B * T * S, V, generator=g)
    labels = torch.randint(1, V, (B, U1 - 1), generator=g, dtype=torch.int32)
    tl, ul = _lens(t_len, u_len)
    band = {'s_begin': s.to(DEV), 'S': S}
    lp = torch.empty(B * T * S, 3, device=DEV)
    ops.rnnt_logprob(logits.to(DEV), 0, V, B, T, U1, tl, ul, labels.to(DEV), lp, **band)
    loss, nll, grad = ops.rnnt_loss(lp, B, T, U1, tl, ul, grad_scale=1.0, **band)
    lp = lp.cpu().double().view(B, T, S, 3)
    grad = grad.cpu().double().view(B, T, S, 2)
    x = logits[:, :V].double().view(B, T, S, V)
    for b in range(B):
        Tb, Ub = t_len[b], u_len[b]
        full_b = torch.full((Tb, Ub + 1), float('nan'), dtype=torch.float64)
        full_y = torch.full((Tb, max(Ub, 1)), float('nan'), dtype=torch.float64)
        for t in range(Tb):
            for k in range(S):
                u = int(s[b, t]) + k
                if u > Ub:
                    continue
                lse = torch.logsumexp(x[b, t, k], 0)
                assert abs(float(lp[b, t, k, 1]) - float(x[b, t, k, 0] - lse)) < 1e-5
                full_b[t, u] = lp[b, t, k, 1]
                if u < Ub:
                    assert abs(float(lp[b, t, k, 2]) - float(x[b, t, k, int(labels[b, u])] - lse)) < 1e-5
                    full_y[t, u] = lp[b, t, k, 2]
        a = full_b.clone().requires_grad_(True)
        c = full_y[:, :Ub].clone().requires_grad_(True)
        want = prr.band_nll(a, c, s[b, :Tb].tolist(), S)
        if case == 'no_path' and b == 1:
            assert float(nll[b]) == float('inf') and float(want) == float('inf')
            assert float(grad[b].abs().sum()) == 0
            continue
        assert abs(float(nll[b]) - float(want)) < 1e-5 * abs(float(want))
        (want / B).backward()
        for t in range(Tb):
            for k in range(S):
                u = int(s[b, t]) + k
                if u > Ub:
                    assert float(grad[b, t, k].abs().sum()) == 0
                    continue
                gb = float(a.grad[t, u]) if a.grad is not None else 0.0
                gy = float(c.grad[t, u]) if u < Ub and c.grad is not None else 0.0
                assert abs(float(grad[b, t, k, 0]) - gb) < 1e-5 and abs(float(grad[b, t, k, 1]) - gy) < 1e-5
    if case == 'no_path':
        assert float(loss) == float('inf')


# ------------------------------------------------------------------------------------------------ the model
def _pbuild(p, seed=1234):
    model, sd = _build(p, seed)
    return model, sd


@pytest.mark.parametrize('encoder_type,layers,rate', [('transformer', 1, 0.0), ('transformer', 2, 0.1), ('conformer', 1, 0.0),
                                                      ('conformer', 2, 0.1)])
def test_pruned_training_matches_restatement(encoder_type, layers, rate, monkeypatch):
    """The bands are a selection from fp32 occupancies, so a near-tie between two windows may go either way between the
    GPU and the float64 restatement: the restatement's own bands must agree with the GPU's on almost every frame, and the
    loss and gradients are compared on the GPU's bands."""
    p = _pparams(S=3, alpha=0.5, encoder_type=encoder_type, layers=layers, dropout=rate, rate=rate)
    model, sd = _pbuild(p)
    x, mask, tgt, tlen = _batch()
    seed = torch.tensor([777], dtype=torch.int32, device=DEV)
    T2 = ops.conv_geometry(x.shape[1], 80)[2]
    drop = _replay(model, x.shape[0], T2, tgt.shape[1] - 1, rate, rate, seed) if rate > 0 else None
    seen = []
    ranges = ops.rnnt_prune_ranges
    monkeypatch.setattr(ops, 'rnnt_prune_ranges', lambda *a, **k: seen.append(ranges(*a, **k)) or seen[-1])
    with torch.no_grad():
        loss, g = train.transducer_forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV),
                                                    drop_seed=seed)
    gpu_s = seen[0].cpu()
    own = []
    bands = [gpu_s[b, :T2].tolist() for b in range(x.shape[0])]
    loss_ref, g_ref, _ = prr.loss_and_grads(x, mask, tgt, tlen, sd, p, drop=drop, bands=bands, record=own)
    same = sum(int(a == c) for b, s in enumerate(own) for a, c in zip(s.tolist(), bands[b]))
    frames = sum(len(s) for s in own)
    print(f'bands: {same} of {frames} frames as the restatement picks them')
    assert same >= 0.9 * frames
    assert set(g) == {n for n, _ in model.named_parameters() if g_ref[n] is not None}
    assert {'joint.simple_am_proj.weight', 'joint.simple_am_proj.bias', 'joint.simple_lm_proj.weight',
            'joint.simple_lm_proj.bias'} <= set(g)
    zero = [n for n in g if n.endswith('depthwise_conv.bias')]
    worst = sorted(((_rel(g[n], g_ref[n]), n) for n in g if n not in zero), reverse=True)
    print(f'{encoder_type} layers {layers} rate {rate}: loss gpu {float(loss):.5f} ref {float(loss_ref):.5f}; worst '
          + ', '.join(f'{n} {r:.2e}' for r, n in worst[:4]))
    assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    assert worst[0][0] < REL_L2_GRAD_PRUNED, worst[:3]


def test_wide_band_is_the_full_path():
    """S >= U + 1 with simple_loss_scale 0: the objective and every gradient but the simple projections' are the full
    path's."""
    p = _pparams(S=12, alpha=0.0)
    model, _ = _pbuild(p)
    x, mask, tgt, tlen = _batch()
    pk = train.EncoderPack(model, with_decoder=False)
    op = train.transducer_operands(model, pk)
    out = []
    for o in (op, {k: v for k, v in op.items() if k != 'simple'}):
        with torch.no_grad():
            mem, tr = train._encoder_fwd(model.train(), pk, x.to(DEV), mask.to(DEV), None)
            g = train.Grads()
            loss, dmem = train.transducer_head(model, o, mem, tr.B, tr.T2, tr.lengths, tgt.to(DEV), tlen.to(DEV), g=g)
        out.append((loss, dmem, g))
    assert abs(float(out[0][0]) - float(out[1][0])) <= 1e-6 * abs(float(out[1][0]))
    for n in out[1][2]:
        assert _rel(out[0][2][n], out[1][2][n]) < 1e-5, n
    assert _rel(out[0][1], out[1][1]) < 1e-5


def test_autograd_seam_and_modes():
    p = _pparams()
    model, sd = _pbuild(p)
    x, mask, tgt, tlen = _batch()
    inputs, targets = {'inputs': x.to(DEV), 'mask': mask.to(DEV)}, {'targets': tgt.to(DEV), 'targets_length': tlen.to(DEV)}
    model.train()
    loss, aux = model(inputs, targets)
    assert aux is None and loss.requires_grad
    (loss * 0.5).backward()
    loss_ref, g_ref, _ = prr.loss_and_grads(x, mask, tgt, tlen, sd, p)
    for n in ('joint.simple_am_proj.weight', 'joint.simple_am_proj.bias', 'joint.simple_lm_proj.weight',
              'joint.simple_lm_proj.bias'):
        t = dict(model.named_parameters())[n]
        assert t.grad is not None and _rel(t.grad, 0.5 * g_ref[n]) < REL_L2_GRAD, n
    used = list(model.named_parameters())
    r = _rel(torch.cat([t.grad.reshape(-1) for _, t in used]), 0.5 * torch.cat([g_ref[n].reshape(-1) for n, _ in used]))
    assert r < 2e-2, r
    with torch.no_grad():
        l_nograd, _ = model(inputs, targets)
        model.eval()
        l_eval, _ = model(inputs, targets)
    assert abs(float(l_nograd) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    assert abs(float(l_eval) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    assert 'simple' not in model._pack.get()


def test_batch_with_an_unreachable_utterance():
    """U_b > T_b (S - 1): that utterance's pruned nll is +inf, so the batch loss is +inf, and its pruned gradients are
    zero: the other utterances' gradients are what they are without it."""
    p = _pparams(S=2, alpha=0.5)
    model, _ = _pbuild(p)
    # T' = 2 frames, so at most 2 (S - 1) = 2 labels fit the bands: utterances 0 and 1 have 4 and 6, utterance 2 has one
    x, mask, tgt, tlen = _batch(B=3, T=12, L=8, lens=(12, 12, 12))
    assert ops.conv_geometry(12, 80)[2] == 2 and (tlen - 1).tolist() == [4, 6, 1]
    with torch.no_grad():
        loss, g = train.transducer_forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV))
    assert float(loss) == float('inf')
    assert all(bool(torch.isfinite(t).all()) for t in g.values())


def _trainer_run(p, use_graph, steps=2):
    model, sd = _pbuild(p)
    model.train()
    tr = train.FusedTrainer(model, clip_grad=0.05, accum_steps=2, use_graph=use_graph)
    losses = []
    for _ in range(steps):
        for _ in range(2):
            x, mask, tgt, tlen = _batch(seed=0)
            losses.append(float(tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV))))
    torch.cuda.synchronize()
    return model, sd, tr, losses


def test_fused_trainer_follows_the_oracle_step_graph_and_eager():
    p = _pparams()
    runs = {}
    for use_graph in (False, True):
        model, sd, tr, losses = _trainer_run(p, use_graph)
        assert tr._graphs if use_graph else not tr._graphs
        runs[use_graph] = ({n: t.detach().clone() for n, t in model.named_parameters()}, losses)
    assert runs[False][1] == runs[True][1]
    _, sd = _pbuild(p)
    names = [n for n, _ in tr.params]
    assert 'joint.simple_am_proj.weight' in names and 'joint.simple_lm_proj.bias' in names
    w = {n: sd[n].clone() for n in names}
    m = {n: torch.zeros_like(w[n]) for n in names}
    v = {n: torch.zeros_like(w[n]) for n in names}
    for opt_step in (1, 2):
        acc = None
        for _ in range(2):
            x, mask, tgt, tlen = _batch(seed=0)
            sd_now = dict(sd)
            sd_now.update({n: w[n] for n in names})
            _, g_ref, _ = prr.loss_and_grads(x, mask, tgt, tlen, sd_now, p)
            acc = {n: g_ref[n] / 2 for n in names} if acc is None else {n: acc[n] + g_ref[n] / 2 for n in names}
        lr = ot.transformer_lr(ot.first_step_index() + opt_step - 1, 256, 12000)
        ot.clip_and_adam(w, acc, m, v, opt_step, lr, 0.05)
    for use_graph in (False, True):
        got = runs[use_graph][0]
        num = sum(float(((got[n].cpu() - w[n]) ** 2).sum()) for n in names)
        den = sum(float(((w[n] - sd[n]) ** 2).sum()) for n in names)
        print(f'graph={use_graph}: rel {(num / den) ** 0.5:.3e}')
        assert (num / den) ** 0.5 < 0.3
    num = sum(float(((runs[True][0][n] - runs[False][0][n]) ** 2).sum()) for n in names)
    den = sum(float(((runs[False][0][n].cpu() - sd[n]) ** 2).sum()) for n in names)
    assert (num / den) ** 0.5 < 1e-4


def test_mixspeech_micro_step_matches_oracle():
    p = _pparams()
    model, sd = _pbuild(p)
    model.train()
    tr = train.FusedTrainer(model, accum_steps=1, use_graph=False, mixspeech=True)
    x, mask, tgt, tlen = _batch(B=4, lens=(120, 96, 109, 100), seed=3)
    batch = model.train_batch(x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV))
    tr.flat_bf16.copy_(tr.flat_p)
    loss = tr._micro_mix(batch)
    lam = float(tr.last_lambda)
    xm = lam * x[0::2] + (1 - lam) * x[1::2]
    mm = mask[0::2] | mask[1::2]
    l1, g1, _ = prr.loss_and_grads(xm, mm, tgt[0::2], tlen[0::2], sd, p)
    l2, g2, _ = prr.loss_and_grads(xm, mm, tgt[1::2], tlen[1::2], sd, p)
    want = lam * l1 + (1 - lam) * l2
    assert abs(float(loss) - float(want)) < 2e-2 * abs(float(want))
    names = [n for n, _ in tr.params]
    got = torch.cat([tr.sink[n].reshape(-1).cpu() for n in names])
    ref = torch.cat([(lam * g1[n] + (1 - lam) * g2[n]).reshape(-1) for n in names])
    assert _rel(got, ref) < REL_L2_GRAD


# ------------------------------------------------------------------------------------------------ recognition
@pytest.mark.parametrize('mode', ['greedy', 'alsd'])
def test_checkpoint_with_simple_projections_recognizes_alike(mode):
    p = _pparams()
    pruned, _ = _pbuild(p, seed=21)
    plain = TransducerModel(params()).to(DEV)
    plain.load_state_dict({k: v for k, v in pruned.state_dict().items() if '.simple_' not in k})
    x, mask, _, _ = _batch(lens=(120, 60, 97), seed=5)
    out = []
    for m in (pruned, plain):
        m.eval()
        rec = TransducerRecognizer(m, mode=mode, beam_width=4, max_len=40)
        out.append([t.clone() for t in rec.recognize_ids(x.to(DEV), mask.to(DEV))])
    for a, b in zip(*out):
        assert torch.equal(a, b)
