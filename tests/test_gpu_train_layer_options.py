"""GPU tests of the layer options training takes beside GLU / ReLU and residual_dropout: the gelu, tanh and swish
feed-forward kernels (otb_act_fwd / otb_act_bwd) against float64 autograd, the attention-output dropout as a second mask in
the residual GEMM epilogue and in its backward replay, and whole training passes -- Transformer post- and pre-norm,
Conformer, CTC model, the MWER branch, FusedTrainer eager and graph -- against the fp32 restatement with the product's
masks replayed (the restatement is pinned to the reference by tests/test_train_layer_options.py)."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops, train
    from opentransformer_b200.recognize import second_pass_rows
    DEV = torch.device('cuda:0')

from oracle import speech_model as om
from oracle import train_step as ot
from tests import conformer_train_ref as conf_ref
from tests import ctc_ref
from tests import mwer_ref as mr
from tests.test_gpu_train import REL_L2_GRAD, REL_L2_GRAD_ALL, _batch, _build, _params
from tests.test_gpu_train_kernels import _bf, _keep_np, _rnd, _scale32

BF = torch.bfloat16
P_RES, P_ATTN = 0.1, 0.1
ACTS = ('gelu', 'tanh', 'swish')


def _rel(a, b):
    return float((a.float().cpu() - b.float().cpu()).norm() / (b.float().cpu().norm() + 1e-20))


def _scale2(p, p2):
    """1 / ((1 - p) (1 - p2)) as the kernels compute it: fp32 rates, float64 product, rounded once."""
    return float(np.float32(1.0 / ((1.0 - float(np.float32(p))) * (1.0 - float(np.float32(p2))))))


# ------------------------------------------------------------------------------------------------ activation kernels
def _act64(u, act):
    return {'gelu': F.gelu, 'tanh': torch.tanh, 'swish': lambda x: x * torch.sigmoid(x)}[act](u)


@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('M,N', [(1, 1), (7, 13), (129, 1000), (1000, 2048), (3, 5)])
def test_act_kernels_match_float64(act, M, N):
    """h = act(u) and du = dh act'(u) against float64 autograd on the same bf16 operands: one bf16 rounding of an fp32
    result, at ragged M, N (a tail of M N mod 8 elements)."""
    u = _bf(M, N, scale=3.0, seed=M * 7 + N)
    dh = _bf(M, N, seed=M + N)
    h = ops.act_fwd(u, act)
    du = ops.act_bwd(dh, u, act)
    x = u.double().cpu().requires_grad_(True)
    y = _act64(x, act)
    y.backward(dh.double().cpu())
    for name, got, want in (('h', h, y.detach()), ('du', du, x.grad)):
        err = (got.double().cpu() - want).abs()
        bound = (2.0 ** -8 + 2.0 ** -16) * want.abs() + 1e-6     # half a bf16 ulp of the result, plus the fp32 math
        print(f'{act} M={M} N={N} {name}: max err / bound {float((err / bound).max()):.3f}')
        assert bool((err <= bound).all()), (name, float((err / bound).max()))


def test_act_refuses_an_activation_it_does_not_run():
    u = _bf(4, 8)
    with pytest.raises(KeyError):
        ops.act_fwd(u, 'glu')
    with pytest.raises(RuntimeError, match='16-byte'):
        ops.act_fwd(torch.empty(33, dtype=BF, device=DEV)[1:].view(4, 8), 'gelu')


# ------------------------------------------------------------------------------------------------ two-mask epilogue
# (M, K): 64-wide and 128-wide N tiles, M not a multiple of 128
@pytest.mark.parametrize('p_res,p_attn', [(0.1, 0.1), (0.0, 0.2), (0.3, 0.1), (0.1, 0.0)])
@pytest.mark.parametrize('M,K', [(100, 256), (7968, 256), (1000, 2048)])
def test_two_mask_epilogue_and_backward(p_res, p_attn, M, K):
    """out = resid + alpha keep_res keep_attn (a w^T + b) / ((1 - p_res)(1 - p_attn)) against the masks ops.dropout_mask
    exports for each site (checked against dropout.cuh's keep() restated); the backward is one multiply by the same masks;
    the keep rate is (1 - p_res)(1 - p_attn)."""
    N, site, site2, alpha = 256, 1004, train.ATTN_SITE + 1004, 0.5
    seed = torch.tensor([20241017], dtype=torch.int32, device=DEV)
    a, w = _bf(M, K, seed=30), _bf(N, K, scale=K ** -0.5, seed=31)
    b, resid = _rnd(N, scale=0.1, seed=32), _bf(M, N, seed=33)
    out = ops.linear_dropout_resid(a, w, b, resid, p_res, seed, site, alpha=alpha, p2=p_attn, site2=site2)
    m_res, m_attn = ops.dropout_mask(M, N, p_res, seed, site), ops.dropout_mask(M, N, p_attn, seed, site2)
    assert torch.equal(m_res.cpu(), _keep_np(20241017, site, M, N, p_res))
    assert torch.equal(m_attn.cpu(), _keep_np(20241017, site2, M, N, p_attn))
    mask = m_res * m_attn
    assert torch.equal(ops.dropout_mask(M, N, p_res, seed, site, p2=p_attn, site2=site2), mask)
    scale = _scale2(p_res, p_attn) if p_res > 0 and p_attn > 0 else _scale32(max(p_res, p_attn))
    y = a.float() @ w.float().t() + b
    ref = resid.float() + alpha * (mask.float() * y * scale)
    dropped = mask == 0
    assert torch.equal(out[dropped], resid[dropped]), 'the epilogue dropped other elements than the two replayed masks'
    r = _rel(out, ref)
    keep = float(mask.float().mean())
    want = (1 - p_res) * (1 - p_attn)
    print(f'two masks p_res={p_res} p_attn={p_attn} M={M} K={K}: out rel_l2 {r:.2e}, keep {keep:.5f} (expected {want:.5f})')
    assert r < 4e-3
    assert abs(keep - want) <= 6.0 * (want * (1 - want) / mask.numel()) ** 0.5
    dy = _bf(M, N, seed=34)
    got = ops.dropout_bwd(dy, p_res, seed, site, p2=p_attn, site2=site2)
    assert torch.equal(got, (dy.float() * mask.float() * scale).to(BF)), 'the backward is one fp32 multiply and one rounding'


def test_attention_rate_zero_is_the_one_mask_call_bit_for_bit():
    """p_attn = 0 launches what the one-mask call launches: the same output bits and the same backward, whatever site2."""
    M, K, N, site = 1000, 256, 256, 6
    seed = torch.tensor([4242], dtype=torch.int32, device=DEV)
    a, w = _bf(M, K, seed=40), _bf(N, K, scale=K ** -0.5, seed=41)
    b, resid = _rnd(N, scale=0.1, seed=42), _bf(M, N, seed=43)
    for p in (0.0, 0.1):
        one = ops.linear_dropout_resid(a, w, b, resid, p, seed, site)
        two = ops.linear_dropout_resid(a, w, b, resid, p, seed, site, p2=0.0, site2=train.ATTN_SITE + site)
        assert torch.equal(one, two)
        dy = _bf(M, N, seed=44)
        assert torch.equal(ops.dropout_bwd(dy, p, seed, site), ops.dropout_bwd(dy, p, seed, site, p2=0.0, site2=123))
    # and the residual-only training layer is the plain residual GEMM when every rate is 0
    plain = ops.linear(a, w, b, ops.EPI_RESID, resid=resid)
    assert torch.equal(train._resid(a, train.Lin(w, None, b, '', ''), resid, (0.0, seed, site, (0.0, 0.0)), 0), plain)


# ------------------------------------------------------------------------------------------------ whole passes
def _masks(model, seed, rows, dec_offset=0):
    """(block prefix, sub-layer) -> keep / (1 - p) [rows, 256] of every residual and attention-output dropout site with a
    non-zero rate, the two masks of one sub-layer multiplied; dec_offset moves the decoder's sites (MWER's branch)."""
    n_enc = train._enc_sites(model.encoder)
    out = {}
    for site, part, rate in train.dropout_sites(model) + train.attn_dropout_sites(model):
        if rate == 0.0:
            continue
        base = site - train.ATTN_SITE if site >= train.ATTN_SITE else site
        i, k = divmod(base - (train.ENC_SITE if part == 'encoder' else train.DEC_SITE), n_enc if part == 'encoder' else 3)
        s = site + (dec_offset if part == 'decoder' else 0)
        m = ops.dropout_mask(rows[part], 256, rate, seed, s).cpu().float() / (1.0 - rate)
        key = (f'{part}.blocks.{i}', k)
        out[key] = out[key] * m if key in out else m
    return out


def _drop_fn(masks, B):
    return lambda site, t: t * masks[site].view(B, -1, 256) if site in masks else t


def _compare(tag, loss, g, loss_ref, g_ref, names, tol=REL_L2_GRAD, tol_all=REL_L2_GRAD_ALL):
    worst = sorted(((_rel(g[n], g_ref[n]), n) for n in names), reverse=True)
    r_all = _rel(torch.cat([g[n].reshape(-1).cpu() for n in names]), torch.cat([g_ref[n].reshape(-1) for n in names]))
    print(f'{tag}: loss gpu {float(loss):.5f} oracle {float(loss_ref):.5f}; all grads rel_l2 {r_all:.3e}; worst '
          + ', '.join(f'{n} {r:.2e}' for r, n in worst[:3]))
    assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    assert r_all < tol_all and worst[0][0] < tol, worst[:3]


def _speech_params(act, pre, n_enc=2, n_dec=2):
    p = _params(n_enc=n_enc, n_dec=n_dec)
    for part in ('encoder', 'decoder'):
        p[part].update(activation=act, normalize_before=pre, residual_dropout=P_RES, slf_attn_dropout=P_ATTN)
    p['decoder']['src_attn_dropout'] = P_ATTN
    return p


@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('pre', [False, True])
def test_transformer_pass_matches_restatement(act, pre):
    params = _speech_params(act, pre)
    model, sd = _build(params)
    x, mask, tgt = _batch()
    B, T2, L = x.shape[0], ops.conv_geometry(x.shape[1], 80)[2], tgt.shape[1] - 1
    seed = torch.tensor([12345], dtype=torch.int32, device=DEV)
    masks = _masks(model, seed, {'encoder': B * T2, 'decoder': B * L})
    assert len(masks) == 2 * 2 + 2 * 3
    om.set_dropout(_drop_fn(masks, B))
    try:
        loss_ref, g_ref = ot.loss_and_grads(x, mask, tgt, sd, params)
    finally:
        om.set_dropout(None)
    with torch.no_grad():
        loss, g = train.forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), drop_seed=seed)
    names = [n for n, _ in model.named_parameters()]
    assert set(names) == set(g_ref) == set(g)
    _compare(f'{"pre" if pre else "post"}-norm {act}, residual + attention dropout', loss, g, loss_ref, g_ref, names)


def test_conformer_pass_matches_restatement():
    """A Conformer encoder with a swish macaron feed-forward (residual dropout; its rel-pos attention takes no rate) and a
    Transformer decoder with self- and cross-attention dropout."""
    from tests.test_gpu_conformer_train import _batch as conf_batch, _build as conf_build, _params as conf_params
    params = conf_params(rate=P_RES)
    params['encoder']['activation'] = 'swish'
    params['decoder'].update(activation='swish', slf_attn_dropout=P_ATTN, src_attn_dropout=P_ATTN)
    model, sd = conf_build(params)
    x, mask, tgt, _ = conf_batch()
    B, T2, L = x.shape[0], ops.conv_geometry(x.shape[1], 80)[2], tgt.shape[1] - 1
    seed = torch.tensor([777], dtype=torch.int32, device=DEV)
    masks = _masks(model, seed, {'encoder': B * T2, 'decoder': B * L})
    loss_ref, g_ref, _ = conf_ref.loss_and_grads_train(x, mask, tgt, sd, params, drop=_drop_fn(masks, B))
    with torch.no_grad():
        loss, g = train.forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), drop_seed=seed)
    names = [n for n in g if g_ref.get(n) is not None and not n.endswith('depthwise_conv.bias')]
    _compare('conformer swish, residual dropout + decoder attention dropout', loss, g, loss_ref, g_ref, names)


def test_ctc_model_pass_matches_restatement():
    from tests.test_gpu_ctc_model import _batch as ctc_batch, _build as ctc_build, _params as ctc_params
    params = ctc_params('transformer', P_RES)
    params['encoder'].update(activation='gelu', slf_attn_dropout=P_ATTN)
    model, sd = ctc_build(params)
    x, mask, tgt, tlen = ctc_batch()
    B, T2 = x.shape[0], ops.conv_geometry(x.shape[1], 80)[2]
    seed = torch.tensor([31337], dtype=torch.int32, device=DEV)
    masks = _masks(model, seed, {'encoder': B * T2})
    loss_ref, g_ref, _ = ctc_ref.loss_and_grads_train(x, mask, tgt, tlen, sd, params, drop=_drop_fn(masks, B))
    with torch.no_grad():
        loss, g = train.ctc_forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV), drop_seed=seed)
    _compare('CTC model gelu, residual + attention dropout', loss, g, loss_ref, g_ref, list(g))


def test_mwer_branch_matches_restatement():
    """forward_backward with an n-best: the MWER branch's decoder draws its residual and attention masks at its own sites
    (MWER_SITE + ..., ATTN_SITE + MWER_SITE + ...), replayed in the oracle."""
    from tests.test_gpu_mwer import REL_L2_MWER, REL_L2_MWER_ALL, REL_L2_MWER_LAST_NORM_BIAS, _fixed_nbest, _oracle_mwer
    params = _speech_params('swish', False)
    model, sd = _build(params)
    x, mask, tgt = _batch()
    tlen = (tgt[:, 1:] != 0).sum(1).to(torch.int32)
    B, K, lam = x.shape[0], 4, 0.3
    ids = _fixed_nbest(tgt, K, seed=3)
    hyp_in, hyp_tgt, _, Lp = second_pass_rows(ids.to(DEV))
    hyps = [[mr.cut(ids[b, k]) for k in range(K)] for b in range(B)]
    seed = torch.tensor([778], dtype=torch.int32, device=DEV)
    T2, L = ops.conv_geometry(x.shape[1], 80)[2], tgt.shape[1] - 1
    masks = _masks(model, seed, {'encoder': B * T2, 'decoder': B * L})
    mmasks = {k: v for k, v in _masks(model, seed, {'encoder': 8, 'decoder': B * K * Lp},
                                      dec_offset=train.MWER_SITE - train.DEC_SITE).items() if k[0].startswith('decoder')}
    loss_ref, g_ref = _oracle_mwer(x, mask, tgt, tlen, sd, params, hyp_in.cpu(), hyps, K, lam, False, _drop_fn(masks, B),
                                   _drop_fn(mmasks, B * K))
    with torch.no_grad():
        loss, g = train.forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), truth_length=tlen.to(DEV),
                                         drop_seed=seed, nbest=(hyp_in, hyp_tgt.view(B * K, Lp), K), mwer_ce_weight=lam)
    names = [n for n in g_ref if g_ref[n] is not None]
    # the last norm3.bias carries the MWER term's amplified softmax error (tests/test_gpu_mwer.py): its own bound
    last_bias = f'decoder.blocks.{params["decoder"]["n_blocks"] - 1}.norm3.bias'
    _compare('MWER swish, residual + attention dropout', loss, g, loss_ref, g_ref, [n for n in names if n != last_bias],
             tol=REL_L2_MWER, tol_all=REL_L2_MWER_ALL)
    assert _rel(g[last_bias], g_ref[last_bias]) < REL_L2_MWER_LAST_NORM_BIAS


@pytest.mark.parametrize('use_graph', [False, True])
def test_fused_trainer_follows_the_reference_update(use_graph):
    """gelu feed-forwards and residual + attention dropout through FusedTrainer, three optimizer steps (with the graph: the
    first eager, the second captured, the third replayed): each step's loss against the oracle with that step's masks
    replayed, and the weights after clip + Adam against the oracle's update."""
    params = _speech_params('gelu', False, n_enc=1, n_dec=1)
    model, sd = _build(params)
    model.train()
    tr = train.FusedTrainer(model, lr=1e-3, clip_grad=0.05, model_size=256, warmup_steps=12000, accum_steps=1,
                            use_graph=use_graph)
    names = [n for n, _ in model.named_parameters()]
    w = {n: sd[n].clone() for n in names}
    m = {n: torch.zeros_like(w[n]) for n in names}
    v = {n: torch.zeros_like(w[n]) for n in names}
    losses = []
    for step in (1, 2, 3):
        x, mask, tgt = _batch(seed=10 + step)
        B, T2, L = x.shape[0], ops.conv_geometry(x.shape[1], 80)[2], tgt.shape[1] - 1
        loss = tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV))
        seed = tr.drop_seed.clone()          # the micro-step advances the seed before it draws
        masks = _masks(model, seed, {'encoder': B * T2, 'decoder': B * L})
        sd_now = dict(sd)
        sd_now.update({n: w[n] for n in names})
        sd_now['decoder.output_layer.weight'] = w['decoder.embedding.weight']
        om.set_dropout(_drop_fn(masks, B))
        try:
            loss_ref, g_ref = ot.loss_and_grads(x, mask, tgt, sd_now, params)
        finally:
            om.set_dropout(None)
        losses.append(float(loss))
        assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref)), (step, float(loss), float(loss_ref))
        ot.clip_and_adam(w, g_ref, m, v, step, ot.transformer_lr(ot.first_step_index() + step - 1, 256, 12000), 0.05)
        torch.cuda.synchronize()
        num = sum(float(((p.detach().cpu() - w[n]) ** 2).sum()) for n, p in model.named_parameters())
        den = sum(float(((w[n] - sd[n]) ** 2).sum()) for n in names)
        print(f'graph={use_graph} step {step}: loss {float(loss):.5f} oracle {float(loss_ref):.5f}; '
              f'||w_gpu - w_oracle|| / ||w_oracle - w_init|| = {(num / den) ** 0.5:.3e}')
        assert (num / den) ** 0.5 < 0.3
    assert len(set(losses)) == 3
    if use_graph:
        assert len(tr._graphs) == 1


def test_autograd_seam_with_the_new_options():
    """model.train(); loss.backward() with a tanh feed-forward and attention dropout: every .grad set, and two calls draw
    different masks."""
    params = _speech_params('tanh', True, n_enc=1, n_dec=1)
    model, _ = _build(params)
    x, mask, tgt = _batch()
    model.train()
    inputs, targets = {'inputs': x.to(DEV), 'mask': mask.to(DEV)}, {'targets': tgt.to(DEV), 'targets_length': None}
    l1, _ = model(inputs, targets)
    l2, _ = model(copy.copy(inputs), targets)
    l1.backward()
    assert float(l1) != float(l2)
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in model.parameters())
