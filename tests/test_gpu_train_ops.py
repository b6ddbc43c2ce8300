"""GPU parity of the backward kernels (training step) against torch fp32 autograd on the same bf16-rounded operands."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops
    DEV = torch.device('cuda:0')
BF = torch.bfloat16


def _rel(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-20))


def _bf(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(BF).to(DEV)


@pytest.mark.parametrize('M,N,K', [(7968, 768, 256), (960, 4240, 256), (7968, 256, 2048), (300, 64, 64), (129, 200, 72),
                                   (64, 256, 256), (7968, 4096, 256)])
def test_linear_wgrad(M, N, K):
    dy, x = _bf(M, N, seed=1, scale=0.5), _bf(M, K, seed=2)
    got = ops.linear_wgrad(dy, x)
    ref = dy.float().t() @ x.float()
    r = _rel(got, ref)
    print(f'wgrad M={M} N={N} K={K} rel_l2={r:.2e}')
    assert r < 2e-3 and torch.isfinite(got).all()


def test_linear_wgrad_strided_views():
    M = 1000
    big_dy, big_x = _bf(M, 768, seed=3), _bf(M, 512, seed=4)
    dy, x = big_dy[:, 256:512], big_x[:, 128:384]
    got = ops.linear_wgrad(dy, x)
    assert _rel(got, dy.float().t() @ x.float()) < 2e-3


def test_dgrad_through_transposed_weight():
    M, N, K = 777, 768, 256
    dy, w = _bf(M, N, seed=5), _bf(N, K, seed=6, scale=0.1)
    wt = w.t().contiguous()
    got = ops.linear(dy, wt)                       # dx = dy W
    assert _rel(got, dy.float() @ w.float()) < 5e-3


@pytest.mark.parametrize('M,N', [(7968, 4096), (100, 256), (33, 4240)])
def test_colsum(M, N):
    x = _bf(M, N, seed=7)
    got = ops.colsum(x)
    torch.testing.assert_close(got, x.float().sum(0), rtol=1e-4, atol=1e-2)


@pytest.mark.parametrize('M,N', [(7968, 256), (37, 256), (500, 64)])
def test_layernorm_bwd(M, N):
    z, dy = _bf(M, N, seed=8, scale=2.0), _bf(M, N, seed=9)
    g = torch.randn(N, generator=torch.Generator().manual_seed(1)).to(DEV) * 0.5 + 1.0
    b = torch.randn(N, generator=torch.Generator().manual_seed(2)).to(DEV) * 0.1
    dz, dg, db = ops.layernorm_bwd(dy, z, g)
    zz = z.float().clone().requires_grad_(True)
    gg, bb = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    torch.nn.functional.layer_norm(zz, (N,), gg, bb, 1e-5).backward(dy.float())
    print(f'LN bwd M={M} N={N}: dz {_rel(dz, zz.grad):.2e} dgamma {_rel(dg, gg.grad):.2e} dbeta {_rel(db, bb.grad):.2e}')
    assert _rel(dz, zz.grad) < 6e-3 and _rel(dg, gg.grad) < 1e-3 and _rel(db, bb.grad) < 1e-3


def test_glu_fwd_bwd():
    M, F = 999, 2048
    u, dh = _bf(M, 2 * F, seed=10), _bf(M, F, seed=11)
    h = ops.glu_fwd(u)
    du = ops.glu_bwd(dh, u)
    uu = u.float().clone().requires_grad_(True)
    hr = torch.nn.functional.glu(uu, dim=-1)
    hr.backward(dh.float())
    assert _rel(h, hr) < 4e-3 and _rel(du, uu.grad) < 6e-3


def test_relu_bwd_and_embed_bwd():
    y, dy = _bf(1000, 128, seed=12), _bf(1000, 128, seed=13)
    got = ops.relu_bwd(dy, y)
    assert torch.equal(got, torch.where(y > 0, dy, torch.zeros_like(dy)))
    V, d, n = 50, 256, 400
    tok = torch.randint(0, V, (n,), generator=torch.Generator().manual_seed(3)).to(DEV)
    dx = _bf(n, d, seed=14)
    dE = torch.ones(V, d, device=DEV)
    ops.embed_bwd(tok, dx, dE, 16.0)
    ref = torch.ones(V, d, device=DEV).index_add_(0, tok, dx.float() * 16.0)
    torch.testing.assert_close(dE, ref, rtol=1e-4, atol=1e-2)


def test_ls_ce_train_grad_and_fixed_lr_scheduled_adam():
    rows, V, ld = 90, 4234, 4240
    g = torch.Generator().manual_seed(5)
    logits = torch.zeros(rows, ld, device=DEV)
    logits[:, :V] = (torch.randn(rows, V, generator=g) * 3).to(DEV)
    tgt = torch.randint(1, V, (rows,), generator=g).to(DEV)
    tgt[::7] = 0
    loss, dl = ops.ls_cross_entropy_train(logits, tgt, V, 0.1, 0)
    x = logits[:, :V].clone().requires_grad_(True)
    conf = torch.full((rows, V), 0.1 / (V - 1), device=DEV)
    conf.scatter_(1, tgt.unsqueeze(1), 0.9)
    logp = torch.log_softmax(x, -1)
    per = (conf * (conf.log() - logp)).sum(-1).masked_fill(tgt == 0, 0.0)
    ref = per.sum() / (tgt != 0).sum()
    ref.backward()
    assert abs(float(loss) - float(ref)) < 1e-4 * abs(float(ref))
    assert _rel(dl[:, :V], x.grad) < 6e-3 and float(dl[:, V:].abs().max()) == 0.0
    # Adam + clipping vs torch.optim.Adam on a flat buffer
    n = 100003
    p0 = torch.randn(n, generator=g).to(DEV)
    pr = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([pr], lr=1e-3, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6)
    p, m, v = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    ss = torch.zeros(1, device=DEV)
    counters = torch.zeros(3, dtype=torch.int32, device=DEV)
    hyper = torch.zeros(4, device=DEV)

    def adam(grad):   # warmup_steps 0: the fixed lr 1e-3, step count kept on the device
        ops.adam_step_sched(p, grad, m, v, ss, 5.0, 1e-3, 256, 0, 1.0, (0.9, 0.98), 1e-9, 1e-6, counters, hyper)

    for step in range(1, 4):
        gr = (torch.randn(n, generator=g) * (10.0 if step == 2 else 0.01)).to(DEV)
        pr.grad = gr.clone()
        torch.nn.utils.clip_grad_norm_([pr], 5.0)
        opt.step()
        ops.sumsq(gr, ss)
        adam(gr)
        torch.testing.assert_close(p, pr.detach(), rtol=1e-5, atol=1e-6)
    bad = torch.full((n,), float('nan'), device=DEV)
    before = p.clone()
    ops.sumsq(bad, ss)
    adam(bad)
    assert torch.equal(p, before), 'non-finite gradient norm must skip the update (trainer.py:229-230)'


def test_spec_augment_kernel_matches_numpy_slicing():
    import random
    import numpy as np
    from opentransformer_b200.augment import draw_bands, spec_augment_
    B, T, F = 3, 300, 80
    lens = [300, 211, 257]
    x = torch.randn(B, T, F, generator=torch.Generator().manual_seed(1)) + 3.0
    random.seed(5); np.random.seed(6)
    ref = x.clone()
    for b, n in enumerate(lens):           # data/augment.py:28-39 on the un-padded utterance
        bd = draw_bands(n, F)
        for j in range(2):
            ref[b, :, bd[2 * j]:bd[2 * j] + bd[2 * j + 1]] = 0
        for j in range(2, 4):
            ref[b, bd[2 * j]:bd[2 * j] + bd[2 * j + 1], :] = 0
    random.seed(5); np.random.seed(6)
    got = spec_augment_(x.to(DEV).clone(), lens)
    assert torch.equal(got.cpu(), ref)


def test_ctc_loss_and_logit_gradient_vs_torch():
    """otb_ctc_loss = nn.CTCLoss(blank 0, 'mean', zero_infinity=True) (model/ctc.py:31,48-52) and its gradient w.r.t. the
    logits: ragged input lengths, repeated labels, an empty target and an INFEASIBLE utterance (more labels than frames,
    which zero_infinity turns into loss 0 / gradient 0)."""
    B, T, V, L = 6, 37, 50, 9
    g = torch.Generator().manual_seed(21)
    logits = (torch.randn(B * T, 56, generator=g) * 2).to(DEV)
    in_len = torch.tensor([37, 30, 12, 37, 5, 20], dtype=torch.int32)
    tgt = torch.randint(1, V, (B, L), generator=g)
    tgt[0, 3] = tgt[0, 2]                                 # repeated label
    tgt[3, :] = tgt[3, 0]                                 # all labels equal
    tlen = torch.tensor([9, 6, 4, 9, 8, 0], dtype=torch.int32)     # utterance 4: 8 labels in 5 frames -> infeasible; 5: empty
    loss, nll, dl = ops.ctc_loss(logits, B, T, V, in_len.to(DEV), tgt.to(DEV), tlen.to(DEV), 0, want_grad=True)
    x = logits[:, :V].detach().cpu().double().view(B, T, V).requires_grad_(True)
    lp = torch.log_softmax(x, -1).transpose(0, 1)
    ref = F.ctc_loss(lp, tgt, in_len.long(), tlen.long(), blank=0, reduction='mean', zero_infinity=True)
    ref.backward()
    ref_nll = F.ctc_loss(lp.detach(), tgt, in_len.long(), tlen.long(), blank=0, reduction='none', zero_infinity=False)
    print(f'ctc loss gpu {float(loss):.6f} torch {float(ref):.6f}; nll gpu {nll.cpu().tolist()} torch {ref_nll.tolist()}')
    assert abs(float(loss) - float(ref)) < 1e-4 * max(1.0, abs(float(ref)))
    fin = torch.isfinite(ref_nll)
    assert torch.equal(torch.isfinite(nll.cpu()), fin)
    torch.testing.assert_close(nll.cpu()[fin].double(), ref_nll[fin], rtol=1e-4, atol=1e-4)
    got = dl.float().cpu().view(B, T, -1)
    assert float(got[:, :, V:].abs().max()) == 0.0
    assert float(got[4].abs().max()) == 0.0, 'infeasible utterance: zero gradient (zero_infinity)'
    r = _rel(got[:, :, :V], x.grad.float())
    print(f'ctc dlogits rel_l2 {r:.3e}')
    assert r < 6e-3
