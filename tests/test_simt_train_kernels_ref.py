"""Pin the float64 restatements of tests/simt_train_kernels_ref.py (the training step's SIMT kernels) to torch autograd,
torch.optim.Adam and nn.Conv1d + nn.BatchNorm1d in train(), all in float64 on the CPU, and check their edge cases in the
simplest form.  No GPU needed."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import simt_train_kernels_ref as ref

F64 = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _close(a, b, tol=1e-12):
    a, b = a.to(F64), b.to(F64)
    scale = max(float(b.abs().max()) if b.numel() else 0.0, 1.0)
    assert float((a - b).abs().max()) <= tol * scale if a.numel() else True, float((a - b).abs().max())


@pytest.mark.parametrize('M,N', [(1, 8), (5, 136), (7, 256), (3, 1000)])
def test_layernorm_bwd_matches_autograd(M, N):
    g = _g(N)
    z = (torch.randn(M, N, generator=g, dtype=F64) * 2 + 50).requires_grad_()
    gamma = (1 + 0.3 * torch.randn(N, generator=g, dtype=F64)).requires_grad_()
    beta = (0.2 * torch.randn(N, generator=g, dtype=F64)).requires_grad_()
    dy = torch.randn(M, N, generator=g, dtype=F64)
    F.layer_norm(z, (N,), gamma, beta, 1e-5).backward(dy)
    dz, dgamma, dbeta = ref.layernorm_bwd(dy, z.detach(), gamma.detach(), 1e-5)
    _close(dz, z.grad, 1e-10)
    _close(dgamma, gamma.grad)
    _close(dbeta, beta.grad)


def test_glu_matches_autograd():
    g = _g(1)
    u = torch.randn(9, 2 * 24, generator=g, dtype=F64, requires_grad=True)
    dh = torch.randn(9, 24, generator=g, dtype=F64)
    h = F.glu(u, -1)
    h.backward(dh)
    _close(ref.glu(u.detach()), h.detach())
    _close(ref.glu_bwd(dh, u.detach()), u.grad)


@pytest.mark.parametrize('p,p2', [(0.1, 0.0), (0.0, 0.25), (0.1, 0.3), (0.0, 0.0)])
def test_dropout_bwd_is_the_gradient_of_the_masked_scaled_product(p, p2):
    g = _g(2)
    x = torch.randn(6, 10, generator=g, dtype=F64, requires_grad=True)
    k1 = torch.rand(6, 10, generator=g) >= p
    k2 = torch.rand(6, 10, generator=g) >= p2
    dy = torch.randn(6, 10, generator=g, dtype=F64)
    p32, q32 = (float(torch.tensor(v, dtype=torch.float32)) for v in (p, p2))
    (x * k1 / (1 - p32) * k2 / (1 - q32)).backward(dy)
    _close(ref.dropout_bwd(dy, k1 & k2, p, p2), x.grad)


def test_dropout_add_masks_rows_past_their_length():
    g = _g(3)
    M, N, period = 12, 16, 4
    x, r = torch.randn(M, N, generator=g, dtype=F64), torch.randn(M, N, generator=g, dtype=F64)
    keep = torch.rand(M, N, generator=g) >= 0.2
    row_len = torch.tensor([4, 1, 0], dtype=torch.int32)
    got = ref.dropout_add(x, r, keep, 0.2, alpha=0.5, row_len=row_len, row_period=period)
    want = r.clone()
    for row in range(M):
        if row % period < int(row_len[row // period]):
            want[row] += 0.5 * x[row] * keep[row] / (1 - float(torch.tensor(0.2, dtype=torch.float32)))
    _close(got, want)
    _close(ref.dropout_add(x, None, None, 0.0), x)                 # p = 0, no residual, no rows masked: x itself


def test_embed_bwd_matches_autograd_and_skips_out_of_range_ids():
    g = _g(4)
    V, d = 7, 16
    tok = torch.tensor([3, 3, 0, 6, -1, 7, 3, 100])
    dx = torch.randn(tok.numel(), d, generator=g, dtype=F64)
    dE0 = torch.randn(V, d, generator=g, dtype=F64)
    ok = (tok >= 0) & (tok < V)
    E = torch.zeros(V, d, dtype=F64, requires_grad=True)
    (F.embedding(tok[ok], E) * 0.5).backward(dx[ok])
    _close(ref.embed_bwd(tok, dx, dE0, 0.5), dE0 + E.grad)


@pytest.mark.parametrize('max_norm,warmup', [(5.0, 4), (0.0, 0), (1e-3, 1000)])
def test_adam_step_matches_torch_adam(max_norm, warmup):
    """Steps alternate above / below the clip; the third step's gradient holds an Inf: skipped, only counters[2] moves."""
    n, base_lr, d_model, factor, betas, eps, wd = 1025, 1e-3, 256.0, 1.0, (0.9, 0.98), 1e-9, 1e-4
    f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))               # noqa: E731  the kernel's scalar operands
    g = _g(5)
    p0 = torch.randn(n, generator=g, dtype=F64)
    pr = p0.clone().requires_grad_()
    opt = torch.optim.Adam([pr], lr=f32(base_lr), betas=(f32(betas[0]), f32(betas[1])), eps=f32(eps), weight_decay=f32(wd))
    p, m, v = p0.clone(), torch.zeros(n, dtype=F64), torch.zeros(n, dtype=F64)
    counters = [0, 2, 0]
    taken = 0
    for step in range(1, 6):
        gr = torch.randn(n, generator=g, dtype=F64) * (1.0 if step % 2 else 1e-3)
        if step == 3:
            gr[n // 3] = math.inf
        out = ref.adam_step(p, gr, m, v, float((gr * gr).sum()), counters, max_norm, base_lr, d_model, warmup, factor,
                            betas[0], betas[1], eps, wd)
        if step == 3:
            assert out[3] == [counters[0], counters[1], counters[2] + 1] and out[4] is None
            assert torch.equal(out[0], p) and torch.equal(out[1], m) and torch.equal(out[2], v)
            counters = out[3]
            continue
        taken += 1
        lr = ref.transformer_lr(counters[1] + 1, d_model, warmup, factor) if warmup > 0 else f32(base_lr)
        opt.param_groups[0]['lr'] = lr
        pr.grad = gr.clone()
        if max_norm > 0:
            torch.nn.utils.clip_grad_norm_([pr], f32(max_norm))
        opt.step()
        p, m, v, counters, hyper = out
        assert counters == [taken, taken + 2, 1 if step > 3 else 0]
        assert hyper[0] == pytest.approx(lr, rel=1e-15) and hyper[3] == 1.0
        assert hyper[1] == pytest.approx(1 - f32(betas[0]) ** taken, rel=1e-15)
        st = opt.state[pr]
        _close(p, pr.detach(), 1e-13)
        _close(m, st['exp_avg'], 1e-13)
        _close(v, st['exp_avg_sq'], 1e-13)
    assert float((p - p0).abs().max()) > 1e-6


def test_spec_augment_zero_pattern():
    B, T, Fb = 2, 9, 11
    x = torch.arange(1, B * T * Fb + 1, dtype=F64).view(B, T, Fb)
    bands = torch.tensor([[2, 3, 9, 5, 4, 0, 7, 4],                 # f [2, 5), f [9, 11) past the edge; t empty, t [7, 9)
                          [0, 0, 3, 4, 1, 2, 2, 3]], dtype=torch.int32)   # f empty, f [3, 7); t [1, 3) and [2, 5) overlap
    got = ref.spec_augment(x, bands, 2, 2)
    want = x.clone()
    for b, row in enumerate(bands.tolist()):
        for t in range(T):
            for f in range(Fb):
                kill = any(row[2 * j] <= f < row[2 * j] + row[2 * j + 1] for j in range(2))
                kill |= any(row[4 + 2 * j] <= t < row[4 + 2 * j] + row[5 + 2 * j] for j in range(2))
                if kill:
                    want[b, t, f] = 0.0
    assert torch.equal(got, want)
    # nt = 0 / nf = 0: the frequency bands alone, then the time bands alone, make up the same pattern
    both = ref.spec_augment(ref.spec_augment(x, bands[:, :4], 2, 0), bands[:, 4:], 0, 2)
    assert torch.equal(both, want)
    assert torch.equal(ref.spec_augment(x, torch.zeros(B, 0, dtype=torch.int32), 0, 0), x)


# ------------------------------------------------------------------------------------------------ Conformer conv module
def _conv_autograd(x, lens, w, wb, gamma, beta, rm, rv, nbt, dy, B, T):
    """nn.Conv1d (depthwise) + nn.BatchNorm1d in train() + swish on the masked input, in float64, with autograd."""
    d, k = w.shape
    conv = torch.nn.Conv1d(d, d, k, padding=(k - 1) // 2, groups=d, bias=wb is not None).double()
    bn = torch.nn.BatchNorm1d(d, momentum=float(torch.tensor(0.1, dtype=torch.float32)), eps=1e-5).double().train()
    with torch.no_grad():
        conv.weight.copy_(w.to(F64).unsqueeze(1))
        if wb is not None:
            conv.bias.copy_(wb.to(F64))
        bn.weight.copy_(gamma.to(F64))
        bn.bias.copy_(beta.to(F64))
        bn.running_mean.copy_(rm.to(F64))
        bn.running_var.copy_(rv.to(F64))
        bn.num_batches_tracked.fill_(int(nbt))
    mask = ref.frame_mask(lens, B, T)
    X = x.to(F64).view(B, T, d).clone().requires_grad_()
    A = bn(conv((X * mask[..., None]).transpose(1, 2)))
    out = (A * torch.sigmoid(A)).transpose(1, 2) * mask[..., None]
    out.backward(dy.to(F64).view(B, T, d))
    return out.detach().reshape(B * T, d), X.grad.reshape(B * T, d), conv, bn


@pytest.mark.parametrize('B,T,d,k,lens,bias', [
    (3, 13, 16, 5, [13, 8, 3], True),
    (2, 4, 8, 7, [4, 2], True),            # k > T
    (3, 6, 24, 1, [6, 0, 2], False),       # k = 1, an utterance of length 0, no conv bias
    (4, 1, 8, 3, [1, 0, 1, 1], True),      # T = 1
    (2, 5, 8, 3, [9, 6], True),            # lengths above T: every frame valid
])
def test_conv_module_matches_conv1d_batchnorm_autograd(B, T, d, k, lens, bias):
    g = _g(B * 100 + T * 10 + k)
    lens = torch.tensor(lens, dtype=torch.int32)
    x = torch.randn(B * T, d, generator=g, dtype=F64)
    w = 0.4 * torch.randn(d, k, generator=g, dtype=F64)
    wb = 3.0 + 0.2 * torch.randn(d, generator=g, dtype=F64) if bias else None
    gamma, beta = 1 + 0.2 * torch.randn(d, generator=g, dtype=F64), 0.2 * torch.randn(d, generator=g, dtype=F64)
    rm, rv = 0.1 * torch.randn(d, generator=g, dtype=F64), 1 + torch.rand(d, generator=g, dtype=F64)
    dy = torch.randn(B * T, d, generator=g, dtype=F64)
    out, dx, conv, bn = _conv_autograd(x, lens, w, wb, gamma, beta, rm, rv, 5, dy, B, T)
    fw = ref.conv_module_train(x, lens, w, wb, gamma, beta, rm, rv, 5, B, T)
    _close(fw['out'], out, 1e-11)
    _close(fw['running_mean'], bn.running_mean)
    _close(fw['running_var'], bn.running_var)
    assert fw['num_batches'] == int(bn.num_batches_tracked) == 6
    for kw in (dict(wb=wb), dict(c=fw['c'], mean=fw['mean'], invstd=fw['invstd'])):
        bw = ref.conv_module_bwd(dy, x, lens, w, gamma, beta, B, T, **kw)
        _close(bw['dx'], dx, 1e-10)
        _close(bw['dw'], conv.weight.grad.squeeze(1), 1e-10)
        if bias:
            _close(bw['dwb'], conv.bias.grad, 1e-10)
        _close(bw['dgamma'], bn.weight.grad, 1e-10)
        _close(bw['dbeta'], bn.bias.grad, 1e-10)
    mask = ref.frame_mask(lens, B, T).view(-1)
    assert bool((fw['out'][~mask] == 0).all()) and bool((dx[~mask] == 0).all())
    if int(lens.min()) > T:                   # lengths above T are clamped: the same as every frame valid
        full = torch.full_like(lens, T)
        _close(ref.conv_module_train(x, full, w, wb, gamma, beta, rm, rv, 5, B, T)['out'], fw['out'], 0)


def test_conv_module_single_position():
    """B*T = 1 (nn.BatchNorm1d refuses it in train()): c is its own mean, the variance 0, the output swish(beta), and
    running_var takes the biased variance 0."""
    d = 8
    g = _g(7)
    x, w, wb = torch.randn(1, d, generator=g, dtype=F64), torch.randn(d, 3, generator=g, dtype=F64), torch.randn(d, generator=g, dtype=F64)
    gamma, beta = torch.randn(d, generator=g, dtype=F64), torch.randn(d, generator=g, dtype=F64)
    rm, rv = torch.randn(d, generator=g, dtype=F64), torch.rand(d, generator=g, dtype=F64)
    fw = ref.conv_module_train(x, torch.tensor([1], dtype=torch.int32), w, wb, gamma, beta, rm, rv, 0, 1, 1)
    _close(fw['c'], x * w[:, 1] + wb)
    _close(fw['out'], (beta * torch.sigmoid(beta))[None])
    _close(fw['running_var'], 0.9 * rv + 0.0, 1e-8)
    _close(fw['running_mean'], 0.9 * rm + 0.1 * fw['c'][0], 1e-8)
    bw = ref.conv_module_bwd(torch.randn(1, d, generator=g, dtype=F64), x, torch.tensor([1], dtype=torch.int32), w, gamma, beta,
                             1, 1, wb=wb)
    assert float(bw['dx'].abs().max()) == 0.0 and float(bw['dw'].abs().max()) == 0.0 and float(bw['dgamma'].abs().max()) == 0.0
