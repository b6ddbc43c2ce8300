"""The training step's kernels one at a time, against plain fp32 / fp64 torch versions of the same operation on the same
bf16-rounded operands (only accumulation order and output rounding may differ; where a kernel only moves data or does one
multiply, equality is exact):
  * conv front-end backward: im2col, col2im + ReLU', the conv1 weight gradient, and the whole chain against autograd;
  * residual dropout: the mask drawn in the GEMM epilogue, its replay in the backward, and the mask's properties;
  * gradient accumulation (`accumulate=True` / a pre-filled `grad_sink`), op by op and through a whole training step;
  * the device-scheduled Adam step (Noam LR and step counters on the device, skip on a non-finite norm).
The attention backward is tested element by element in tests/test_gpu_attention.py.
Run with -m gpu on an H100."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops, train
    DEV = torch.device('cuda:0')

from tests.test_gpu_ops import _rnd, _report
from tests.test_gpu_train import _params, _build, _batch

BF = torch.bfloat16
torch.backends.cudnn.allow_tf32 = False        # the fp32 checkers must not silently run in TF32
torch.backends.cuda.matmul.allow_tf32 = False


def _bf(*shape, scale=1.0, seed=0):
    return _rnd(*shape, scale=scale, seed=seed).to(BF)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


# ------------------------------------------------------------------------------------------------ conv front-end backward
# (B, T, F, C1p, ragged lengths or None); C2 = 128 throughout
CONV_GEOMS = {
    'bench': (32, 1000, 80, 64, None),                 # bench.py --workload train: B 32 x 1000 frames
    'smallest_T': (2, 7, 80, 64, None),                # T2 = 1
    'T8_F40': (3, 8, 40, 128, None),
    'T91_F83': (3, 91, 83, 64, None),
    'T91_F81_C192': (2, 91, 81, 192, None),            # F1 = 41 is odd: conv2 reads the zero column f1 = F1
    'ragged': (4, 200, 80, 64, (200, 131, 77, 160)),
    'C256': (2, 120, 80, 256, None),                   # conformer_baseline mid_channel
}


def _ulp_bf16(x):
    """Spacing of bf16 numbers at |x| (x fp32)."""
    _, e = torch.frexp(x)
    return torch.ldexp(torch.ones_like(x), e - 8)


@pytest.mark.parametrize('geom', list(CONV_GEOMS))
def test_conv_frontend_backward(geom):
    B, T, Fq, C, lens = CONV_GEOMS[geom]
    C2 = 128
    T1, F1, T2, F2 = ops.conv_geometry(T, Fq)
    T1p, F1p = 2 * (T2 + 1), 2 * F2
    x = _rnd(B, T, Fq, seed=1)
    if lens is not None:
        x = x * (torch.arange(T, device=DEV)[None] < torch.tensor(lens, device=DEV)[:, None]).unsqueeze(2)
    w1, b1 = _rnd(C, 1, 3, 3, scale=0.4, seed=2), _rnd(C, scale=0.1, seed=3)
    w2 = _bf(C2, 9 * C, scale=(9 * C) ** -0.5, seed=4)            # [C2, (kh*3+kw)*C + c]
    b2 = _rnd(C2, scale=0.05, seed=5)
    h1 = ops.conv1_relu(x, w1, b1)
    assert h1.shape == (B, T1p, F1p, C)

    # im2col: a pure gather, bit for bit
    col = ops.conv_im2col(h1, B, T, Fq, C)
    hp = F.pad(h1, (0, 0, 1, 0))                                   # f = -1 is the zero padding
    ref_col = torch.stack([hp[:, kh:kh + 2 * T2:2, kw:kw + 2 * F2:2, :] for kh in range(3) for kw in range(3)], 3)
    assert torch.equal(col, ref_col.reshape(B * T2 * F2, 9 * C)), f'{geom}: im2col differs from the gather'

    # col2im + ReLU': fp32 scatter-add of the taps, within one bf16 ulp; positions outside [0,T1) x [0,F1) exactly zero
    dcol = _bf(B * T2 * F2, 9 * C, seed=6)
    got = ops.conv_col2im_relu(dcol, h1, B, T, Fq, C).float()
    acc = torch.zeros(B, T1p, F1p + 1, C, device=DEV)
    dv = dcol.float().view(B, T2, F2, 9, C)
    for kh in range(3):
        for kw in range(3):
            acc[:, kh:kh + 2 * T2:2, kw:kw + 2 * F2:2, :] += dv[:, :, :, kh * 3 + kw, :]
    ref = acc[:, :, 1:, :].clone()
    ref[:, T1:] = 0.0
    ref[:, :, F1:] = 0.0
    ref = ref * (h1 > 0).float()
    if T1 < T1p:
        assert torch.equal(got[:, T1:], torch.zeros_like(got[:, T1:])), f'{geom}: rows t1 >= T1 must be written as zero'
    if F1 < F1p:
        assert torch.equal(got[:, :, F1:], torch.zeros_like(got[:, :, F1:])), f'{geom}: columns f1 >= F1 must be written as zero'
    err = (got - ref).abs()
    n_off = int((err > 0).sum())
    worst_ulps = float((err / _ulp_bf16(ref)).max())
    print(f'col2im {geom}: {n_off} of {ref.numel()} elements not bit-equal to the rounded fp32 sum, worst {worst_ulps:.2f} ulp '
          f'(limit 1)')
    assert worst_ulps <= 1.0

    # conv1 weight / bias gradient against an fp64 sum over the same bf16 dpre1 (its padding positions hold noise that
    # the kernel must not read)
    dpre1 = _bf(B, T1p, F1p, C, seed=7)
    g1 = ops.conv1_wgrad(dpre1, x, B, T, Fq, C)
    xp = F.pad(x.double(), (1, 1))
    d = dpre1[:, :T1, :F1, :].double()
    taps = [torch.einsum('btfc,btf->c', d, xp[:, kh:kh + 2 * T1 - 1:2, kw:kw + 2 * F1 - 1:2]) for kh in range(3) for kw in range(3)]
    ref_g1 = torch.stack(taps + [d.sum((0, 1, 2))], 1)
    r = _rel(g1, ref_g1)
    print(f'conv1_wgrad {geom}: rel_l2 {r:.2e} (limit 1e-5); bias rel_l2 {_rel(g1[:, 9], ref_g1[:, 9]):.2e}')
    assert r <= 1e-5 and _rel(g1[:, 9], ref_g1[:, 9]) <= 1e-5

    # the whole front-end backward, chained as train.forward_backward does, against autograd through the fp32 convolutions
    # on the same weights; h1 is rounded to bf16 straight-through as the kernel stores it, so both sides take the same
    # ReLU branches
    G = _bf(B, C2, T2, F2, seed=8).float()
    w1r, b1r = w1.clone().requires_grad_(True), b1.clone().requires_grad_(True)
    w2r = w2.float().view(C2, 3, 3, C).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    b2r = b2.clone().requires_grad_(True)
    h1r = torch.relu(F.conv2d(x[:, None], w1r, b1r, stride=2, padding=(0, 1)))
    h1r = h1r + (h1r.to(BF).float() - h1r).detach()
    h2r = torch.relu(F.conv2d(h1r, w2r, b2r, stride=2, padding=(0, 1)))
    (h2r * G).sum().backward()
    h2 = ops.conv2_relu(h1, w2, b2, B, T, Fq)                                          # [B*T2, F2*C2]
    dpre2 = ops.relu_bwd(G.permute(0, 2, 3, 1).reshape(B * T2, F2 * C2).to(BF).contiguous(), h2).view(B * T2 * F2, C2)
    dw2 = ops.linear_wgrad(dpre2, col)
    dcol = ops.linear(dpre2, w2.t().contiguous())
    dpre1 = ops.conv_col2im_relu(dcol, h1, B, T, Fq, C)
    g1 = ops.conv1_wgrad(dpre1, x, B, T, Fq, C)
    r_w1 = _rel(g1[:, :9].reshape(C, 1, 3, 3), w1r.grad)
    r_b1 = _rel(g1[:, 9], b1r.grad)
    r_w2 = _rel(dw2.view(C2, 3, 3, C).permute(0, 3, 1, 2), w2r.grad)
    print(f'front-end backward {geom}: dW1 {r_w1:.2e} db1 {r_b1:.2e} dW2 {r_w2:.2e} (limit 5e-3)')
    assert r_w1 <= 5e-3 and r_b1 <= 5e-3 and r_w2 <= 5e-3


# ------------------------------------------------------------------------------------------------ residual dropout
def _keep_np(seed, site, M, N, p):
    """dropout.cuh's keep(seed, site, row, col) restated in numpy (uint32 arithmetic in uint64 with explicit wrap)."""
    m32 = 0xFFFFFFFF
    t = float(np.float32(p)) * 4294967296.0
    thresh = 0 if p <= 0 else (m32 if t >= 4294967295.0 else int(t))
    rows = np.arange(M, dtype=np.uint64)[:, None]
    cols = np.arange(N, dtype=np.uint64)[None, :]
    h = np.uint64((seed * 0x9E3779B1 + site * 0x85EBCA77 + 0x27D4EB2F) & m32)
    h = h ^ ((rows * 0xC2B2AE3D) & m32)
    h = ((h ^ (h >> 16)) * 0x7FEB352D) & m32
    h = h ^ ((cols * 0x165667B1) & m32)
    h = ((h ^ (h >> 15)) * 0x846CA68B) & m32
    h = h ^ (h >> 16)
    return torch.from_numpy((h >= thresh).astype(np.uint8))


def _scale32(p):
    """1 / (1 - p) as the kernels compute it, in fp32."""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))


# (M, K, p, alpha): M = 100 takes 64-wide N tiles, M = 7968 128-wide ones (choose_bn); neither is a multiple of 128
@pytest.mark.parametrize('M,K,p,alpha', [(100, 256, 0.1, 1.0), (100, 256, 0.5, 0.5), (7968, 256, 0.1, 1.0), (7968, 2048, 0.5, 0.5),
                                         (1000, 256, 0.1, 0.5)])
def test_linear_dropout_resid(M, K, p, alpha):
    N, site = 256, 1004
    seed = torch.tensor([20240917], dtype=torch.int32, device=DEV)
    a, w = _bf(M, K, seed=30), _bf(N, K, scale=K ** -0.5, seed=31)
    b, resid = _rnd(N, scale=0.1, seed=32), _bf(M, N, seed=33)
    out = ops.linear_dropout_resid(a, w, b, resid, p, seed, site, alpha=alpha)
    mask = ops.dropout_mask(M, N, p, seed, site)
    assert torch.equal(mask.cpu(), _keep_np(20240917, site, M, N, p)), 'exported mask differs from dropout.cuh keep()'
    y = a.float() @ w.float().t() + b
    ref = resid.float() + alpha * (mask.float() * y * _scale32(p))
    dropped = mask == 0
    # a dropped element is resid + alpha * 0: the residual itself, bit for bit -- so the epilogue's mask is the replayed one
    assert torch.equal(out[dropped], resid[dropped]), 'the GEMM epilogue dropped other elements than the replayed mask'
    print(f'linear_dropout_resid M={M} K={K} p={p} alpha={alpha}: ' + _report('out', out, ref, 4e-3)
          + f'; dropped {float(dropped.float().mean()):.4f}')


@pytest.mark.parametrize('M,N,p', [(7968, 256, 0.1), (100, 256, 0.5), (37, 2048, 0.1)])
def test_dropout_bwd_is_one_multiply(M, N, p):
    seed = torch.tensor([99], dtype=torch.int32, device=DEV)
    dy = _bf(M, N, seed=34)
    got = ops.dropout_bwd(dy, p, seed, 7)
    mask = ops.dropout_mask(M, N, p, seed, 7)
    assert torch.equal(mask.cpu(), _keep_np(99, 7, M, N, p))
    ref = (dy.float() * mask.float() * _scale32(p)).to(BF)
    assert torch.equal(got, ref), 'dropout_bwd must be exactly one fp32 multiply and one rounding'


def test_dropout_mask_properties():
    seed = torch.tensor([12345], dtype=torch.int32, device=DEV)
    N = 256
    for p in (0.1, 0.5):
        m_big = ops.dropout_mask(7968, N, p, seed, 3)
        n = m_big.numel()
        keep = float(m_big.float().mean())
        bound = 6.0 * math.sqrt(p * (1 - p) / n)
        print(f'dropout p={p}: keep rate {keep:.5f}, expected {1 - p} +- {bound:.5f} (6 sigma)')
        assert abs(keep - (1 - p)) <= bound
        # row r's mask does not depend on how many rows the launch has
        assert torch.equal(ops.dropout_mask(100, N, p, seed, 3), m_big[:100])
        assert not torch.equal(ops.dropout_mask(7968, N, p, seed, 4), m_big), 'different sites must draw different masks'
        seed2 = torch.tensor([12346], dtype=torch.int32, device=DEV)
        assert not torch.equal(ops.dropout_mask(7968, N, p, seed2, 3), m_big), 'different seeds must draw different masks'
    assert bool((ops.dropout_mask(1000, N, 0.0, seed, 3) == 1).all()), 'p = 0 keeps everything'
    dy = _bf(1000, N, seed=35)
    assert torch.equal(ops.dropout_bwd(dy, 0.0, seed, 3), dy)


# ------------------------------------------------------------------------------------------------ accumulation, op level
# (M, N, K): split-K > 1 / split-K = 1 with few k-blocks / split-K = 1 with many tiles (the output layer's shape)
@pytest.mark.parametrize('M,N,K', [(7968, 768, 256), (64, 256, 256), (960, 4240, 256)])
@pytest.mark.parametrize('strided', [False, True])
def test_linear_wgrad_accumulate_and_overwrite(M, N, K, strided):
    dy, x = _bf(M, N, scale=0.5, seed=40), _bf(M, K, seed=41)
    ref = (dy.double().t() @ x.double())
    pad = 16 if strided else 0

    def out_buffer(fill):
        big = torch.full((N, K + pad), float('nan'), device=DEV)
        big[:, pad // 2:pad // 2 + K] = fill
        return big, big[:, pad // 2:pad // 2 + K]

    s0 = _rnd(N, K, scale=float(ref.std()), seed=42)
    big, out = out_buffer(s0)
    ops.linear_wgrad(dy, x, out=out, accumulate=True)
    r_acc = _rel(out - s0, ref)
    big2, out2 = out_buffer(float('nan'))
    ops.linear_wgrad(dy, x, out=out2, accumulate=False)
    r_new = _rel(out2, ref)
    print(f'wgrad M={M} N={N} K={K} pitch {K + pad}: accumulate rel_l2 {r_acc:.2e}, overwrite rel_l2 {r_new:.2e} (limit 2e-3)')
    assert torch.isfinite(out2).all(), 'without accumulate every element must be written'
    assert r_acc < 2e-3 and r_new < 2e-3
    if pad:    # the columns around the view stay untouched
        assert torch.isnan(big[:, :pad // 2]).all() and torch.isnan(big[:, pad // 2 + K:]).all()
        assert torch.isnan(big2[:, :pad // 2]).all() and torch.isnan(big2[:, pad // 2 + K:]).all()


@pytest.mark.parametrize('M,N', [(7968, 4096), (100, 256), (33, 4240)])
def test_colsum_accumulate_and_overwrite(M, N):
    x = _bf(M, N, seed=43)
    ref = x.double().sum(0)
    s0 = _rnd(N, scale=float(ref.std()), seed=44)
    out = s0.clone()
    ops.colsum(x, out=out, accumulate=True)
    out2 = torch.full((N,), float('nan'), device=DEV)
    ops.colsum(x, out=out2, accumulate=False)
    print(f'colsum M={M} N={N}: ' + _report('accumulate', out - s0, ref, 1e-5) + '; ' + _report('overwrite', out2, ref, 1e-5))


@pytest.mark.parametrize('M,N', [(7968, 256), (37, 256), (500, 64)])
def test_layernorm_bwd_accumulate_and_overwrite(M, N):
    z, dy = _bf(M, N, scale=2.0, seed=45), _bf(M, N, seed=46)
    gamma = _rnd(N, scale=0.5, seed=47) + 1.0
    zd = z.double()
    xh = (zd - zd.mean(1, keepdim=True)) / torch.sqrt(zd.var(1, unbiased=False, keepdim=True) + 1e-5)
    ref_g, ref_b = (dy.double() * xh).sum(0), dy.double().sum(0)
    sg, sb = _rnd(N, scale=float(ref_g.std()), seed=48), _rnd(N, scale=float(ref_b.std()), seed=49)
    dg, db = sg.clone(), sb.clone()
    dz, _, _ = ops.layernorm_bwd(dy, z, gamma, dgamma=dg, dbeta=db, accumulate=True)
    nan = torch.full((N,), float('nan'), device=DEV)
    dz2, dg2, db2 = ops.layernorm_bwd(dy, z, gamma, dgamma=nan.clone(), dbeta=nan.clone(), accumulate=False)
    assert torch.equal(dz, dz2), 'dz must not depend on the accumulate flag'
    print(f'LN bwd M={M} N={N}: ' + '; '.join([_report('dgamma acc', dg - sg, ref_g, 1e-4), _report('dbeta acc', db - sb, ref_b, 1e-5),
                                              _report('dgamma new', dg2, ref_g, 1e-4), _report('dbeta new', db2, ref_b, 1e-5)]))


@pytest.mark.parametrize('n', [30_000_000, 1_000_003])
def test_sumsq_adds_to_the_running_value(n):
    g = _rnd(n, scale=0.01, seed=50)
    ref = float((g.double() ** 2).sum())
    buf = torch.tensor([0.75 * ref], device=DEV)
    ops.sumsq(g, buf, zero_first=False)
    r_acc = abs(float(buf) - 1.75 * ref) / (1.75 * ref)
    buf2 = torch.tensor([float('nan')], device=DEV)
    ops.sumsq(g, buf2, zero_first=True)
    r_new = abs(float(buf2) - ref) / ref
    print(f'sumsq n={n}: accumulate rel {r_acc:.2e}, zero-first rel {r_new:.2e} (limit 1e-5)')
    assert r_acc <= 1e-5 and r_new <= 1e-5


def test_embed_bwd_repeats_and_out_of_range_ids():
    V, d, scale = 50, 256, 16.0
    g = torch.Generator().manual_seed(51)
    tok = torch.randint(0, V, (400,), generator=g)
    tok[::7] = 3                                       # a heavily repeated id
    tok[5], tok[77], tok[200] = -1, V, -1              # skipped by the kernel
    dx = _bf(400, d, seed=52)
    big = _rnd(V + 2, d, seed=53)                      # guard rows 0 and V + 1 sit where ids -1 and V would land
    before = big.clone()
    ops.embed_bwd(tok.to(DEV), dx, big[1:V + 1], scale)
    ok = (tok >= 0) & (tok < V)
    ref = before[1:V + 1].double().index_add_(0, tok[ok].to(DEV), dx.double()[ok.to(DEV)] * scale)
    assert torch.equal(big[0], before[0]) and torch.equal(big[V + 1], before[V + 1]), 'out-of-range ids must be skipped'
    untouched = torch.ones(V, dtype=torch.bool)
    untouched[tok[ok]] = False
    assert torch.equal(big[1:V + 1][untouched.to(DEV)], before[1:V + 1][untouched.to(DEV)])
    print('embed_bwd: ' + _report('dE', big[1:V + 1] - before[1:V + 1], ref - before[1:V + 1].double(), 1e-5))


# ------------------------------------------------------------------------------------------------ accumulation, whole step
@pytest.mark.parametrize('tied', [True, False])
@pytest.mark.parametrize('rdrop', [0.0, 0.1])
@pytest.mark.parametrize('ctc', [0.0, 0.3])
def test_grad_sink_accumulates_every_gradient(tied, rdrop, ctc):
    """sink - S0 == 0.5 g_plain for every parameter: the scale is exact in bf16, so only the order of fp32 atomics differs;
    a kernel that ignored its accumulate flag would be off by about 100 %."""
    params = _params(n_enc=2, n_dec=1, tied=tied)
    for part in ('encoder', 'decoder'):
        params[part]['residual_dropout'] = rdrop
    kw = {}
    if ctc:
        params['ctc_weight'] = ctc
        params['encoder_output_size'] = 256
    model, _ = _build(params)
    model.train()
    x, mask, tgt = _batch()
    if ctc:
        kw['truth_length'] = torch.tensor([int((tgt[b, 1:] != 0).sum()) for b in range(tgt.shape[0])], dtype=torch.int32).to(DEV)
    seed = torch.tensor([4242], dtype=torch.int32, device=DEV)
    args = (model, x.to(DEV), mask.to(DEV), tgt.to(DEV))
    with torch.no_grad():
        loss, g = train.forward_backward(*args, drop_seed=seed, **kw)
        g = {n: t.clone() for n, t in g.items()}
        names = [n for n, _ in model.named_parameters()]
        # FusedTrainer's own sink (views into its flat fp32 buffer) and bf16 weight views, as in its micro-step
        tr = train.FusedTrainer(model, use_graph=False)
        sink, s0 = tr.sink, {}
        for i, n in enumerate(names):
            sink[n].copy_(_rnd(*sink[n].shape, seed=100 + i) * (float(g[n].float().pow(2).mean().sqrt()) + 1e-6))
            s0[n] = sink[n].clone()
        tr.flat_bf16.copy_(tr.flat_p)
        loss2, _ = train.forward_backward(*args, grad_sink=sink, grad_scale=0.5, bf16_of=tr._bf16_of, drop_seed=seed, **kw)
    assert abs(float(loss2) - float(loss)) <= 1e-6 * abs(float(loss))
    worst = sorted(((_rel(sink[n] - s0[n], 0.5 * g[n]), n) for n in names), reverse=True)
    print(f'grad_sink tied={tied} residual_dropout={rdrop} ctc={ctc}: worst ' + ', '.join(f'{n} {r:.2e}' for r, n in worst[:3])
          + ' (limit 1e-5)')
    assert set(names) == set(g)
    assert worst[0][0] <= 1e-5, worst[:3]


# ------------------------------------------------------------------------------------------------ device-scheduled Adam
BETAS, EPS, WD, MAX_NORM, D_MODEL = (0.9, 0.98), 1e-9, 1e-6, 5.0, 256


def _adam_pair(n, seed):
    p0 = _rnd(n, seed=seed)
    pr = p0.clone().requires_grad_(True)
    return p0.clone(), pr, torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)


def _sched_step(p, g, m, v, ss, counters, hyper, base_lr, warmup):
    ops.sumsq(g, ss)
    ops.adam_step_sched(p, g, m, v, ss, MAX_NORM, base_lr, D_MODEL, warmup, 1.0, BETAS, EPS, WD, counters, hyper)


# warmup 4: lr(3), lr(4) on the warm-up ramp, lr(5), lr(6) on the decay (at warmup 12000 the first updates are ~1e-7,
# below what rtol 1e-5 on the weights can see); warmup 0: constant LR
@pytest.mark.parametrize('warmup', [4, 0])
def test_adam_step_sched_matches_torch_adam(warmup):
    """clip_grad_norm_ + torch.optim.Adam with lr = transformer_lr(global step), counters starting at [0, 2, 0] as
    FusedTrainer's (first update at lr(3)).  Steps alternate above / below the clip."""
    n, base_lr = 100003, 1e-3
    p, pr, m, v = _adam_pair(n, 60)
    opt = torch.optim.Adam([pr], lr=base_lr, betas=BETAS, eps=EPS, weight_decay=WD)
    counters = torch.tensor([0, 2, 0], dtype=torch.int32, device=DEV)
    hyper, ss = torch.zeros(4, device=DEV), torch.zeros(1, device=DEV)
    p0 = p.clone()
    for step in range(1, 5):
        gr = _rnd(n, scale=0.1 if step % 2 else 1e-3, seed=60 + step)        # norm ~32 (clipped to 5) / ~0.3 (not clipped)
        lr = train.transformer_lr(step + 2, D_MODEL, warmup) if warmup else base_lr
        opt.param_groups[0]['lr'] = lr
        pr.grad = gr.clone()
        norm = float(torch.nn.utils.clip_grad_norm_([pr], MAX_NORM))
        opt.step()
        _sched_step(p, gr, m, v, ss, counters, hyper, base_lr, warmup)
        assert counters.tolist() == [step, step + 2, 0]
        assert abs(float(hyper[0]) - lr) <= 1e-6 * lr
        err = float((p - pr.detach()).abs().max())
        print(f'adam sched warmup={warmup} step {step}: grad norm {norm:.3g}, lr {lr:.4g}, max abs diff {err:.2e}')
        torch.testing.assert_close(p, pr.detach(), rtol=1e-5, atol=1e-6)
    assert float((p - p0).abs().max()) > 1e-3, 'the updates must be large enough for the comparison to see them'


def test_adam_step_sched_skips_a_non_finite_step():
    """trainer.py:229-233: a NaN gradient norm skips the optimizer AND the scheduler step; only the skip count advances."""
    n, warmup = 5000, 4
    p, pr, m, v = _adam_pair(n, 70)
    p0 = p.clone()
    opt = torch.optim.Adam([pr], lr=1e-3, betas=BETAS, eps=EPS, weight_decay=WD)
    counters = torch.tensor([0, 2, 0], dtype=torch.int32, device=DEV)
    hyper, ss = torch.zeros(4, device=DEV), torch.zeros(1, device=DEV)
    lrs = {1: 3, 2: 4, 4: 5}
    for step in (1, 2, 3, 4):
        gr = _rnd(n, scale=0.1, seed=70 + step)
        if step == 3:
            gr[n // 2] = float('nan')
            before = (p.clone(), m.clone(), v.clone())
            _sched_step(p, gr, m, v, ss, counters, hyper, 1e-3, warmup)
            assert torch.equal(p, before[0]) and torch.equal(m, before[1]) and torch.equal(v, before[2])
            assert counters.tolist() == [2, 4, 1], counters.tolist()
            continue
        opt.param_groups[0]['lr'] = train.transformer_lr(lrs[step], D_MODEL, warmup)
        pr.grad = gr.clone()
        torch.nn.utils.clip_grad_norm_([pr], MAX_NORM)
        opt.step()                         # torch's 3rd step: bias correction t = 3
        _sched_step(p, gr, m, v, ss, counters, hyper, 1e-3, warmup)
        torch.testing.assert_close(p, pr.detach(), rtol=1e-5, atol=1e-6)
    assert float((p - p0).abs().max()) > 1e-2, 'the updates must be large enough for the comparison to see them'
    assert counters.tolist() == [3, 5, 1]
    assert abs(float(hyper[0]) - train.transformer_lr(5, D_MODEL, warmup)) <= 1e-6 * float(hyper[0])


def test_fused_trainer_skips_a_step_on_nan_input():
    params = _params(n_enc=1, n_dec=1)
    model, _ = _build(params)
    model.train()
    tr = train.FusedTrainer(model, accum_steps=1, use_graph=False)
    x, mask, tgt = _batch()
    bad = x.clone()
    bad[1, 17, 5] = float('nan')       # reaches the gradient norm through the conv1 weight gradient (x enters it directly)
    w0, m0, v0 = tr.flat_p.clone(), tr.m.clone(), tr.v.clone()
    loss = tr.step(bad.to(DEV), mask.to(DEV), tgt.to(DEV))
    torch.cuda.synchronize()
    print(f'FusedTrainer NaN step: loss {float(loss)}, counters {tr.counters.tolist()}')
    assert torch.equal(tr.flat_p, w0) and torch.equal(tr.m, m0) and torch.equal(tr.v, v0)
    assert tr.skipped_steps == 1 and tr.global_step == 2 and tr.opt_steps == 0
    assert float(tr.flat_g.abs().max()) == 0.0, 'the gradient buffer is cleared for the next step'
    tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV))                  # the next finite step is the first update, at lr(3)
    assert tr.skipped_steps == 1 and tr.global_step == 3 and tr.opt_steps == 1
    assert abs(tr.lr() - train.transformer_lr(3, 256, 12000)) < 1e-12
    assert not torch.equal(tr.flat_p, w0)
