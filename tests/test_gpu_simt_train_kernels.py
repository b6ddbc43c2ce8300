"""The SIMT kernels of the training step at every configuration they accept, against the float64 restatements of
tests/simt_train_kernels_ref.py on the same bf16 / f32 operands:
  * otb_layernorm_bwd: N 8 to 256 (idle lanes past N), row pitches wider than N, more rows than one grid pass, rows whose
    mean is large against their spread, dgamma / dbeta zeroed by the launcher or accumulated;
  * otb_glu_fwd / otb_glu_bwd;
  * otb_dropout_bwd with one and two masks (both template instances) and p = 0 < p2, its masks against ops.dropout_mask and
    against the masks the forward epilogue (otb_linear_dropout_resid) drew; otb_dropout_add with row_len / row_period;
  * otb_embed_bwd at d 8 to 520 (the lane loop and its tail), repeated and out-of-range ids;
  * otb_adam_step_sched at n 1 to past one grid pass, clip on / off / max_norm 0, weight decay, the skipped step, and the
    gradient-noise instance with an empty noise mask;
  * otb_spec_augment with bands past the edge, empty and overlapping bands, nf = 0 and nt = 0;
  * otb_conformer_conv_train / _bwd at d not a multiple of 256, k = 1 and k > T, T = 1, B*T = 1, an utterance of length 0, a
    batch past the reduction grid's cap, no conv bias, accumulate, channels with a mean far above their spread, and lengths
    above T.
Bounds follow from the output type: a bf16 output is within one bf16 ulp of the float64 value plus the error of the f32
arithmetic before the rounding; an f32 output is within c * u * scale, u = 2^-24, the scale taken from the row or column.
Every case prints its measured error.  Outputs sit in NaN-filled buffers with wider pitches and extra rows; the canaries
must survive.  Run with -m gpu on an H100."""
import ctypes
import math

import pytest
import torch

from tests import simt_train_kernels_ref as ref

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import _lib, ops
    DEV = torch.device('cuda:0')

BF = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
U = 2.0 ** -24           # f32 unit roundoff
NAN = float('nan')


def _f32(v):
    return float(torch.tensor(v, dtype=F32))


def _rnd(*shape, scale=1.0, seed=0, dtype=F32):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dtype)


def _canvas(rows, cols, dtype):
    return torch.full((rows, cols), NAN, dtype=dtype, device=DEV)


def _ulp(want):
    """Spacing of bf16 numbers at |want| (float64)."""
    _, e = torch.frexp(want.abs().clamp(min=2.0 ** -120))
    return torch.ldexp(torch.ones_like(want), e - 8)


def _check_bf16(name, got, want, abs_tol=0.0):
    """bf16 `got` within one bf16 ulp of the float64 `want`, plus abs_tol: the error of the f32 arithmetic before the final
    rounding (a float or a tensor broadcast against `want`)."""
    err = (got.double() - want).abs()
    ulp = _ulp(want)
    bound = ulp + abs_tol
    bad = (err > bound) | torch.isnan(got)
    if got.numel():
        over = ((err - ulp).clamp(min=0) / torch.as_tensor(abs_tol, dtype=F64, device=err.device).clamp(min=1e-300)).max().item()
        print(f'{name}: max |err| / ulp {(err / ulp).max().item():.3f}, max |err| / (ulp + abs) {(err / bound).max().item():.3f}, '
              f'max (|err| - ulp) / abs {over:.3g}')
    if bad.any():
        i = torch.nonzero(bad)[:6].tolist()
        raise AssertionError(f'{name}: {int(bad.sum())} elements off by more than one bf16 ulp + abs, first at {i}: '
                             f'got {[got[tuple(j)].item() for j in i]} want {[want[tuple(j)].item() for j in i]}')


def _check_f32(name, got, want, scale, c):
    """f32 `got` within c * u * scale of the float64 `want` (scale broadcast against `want`)."""
    assert not torch.isnan(got).any(), f'{name}: NaN in the output'
    ratio = (got.double() - want).abs() / (U * scale.expand_as(want).clamp(min=1e-300))
    worst = ratio.max().item() if ratio.numel() else 0.0
    print(f'{name}: max |err| / (u * scale) {worst:.2f} (bound {c})')
    assert worst <= c, f'{name}: error {worst:.2f} u * scale exceeds {c} at flat index {int(ratio.argmax())}'


def _nan_tail(t, name):
    assert bool(torch.isnan(t.float()).all()), f'{name}: a canary past the written area changed'


def _refused(fn, what):
    with pytest.raises(RuntimeError, match=what):
        fn()
    torch.cuda.synchronize()


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _seed(v):
    return torch.tensor([v], dtype=torch.int32, device=DEV)


# ------------------------------------------------------------------------------------------------ LayerNorm backward
LNB_C = 3.5          # dz, dgamma, dbeta: u * scale (see _lnb_scales); 2.19 measured on an H100 SXM (700 W)


def _layernorm_bwd(dy, lddy, z, ldz, gamma, dz, lddz, dg, db, eps, M, N, accumulate):
    _lib.check(_lib.lib().otb_layernorm_bwd(ops._p(dy), lddy, ops._p(z), ldz, ops._p(gamma), ops._p(dz), lddz, ops._p(dg),
                                            ops._p(db), eps, M, N, 1 if accumulate else 0, ops._stream()), 'otb_layernorm_bwd')


def _lnb_rows(M, N, seed):
    z = _rnd(M, N, scale=2.0, seed=seed) + _rnd(M, 1, scale=1.0, seed=seed + 1)
    if M >= 2:
        z[M - 1] = 256.0 + _rnd(N, scale=8.0, seed=seed + 2)          # mean 32 times the spread (bf16 steps of 2 there)
    if M >= 4:
        z[1] = 4096.0 + _rnd(N, scale=64.0, seed=seed + 3)
    return z.to(BF)


def _lnb_scales(dy, z, gamma, eps):
    """Per-row scale of dz and per-column scales of dgamma / dbeta: the f32 statistics are off by u * max|z| in the mean,
    which moves xhat by u * max|z| * rstd."""
    z, dy = z.double(), dy.double()
    mean = z.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((z - mean) ** 2).mean(-1, keepdim=True) + eps)
    xh = (z - mean) * rstd
    g = dy * gamma.double()
    cond = 1.0 + z.abs().amax(-1, keepdim=True) * rstd
    s_dz = rstd * (g.abs().amax(-1, keepdim=True) + g.abs().mean(-1, keepdim=True)
                   + xh.abs().amax(-1, keepdim=True) * (g * xh).abs().mean(-1, keepdim=True)) * cond
    return s_dz, (dy.abs() * (xh.abs() + z.abs() * rstd)).sum(0), dy.abs().sum(0)


@pytest.mark.parametrize('N', [8, 64, 136, 248, 256])
def test_layernorm_bwd(N):
    gamma = 1 + 0.3 * _rnd(N, seed=N)
    eps = _f32(1e-5)
    for M in (1, 7, 8, 9, 4 * _sms() * 8 + 37):                          # the last: more rows than one grid pass
        z, dy = _lnb_rows(M, N, seed=M), _rnd(M, N, seed=M + 7, dtype=BF)
        want_dz, want_dg, want_db = ref.layernorm_bwd(dy, z, gamma, eps)
        s_dz, s_dg, s_db = _lnb_scales(dy, z, gamma, eps)
        for lddy, ldz, lddz in ((N, N, N), (N + 16, N + 8, N + 24)):
            name = f'layernorm_bwd N={N} M={M} ld={lddy},{ldz},{lddz}'
            dyb, zb = _canvas(M, lddy, BF), _canvas(M, ldz, BF)       # NaN past column N: an idle lane must not read it
            dyb[:, :N], zb[:, :N] = dy, z
            dzb = _canvas(M + 1, lddz, BF)
            dg, db = torch.full((N + 8,), NAN, device=DEV), torch.full((N + 8,), NAN, device=DEV)
            _layernorm_bwd(dyb, lddy, zb, ldz, gamma, dzb, lddz, dg, db, eps, M, N, False)
            _check_bf16(f'{name} dz', dzb[:M, :N], want_dz, LNB_C * U * s_dz)
            _check_f32(f'{name} dgamma', dg[:N], want_dg, s_dg, LNB_C)
            _check_f32(f'{name} dbeta', db[:N], want_db, s_db, LNB_C)
            _nan_tail(dzb[:, N:], name), _nan_tail(dzb[M], name), _nan_tail(dg[N:], name), _nan_tail(db[N:], name)
            prev_g, prev_b = _rnd(N, seed=1), _rnd(N, seed=2)
            dg[:N], db[:N] = prev_g, prev_b
            _layernorm_bwd(dyb, lddy, zb, ldz, gamma, dzb, lddz, dg, db, eps, M, N, True)
            _check_f32(f'{name} dgamma accumulate', dg[:N], prev_g.double() + want_dg, s_dg + prev_g.double().abs(), LNB_C)
            _check_f32(f'{name} dbeta accumulate', db[:N], prev_b.double() + want_db, s_db + prev_b.double().abs(), LNB_C)
            _nan_tail(dg[N:], name), _nan_tail(db[N:], name)


def test_layernorm_bwd_refusals():
    x = _rnd(4, 272, dtype=BF)
    g, o = _rnd(272), torch.empty(4, 272, dtype=BF, device=DEV)
    dg, db = torch.empty(272, device=DEV), torch.empty(272, device=DEV)
    _refused(lambda: _layernorm_bwd(x, 272, x, 272, g, o, 272, dg, db, 1e-5, 4, 264, False), '<= 256')
    _refused(lambda: _layernorm_bwd(x, 272, x, 272, g, o, 272, dg, db, 1e-5, 4, 60, False), 'multiple of 8')


# ------------------------------------------------------------------------------------------------ GLU
GLU_C = 8            # u * |value| * (2 + |g|): the f32 arithmetic with __expf in the sigmoid


@pytest.mark.parametrize('F', [8, 136, 1024])
def test_glu(F):
    for M in (1, 37):
        u = _rnd(M, 2 * F, scale=3.0, seed=F + M, dtype=BF)
        dh = _rnd(M, F, seed=F + M + 1, dtype=BF)
        a, g = u.double().chunk(2, -1)
        s = torch.sigmoid(g)
        amp = 2 + g.abs()
        hb = _canvas(M + 1, F, BF)
        _lib.check(_lib.lib().otb_glu_fwd(ops._p(u), ops._p(hb), M, F, ops._stream()), 'otb_glu_fwd')
        _check_bf16(f'glu F={F} M={M} h', hb[:M], ref.glu(u), GLU_C * U * (a * s).abs() * amp)
        _nan_tail(hb[M], f'glu F={F} M={M}')
        dub = _canvas(M + 1, 2 * F, BF)
        _lib.check(_lib.lib().otb_glu_bwd(ops._p(dh), ops._p(u), ops._p(dub), M, F, ops._stream()), 'otb_glu_bwd')
        d = dh.double()
        tol = torch.cat([(d * s).abs() * amp, (d * a * s).abs() * amp], -1)
        _check_bf16(f'glu_bwd F={F} M={M} du', dub[:M], ref.glu_bwd(dh, u), GLU_C * U * tol)
        _nan_tail(dub[M], f'glu_bwd F={F} M={M}')


# ------------------------------------------------------------------------------------------------ dropout
DROP_C = 3           # u * |value|: the f32 scale and one product


def _dropout_bwd(dy, lddy, out, ldo, mask, M, N, p, seed, site, p2, site2):
    _lib.check(_lib.lib().otb_dropout_bwd(ops._p(dy), lddy, ops._p(out), ldo, ops._p(mask), M, N, float(p), ops._p(seed), int(site),
                                          float(p2), int(site2), ops._stream()), 'otb_dropout_bwd')


@pytest.mark.parametrize('p,p2', [(0.1, 0.0), (0.0, 0.3), (0.1, 0.3), (0.5, 0.5), (0.0, 0.0)])
def test_dropout_bwd(p, p2):
    seed, site, site2 = _seed(9876), 7, 1003
    for M, N in ((1, 2), (33, 6), (70, 258)):
        name = f'dropout_bwd p={p} p2={p2} M={M} N={N}'
        dy = _rnd(M, N, seed=M * N, dtype=BF)
        dyb = _canvas(M, N + 4, BF)
        dyb[:, :N] = dy
        ob = _canvas(M + 1, N + 2, BF)
        mb = torch.full((M + 1, N), 0xAB, dtype=torch.uint8, device=DEV)
        _dropout_bwd(dyb, N + 4, ob, N + 2, mb, M, N, p, seed, site, p2, site2)
        keep = mb[:M]
        assert torch.equal(keep, ops.dropout_mask(M, N, p, seed, site, p2, site2)), f'{name}: mask differs from dropout_mask'
        one = (ops.dropout_mask(M, N, p, seed, site) if p > 0 else torch.ones_like(keep)) & \
            (ops.dropout_mask(M, N, p2, seed, site2) if p2 > 0 else torch.ones_like(keep))
        assert torch.equal(keep, one), f'{name}: the mask is not the product of the masks of both sites'
        assert bool((mb[M] == 0xAB).all()), f'{name}: wrote past mask row M'
        want = ref.dropout_bwd(dy, keep.bool(), p, p2)
        _check_bf16(name, ob[:M, :N], want, DROP_C * U * want.abs())
        assert bool((ob[:M, :N][keep == 0] == 0).all()), f'{name}: a dropped element is not zero'
        _nan_tail(ob[:, N:], name), _nan_tail(ob[M], name)
        # with only out (no mask) the same values
        ob2 = _canvas(M, N + 2, BF)
        _dropout_bwd(dyb, N + 4, ob2, N + 2, None, M, N, p, seed, site, p2, site2)
        assert torch.equal(ob2[:, :N], ob[:M, :N]), f'{name}: out without the mask export differs'
    big = ops.dropout_mask(256, 1024, p, seed, site, p2, site2).float().mean().item()
    assert abs(big - (1 - p) * (1 - p2)) < 0.01, f'kept fraction {big:.4f}, want {(1 - p) * (1 - p2):.4f}'


@pytest.mark.parametrize('p,p2', [(0.1, 0.0), (0.0, 0.3), (0.1, 0.3)])
@pytest.mark.parametrize('N', [256, 384])
def test_dropout_bwd_replays_the_forward_epilogue_masks(p, p2, N):
    """otb_linear_dropout_resid with a @ w^T = 1, no bias, zero residual: out = keep * scale, so its zero pattern is the mask
    the forward drew, which the backward must replay."""
    M, K = 130, 64
    seed, site, site2 = _seed(2024), 11, 2011
    a = torch.ones(M, K, dtype=BF, device=DEV)
    w = torch.full((N, K), 1.0 / K, dtype=BF, device=DEV)
    resid = torch.zeros(M, N, dtype=BF, device=DEV)
    out = ops.linear_dropout_resid(a, w, None, resid, p, seed, site, p2=p2, site2=site2)
    fwd_keep = (out != 0).to(torch.uint8)
    assert torch.equal(fwd_keep, ops.dropout_mask(M, N, p, seed, site, p2, site2)), 'forward and backward masks differ'
    kept = out[out != 0].double()
    scale = ref.dropout_scale(p, p2)
    assert kept.unique().numel() == 1 and abs(float(kept[0]) - scale) <= 2.0 ** -8 * scale, 'kept values are not the scale'
    dy = torch.ones(M, N, dtype=BF, device=DEV)
    assert torch.equal(ops.dropout_bwd(dy, p, seed, site, p2, site2) != 0, out != 0)


def _dropout_add(x, ldx, resid, ldr, out, ldo, M, N, alpha, p, seed, site, row_len, row_period):
    _lib.check(_lib.lib().otb_dropout_add(ops._p(x), ldx, ops._p(resid), ldr, ops._p(out), ldo, M, N, float(alpha), float(p),
                                          ops._p(seed), int(site), ops._p(row_len), int(row_period), ops._stream()), 'otb_dropout_add')


@pytest.mark.parametrize('p', [0.0, 0.2])
@pytest.mark.parametrize('with_resid', [False, True], ids=['no_resid', 'resid'])
def test_dropout_add(p, with_resid):
    seed, site = _seed(555), 23
    for M, N, period, lens in ((20, 8, 5, [5, 2, 0, 7]), (7, 136, 1, [1, 0, 1, 1, 0, 0, 1]), (40, 256, 0, None),
                               (36, 64, 12, [12, 3, 30])):
        name = f'dropout_add p={p} resid={with_resid} M={M} N={N} period={period}'
        x = _rnd(M, N, seed=M + N, dtype=BF)
        xb = _canvas(M, N + 8, BF)
        xb[:, :N] = x
        r = _rnd(M, N, seed=M + N + 1, dtype=BF) if with_resid else None
        rb = None
        if with_resid:
            rb = _canvas(M, N + 16, BF)
            rb[:, :N] = r
        ob = _canvas(M + 1, N + 24, BF)
        row_len = torch.tensor(lens, dtype=torch.int32, device=DEV) if lens else None
        _dropout_add(xb, N + 8, rb, N + 16 if with_resid else 0, ob, N + 24, M, N, 0.5, p, seed if p > 0 else None, site, row_len,
                     period)
        keep = ops.dropout_mask(M, N, p, seed, site).bool() if p > 0 else None
        want = ref.dropout_add(x, r, keep, p, 0.5, row_len, period)
        mag = ref.dropout_add(x.abs(), None if r is None else r.abs(), keep, p, 0.5, row_len, period)
        got = ob[:M, :N]
        _check_bf16(name, got, want, DROP_C * U * mag)
        dead = ~ref.row_live(M, row_len, period, DEV)
        if dead.any():                                      # masked rows: exactly the residual, or exactly zero
            assert torch.equal(got[dead], r[dead] if with_resid else torch.zeros_like(got[dead])), f'{name}: masked row'
        _nan_tail(ob[:, N:], name), _nan_tail(ob[M], name)


# ------------------------------------------------------------------------------------------------ embedding backward
EMB_C = 4            # u * (|dE| + sum |scale dx|) of the element; 2.51 measured on an H100 SXM (700 W) (the atomics'
                     # order varies: 2.14 in another run)


@pytest.mark.parametrize('d', [8, 256, 264, 384, 520])
def test_embed_bwd(d):
    V = 11
    for n_tok in (1, 37):
        tok = torch.randint(0, V, (n_tok,), generator=torch.Generator().manual_seed(d + n_tok)).to(DEV)
        if n_tok > 1:
            tok[1::5] = 3                                       # repeats
            tok[2], tok[4], tok[6] = -1, V, 1 << 40             # out of range: add nothing
        dx = _rnd(n_tok, d, seed=d, dtype=BF)
        dE = _canvas(V + 1, d, F32)                             # row V: canary, id V is out of range
        dE0 = _rnd(V, d, seed=d + 1)
        dE[:V] = dE0
        scale = math.sqrt(d)
        _lib.check(_lib.lib().otb_embed_bwd(ops._p(tok), ops._p(dx), ops._p(dE), n_tok, d, V, ctypes.c_float(scale),
                                            ops._stream()), 'otb_embed_bwd')
        want = ref.embed_bwd(tok, dx, dE0, _f32(scale))
        s = ref.embed_bwd(tok, dx.abs(), dE0.abs(), _f32(scale))
        _check_f32(f'embed_bwd d={d} N={n_tok}', dE[:V], want, s, EMB_C)
        _nan_tail(dE[V], f'embed_bwd d={d}')


# ------------------------------------------------------------------------------------------------ Adam
ADAM_C = 7           # p, m, v: u * scale (see test_adam_step_sched); 4.72 measured on an H100 SXM (700 W)
BETAS, EPS = (0.9, 0.98), 1e-9


def _adam(p, g, m, v, n, ss, max_norm, base_lr, model_size, warmup, factor, wd, counters, hyper, noise=0.0, noise_seed=None,
          noise_mask=None):
    _lib.check(_lib.lib().otb_adam_step_sched(ops._p(p), ops._p(g), ops._p(m), ops._p(v), n, ops._p(ss), max_norm, base_lr,
                                              float(model_size), float(warmup), factor, BETAS[0], BETAS[1], EPS, wd,
                                              ops._p(counters), ops._p(hyper), float(noise), ops._p(noise_seed), ops._p(noise_mask),
                                              ops._stream()), 'otb_adam_step_sched')


@pytest.mark.parametrize('max_norm,wd,warmup', [(5.0, 1e-4, 4), (1e6, 0.0, 0), (0.0, 1e-2, 25000), (0.5, 0.0, 0)])
def test_adam_step_sched(max_norm, wd, warmup):
    """Three calls per n: a step, a skipped step (non-finite sumsq), a step; each against the restatement from the kernel's
    own state before it."""
    base_lr, model_size, factor = 1e-3, 256, 1.0
    grid_pass = 8 * _sms() * 1024
    for n in (1, 1023, 1025, 100003, 2 * grid_pass + 4097):
        name = f'adam max_norm={max_norm} wd={wd} warmup={warmup} n={n}'
        bufs = [torch.full((n + 8,), NAN, device=DEV) for _ in range(4)]
        p, g, m, v = (b[:n] for b in bufs)
        p.copy_(_rnd(n, seed=n)), m.copy_(_rnd(n, scale=0.01, seed=n + 1)), v.copy_(_rnd(n, scale=1e-3, seed=n + 2).abs())
        counters = torch.tensor([9, 40, 3], dtype=torch.int32, device=DEV)
        hyper, ss = torch.zeros(4, device=DEV), torch.zeros(1, device=DEV)
        for call, sumsq in enumerate((None, math.inf, None)):
            g.copy_(_rnd(n, scale=3.0 / math.sqrt(n), seed=n + 10 + call))           # norm about 3
            ss.fill_(float((g.double() ** 2).sum()) if sumsq is None else sumsq)
            before = [t.clone() for t in (p, m, v)]
            c0 = counters.tolist()
            _adam(p, g, m, v, n, ss, max_norm, base_lr, model_size, warmup, factor, wd, counters, hyper)
            wp, wm, wv, wc, wh = ref.adam_step(*before[:1], g, *before[1:], float(ss), c0, max_norm, base_lr, model_size, warmup,
                                                factor, BETAS[0], BETAS[1], EPS, wd)
            assert counters.tolist() == wc, f'{name} call {call}: counters {counters.tolist()}, want {wc}'
            for b in bufs:
                _nan_tail(b[n:], name)
            if wh is None:
                assert float(hyper[3]) == 0.0
                assert all(torch.equal(a, b) for a, b in zip((p, m, v), before)), f'{name}: a skipped step changed the state'
                continue
            h = hyper.double().cpu()
            for j in range(3):
                assert abs(float(h[j]) - wh[j]) <= U * abs(wh[j]), f'{name}: hyper[{j}] {float(h[j])!r}, want {wh[j]!r}'
            assert float(h[3]) == 1.0
            b1, b2 = _f32(BETAS[0]), _f32(BETAS[1])
            total = math.sqrt(float(ss))
            coef = min(1.0, _f32(max_norm) / (total + 1e-6)) if max_norm > 0 else 1.0
            gd = g.double().abs() * coef + _f32(wd) * before[0].double().abs()
            s_m = b1 * before[1].double().abs() + (1 - b1) * gd
            s_v = b2 * before[2].double().abs() + (1 - b2) * gd * gd
            upd = (wp - before[0].double()).abs()
            _check_f32(f'{name} call {call} p', p, wp, before[0].double().abs() + upd, ADAM_C)
            _check_f32(f'{name} call {call} m', m, wm, s_m, ADAM_C)
            _check_f32(f'{name} call {call} v', v, wv, s_v, ADAM_C)
            assert float(upd.max()) > 0


def test_adam_noise_instance_with_an_empty_mask_is_the_plain_step():
    """adam_kernel<true> with noise_mask all zero draws no noise into any element: bit-identical to adam_kernel<false>."""
    n = 8 * _sms() * 1024 + 1025
    outs = []
    for noise in (0.0, 0.5):
        p, m = _rnd(n, seed=1), _rnd(n, scale=0.01, seed=2)
        v, g = _rnd(n, scale=1e-3, seed=3).abs(), _rnd(n, scale=1e-2, seed=4)
        counters = torch.tensor([4, 6, 0], dtype=torch.int32, device=DEV)
        hyper, ss = torch.zeros(4, device=DEV), torch.full((1,), float((g.double() ** 2).sum()), device=DEV)
        mask = torch.zeros((n + 7) // 8, dtype=torch.uint8, device=DEV)
        _adam(p, g, m, v, n, ss, 1.0, 1e-3, 256, 4, 1.0, 1e-4, counters, hyper, noise, _seed(77) if noise else None,
              mask if noise else None)
        outs.append((p, m, v, counters, hyper))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ SpecAugment
@pytest.mark.parametrize('nf,nt', [(2, 2), (0, 2), (2, 0), (0, 0), (3, 1)])
def test_spec_augment(nf, nt):
    B, T, F = 3, 17, 80
    x0 = _rnd(B, T, F, seed=nf * 10 + nt) + 10.0                                 # no zero before the masking
    buf = torch.full((B * T * F + 64,), NAN, device=DEV)
    buf[:B * T * F] = x0.view(-1)
    rows = []
    for b in range(B):
        fb = [(70, 30), (5, 0), (10, 8), (60, 20), (75, 5)][:nf] if b != 1 else [(0, F), (3, 2), (4, 9)][:nf]
        tb = [(15, 9), (2, 0), (1, 5)][:nt] if b != 2 else [(0, 4)][:nt]         # past the edge, empty; overlapping f bands
        fb += [(0, 0)] * (nf - len(fb))
        tb += [(0, 0)] * (nt - len(tb))
        rows.append([v for band in fb + tb for v in band])
    bands = torch.tensor(rows, dtype=torch.int32).view(B, 2 * (nf + nt)).to(DEV)
    arg = bands if bands.numel() else torch.zeros(1, dtype=torch.int32, device=DEV)    # the launcher wants a pointer
    _lib.check(_lib.lib().otb_spec_augment(ops._p(buf), ops._p(arg), B, T, F, nf, nt, ops._stream()), 'otb_spec_augment')
    got = buf[:B * T * F].view(B, T, F)
    want = ref.spec_augment(x0, bands.cpu(), nf, nt).to(DEV)
    assert torch.equal(got == 0, want == 0), f'spec_augment nf={nf} nt={nt}: zero pattern differs'
    assert torch.equal(got.double(), want), f'spec_augment nf={nf} nt={nt}: a kept value changed'
    print(f'spec_augment nf={nf} nt={nt}: {int((got == 0).sum())} of {got.numel()} zeroed, exact')
    _nan_tail(buf[B * T * F:], 'spec_augment')


# ------------------------------------------------------------------------------------------------ Conformer conv module
CONV_C = 7.5         # every f32 output and the bf16 outputs' f32 part, in u * scale (see _conv_case); 4.98 measured on an
                     # H100 SXM (700 W), the batch mean over 5200 rows


def _tconv(s, w, B, T, transposed=False):
    """|w| (transposed) depthwise conv of a non-negative [B*T, d] scale: the error scale of a conv of s."""
    d, k = w.shape
    pad = (k - 1) // 2
    sp = torch.nn.functional.pad(s.view(B, T, d), (0, 0, pad, pad))
    out = torch.zeros(B, T, d, dtype=F64, device=s.device)
    for tap in range(k):
        j = 2 * pad - tap if transposed else tap
        out = out + sp[:, j:j + T] * w[:, tap].double().abs()
    return out.view(B * T, d)


def _conv_fwd(x, lens, w, wb, gamma, beta, rm, rv, nbt, c, stats, out, B, T, eps):
    d, k = w.shape
    _lib.check(_lib.lib().otb_conformer_conv_train(ops._p(x), ops._p(lens), ops._p(w), ops._p(wb), ops._p(gamma), ops._p(beta),
                                                   ops._p(rm), ops._p(rv), ops._p(nbt), 0.1, eps, ops._p(c), ops._p(stats),
                                                   ops._p(out), B, T, d, k, ops._stream()), 'otb_conformer_conv_train')


def _conv_bwd(dy, x, lens, w, gamma, beta, c, stats, red, dc, dx, dw, dwb, dg, db, accumulate, B, T):
    d, k = w.shape
    _lib.check(_lib.lib().otb_conformer_conv_bwd(ops._p(dy), ops._p(x), ops._p(lens), ops._p(w), ops._p(gamma), ops._p(beta),
                                                 ops._p(c), ops._p(stats), ops._p(red), ops._p(dc), ops._p(dx), ops._p(dw),
                                                 ops._p(dwb), ops._p(dg), ops._p(db), 1 if accumulate else 0, B, T, d, k,
                                                 ops._stream()), 'otb_conformer_conv_bwd')


def _vec(n, extra=8):
    return torch.full((n + extra,), NAN, device=DEV)


def _conv_case(name, B, T, d, k, lens, bias=True, big_mean=False, ref_lens=None, seed=0):
    lens = torch.tensor(lens, dtype=torch.int32, device=DEV)
    ref_lens = lens if ref_lens is None else torch.tensor(ref_lens, dtype=torch.int32, device=DEV)
    M = B * T
    eps = _f32(1e-5)
    x = _rnd(M, d, seed=seed, dtype=BF)
    w = 0.3 * _rnd(d, k, seed=seed + 1)
    wb = 0.2 * _rnd(d, seed=seed + 2) if bias else None
    if big_mean:                                  # every other channel: conv output mean ~1000, spread ~1
        wb[::2] += 1000.0
    gamma, beta = 1 + 0.2 * _rnd(d, seed=seed + 3), 0.2 * _rnd(d, seed=seed + 4)
    rm0, rv0 = 0.1 * _rnd(d, seed=seed + 5), 1 + 0.1 * _rnd(d, seed=seed + 6).abs()
    dy = _rnd(M, d, seed=seed + 7, dtype=BF)
    # forward, into NaN buffers with a canary row / tail
    cb, ob, stats = _canvas(M + 1, d, F32), _canvas(M + 1, d, BF), _vec(2 * d)
    rmb, rvb = _vec(d), _vec(d)
    rmb[:d], rvb[:d] = rm0, rv0
    nbt = torch.tensor([41, 12345], dtype=torch.int64, device=DEV)
    _conv_fwd(x, lens, w, wb, gamma, beta, rmb, rvb, nbt, cb, stats, ob, B, T, eps)
    fw = ref.conv_module_train(x, ref_lens, w, wb, gamma, beta, rm0, rv0, 41, B, T, eps=eps)
    mask = ref.frame_mask(ref_lens, B, T).view(M)
    xm = x.double() * mask[:, None]
    s_c = _tconv(xm.abs(), w, B, T) + (wb.double().abs() if bias else 0.0)
    cond = 1.0 + s_c.amax(0) * fw['invstd']                                        # per channel
    _check_f32(f'{name} c', cb[:M], fw['c'], s_c, CONV_C)
    _check_f32(f'{name} mean', stats[:d], fw['mean'], fw['c'].abs().mean(0), CONV_C)
    _check_f32(f'{name} invstd', stats[d:2 * d], fw['invstd'], fw['invstd'] * cond, CONV_C)
    xh = (fw['c'] - fw['mean']) * fw['invstd']
    a = xh * gamma.double() + beta.double()
    s_out = gamma.double().abs() * (xh.abs() + cond) + beta.double().abs() + a.abs()
    _check_bf16(f'{name} out', ob[:M], fw['out'], CONV_C * U * 1.1 * s_out)
    assert bool((ob[:M][~mask] == 0).all()), f'{name}: a padded frame of out is not exactly zero'
    _check_f32(f'{name} running_mean', rmb[:d], fw['running_mean'], 0.9 * rm0.double().abs() + 0.1 * fw['c'].abs().mean(0), CONV_C)
    var_unb = ((fw['c'] - fw['mean']) ** 2).sum(0) / max(M - 1, 1)
    _check_f32(f'{name} running_var', rvb[:d], fw['running_var'], 0.9 * rv0.double().abs() + 0.1 * var_unb * cond, CONV_C)
    assert nbt.tolist() == [42, 12345], f'{name}: num_batches_tracked {nbt.tolist()}'
    for t in (cb[M], ob[M], stats[2 * d:], rmb[d:], rvb[d:]):
        _nan_tail(t, name)
    # backward from the forward kernel's own c and statistics
    c, st = cb[:M], stats[:2 * d].view(2, d)
    bw = ref.conv_module_bwd(dy, x, ref_lens, w, gamma, beta, B, T, c=c, mean=st[0], invstd=st[1])
    a = bw['xh'] * gamma.double() + beta.double()
    s_da = dy.double().abs() * (1 + a.abs()) * mask[:, None]
    s_dg, s_db = (s_da * bw['xh'].abs()).sum(0), s_da.sum(0)
    s_dc = gamma.double().abs() * st[1].double() * (s_da + s_da.mean(0) + bw['xh'].abs() * (s_da * bw['xh'].abs()).mean(0))
    s_dx = _tconv(s_dc, w, B, T, transposed=True) * mask[:, None]
    xp = torch.nn.functional.pad(xm.abs().view(B, T, d), (0, 0, (k - 1) // 2, (k - 1) // 2))
    s_dw = torch.stack([(s_dc.view(B, T, d) * xp[:, tap:tap + T]).sum((0, 1)) for tap in range(k)], 1)
    s_dwb = s_dc.sum(0)
    red, dcb = _vec(2 * d), _canvas(M + 1, d, F32)
    dxb = _canvas(M + 1, d, BF)
    dwv, dwbv, dgv, dbv = _vec(d * k), _vec(d), _vec(d), _vec(d)
    dw = dwv[:d * k].view(d, k)
    for accumulate in (False, True):
        tag = f'{name} {"accumulate" if accumulate else "overwrite"}'
        prev = {}
        if accumulate:
            for key, t, sd in (('dw', dw, 11), ('dwb', dwbv[:d], 12), ('dgamma', dgv[:d], 13), ('dbeta', dbv[:d], 14)):
                if key == 'dwb' and not bias:
                    continue
                t.copy_(_rnd(*t.shape, seed=seed + sd))
                prev[key] = t.double().clone()
        _conv_bwd(dy, x, lens, w, gamma, beta, c, st, red, dcb, dxb, dw, dwbv if bias else None, dgv, dbv, accumulate, B, T)
        _check_bf16(f'{tag} dx', dxb[:M], bw['dx'], CONV_C * U * s_dx)
        assert bool((dxb[:M][~mask] == 0).all()), f'{tag}: a padded frame of dx is not exactly zero'
        outs = [('dw', dw, bw['dw'], s_dw), ('dgamma', dgv[:d], bw['dgamma'], s_dg), ('dbeta', dbv[:d], bw['dbeta'], s_db)]
        if bias:
            outs.append(('dwb', dwbv[:d], bw['dwb'], s_dwb))
        for key, got, want, s in outs:
            p0 = prev.get(key)
            _check_f32(f'{tag} {key}', got, want if p0 is None else p0 + want, s if p0 is None else s + p0.abs(), CONV_C)
        for t in (dxb[M], dcb[M], red[2 * d:], dwv[d * k:], dgv[d:], dbv[d:]) + (() if bias else (dwbv,)):
            _nan_tail(t, tag)
        if bias:
            _nan_tail(dwbv[d:], tag)


CONV_CASES = {
    'd256_k15': (3, 61, 256, 15, [61, 40, 17]),
    'd8_k1': (2, 5, 8, 1, [5, 3]),
    'd136_k31_gt_T_len0': (3, 9, 136, 31, [9, 0, 4]),
    'd264_T1': (4, 1, 264, 3, [1, 0, 1, 1]),
    'M1': (1, 1, 16, 5, [1]),
    'd384_M5200': (40, 130, 384, 15, [130 - 3 * i for i in range(40)]),     # reduce_grid caps gy at 128
}


@pytest.mark.parametrize('case', list(CONV_CASES))
def test_conformer_conv(case):
    B, T, d, k, lens = CONV_CASES[case]
    _conv_case(f'conformer_conv {case}', B, T, d, k, lens, seed=d + k)


def test_conformer_conv_without_bias():
    _conv_case('conformer_conv no bias', 3, 20, 136, 5, [20, 11, 6], bias=False, seed=5)


def test_conformer_conv_mean_far_above_spread():
    _conv_case('conformer_conv big mean', 3, 24, 264, 7, [24, 24, 10], big_mean=True, seed=6)


def test_conformer_conv_lengths_above_T():
    """Lengths above T (the last utterance's included) mean every frame is valid: no tap reads the next utterance's rows
    or past the end of x."""
    _conv_case('conformer_conv lengths > T', 3, 12, 136, 7, [13, 20, 100], ref_lens=[12, 12, 12], seed=7)


def test_conformer_conv_refusals():
    x = _rnd(6, 16, dtype=BF)
    lens = torch.tensor([3, 3], dtype=torch.int32, device=DEV)
    g = _rnd(16)
    c, st, out = torch.empty(6, 16, device=DEV), torch.empty(2, 16, device=DEV), torch.empty(6, 16, dtype=BF, device=DEV)
    _refused(lambda: _conv_fwd(x, lens, _rnd(16, 4), None, g, g, None, None, None, c, st, out, 2, 3, 1e-5), 'odd')
    _refused(lambda: _conv_fwd(x[:, :12], lens, _rnd(12, 3), None, g, g, None, None, None, c, st, out, 2, 3, 1e-5), 'multiple of 8')
