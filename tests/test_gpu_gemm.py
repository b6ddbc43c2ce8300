"""Every configuration the wgmma GEMM (csrc/gemm_tc.cu) can launch, against an fp64 reference on the same bf16-rounded
operands, element by element.

Which kernel instantiation runs is decided on the host (choose_bn) from M, N, the epilogue, the output type, the SM count
and the tile policy.  The cases below are chosen so that, under each of the two tile policies, they reach every
(epilogue, tile width, output type) cell of REACHABLE; test_cases_reach_every_configuration checks that through
otb_gemm_config, and test_dispatcher_stays_inside_the_tested_set fails when the dispatcher can answer a configuration
that has no case here.

Bounds (per element; ref is the fp64 result, acc = K 2^-23 (|a| |w|^T + |b|) bounds the fp32 accumulation):
  bf16 output  |got - ref| <= 2^-8 |ref| + L acc          fp32 output  |got - ref| <= 2^-21 |ref| + L acc
with L the Lipschitz constant of the epilogue (|alpha| for TABLE / RESID), plus
  GLU, swish   2^-10 |value|  for the tanh.approx sigmoid (|error| <= 2^-12 in sigmoid)
  GELU         2^-22 |v|      1 + erf(v / sqrt 2) cancels for negative v: fp32 erff's last-bit error is magnified
                              there, an absolute error of about ulp(1) |v| / 2 that no relative bound covers
  RESID_LN     two bf16 ulps of the fp64 result, plus |gamma| rstd (acc + 2^-20 max_row |x|) + 2^-20 |beta|: the
               fp32 error of x, of the row mean and of the affine step, which only matters for outputs near 0.
Measured on an H100 80GB HBM3 at a 400 W power limit, the largest err/bound is 0.99 for bf16 outputs (the output rounding
alone reaches 2^-8 |ref| just above a power of two), 0.075 for fp32 GELU and 0.25 for RESID_LN; a one-pass variance
(E[x^2] - mean^2) with no recentring reached 7.5 on the rows offset by 256x their spread.
Every output lives in a NaN-filled buffer with a wider pitch; everything outside the [M, N] window must stay NaN."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops
    DEV = torch.device('cuda:0')
BF = torch.bfloat16
torch.backends.cuda.matmul.allow_tf32 = False

BIAS, RELU, GLU, TABLE, RESID, RESID_LN, SWISH, GELU, TANH = range(9)
NAMES = ['bias', 'relu', 'glu', 'table', 'resid', 'resid_ln', 'swish', 'gelu', 'tanh']
ELEMENTWISE = (BIAS, RELU, TABLE, SWISH, GELU, TANH)

# (epilogue, tile width, fp32 output) of every kernel instantiation the dispatcher may launch
REACHABLE = ({(e, bn, f32) for e in ELEMENTWISE for bn in (64, 128) for f32 in (False, True)}
             | {(RESID, bn, False) for bn in (64, 128)}
             | {(GLU, 128, f32) for f32 in (False, True)}
             | {(RESID_LN, bn, False) for bn in (64, 128, 256)})

# (M, N, K, options).  Tile widths on 132 SMs, latency / throughput policy.  Options: 'views' = A, W (and the residual)
# are column views of wider matrices; 'mask' = row mask (row_len, row_period).
#   M 1, 63, 127: one row block; latency takes 64, throughput 128 once N > 64
#   M 300 N 4234: 128 under both; M 513: 64 under both, 5 row blocks x 67 column tiles = 335 tiles, so each CTA walks
#   two or three tiles; M 7968 N 768: 128 under both, 378 tiles
SHAPES = [
    (1, 4234, 72, ''),          # one row; N 4234: last tile 10 columns (2-byte copy-out for bf16 and fp32)
    (63, 184, 8, 'mask'),       # last tile 56 columns at both widths; K 8: one k-block, mostly TMA zero fill
    (65, 8, 384, ''),           # a single 8-column tile; K 384 = 6 k-blocks = STAGES of the 64-wide tile
    (127, 120, 448, 'mask'),    # last tile 56 (64-wide) or 120 columns; K 448 = STAGES + 1 of the 64-wide tile
    (129, 136, 2056, ''),       # second row block holds one row; last tile 8 columns; K 2056 = 32 k-blocks + 8
    (300, 4234, 256, 'mask'),   # K 256 = STAGES of the 128-wide tile
    (513, 100, 200, 'views'),   # N 100: 200-byte rows, 2-byte copy-out, per-element residual load; K 200
    (513, 4234, 64, ''),        # 335 tiles: the producer runs ahead across tiles
    (7968, 768, 320, 'views'),  # K 320 = STAGES + 1 of the 128-wide tile
]
LN_SHAPES = [   # N must be 64, 128 or 256: the tile spans the row
    (1, 64, 72, ''),
    (65, 256, 192, ''),         # 64-row tiles of the 256-wide configuration: the second tile holds one row; K = STAGES
    (127, 64, 448, 'mask'),
    (129, 128, 256, 'views'),   # K 256 = STAGES of the 128-wide tile
    (300, 128, 2056, 'mask'),
    (513, 256, 8, 'mask'),
    (16900, 256, 256, 'views'),  # 265 tiles of 64 rows; K 256 = STAGES + 1 of the 256-wide tile
    (20000, 128, 320, ''),      # 157 tiles
    (20000, 64, 384, ''),
]
CASES = ([(e, M, N, K, f32, opt) for e in ELEMENTWISE for f32 in (False, True) for (M, N, K, opt) in SHAPES]
         + [(GLU, M, N, K, f32, opt) for f32 in (False, True) for (M, N, K, opt) in SHAPES]
         + [(RESID, M, N, K, False, opt) for (M, N, K, opt) in SHAPES]
         + [(RESID_LN, M, N, K, False, opt) for (M, N, K, opt) in LN_SHAPES])


def _id(c):
    e, M, N, K, f32, opt = c
    return f'{NAMES[e]}-{M}x{N}x{K}-{"f32" if f32 else "bf16"}' + (f'-{opt}' if opt else '')


@pytest.fixture(scope='module', params=['latency', 'throughput'])
def policy(request):
    ops.set_tile_policy(request.param)
    try:
        yield request.param
    finally:
        ops.set_tile_policy('latency')


def _rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def _bf_matrix(rows, cols, scale, seed, view):
    """bf16 [rows, cols]; with view, columns 8.. of a wider matrix (16-byte-aligned offset, pitch > cols)."""
    x = _rnd(rows, cols, scale=scale, seed=seed).to(BF)
    if not view:
        return x
    full = torch.full((rows, (cols + 7) // 8 * 8 + 24), float('nan'), dtype=BF, device=DEV)
    full[:, 8:8 + cols] = x
    return full[:, 8:8 + cols]


def _guarded(rows, cols, dtype, fill=float('nan')):
    """A NaN-filled buffer and a [rows, cols] window of it one row down and 16 bytes in, with a wider pitch."""
    c0 = 16 // torch.tensor([], dtype=dtype).element_size()
    buf = torch.full((rows + 2, (cols + c0 - 1) // c0 * c0 + 2 * c0), float('nan'), dtype=dtype, device=DEV)
    win = buf[1:1 + rows, c0:c0 + cols]
    if fill == fill:
        win.fill_(fill)
    return buf, win


def _assert_window_only(buf, win):
    inside = torch.zeros(buf.shape, dtype=torch.bool, device=DEV)
    r0, c0 = divmod((win.data_ptr() - buf.data_ptr()) // buf.element_size(), buf.stride(0))
    inside[r0:r0 + win.shape[0], c0:c0 + win.shape[1]] = True
    outside_written = (~torch.isnan(buf.float())) & ~inside
    assert not outside_written.any(), f'written outside the output window at {torch.nonzero(outside_written)[:8].tolist()}'


def _bf16_ulp(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def _check(name, got, ref, tol):
    got = got.double()
    err = (got - ref).abs()
    bad = ~(err <= tol)       # NaN in got counts as bad
    ratio = float((err / tol.clamp_min(1e-300)).nan_to_num(float('inf')).max())
    msg = f'{name}: worst err/bound {ratio:.3f}, max |err| {float(err.nan_to_num(float("inf")).max()):.3e}'
    if bad.any():
        idx = torch.nonzero(bad)[:8].tolist()
        detail = [(i, float(got[i[0], i[1]]), float(ref[i[0], i[1]]), float(tol[i[0], i[1]])) for i in idx]
        raise AssertionError(f'{msg}; {int(bad.sum())} elements out of bound, first (idx, got, ref, bound): {detail}')
    return msg


def _row_mask(M, seed):
    """row_len / row_period of a ragged batch covering M rows: lengths 0, full and in between."""
    period = 50 if M > 50 else max(M // 2, 1)
    B = (M + period - 1) // period
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(0, period + 1, (B,), generator=g)
    lens[0] = period
    if B > 1:
        lens[1] = 0
    lens = lens.to(torch.int32).to(DEV)
    live = (torch.arange(B * period, device=DEV).view(B, period) % period < lens[:, None].long()).reshape(-1)[:M]
    return lens, period, live


def _run_case(case, offset=0.0):
    epi, M, N, K, f32, opt = case
    views, masked = 'views' in opt, 'mask' in opt
    seed = 17 * M + N + K + epi
    n_w = 2 * N if epi == GLU else N
    a = _bf_matrix(M, K, 1.0, seed, views)
    w = _bf_matrix(n_w, K, K ** -0.5, seed + 1, views)
    b = _rnd(n_w, scale=0.5, seed=seed + 2)
    kw = {}
    A, W = a.double(), w.double()
    v = A @ W.t() + b.double()
    acc = K * 2.0 ** -23 * (A.abs() @ W.abs().t() + b.double().abs())
    live = None
    if masked:
        lens, period, live = _row_mask(M, seed + 3)
        kw.update(row_len=lens, row_period=period)
    if epi in (RESID, RESID_LN):
        res = _bf_matrix(M, N, 1.0, seed + 4, views or N % 8 != 0)   # the residual pitch must be a multiple of 8
        if offset:   # rows whose common offset is `offset` x the spread of the GEMM result (exact in bf16)
            res = torch.where(torch.arange(M, device=DEV)[:, None] % 3 == 1, -offset, offset).to(BF).expand(M, N).contiguous()
        kw['resid'] = res
    if epi == RESID:
        kw['alpha'] = -0.75
    if epi == RESID_LN:
        kw.update(gamma=1 + 0.2 * _rnd(N, seed=seed + 5), beta=0.2 * _rnd(N, seed=seed + 6), eps=1e-5)
    if epi == TABLE:
        period = 7 if M > 7 else M + 3       # period != M: rows wrap around the table (or never reach its end)
        kw.update(alpha=math.sqrt(N), table=_rnd(period, N, seed=seed + 7), period=period)

    buf, out = _guarded(M, N, torch.float32 if f32 else BF)
    ops.linear(a, w, b, epi, out=out, **kw)
    torch.cuda.synchronize()

    L = 1.0
    extra = torch.zeros((), dtype=torch.float64, device=DEV)
    if epi == BIAS:
        ref = v
    elif epi == RELU:
        ref = v.clamp_min(0)
    elif epi == TANH:
        ref = torch.tanh(v)
    elif epi == GELU:
        ref = 0.5 * v * (1 + torch.erf(v / math.sqrt(2)))
        L, extra = 1.13, 2.0 ** -22 * v.abs()
    elif epi == SWISH:
        ref = v * torch.sigmoid(v)
        L, extra = 1.1, 2.0 ** -10 * v.abs()
    elif epi == TABLE:
        ref = v * kw['alpha'] + kw['table'].double()[torch.arange(M, device=DEV) % kw['period']]
        L = kw['alpha']
    elif epi == GLU:
        va, vg = v[:, :N], v[:, N:]
        ref = va * torch.sigmoid(vg)
        acc = acc[:, :N] + va.abs() / 4 * acc[:, N:]
        extra = 2.0 ** -10 * va.abs()
    elif epi == RESID:
        ref = res.double() + kw['alpha'] * torch.where(live[:, None], v, 0.0) if masked else res.double() + kw['alpha'] * v
        L = abs(kw['alpha'])
    if epi == RESID_LN:
        x = res.double() + (torch.where(live[:, None], v, 0.0) if masked else v)
        mean = x.mean(1, keepdim=True)
        rstd = torch.rsqrt(x.var(1, unbiased=False, keepdim=True) + kw['eps'])
        g, be = kw['gamma'].double(), kw['beta'].double()
        ref = (x - mean) * rstd * g + be
        if masked:
            acc = torch.where(live[:, None], acc, 0.0)
        prop = g.abs() * rstd * (acc + 2.0 ** -20 * x.abs().amax(1, keepdim=True)) + 2.0 ** -20 * be.abs()
        tol = 2 * _bf16_ulp(ref) + prop
    else:
        if masked and epi != RESID:
            ref = torch.where(live[:, None], ref, 0.0)
        if masked:
            acc = torch.where(live[:, None], acc, 0.0)
        tol = (2.0 ** -21 if f32 else 2.0 ** -8) * ref.abs() + L * acc + extra
    msg = _check(_id(case), out, ref, tol)
    if masked and epi == RESID:        # a masked row is the residual, exactly
        assert torch.equal(out[~live], res[~live]), 'masked rows must equal the residual'
    elif masked and epi != RESID_LN:   # every other epilogue writes 0 (TABLE too: not the table row)
        assert bool((out[~live] == 0).all()), 'masked rows must be 0'
    _assert_window_only(buf, out)
    return msg


# ------------------------------------------------------------------------------------------------ configuration set
def test_cases_reach_every_configuration(policy):
    reached = {}
    for c in CASES:
        epi, M, N, K, f32, opt = c
        reached.setdefault((epi, ops.gemm_config(M, N, epi, f32), f32), []).append(_id(c))
    print(f'\n{policy} policy, {ops.num_sms()} SMs: configuration -> cases')
    for key in sorted(reached):
        print(f'  {NAMES[key[0]]:9s} bn {key[1]:3d} {"f32 " if key[2] else "bf16"}: {len(reached[key])} cases')
    assert set(reached) - REACHABLE == set(), 'a case reaches a configuration REACHABLE does not list'
    missing = REACHABLE - set(reached)
    assert not missing, f'{policy}: no case reaches {sorted((NAMES[e], bn, f) for e, bn, f in missing)}'
    # the policy must change the choice somewhere, or the two passes over CASES test the same kernels twice
    other = 'throughput' if policy == 'latency' else 'latency'
    here = [ops.gemm_config(c[1], c[2], c[0], c[4]) for c in CASES]
    ops.set_tile_policy(other)
    try:
        there = [ops.gemm_config(c[1], c[2], c[0], c[4]) for c in CASES]
    finally:
        ops.set_tile_policy(policy)
    changed = sum(h != t for h, t in zip(here, there))
    print(f'  {changed} of {len(CASES)} cases take another tile under the {other} policy')
    assert changed > 0


def test_dispatcher_stays_inside_the_tested_set(policy):
    for epi in range(9):
        for f32 in (False, True):
            for M in (1, 64, 129, 512, 513, 7968):
                for N in (8, 64, 100, 256, 384, 768, 4234):
                    try:
                        bn = ops.gemm_config(M, N, epi, f32)
                    except RuntimeError:
                        assert epi in (RESID, RESID_LN), (NAMES[epi], M, N, f32)
                        continue
                    assert (epi, bn, f32) in REACHABLE, (policy, NAMES[epi], M, N, f32, bn)


# ------------------------------------------------------------------------------------------------ forward GEMM
@pytest.mark.parametrize('case', CASES, ids=_id)
def test_gemm_matches_fp64(policy, case):
    print(_run_case(case), f'[{policy}, bn {ops.gemm_config(case[1], case[2], case[0], case[4])}]')


@pytest.mark.parametrize('M,N,K', [(512, 256, 256), (300, 128, 320), (129, 64, 72)])
@pytest.mark.parametrize('offset', [4.0, 16.0, 256.0])
def test_layernorm_epilogue_with_large_row_offset(policy, M, N, K, offset):
    """Rows whose common offset is 4x, 16x and 256x their spread: on either side of the point where the epilogue stops
    trusting E[x^2] - mean^2 and recomputes the variance of the centred values."""
    print(_run_case((RESID_LN, M, N, K, False, ''), offset=offset))


def test_residual_epilogue_refuses_fp32_output():
    a = _rnd(64, 64, seed=1).to(BF)
    w = _rnd(64, 64, seed=2).to(BF)
    res = _rnd(64, 64, seed=3).to(BF)
    with pytest.raises(RuntimeError, match='residual epilogue writes bf16'):
        ops.linear(a, w, None, ops.EPI_RESID, resid=res, out_f32=True)
    out = ops.linear(a, w, None, ops.EPI_RESID, resid=res)      # the context is still usable
    torch.cuda.synchronize()
    A, W = a.double(), w.double()
    ref = res.double() + A @ W.t()
    print(_check('resid after the refusal', out, ref, 2.0 ** -8 * ref.abs() + 64 * 2.0 ** -23 * (A.abs() @ W.abs().t())))


# ------------------------------------------------------------------------------------------------ weight gradient
def _wgrad_splits(Mact, Nw, Kw):
    """Split-K count gemm_wgrad_launch picks (csrc/gemm_tc.cu)."""
    bn = 128 if Kw > 64 else 64
    tiles = ((Nw + 127) // 128) * ((Kw + bn - 1) // bn)
    num_kb = (Mact + 63) // 64
    return max(min(ops.num_sms() // tiles, num_kb // 4), 1)


@pytest.mark.parametrize('Kw', [64, 70, 72, 130, 256])
@pytest.mark.parametrize('Mact', [300, 4000])       # 5 k-blocks: one split; 63 k-blocks: split-K > 1
@pytest.mark.parametrize('accumulate', [False, True])
def test_wgrad_matches_fp64(Kw, Mact, accumulate):
    """dW[Nw, Kw] (+)= dy^T x with x a Kw-column view (pitch a multiple of 8) and dW a window of a NaN-filled buffer."""
    Nw = 192
    splits = _wgrad_splits(Mact, Nw, Kw)
    assert (splits > 1) == (Mact == 4000)
    dy = _rnd(Mact, Nw, scale=0.5, seed=Kw).to(BF)
    x = _bf_matrix(Mact, Kw, 1.0, Kw + 1, False)
    if Kw % 8:   # NaN in the pad columns: a read past column Kw would poison dW
        full = torch.full((Mact, (Kw + 7) // 8 * 8), float('nan'), dtype=BF, device=DEV)
        full[:, :Kw] = x
        x = full[:, :Kw]
    prior = _rnd(Nw, Kw, scale=4.0, seed=Kw + 2) if accumulate else None
    buf, out = _guarded(Nw, Kw, torch.float32, fill=float('nan') if prior is None else 0.0)
    if prior is not None:
        out.copy_(prior)
    ops.linear_wgrad(dy, x, out=out, accumulate=accumulate)
    torch.cuda.synchronize()
    D, X = dy.double(), x.double()
    ref = D.t() @ X
    tol = 2.0 ** -21 * ref.abs() + Mact * 2.0 ** -23 * (D.abs().t() @ X.abs())
    if prior is not None:
        ref = ref + prior.double()
        tol = tol + 2.0 ** -22 * prior.double().abs()
    print(_check(f'wgrad Kw {Kw} Mact {Mact} split-K {splits} accumulate {accumulate}', out, ref, tol))
    _assert_window_only(buf, out)
