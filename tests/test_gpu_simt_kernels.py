"""The SIMT inference and loss kernels at every configuration they accept, against the float64 restatements of
tests/simt_kernels_ref.py on the same bf16 / f32 operands:
  * otb_layernorm: every instantiation (N <= 256, and 2, 3, 4 chunks of 256 per lane), row pitches wider than N;
  * otb_log_softmax and otb_logsoftmax_topk: vocabulary edges of the 8 per-warp slices, ties, -inf, k up to 16;
  * otb_ls_ce: PAD ids, targets outside [0, V), smoothing 0 / 1, f32 and bf16 gradients;
  * otb_embed_posenc / otb_embedding, otb_scale_add_table, otb_dwconv_swish;
  * otb_decode_self_attn: d_k 64 and 96, both cache layouts, 1 to 8 heads, prefixes up to 1023 positions.
Bounds follow from the output type: a bf16 output is within one bf16 ulp of the float64 value plus the error of the f32
arithmetic before the rounding; an f32 output is within c * u * (the row's scale), u = 2^-24.  Every case prints its
measured error.  Output columns and rows past the written area hold NaN canaries that must survive.  Run with -m gpu on an
H100."""
import math

import pytest
import torch

from tests import simt_kernels_ref as ref

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import _lib, ops
    DEV = torch.device('cuda:0')

BF = torch.bfloat16
F64 = torch.float64
U = 2.0 ** -24           # f32 unit roundoff
NAN = float('nan')


def _rnd(*shape, scale=1.0, seed=0, dtype=torch.float32):
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
    print(f'{name}: max |err| {err.max().item():.3e}, max |err| / ulp {(err / ulp).max().item():.3f}, '
          f'max |err| / (ulp + abs) {(err / bound).max().item():.3f}')
    if bad.any():
        i = torch.nonzero(bad)[:6].tolist()
        raise AssertionError(f'{name}: {int(bad.sum())} elements off by more than one bf16 ulp + abs, first at {i}: '
                             f'got {[got[tuple(j)].item() for j in i]} want {[want[tuple(j)].item() for j in i]}')


def _check_f32(name, got, want, scale, c):
    """f32 `got` within c * u * scale of the float64 `want` (scale: the row's magnitude, broadcast against `want`); the
    non-finite entries must be the same non-finite values."""
    fin = torch.isfinite(want)
    assert torch.equal(fin, torch.isfinite(got)), f'{name}: finite pattern differs'
    g, w = got.double()[~fin], want[~fin]
    assert torch.equal(torch.isnan(g), torch.isnan(w)) and torch.equal(g[~torch.isnan(g)], w[~torch.isnan(w)]), \
        f'{name}: non-finite values differ'
    if not fin.any():
        print(f'{name}: all non-finite, equal')
        return
    ratio = ((got.double() - want).abs() / (U * scale.expand_as(want)))[fin]
    worst = ratio.max().item()
    print(f'{name}: max |err| / (u * row scale) {worst:.2f} (bound {c})')
    assert worst <= c, f'{name}: error {worst:.2f} u * scale exceeds {c} at flat index {int(ratio.argmax())}'


def _refused(fn, what):
    with pytest.raises(RuntimeError, match=what):
        fn()
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ LayerNorm
LN_N = [8, 64, 136, 256,          # layernorm256_kernel (4 rows per warp)
        264, 384, 512,            # layernorm_kernel<2>
        520, 768,                 # layernorm_kernel<3>
        776, 1024]                # layernorm_kernel<4>
LN_M = [1, 3, 4, 5, 31, 32, 33, 1000]
LN_C = 4                          # f32 bound, in u * (the row's max |x| / std, times max |gamma|, plus max |beta|);
                                  # 2.67 measured on an H100 SXM (700 W)


def _layernorm(x, ldx, out, ldo, g1, b1, g2, b2, eps, M, N):
    """otb_layernorm on row-pitched buffers (the ops wrapper takes only contiguous rows)."""
    _lib.check(_lib.lib().otb_layernorm(ops._p(x), ldx, ops._p(out), ldo, 1 if out.dtype == torch.float32 else 0, ops._p(g1),
                                        ops._p(b1), ops._p(g2), ops._p(b2), eps, M, N, ops._stream()), 'otb_layernorm')


def _ln_rows(M, N, seed):
    x = _rnd(M, N, scale=3.0, seed=seed) + _rnd(M, 1, scale=2.0, seed=seed + 1)
    if M >= 3:
        x[M // 2] = 0.75                                                  # variance 0: exactly beta
    if M >= 2:
        x[M - 1] = 1000.0 + _rnd(N, scale=4.0, seed=seed + 2)             # large offset: 1000 + noise
    return x.to(BF)


def _ln_tol(x, g, b, eps):
    """Per-row f32 error scale of one LayerNorm: the condition max|x| / std times max|gamma|, plus max|beta|."""
    x = x.double()
    std = torch.sqrt(x.var(-1, unbiased=False, keepdim=True) + eps)
    return x.abs().amax(-1, keepdim=True) / std * g.abs().max().double() + b.abs().max().double()


@pytest.mark.parametrize('double', [False, True], ids=['single', 'double'])
@pytest.mark.parametrize('out_dtype', [torch.float32, BF], ids=['f32', 'bf16'])
@pytest.mark.parametrize('N', LN_N)
def test_layernorm(N, out_dtype, double):
    g1, b1 = 1 + 0.3 * _rnd(N, seed=2), 0.3 * _rnd(N, seed=3)
    g2, b2 = (1 + 0.3 * _rnd(N, seed=4), 0.3 * _rnd(N, seed=5)) if double else (None, None)
    f32 = out_dtype == torch.float32
    for M in LN_M:
        x = _ln_rows(M, N, seed=M)
        for ldx, ldo, eps in ((N, N, 1e-5), (N + 16, N + (4 if f32 else 8), 1e-5 if M != 33 else 1e-12)):
            xb = _canvas(M, ldx, BF)
            xb[:, :N] = x
            ob = _canvas(M + 1, ldo, out_dtype)                           # one canary row past M
            _layernorm(xb, ldx, ob, ldo, g1, b1, g2, b2, eps, M, N)
            got = ob[:M, :N]
            want = ref.layernorm(x, g1, b1, g2, b2, eps)
            scale = _ln_tol(x, g1, b1, eps)
            if double:
                y1 = ref.layernorm(x, g1, b1, eps=eps)
                scale = _ln_tol(y1, g2, b2, eps) + 2 * scale * g2.abs().max().double() / torch.sqrt(
                    y1.var(-1, unbiased=False, keepdim=True) + eps)
            name = f'layernorm N={N} M={M} ldx={ldx} ldo={ldo} eps={eps:g}'
            const = M // 2 if M >= 3 else None
            if const is not None:
                if not double:                                            # exactly beta, in the output type
                    assert torch.equal(got[const], b1.to(out_dtype)), f'{name}: constant row is not beta'
                keep = torch.ones(M, dtype=torch.bool, device=DEV)
                keep[const] = False
                got, want, scale = got[keep], want[keep], scale[keep]
            if f32:
                _check_f32(name, got, want, scale, LN_C)
            else:
                _check_bf16(name, got, want, LN_C * U * scale)
            assert bool(torch.isnan(ob[:, N:].float()).all()) and bool(torch.isnan(ob[M].float()).all()), \
                f'{name}: wrote past column N or row M'


def test_layernorm_refusals():
    x = _rnd(4, 1040, dtype=BF)
    g, b = _rnd(1040), _rnd(1040)
    o = torch.empty(4, 1040, dtype=BF, device=DEV)
    _refused(lambda: _layernorm(x, 12, o, 12, g, b, None, None, 1e-5, 4, 12), 'multiple of 8')
    _refused(lambda: _layernorm(x, 1040, o, 1040, g, b, None, None, 1e-5, 4, 1032), '<= 1024')
    _refused(lambda: _layernorm(x, 68, o, 64, g, b, None, None, 1e-5, 4, 64), 'multiple of 8')      # ldx % 8
    _refused(lambda: _layernorm(x, 64, o, 68, g, b, None, None, 1e-5, 4, 64), 'output stride')      # bf16 ldo % 8
    of = torch.empty(4, 1040, device=DEV)
    _refused(lambda: _layernorm(x, 64, of, 66, g, b, None, None, 1e-5, 4, 64), 'output stride')     # f32 ldo % 4


# ------------------------------------------------------------------------------------------------ log-softmax
LSM_C = 2          # bound in u * (max |finite x| + |lse|) of the row; 1.41 measured on an H100 SXM (700 W)


def _lsm_rows(V, seed):
    x = _rnd(6, V, scale=4.0, seed=seed)
    if V >= 2:
        x[1, ::3] = -math.inf
    x[2] = -math.inf
    x[2, V // 2] = 3.0                                                    # one finite entry: 0 there, -inf elsewhere
    x[3] = -math.inf                                                      # no finite entry: NaN, as torch
    x[4, 0] = 1e30
    if V >= 2:
        x[4, 1:] = -1e30
    x[5] *= 20
    return x


def _row_scale(x, with_lse=True):
    """max |finite x| of each row, plus |log sum exp x| where that is finite."""
    x = x.double()
    zero = torch.zeros((), dtype=F64, device=x.device)
    s = torch.where(torch.isfinite(x), x.abs(), zero).amax(-1, keepdim=True)
    if with_lse:
        lse = torch.logsumexp(x, -1, keepdim=True)
        s = s + torch.where(torch.isfinite(lse), lse.abs(), zero)
    return s


@pytest.mark.parametrize('V', [1, 2, 255, 256, 257, 4234, 50000])
def test_log_softmax(V):
    x = _lsm_rows(V, seed=V)
    xb = _canvas(6, V + 5, torch.float32)
    xb[:, :V] = x
    ob = _canvas(7, V + 3, torch.float32)
    ops.log_softmax(xb, V, out=ob[:6, :V])
    got = ob[:6, :V]
    want = ref.log_softmax(x)
    _check_f32(f'log_softmax V={V}', got, want, _row_scale(x), LSM_C)
    assert bool((got[2, V // 2] == 0).all()) and (V == 1 or bool(torch.isneginf(got[2, :V // 2]).all()))
    assert bool(torch.isnan(got[3]).all())
    if V == 1:
        assert bool((got[[0, 1, 4, 5]] == 0).all())
    assert bool(torch.isnan(ob[:, V:]).all()) and bool(torch.isnan(ob[6]).all()), 'wrote past V or past the last row'


# ------------------------------------------------------------------------------------------------ log-softmax + top-k
TOPK_C = 3         # values and out_logp, in u * (max |finite x| + |lse| + lm_weight * max |finite lm|) of the row;
                   # 1.87 measured on an H100 SXM (700 W)
TOPK_V = [lambda k: k, lambda k: 8 * k - 1, lambda k: 8 * k + 1, lambda k: 40, lambda k: 257, lambda k: 4234,
          lambda k: 49152]
TOPK_CASES = sorted({(k, f(k)) for k in range(1, 17) for f in TOPK_V if f(k) >= k})


def _topk_rows(V, k, seed):
    """Rows: random; equal maxima spread over the 8 warp slices in reverse slice order; fewer than k finite values; a
    constant row; a wide random row."""
    x = _rnd(5, V, scale=4.0, seed=seed)
    x[1] /= 4
    per = (V + 7) // 8
    top = [(7 - j) * per + j % per for j in range(8)]
    x[1, [i for i in top if i < V]] = 12.0
    x[1, [i for i in ((7 - j) * per + (j + 1) % per for j in range(8)) if i < V and i not in top]] = 11.0
    x[2] = -math.inf
    x[2, torch.arange(0, V, max(1, V // max(1, k // 2)))[:max(1, k // 2)]] = 1.0
    x[3] = 0.5
    x[4] *= 10
    return x


def _clusters(vals, tol):
    """Ranks of one sorted row split where neighbours differ by more than tol -> [(first, last, all_equal)]."""
    out, a = [], 0
    v = vals.tolist()
    for r in range(1, len(v) + 1):
        if r == len(v) or not (v[r - 1] == v[r] or v[r - 1] - v[r] <= tol):
            out.append((a, r - 1, all(v[i] == v[a] for i in range(a, r))))
            a = r
    return out


def _check_topk_ids(name, idx, fused, k, tol):
    """Ids equal the stable float64 top-k wherever the order is decided by more than tol; candidates closer than that may
    come in either order, but a group that lies inside the top k holds the same ids; exact ties go to the lower id."""
    sv, si = ref.stable_topk(fused, min(k + 1, fused.shape[1]))
    idx, sv, si = idx.cpu(), sv.cpu(), si.cpu()
    for r in range(idx.shape[0]):
        for a, b, exact in _clusters(sv[r], float(tol[r])):
            if a >= k:
                break
            hi = min(b, k - 1)
            if exact:
                assert idx[r, a:hi + 1].tolist() == si[r, a:hi + 1].tolist(), f'{name}: row {r} ranks {a}..{hi} (tie)'
            elif b < k:
                assert sorted(idx[r, a:b + 1].tolist()) == sorted(si[r, a:b + 1].tolist()), f'{name}: row {r} ranks {a}..{b}'


@pytest.mark.parametrize('k,V', TOPK_CASES)
def test_logsoftmax_topk(k, V):
    x = _topk_rows(V, k, seed=k * 100003 + V)
    rows = x.shape[0]
    lm = torch.log_softmax(_rnd(rows, V, seed=V + 7), -1)
    lm_inf = lm.clone()
    lm_inf[0, ::2] = -math.inf                                            # an LM that rules tokens out
    lm_inf[4] = -math.inf
    lm_inf[4, V - min(V, max(1, k // 2)):] = 0.0                          # fewer than k finite values through the LM
    xb = _canvas(rows, V + 3, torch.float32)
    xb[:, :V] = x
    for lm_w, lmt in ((0.0, None), (0.0, lm), (0.3, lm_inf)):
        name = f'topk k={k} V={V} lm_weight={lm_w}{"" if lmt is None else " lm"}'
        lpb = _canvas(rows, V + 5, torch.float32)
        lmb = None
        if lmt is not None:
            lmb = _canvas(rows, V + 1, torch.float32)
            lmb[:, :V] = lmt
        val, idx = ops.logsoftmax_topk(xb, V, k, lmb, lm_w, out_logp=lpb[:, :V])
        lp = lpb[:, :V]
        fused = ref.fused_logp(x, lmt, lm_w)
        scale = _row_scale(x)
        if lmt is not None:
            scale = scale + lm_w * _row_scale(lmt, with_lse=False)
        _check_f32(name + ' out_logp', lp, fused, scale, TOPK_C)
        assert bool(torch.isnan(lpb[:, V:]).all()), f'{name}: out_logp written past V'
        # top-k over the kernel's own log-probs: bit-identical
        ov, oi = ref.stable_topk(lp, k)
        assert torch.equal(idx.long(), oi), f'{name}: ids differ from the stable top-k of out_logp'
        assert torch.equal(val.double(), ov), f'{name}: values differ from the stable top-k of out_logp'
        # against float64: values within the bound, ids wherever the order is decided by more than twice the bound
        sv, _ = ref.stable_topk(fused, k)
        _check_f32(name + ' values', val, sv, scale, TOPK_C)
        _check_topk_ids(name, idx, fused, k, (2 * TOPK_C * U * scale).view(-1).tolist())
        if lm_w == 0.0 and lmt is None:
            n = min(k, int((x[1] >= 11).sum()))                           # equal maxima across slices: lower id first
            ties = ref.stable_topk(x[1:2].double(), k)[1][0, :n]
            assert torch.equal(idx[1, :n].long(), ties), f'{name}: tie order across warp slices'
        val2, idx2 = ops.logsoftmax_topk(xb, V, k, lmb, lm_w)             # without materialising the log-probs
        assert torch.equal(val2, val) and torch.equal(idx2, idx), f'{name}: out_logp changes the result'


def test_logsoftmax_topk_refusals():
    x = torch.zeros(2, 49160, device=DEV)
    _refused(lambda: ops.logsoftmax_topk(x, 49153, 4), 'vocabulary too large')
    _refused(lambda: ops.logsoftmax_topk(x, 3, 5), 'must not exceed')     # k > V
    _refused(lambda: ops.logsoftmax_topk(x, 16, 17), r'\[1,16\]')
    _refused(lambda: ops.logsoftmax_topk(x, 16, 0), 'otb_logsoftmax_topk')
    val, idx = ops.logsoftmax_topk(x, 5, 5)                               # k == V: every id once, in order (all tied)
    assert idx.tolist() == [[0, 1, 2, 3, 4]] * 2


# ------------------------------------------------------------------------------------------------ label-smoothed CE
LSCE_C = 4         # bound in u * scale (scale: the magnitudes the per-token formula adds; see _lsce_scale);
                   # 2.48 measured on an H100 SXM (700 W), f32 dlogits


def _ls_ce(logits, ldl, tgt, V, smoothing, pad_id, dl, ldd, bf16_grad):
    rows = tgt.numel()
    tok = _canvas(rows + 1, 1, torch.float32).view(-1)
    loss = torch.full((1,), NAN, device=DEV)
    nv = torch.full((1,), -7, dtype=torch.int32, device=DEV)
    _lib.check(_lib.lib().otb_ls_ce(ops._p(logits), ldl, ops._p(tgt), rows, V, smoothing, pad_id, ops._p(tok), ops._p(loss),
                                    ops._p(nv), ops._p(dl), ldd, 1 if bf16_grad else 0, ops._stream()), 'otb_ls_ce')
    assert bool(torch.isnan(tok[rows])), 'tok_loss written past rows'
    return loss[0], tok[:rows], int(nv)


def _lsce_scale(x, tgt, V, smoothing):
    """Per-row magnitude of the terms the kernel adds: lo * (sum |x| + V |lse|), (hi - lo) * (|x_t| + |lse|) and the
    constant sum conf log conf, times the summation length's growth (V / 256 per thread, then 8 warps)."""
    x = x.double()
    lse = torch.logsumexp(x, -1)
    lo, hi = smoothing / (V - 1), 1.0 - smoothing
    t = tgt.clamp(0, V - 1)
    xt = x.gather(1, t[:, None]).view(-1)
    c = abs((V - 1) * lo * math.log(lo) if lo > 0 else 0.0) + abs(hi * math.log(hi) if hi > 0 else 0.0)
    s = c + lo * (x.abs().sum(-1) + V * lse.abs()) + abs(hi - lo) * (xt.abs() + lse.abs()) + lse.abs()
    return s * (1 + V / 256)


@pytest.mark.parametrize('pad_mode', ['pad0', 'pad_mid'])
@pytest.mark.parametrize('smoothing', [0.0, 0.1, 1.0])
@pytest.mark.parametrize('V', [2, 3, 257, 4234, 30000])
def test_ls_ce(V, smoothing, pad_mode):
    pad_id = 0 if pad_mode == 'pad0' else V // 2
    rows = 40
    g = torch.Generator().manual_seed(V * 7 + int(smoothing * 10))
    tgt = torch.randint(0, V, (rows,), generator=g)
    tgt[0], tgt[1] = 0, (pad_id + 1) % V                                  # token 0, then a real token
    tgt[2], tgt[3], tgt[4], tgt[5] = V - 1, -3, V, pad_id                 # last id, out of range both ways, PAD
    tgt[7::9] = pad_id
    tgt = tgt.to(DEV)
    ldl = V + 1
    x = _rnd(rows, V, scale=3.0, seed=V + 1)
    xb = _canvas(rows, ldl, torch.float32)
    xb[:, :V] = x
    want_loss, want_tok, want_n, want_g = ref.ls_ce(x, tgt, V, smoothing, pad_id)
    scale = _lsce_scale(x, tgt, V, smoothing)
    name = f'ls_ce V={V} smoothing={smoothing} pad_id={pad_id}'
    for bf16_grad in (False, True):
        ldd = (V + 7) // 8 * 8 + 8 if bf16_grad else V + 3
        db = _canvas(rows + 1, ldd, BF if bf16_grad else torch.float32)
        loss, tok, n = _ls_ce(xb, ldl, tgt, V, smoothing, pad_id, db, ldd, bf16_grad)
        assert n == want_n, f'{name}: n_valid {n}, want {want_n} (rows with a target in [0, V) other than PAD)'
        _check_f32(name + ' tok_loss', tok, want_tok, scale, LSCE_C)
        _check_f32(name + ' loss', loss.view(1), want_loss.view(1), scale.sum().view(1) / max(n, 1), LSCE_C)
        # d(mean)/dlogits: (softmax - conf) / n_valid with softmax's error (|x| + |lse| + 1) * u relative
        p = torch.softmax(x.double(), -1)
        gscale = ((x.double().abs() + torch.logsumexp(x.double(), -1, keepdim=True).abs() + 1) * p + (want_g.abs() * max(n, 1))
                  ) / max(n, 1)
        gname = f'{name} dlogits {"bf16" if bf16_grad else "f32"}'
        if bf16_grad:
            _check_bf16(gname, db[:rows, :V], want_g, LSCE_C * U * gscale)
            assert bool((db[:rows, V:] == 0).all()), f'{gname}: pad columns not zero'
        else:
            _check_f32(gname, db[:rows, :V], want_g, gscale, LSCE_C)
            assert bool(torch.isnan(db[:rows, V:]).all()), f'{gname}: wrote past V'
        assert bool(torch.isnan(db[rows].float()).all()), f'{gname}: wrote past the last row'
        bad = (tgt == pad_id) | (tgt < 0) | (tgt >= V)
        assert bool((tok[bad] == 0).all()) and bool((db[:rows, :V][bad] == 0).all()), f'{gname}: unscored rows not zero'
    # an all-PAD batch: loss 0, gradient 0, n_valid 0
    allpad = torch.full((rows,), pad_id, dtype=torch.long, device=DEV)
    db = _canvas(rows + 1, V, torch.float32)
    loss, tok, n = _ls_ce(xb, ldl, allpad, V, smoothing, pad_id, db, V, False)
    assert n == 0 and float(loss) == 0.0 and bool((tok == 0).all()) and bool((db[:rows] == 0).all()), f'{name}: all PAD'


# ------------------------------------------------------------------------------------------------ embedding + posenc
@pytest.mark.parametrize('mode', ['period', 'step', 'row_pos'])
@pytest.mark.parametrize('d', [8, 64, 256, 264, 384, 520])
def test_embed_posenc(d, mode):
    vocab, N, n_pos = 37, 45, 64
    emb = _rnd(vocab, d, seed=d, dtype=BF)
    table = _rnd(n_pos, d, seed=d + 1)
    g = torch.Generator().manual_seed(d)
    tok = torch.randint(0, vocab, (N, 2), generator=g)
    tok[:, 1] = (tok[:, 0] + 5) % vocab                                   # the skipped column holds other ids
    tok[3, 0], tok[10, 0], tok[44, 0] = -1, vocab, vocab - 1              # out of range ids read row 0
    tok = tok.to(DEV)
    kw, rkw = {}, {}
    if mode == 'period':
        kw, rkw = {'period': 7}, {'period': 7}
    elif mode == 'step':
        kw, rkw = {'step_ptr': torch.tensor([n_pos - 1], dtype=torch.int32, device=DEV)}, {'step': n_pos - 1}
    else:
        rp = torch.randint(0, n_pos, (N,), generator=g, dtype=torch.int32)
        rp[::6] = -1                                                      # no position: reads position 0
        rp[1] = n_pos - 1
        rp = rp.to(DEV)
        kw, rkw = {'row_pos': rp}, {'row_pos': rp}
    ob = _canvas(N + 1, d, BF)
    ops.embed_posenc(tok, emb, table, N, d, tok_stride=2, out=ob[:N], **kw)
    want = ref.embed_posenc(tok, emb, table, d, tok_stride=2, **rkw)
    # f32 e * sqrt(d) + pe: three roundings of terms of size |e| sqrt(d) + |pe|
    t = torch.where((tok[:, 0] >= 0) & (tok[:, 0] < vocab), tok[:, 0], torch.zeros_like(tok[:, 0]))
    mag = emb.double()[t].abs() * math.sqrt(d) + (want - emb.double()[t] * math.sqrt(d)).abs()
    _check_bf16(f'embed_posenc d={d} {mode}', ob[:N], want, 4 * U * mag)
    assert bool(torch.isnan(ob[N].float()).all()), 'wrote past row N'
    if mode == 'period':
        eb = _canvas(N + 1, d, BF)
        ops.embedding(tok[:, 0].contiguous(), emb, out=eb[:N])
        assert torch.equal(eb[:N], emb[t]), f'embedding d={d}: not the gathered rows'
        assert bool(torch.isnan(eb[N].float()).all())


# ------------------------------------------------------------------------------------------------ x * alpha + table
@pytest.mark.parametrize('alpha_dev', [False, True], ids=['alpha', 'alpha_dev'])
@pytest.mark.parametrize('period', [None, 1, 'T', 'M'])
@pytest.mark.parametrize('x_dtype', [torch.float32, BF], ids=['x_f32', 'x_bf16'])
def test_scale_add_table(x_dtype, period, alpha_dev):
    T, M, N = 9, 45, 40                                                   # M * N = 1800: not a multiple of 256
    per = {None: 1, 1: 1, 'T': T, 'M': M}[period]
    x = _rnd(M, N, scale=2.0, seed=1, dtype=x_dtype)
    xb = _canvas(M, N + 3, x_dtype)
    xb[:, :N] = x
    table = _rnd(per, N, seed=2) if period is not None else None
    sd = torch.tensor([0.25], device=DEV) if alpha_dev else None
    ob = _canvas(M + 1, N + 5, BF)
    ops.scale_add_table(xb[:, :N], 3.5, table, per, out=ob[:M, :N], scale_dev=sd)
    alpha = 3.5 * (0.25 if alpha_dev else 1.0)
    want = ref.scale_add_table(x, alpha, table, per)
    mag = x.double().abs() * alpha + (want - x.double() * alpha).abs()
    _check_bf16(f'scale_add_table {x_dtype} period={period} alpha_dev={alpha_dev}', ob[:M, :N], want, 4 * U * mag)
    assert bool(torch.isnan(ob[:, N:].float()).all()) and bool(torch.isnan(ob[M].float()).all()), 'canaries overwritten'


# ------------------------------------------------------------------------------------------------ depthwise conv + swish
@pytest.mark.parametrize('d', [8, 64, 384, 520])
@pytest.mark.parametrize('k', [1, 3, 15, 31])
def test_dwconv_swish(k, d):
    B = 3
    w = _rnd(k, d, scale=k ** -0.5, seed=k + d)
    b = _rnd(d, scale=2.0, seed=k + d + 1)
    b[::5] = -100.0                                                       # pre-activations down to -100
    b[1::7] = 30.0
    for T in sorted({1, 2, max(1, k - 1), 249}):
        x = _rnd(B, T, d, seed=T, dtype=torch.float32)
        x[1] *= 8                                                         # utterances differ in scale: a leaked tap shows
        x = x.view(B * T, d).to(BF)
        ob = _canvas(B * T + 1, d, BF)
        ops.dwconv_swish(x, w, b, B, T, out=ob[:B * T])
        want = ref.dwconv_swish(x, w, b, B, T)
        # f32 sum of k + 1 terms (error (k + 1) u sum |terms|, through swish' <= 1.1) and the fast sigmoid (2^-20 relative)
        pad = (k - 1) // 2
        xp = torch.nn.functional.pad(x.double().view(B, T, d).abs(), (0, 0, pad, pad))
        s = b.double().abs().expand(B, T, d).clone()
        for tap in range(k):
            s = s + xp[:, tap:tap + T] * w[tap].double().abs()
        abs_tol = 1.1 * (k + 1) * U * s.view(B * T, d) + 2.0 ** -20 * want.abs()
        _check_bf16(f'dwconv_swish k={k} T={T} d={d}', ob[:B * T], want, abs_tol)
        assert bool(torch.isnan(ob[B * T].float()).all()), 'wrote past the last row'


def test_dwconv_swish_refuses_even_k():
    x = torch.zeros(4, 8, dtype=BF, device=DEV)
    _refused(lambda: ops.dwconv_swish(x, torch.zeros(2, 8, device=DEV), torch.zeros(8, device=DEV), 1, 4), 'k odd')


# ------------------------------------------------------------------------------------------------ decode self-attention
ATT_ABS = 2.0 ** -16      # abs term of the bf16 bound, times max |v| of the cache (f32 P.V sums and __expf)
STEPS = {False: (128, [0, 31, 32, 127]),                 # Lmax <= 128: one chunk (127 = the last unchunked position)
         True: (1023, [128, 129, 255, 256, 1022])}       # chunked: 128-key chunks with an online softmax


@pytest.mark.parametrize('H', [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize('chunked', [False, True], ids=['unchunked', 'chunked'])
@pytest.mark.parametrize('layout', ['step_ptr', 'row_pos'])
@pytest.mark.parametrize('dk', [64, 96])
def test_decode_self_attn(dk, layout, chunked, H):
    Lmax, steps = STEPS[chunked]
    d = H * dk
    for N in (1, 7, 160):
        seed = N * 1000 + H * 10 + dk
        g = torch.Generator().manual_seed(seed)
        if layout == 'step_ptr':
            kc, vc = _rnd(Lmax, N, d, seed=seed, dtype=BF), _rnd(Lmax, N, d, seed=seed + 1, dtype=BF)
            anc = torch.randint(0, N, (2, N, Lmax), generator=g, dtype=torch.int32).to(DEV)   # shared rows
            cases = [(s, None) for s in steps]
        else:
            pool = 64                                                     # prefix rows, shared by many rows and positions
            kc, vc = _rnd(pool + N, d, seed=seed, dtype=BF), _rnd(pool + N, d, seed=seed + 1, dtype=BF)
            anc = torch.randint(0, pool, (N, Lmax), generator=g, dtype=torch.int32)
            if N == 1:
                cases = [(None, [p]) for p in steps + [-1]]
            else:
                pos = [steps[i % len(steps)] for i in range(N)]
                pos[5::6] = [-1] * len(pos[5::6])
                cases = [(None, pos)]
            anc = anc.to(DEV)
        for step, pos in cases:
            qkv = _rnd(N, 3 * d, seed=seed + 2 + (step or 0), dtype=torch.float32)
            qkv[:, :d] *= 4                                               # peaked scores: chunk rescaling matters
            qkv = qkv.to(BF)
            ob = _canvas(N + 1, d, BF)
            if pos is None:
                ctrl = torch.tensor([step, 0, 0, 0], dtype=torch.int32, device=DEV)
                kc0, vc0 = kc.clone(), vc.clone()
                ops.decode_self_attn(qkv, kc, vc, anc, ctrl, N, H, Lmax, out=ob[:N])
                want = ref.decode_self_attn(qkv, kc0, vc0, anc, H, step=step)
                kc0[step], vc0[step] = qkv[:, d:2 * d], qkv[:, 2 * d:]    # the newest K/V land in kc[step, n]
                name = f'decode_self_attn dk={dk} H={H} N={N} step={step}'
                live = torch.ones(N, dtype=torch.bool, device=DEV)
            else:
                rp = torch.tensor(pos, dtype=torch.int32, device=DEV)
                live = rp >= 0
                for n in torch.nonzero(live).view(-1).tolist():
                    anc[n, pos[n]] = 64 + n                                     # the newest K/V go to a row of its own
                kc0, vc0 = kc.clone(), vc.clone()
                ops.decode_self_attn(qkv, kc, vc, anc, None, N, H, Lmax, out=ob[:N], row_pos=rp)
                want = ref.decode_self_attn(qkv, kc0, vc0, anc, H, row_pos=rp)
                rows_new = 64 + torch.nonzero(live).view(-1)
                kc0[rows_new], vc0[rows_new] = qkv[live, d:2 * d], qkv[live, 2 * d:]   # kc[anc[n][pos]], live rows only
                name = f'decode_self_attn dk={dk} H={H} N={N} row_pos={sorted(set(pos))}'
            if live.any():
                _check_bf16(name + f' Lmax={Lmax}', ob[:N][live], want[live], ATT_ABS * vc0.abs().amax().double())
            assert bool((ob[:N][~live] == 0).all()), f'{name}: a row at -1 is not zero'
            assert torch.equal(kc, kc0) and torch.equal(vc, vc0), f'{name}: the cache differs outside the newest slots'
            assert bool(torch.isnan(ob[N].float()).all()), f'{name}: wrote past row N'
