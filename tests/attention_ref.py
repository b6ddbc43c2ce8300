"""Float64 restatement of the tensor-core attention forward (csrc/attn_tc.cu, otb_attention) and backward
(csrc/attn_bwd.cu, otb_attention_bwd), the per-element bound of each kernel output, the checker, a CPU emulation of the
kernels' arithmetic, and the case table and inputs of tests/test_gpu_attention.py.  Needs no GPU.

Conventions (those of attn_tc.cu): key j is visible from query row i of batch b when j < min(kv_len[b], Tk) and, with
causal, j <= i (for any Tq, Tk).  The raw score is t_ij = q_i . k_j, plus BD[h, b Tq + i, j - i + Tq - 1] with the rel-pos
band (Tq == Tk, not causal); P = softmax_j(t / sqrt(d_k)) over the visible keys; L = log2 sum_j exp(t_ij / sqrt(d_k)), the
row log-sum-exp in log2 units, +inf on a row without a visible key, whose output and gradients are zero.

Bounds, per element; u = 2^-24 (fp32 rounding), 2^-8 (bf16 rounding), c = log2(e) / sqrt(d_k):
  score      |t^ - t| <= E_ij = d_k 2^-23 sum_d |q_id| |k_jd| + 2^-24 |t_ij|: the wgmma accumulation model of
             tests/test_gpu_gemm.py, plus the fp32 add of the band.
  exponent   p^ = ex2.approx(fma(t^, c^, -m)): the argument is off by c E + (|c^ - c| / c) c |t| + 2^-24 (c |t| + |m|)
             (c^ is c rounded to fp32: log2(e) rounded, and at d_k 96 sqrtf and the division, 3 u; |m| <= max_row c |t|),
             and the PTX ISA gives ex2.approx.f32 a maximum relative error of 2^-22 (EPS_EX2), so
             delta_ij = 2^arg_err (1 + 2^-22) - 1 bounds |p^ / p - 1|.  Results below 2^-126 are flushed (.ftz): an
             absolute Tk 2^-126 max|v| on the output.
  forward    O = (sum_j bf16(p^_j) v_j) / l with l = sum_j p^_j in fp32.  Each key block rescales o and l by the same
             alpha, so alpha's own error cancels in o / l; the two products are rounded separately, u each per block, a
             relative 2 nblk u on o / l (nblk = Tk / 128 rounded up).  With lam = (1 + max delta)(1 + n u / (1 - n u)) - 1
             (n: keys summed), rho = (1 + max delta)(1 + 2^-8) / (1 - lam) - 1, and K = Tk rounded up to the 128-key block:
               e1 = (rho + (K 2^-23 + 2^-23 + 2 nblk 2^-24)(1 + rho)) (P* |V|) + Tk 2^-126 max|v|
             (P rounding, P error and l; the PV accumulation; fl(1/l) and the multiply by it; the rescales)
               e2 = e1 + 2^-24 (|O* + r| + e1)                                        (the resid add)
               |O - O*| <= e2 + 2^-8 (|O* + r| + e2)                                  (the bf16 output)
  lse        L = m + log2f(l): |L - L*| <= -log2(1 - max delta - n u / (1 - n u) - nblk a) + 2^-23 (log2 K + 1)
             + 2^-24 (|L*| + 1), with a = (1 + 2^-22) 2^(2^-23 max c|t|) (1 + 2^-24) - 1 the error of one alpha rescale
             and 2^-23 |log2 l| the 1-ulp error of log2f.
  dsum       D = sum_d dO_d O_d over the bf16 out passed in: products of bf16 values are exact in fp32, so
             |D - D*| <= d_k 2^-24 sum_d |dO_d| |O_d|.
  dS         P^ = ex2(fma(t^, c, -L^)) is off from P* by pi = 2^(c E + 2^-24 (c|t| + |L|) + u c|t| + dL) (1 + 2^-22) - 1
             (dL the lse bound); dP = dO . v_j is off by d_k 2^-23 sum |dO| |v_j|; D by the dsum bound plus
             sum_d |dO_d| (forward bound of O_d).  With g = dP* - D* and eg those two errors plus 2^-24 (|g| + eg):
               eS = P* ((1 + pi)(|g| + eg)(1 + 2^-24)^2 - |g|) / sqrt(d_k);   dBD = bf16(dS): eS + 2^-8 (|dS*| + eS).
  dQ, dK, dV dQ = bf16(dS) K, dK = bf16(dS)^T Q, dV = bf16(P)^T dO: the operand error times |K|, |Q| or |dO|, the
             accumulation K 2^-23 (|operand| |other|) over the keys (queries) the chain runs through, and the bf16 output
             2^-8 (|ref| + e).
Nothing here is a tolerance: every term is one of the roundings above."""
import math

import torch

U = 2.0 ** -24          # fp32 unit roundoff
ACC = 2.0 ** -23        # per-term wgmma fp32 accumulation error (tests/test_gpu_gemm.py)
UB = 2.0 ** -8          # bf16 unit roundoff
EPS_EX2 = 2.0 ** -22    # ex2.approx.f32 maximum relative error, PTX ISA
LN2 = math.log(2.0)
LOG2E = 1.0 / LN2


def _pad128(n):
    return (n + 127) // 128 * 128


def heads(m, col0, B, H, T, dk):
    """Columns [col0, col0 + H dk) of the first B T rows of a matrix -> float64 [B, H, T, dk]."""
    return m[:B * T, col0:col0 + H * dk].double().reshape(B, T, H, dk).transpose(1, 2)


def flat(t):
    """[B, H, T, dk] -> [B T, H dk]."""
    B, H, T, dk = t.shape
    return t.transpose(1, 2).reshape(B * T, H * dk)


def visible(B, Tq, Tk, kv_len, causal, device, mutate=None):
    """bool [B, 1, Tq, Tk]: key j visible from query row i of batch b."""
    j = torch.arange(Tk, device=device)
    i = torch.arange(Tq, device=device)
    lim = torch.full((B,), Tk, device=device) if kv_len is None else kv_len.to(device).long().clamp(max=Tk)
    vis = (j[None, None, :] < lim[:, None, None]).expand(B, Tq, Tk).clone()
    if causal:
        diag = {'causal_excl_diag': -1, 'causal_plus_one': 1}.get(mutate, 0)
        vis &= j[None, None, :] <= i[None, :, None] + diag
    if mutate == 'drop_last_key':
        vis[torch.arange(B, device=device), :, (lim - 1).clamp(min=0)] = False
    elif mutate in ('drop_key_127', 'drop_key_128'):
        kk = int(mutate[-3:])
        if kk < Tk:
            vis[:, :, kk] = False
    return vis[:, None]


def band(bd, B, H, Tq, Tk, shift=0):
    """The band as [B, H, Tq, Tk]: BD[h, b Tq + i, j - i + Tq - 1] (Tq == Tk)."""
    ld = bd.shape[-1]
    b4 = bd[:, :B * Tq].double().reshape(H, B, Tq, ld).transpose(0, 1)
    idx = (torch.arange(Tk, device=bd.device)[None, :] - torch.arange(Tq, device=bd.device)[:, None] + Tq - 1 + shift)
    return torch.gather(b4, 3, idx.clamp(0, ld - 1).expand(B, H, Tq, Tk))


def forward(q, k, v, B, H, Tq, Tk, kv_len, causal, col0s, bd=None, resid=None, d_k=64, mutate=None):
    """Float64 forward -> dict: out [B Tq, H dk] (O + resid), lse [B, H, Tq] (log2 units, +inf without a visible key),
    pv [B Tq, H dk] = P |V|, and the per-head intermediates the bounds and the backward use."""
    qh, kh, vh = heads(q, col0s[0], B, H, Tq, d_k), heads(k, col0s[1], B, H, Tk, d_k), heads(v, col0s[2], B, H, Tk, d_k)
    vis = visible(B, Tq, Tk, kv_len, causal, q.device, mutate)
    t = qh @ kh.transpose(-1, -2)
    if bd is not None:
        t = t + band(bd, B, H, Tq, Tk, shift=1 if mutate == 'band_shift' else 0)
    t = t.masked_fill(~vis, 0.0)
    scale = 0.125 if mutate == 'scale_64' else 1.0 / math.sqrt(d_k)
    z = (t * scale).masked_fill(~vis, float('-inf'))
    m = z.amax(-1, keepdim=True)
    m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    e = torch.exp(z - m)
    l = e.sum(-1, keepdim=True)
    P = e / torch.where(l > 0, l, torch.ones_like(l))
    O = P @ vh
    any_vis = vis.any(-1).expand(B, H, Tq)
    lse = (m + torch.log(torch.where(l > 0, l, torch.ones_like(l)))).squeeze(-1) * LOG2E
    lse = torch.where(any_vis, lse, torch.full_like(lse, float('inf')))
    if mutate == 'lse_natural':
        lse = lse * LN2
    out = flat(O)
    rh = None
    if resid is not None:
        rh = heads(resid, 0, B, H, Tq, d_k)
        out = out + flat(rh)
    return dict(out=out, lse=lse, pv=flat(P @ vh.abs()), O=O, P=P, t=t, vis=vis, qh=qh, kh=kh, vh=vh, rh=rh,
                dims=(B, H, Tq, Tk, d_k), causal=causal, kv_len=kv_len)


def _c_err(d_k):
    """Relative error of the fp32 c = log2(e) / sqrt(d_k) the host computes: log2(e) rounded, and at d_k 96 sqrtf and the
    division rounded too (d_k 64: both exact)."""
    return U if d_k == 64 else 3 * U


def _sum_err(n):
    return n * U / (1 - n * U)


def forward_bounds(F):
    """-> dict out [B Tq, H dk], lse [B, H, Tq] (module docstring)."""
    B, H, Tq, Tk, d_k = F['dims']
    vis, t = F['vis'], F['t']
    c = LOG2E / math.sqrt(d_k)
    E = d_k * ACC * (F['qh'].abs() @ F['kh'].abs().transpose(-1, -2)) + U * t.abs()
    ct = (c * t.abs()).masked_fill(~vis, 0.0)
    M = ct.amax(-1, keepdim=True)                                     # |m| <= max_row c |t|
    arg = c * E + _c_err(d_k) * ct + U * (ct + M)
    delta = (torch.exp2(arg) * (1 + EPS_EX2) - 1).masked_fill(~vis, 0.0)
    dmax = delta.amax(-1, keepdim=True)
    K = _pad128(Tk)
    lam = (1 + dmax) * (1 + _sum_err(K)) - 1
    rho = (1 + dmax) * (1 + UB) / (1 - lam) - 1
    nblk = math.ceil(Tk / 128)
    coef = rho + (K * ACC + 2 * U + 2 * nblk * U) * (1 + rho)
    flush = Tk * 2.0 ** -126 * float(F['vh'].abs().max()) if F['vh'].numel() else 0.0
    e1 = flat(coef.expand(B, H, Tq, d_k)) * F['pv'] + flush
    y = F['out'].abs()
    e2 = e1 + U * (y + e1)
    out = e2 + UB * (y + e2)
    a = (1 + EPS_EX2) * torch.exp2(2 * U * M) * (1 + U) - 1
    x = dmax + _sum_err(K) + nblk * a
    lse = (-torch.log2(1 - x) + 2 * U * (math.log2(K) + 1)).squeeze(-1) + U * (F['lse'].abs() + 1)
    any_vis = vis.any(-1).expand(B, H, Tq)
    lse = torch.where(any_vis, lse, torch.zeros_like(lse))
    return dict(out=out, lse=lse, E=E, ct=ct)


def backward(F, dout, mutate=None):
    """True float64 gradients of sum(out * dout) -> dict dq [B Tq, H dk], dk, dv [B Tk, H dk], D [B, H, Tq] (from the exact
    O), dS [B, H, Tq, Tk] (the gradient of the raw score t, so also of the band: dBD)."""
    B, H, Tq, Tk, d_k = F['dims']
    do = heads(dout, 0, B, H, Tq, d_k)
    P, O = F['P'], F['O']
    D = (do * (F['vh'][..., :Tq, :] if mutate == 'D_from_dOV' else O)).sum(-1)
    dP = do @ F['vh'].transpose(-1, -2)
    scale = 1.0 if mutate == 'ds_no_scale' else 1.0 / math.sqrt(d_k)
    dS = P * (dP - D[..., None]) * scale
    dq, dk, dv = dS @ F['kh'], dS.transpose(-1, -2) @ F['qh'], P.transpose(-1, -2) @ do
    return dict(dq=flat(dq), dk=flat(dk), dv=flat(dv), D=D, dS=dS, do=do, dP=dP)


def dsum_ref(out, dout, B, H, Tq, d_k=64):
    """D over the bf16 out the backward is given, and its bound -> (D [B, H, Tq], bound)."""
    o, do = heads(out, 0, B, H, Tq, d_k), heads(dout, 0, B, H, Tq, d_k)
    return (do * o).sum(-1), d_k * U * (do.abs() * o.abs()).sum(-1)


def backward_bounds(F, G, FB, out):
    """Bounds of dq, dk, dv, dS (= dBD) and D from the forward F, its bounds FB, the gradients G and the bf16 out the
    backward reads (module docstring)."""
    B, H, Tq, Tk, d_k = F['dims']
    vis, P, do = F['vis'], F['P'], G['do']
    c = LOG2E / math.sqrt(d_k)
    oh = heads(out, 0, B, H, Tq, d_k)
    dL = torch.where(torch.isfinite(F['lse']), FB['lse'], torch.zeros_like(FB['lse']))
    L = torch.where(torch.isfinite(F['lse']), F['lse'], torch.zeros_like(F['lse']))
    arg = c * FB['E'] + U * (FB['ct'] + L.abs()[..., None] + dL[..., None]) + _c_err(d_k) * FB['ct'] + dL[..., None]
    pi = (torch.exp2(arg) * (1 + EPS_EX2) - 1).masked_fill(~vis, 0.0)
    edp = d_k * ACC * (do.abs() @ F['vh'].abs().transpose(-1, -2))
    eD = d_k * U * (do.abs() * oh.abs()).sum(-1) + (do.abs() * heads(FB['out'], 0, B, H, Tq, d_k)).sum(-1)
    g = (G['dP'] - G['D'][..., None]).abs()
    eg = edp + eD[..., None]
    eg = eg + U * (g + eg)
    s = 1.0 / math.sqrt(d_k)
    eS = (P * ((1 + pi) * (g + eg) * (1 + U) ** 2 - g) * s).masked_fill(~vis, 0.0)
    aS = G['dS'].abs()
    eSb = eS + UB * (aS + eS)
    aSb = aS + eSb
    Kk, Kq = _pad128(Tk), _pad128(Tq)

    def out_round(e, ref):
        return e + UB * (ref.abs() + e)
    kh, qh = F['kh'].abs(), F['qh'].abs()
    dq = out_round(flat(eSb @ kh + Kk * ACC * (aSb @ kh)), G['dq'])
    dk = out_round(flat(eSb.transpose(-1, -2) @ qh + Kq * ACC * (aSb.transpose(-1, -2) @ qh)), G['dk'])
    eP = P * ((1 + pi) * (1 + UB) - 1)
    aP = P + eP
    dv = out_round(flat(eP.transpose(-1, -2) @ do.abs() + Kq * ACC * (aP.transpose(-1, -2) @ do.abs())), G['dv'])
    return dict(dq=dq, dk=dk, dv=dv, dS=eSb)


def band_layout(x, vis, B, H, Tq, ld):
    """[B, H, Tq, Tk] values at the visible (i, j) -> ([H, B Tq, ld] with them at column j - i + Tq - 1, written mask)."""
    dev = x.device
    outv = torch.zeros(H, B * Tq, ld, dtype=x.dtype, device=dev)
    written = torch.zeros(H, B * Tq, ld, dtype=torch.bool, device=dev)
    idx = (torch.arange(Tq, device=dev)[None, :] - torch.arange(Tq, device=dev)[:, None] + Tq - 1).expand(B, H, Tq, Tq)
    v4 = vis.expand(B, H, Tq, Tq)
    o4 = outv.view(H, B, Tq, ld).transpose(0, 1)
    w4 = written.view(H, B, Tq, ld).transpose(0, 1)
    o4.scatter_(3, idx, x.masked_fill(~v4, 0.0))
    w4.scatter_(3, idx, v4)
    return outv, written


def check(name, got, ref, bound):
    """|got - ref| <= bound element by element (inf == inf counts as exact; NaN fails).  Prints the worst err/bound and
    the worst |err|, returns the worst err/bound, and raises AssertionError naming the first offending indices."""
    got = got.double()
    same = got == ref
    err = torch.where(same, torch.zeros_like(got), (got - ref).abs())
    ok = err <= bound
    ratio = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                        torch.where(err > 0, torch.full_like(err, float('inf')), torch.zeros_like(err)))
    ratio = torch.where(torch.isnan(err), torch.full_like(err, float('inf')), ratio)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    fin = err[torch.isfinite(err)]
    print(f'  {name}: worst err/bound {worst:.3g}, worst |err| {float(fin.max()) if fin.numel() else 0.0:.3g}')
    if not bool(ok.all()):
        bad = (~ok).nonzero()[:4].tolist()
        first = tuple(bad[0])
        raise AssertionError(f'{name}: {int((~ok).sum())} elements out of bound, first at {bad}: got {float(got[first])}, '
                             f'ref {float(ref[first])}, bound {float(bound[first])}')
    return worst


# ------------------------------------------------------------------------------------------------ the case table
# (name, d_k, B, H, Tq, Tk, kv_len (list or None), causal, band, resid, train (lse + backward), layout, pitch pad, Q scale,
#  input patterns).  layout: 'qkv' one [M, 3d] buffer; 'relpos' [M, 4d] with k_col0 = 2d, v_col0 = 3d; 'sep' q and a
#  [M, 2d] K|V buffer.  Patterns: 'rising' scores rise along the keys (the running max moves in every block); 'block0'
#  the maximum in block 0 and every later block underflows; 'flat' rows whose visible scores are all equal; 'garbage'
#  finite +-1e4 in the K/V rows past kv_len; 'band50' a band of +-50.  Every case also plants one query row per edge key.
CASES = [
    ('enc_bench', 64, 32, 4, 249, 249, 'ragged', False, False, False, True, 'qkv', 0, 1.0, ()),
    ('dec_self_bench', 64, 32, 4, 31, 31, None, True, False, False, True, 'qkv', 0, 1.0, ()),
    ('cross_bench', 64, 32, 4, 31, 249, 'ragged', False, False, False, True, 'sep', 0, 1.0, ('garbage',)),
    ('mwer_self', 64, 40, 4, 31, 31, None, True, False, False, True, 'qkv', 0, 1.0, ()),
    ('mwer_cross', 64, 8, 4, 124, 249, 'ragged', False, False, False, True, 'sep', 0, 1.0, ()),
    ('enc_full', 64, 32, 4, 249, 249, None, False, False, False, True, 'qkv', 0, 1.0, ()),
    ('peaked_249', 64, 3, 4, 249, 249, 'ragged', False, False, False, True, 'qkv', 0, 4.0, ()),
    ('kv_edges', 64, 9, 2, 257, 257, [0, 1, 127, 128, 129, 255, 256, 257, 262], False, False, False, True, 'sep', 16, 1.0,
     ('garbage', 'flat')),
    ('causal_300', 64, 2, 2, 300, 300, None, True, False, False, True, 'qkv', 8, 4.0, ('rising',)),
    ('exact_128', 64, 1, 4, 128, 128, None, False, False, False, True, 'qkv', 0, 1.0, ()),
    ('cross_257_130', 64, 3, 1, 257, 130, [130, 0, 129], False, False, False, True, 'sep', 0, 1.0, ()),
    ('kv_edges_cross', 64, 7, 2, 40, 257, [0, 1, 127, 128, 129, 255, 256], False, False, False, True, 'sep', 8, 1.0,
     ('garbage',)),
    ('causal_q_gt_k', 64, 3, 2, 257, 129, [129, 7, 128], True, False, False, True, 'sep', 0, 1.0, ()),
    ('causal_q_lt_k', 64, 3, 2, 129, 257, [257, 200, 1], True, False, False, True, 'sep', 8, 1.0, ('block0',)),
    ('peaked_1000', 64, 2, 2, 1000, 1000, [999, 1000], False, False, False, True, 'qkv', 0, 4.0, ('garbage',)),
    ('tiny', 64, 3, 2, 1, 1, None, False, False, False, True, 'qkv', 0, 1.0, ()),
    ('tiny_cross', 64, 3, 2, 1, 7, [7, 0, 3], False, False, False, True, 'sep', 0, 1.0, ()),
    ('band64_train', 64, 3, 4, 255, 255, [255, 170, 0], False, True, False, True, 'relpos', 0, 1.0, ('band50',)),
    ('band64_128', 64, 2, 2, 128, 128, [128, 127], False, True, False, True, 'relpos', 8, 1.0, ('band50', 'garbage')),
    ('band64_7', 64, 2, 4, 7, 7, [7, 1], False, True, False, True, 'relpos', 0, 1.0, ()),
    ('band64_200', 64, 3, 4, 200, 200, [200, 133, 0], False, True, False, True, 'relpos', 0, 1.0, ()),
    ('band64_249', 64, 3, 4, 249, 249, [249, 166, 0], False, True, False, True, 'relpos', 0, 1.0, ()),
    ('band64_300', 64, 3, 4, 300, 300, [300, 200, 0], False, True, False, True, 'relpos', 0, 1.0, ()),
    ('band96_resid', 96, 3, 4, 249, 249, 'ragged', False, True, True, False, 'relpos', 8, 1.0, ('band50',)),
    ('band96_256', 96, 2, 4, 256, 256, [256, 129], False, True, True, False, 'relpos', 0, 1.0, ('flat',)),
    ('dk96_1000', 96, 2, 4, 999, 999, [999, 500], False, False, True, False, 'qkv', 8, 1.0, ('rising', 'garbage')),
    ('dk96_causal', 96, 2, 4, 257, 257, None, True, False, False, False, 'qkv', 0, 4.0, ('block0',)),
    ('dk96_cross', 96, 3, 4, 7, 1000, [1000, 0, 128], False, False, False, False, 'sep', 16, 1.0, ('flat', 'garbage')),
    ('dk64_resid_127', 64, 3, 2, 127, 127, [127, 126, 0], False, False, True, False, 'sep', 8, 1.0, ()),
]
NAMES = [c[0] for c in CASES]
CASE = {c[0]: c for c in CASES}


def kv_list(c):
    name, dk, B, H, Tq, Tk, kv = c[:7]
    if kv == 'ragged':
        return [Tk - (7 * i) % max(1, Tk // 2) for i in range(B)]
    return kv


# ------------------------------------------------------------------------------------------------ what the table reaches
FWD_BRANCHES = ('causal', 'kv_len', 'resid', 'no_block', 'multiblock', 'tail')
DKV_BRANCHES = ('causal_iblk0', 'dead_tile', 'tq_gt_tk', 'tq_lt_tk')
# every instantiation and runtime branch the host and the kernels can take
REACHABLE = ({('fwd', dk, 'band' if bd else 'plain') for dk in (64, 96) for bd in (False, True)}
             | {('fwd', dk, br) for dk in (64, 96) for br in FWD_BRANCHES} | {('fwd', 64, 'lse')}
             | {('bwd', 'band' if bd else 'plain') for bd in (False, True)} | {('dkv', br) for br in DKV_BRANCHES})


def cells(c):
    """The cells of REACHABLE case c reaches, read off attn_tc.cu / attn_bwd.cu's control flow; a configuration the host
    refuses yields a cell outside REACHABLE."""
    name, dk, B, H, Tq, Tk, kv, causal, bd, resid, train = c[:11]
    lens = [min(x, Tk) for x in (kv_list(c) or [Tk] * B)]
    out = {('fwd', dk, 'band' if bd else 'plain')}
    if bd and (causal or Tq != Tk):
        out.add(('fwd', dk, 'band_needs_self_noncausal'))
    br = set()
    if causal:
        br.add('causal')
    if kv is not None:
        br.add('kv_len')
    if resid:
        br.add('resid')
    if Tq % 128:
        br.add('tail')
    for L in lens:
        for q0 in range(0, Tq, 128):
            kv_end = min(L, q0 + 128) if causal else L
            br.add('no_block' if kv_end == 0 else ('multiblock' if kv_end > 128 else 'one_block'))
    br.discard('one_block')
    out |= {('fwd', dk, x) for x in br}
    if train:
        out.add(('fwd', dk, 'lse'))
        out.add(('bwd', 'band' if bd else 'plain'))
        if resid:
            out.add(('bwd', 'resid'))
        nq = (Tq + 127) // 128
        for L in lens:
            for j0 in range(0, Tk, 128):
                if j0 >= L:
                    out.add(('dkv', 'dead_tile'))
                elif causal and j0 // 128 > 0 and j0 // 128 < nq:
                    out.add(('dkv', 'causal_iblk0'))
        if Tq > Tk:
            out.add(('dkv', 'tq_gt_tk'))
        if Tq < Tk:
            out.add(('dkv', 'tq_lt_tk'))
    return out


# ------------------------------------------------------------------------------------------------ inputs
def edge_keys(L, Tk):
    return sorted({j for j in (0, 127, 128, L - 1) if 0 <= j < L})


def make_inputs(c, seed=0):
    """bf16 CPU operands of case c in its layout: dict q, k, v (matrices), col0s, kv_len (int32 or None), bd (f32
    [H, B Tq, ld] or None), resid, dout, and planted [(b, i, j)]: query rows aimed at an edge key."""
    name, dk, B, H, Tq, Tk, kv, causal, bd_on, resid_on, train, layout, pad, qs, pats = c
    g = torch.Generator().manual_seed(seed + sum(map(ord, name)))
    d = H * dk
    lens = kv_list(c)
    kv_len = torch.tensor(lens, dtype=torch.int32) if lens is not None else None
    lim = [min(x, Tk) for x in (lens or [Tk] * B)]
    qh = torch.randn(B, H, Tq, dk, generator=g) * qs
    kh = torch.randn(B, H, Tk, dk, generator=g)
    vh = torch.randn(B, H, Tk, dk, generator=g)
    if 'rising' in pats:        # + 32 j / Tk on every score: the running max moves in every key block
        qh[..., 0] = 4.0
        kh[..., 0] = 8.0 * torch.arange(Tk) / Tk
    if 'block0' in pats:        # +-512 from two dims: block 0 holds the maximum, the later blocks underflow to 0
        qh[..., :2] = 16.0
        kh[..., :2] = torch.where(torch.arange(Tk) < 128, 16.0, -16.0)[:, None]
    if 'flat' in pats:          # q = 0: every visible score of the row equal
        qh[:, :, 2::5] = 0.0
    planted = []
    for b in range(B):
        L = lim[b]
        targets = edge_keys(L, Tk)
        if causal:
            targets += [j for j in (min(L, Tq) - 1, 128, 129) if 0 <= j < min(L, Tq)]   # the diagonal
        used = set()
        for j in targets:
            # a query row that sees key j: on the diagonal for causal rows aimed at the diagonal, else any free row
            cand = [i for i in range(Tq) if i not in used and (not causal or j <= i)]
            if causal and j < Tq and j not in used:
                cand = [j] + cand
            if not cand:
                continue
            i = cand[0] if causal else cand[(7 * j + 3) % len(cand)]
            used.add(i)
            n = max(1, min(L, i + 1) if causal else L)
            kn2 = (kh[b, :, j] ** 2).sum(-1, keepdim=True)
            target = math.log(4.5 * n + 1) + 1.0                   # P_ij about 0.6-0.9
            qh[b, :, i] = kh[b, :, j] * (target * math.sqrt(dk) / kn2)
            planted.append((b, i, j))
    if 'garbage' in pats:
        for b in range(B):
            kh[b, :, lim[b]:] = 1e4 * torch.sign(torch.randn(H, Tk - lim[b], dk, generator=g))
            vh[b, :, lim[b]:] = -1e4 * torch.sign(torch.randn(H, Tk - lim[b], dk, generator=g))
    to_m = lambda t: t.transpose(1, 2).reshape(t.shape[0] * t.shape[2], H * dk)   # noqa: E731
    Q, Kt, V = to_m(qh), to_m(kh), to_m(vh)
    nan = float('nan')
    if layout == 'qkv':
        assert Tq == Tk
        m = torch.full((B * Tq, 3 * d + pad), nan)
        m[:, :d], m[:, d:2 * d], m[:, 2 * d:3 * d] = Q, Kt, V
        m = m.to(torch.bfloat16)
        q = k = v = m
        col0s = (0, d, 2 * d)
    elif layout == 'relpos':
        assert Tq == Tk
        m = torch.full((B * Tq, 4 * d + pad), nan)
        m[:, :d] = Q
        m[:, d:2 * d] = torch.randn(B * Tq, d, generator=g)
        m[:, 2 * d:3 * d], m[:, 3 * d:4 * d] = Kt, V
        m = m.to(torch.bfloat16)
        q = k = v = m
        col0s = (0, 2 * d, 3 * d)
    else:
        q = torch.full((B * Tq, d + pad), nan)
        q[:, :d] = Q
        kvm = torch.full((B * Tk, 2 * d + pad), nan)
        kvm[:, :d], kvm[:, d:2 * d] = Kt, V
        q, k = q.to(torch.bfloat16), kvm.to(torch.bfloat16)
        v = k
        col0s = (0, 0, d)
    bd = None
    if bd_on:
        ld = (2 * Tq - 1 + 3) // 4 * 4
        amp = 50.0 if 'band50' in pats else 2.0
        bd = torch.zeros(H, B * Tq, ld)
        bd[..., :2 * Tq - 1] = amp * (2 * torch.rand(H, B * Tq, 2 * Tq - 1, generator=g) - 1)
        for b, i, _ in planted:            # planted rows keep their aim
            bd[:, b * Tq + i] = 0.0
    resid = torch.randn(B * Tq, d, generator=g).to(torch.bfloat16) if resid_on else None
    dout = torch.randn(B * Tq, d, generator=g).to(torch.bfloat16)
    return dict(q=q, k=k, v=v, col0s=col0s, kv_len=kv_len, bd=bd, resid=resid, dout=dout, planted=planted)


def run_reference(c, X, device, mutate=None):
    """The float64 forward (the dict of forward()) of case c on inputs X, on `device`."""
    name, dk, B, H, Tq, Tk, kv, causal = c[:8]
    to = lambda t: t.to(device) if t is not None else None   # noqa: E731
    F = forward(to(X['q']), to(X['k']), to(X['v']), B, H, Tq, Tk, to(X['kv_len']), causal, X['col0s'], to(X['bd']),
                to(X['resid']), dk, mutate=mutate)
    return F


# ------------------------------------------------------------------------------------------------ emulation
def emulate(c, X):
    """The kernels' arithmetic on the CPU: fp32 scores from the bf16 operands, the max and exp2 in fp32, P rounded to bf16
    before PV, an fp32 row sum of the unrounded p, bf16 outputs; the backward recomputes P from the fp32 lse, takes D
    from the bf16 O and rounds dS (and P for dV) to bf16 before the GEMMs.  -> dict out, lse (+ dsum, dq, dk, dv, dS)."""
    name, dk, B, H, Tq, Tk, kv, causal, bd_on, resid_on, train = c[:11]
    f = torch.float32
    qh, kh, vh = (heads(X['q'], X['col0s'][0], B, H, Tq, dk).float(), heads(X['k'], X['col0s'][1], B, H, Tk, dk).float(),
                  heads(X['v'], X['col0s'][2], B, H, Tk, dk).float())
    vis = visible(B, Tq, Tk, X['kv_len'], causal, 'cpu')
    vh = vh.masked_fill(~vis.any(2)[..., None].expand(B, 1, Tk, 1), 0.0)   # P = 0 there; keeps 0 * 1e4 out of fp32 sums
    t = qh @ kh.transpose(-1, -2)
    if X['bd'] is not None:
        t = t + band(X['bd'], B, H, Tq, Tk).float()
    cc = torch.tensor(LOG2E, dtype=f) / torch.sqrt(torch.tensor(float(dk), dtype=f))
    s = (t * cc).masked_fill(~vis, float('-inf'))
    m = s.amax(-1, keepdim=True)
    m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    p = torch.exp2(s - m)
    l = p.sum(-1, keepdim=True)
    o = p.to(torch.bfloat16).float() @ vh
    O = o * torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
    out = flat(O)
    if X['resid'] is not None:
        out = out + X['resid'].float()
    out = out.to(torch.bfloat16)
    lse = torch.where(l > 0, m + torch.log2(l), torch.full_like(l, float('inf'))).squeeze(-1)
    R = dict(out=out, lse=lse)
    if not train:
        return R
    do = heads(X['dout'], 0, B, H, Tq, dk).float()
    ob = heads(out, 0, B, H, Tq, dk).float()
    D = (do * ob).sum(-1)
    P = torch.exp2(torch.where(vis, t * cc - lse[..., None].nan_to_num(posinf=0.0), torch.full_like(t, float('-inf'))))
    dP = do @ vh.transpose(-1, -2)
    dS = (P * (dP - D[..., None]) * 0.125).masked_fill(~vis, 0.0).to(torch.bfloat16).float()
    R.update(dsum=D, dS=dS,
             dq=flat(dS @ kh).to(torch.bfloat16),
             dk=flat(dS.transpose(-1, -2) @ qh).to(torch.bfloat16),
             dv=flat(P.to(torch.bfloat16).float().transpose(-1, -2) @ do).to(torch.bfloat16))
    return R
