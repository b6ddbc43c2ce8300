"""The transducer's training kernels (csrc/rnnt.cu, csrc/rnnt_pruned.cu) restated in float64 on the kernels' own f32 or
bf16 operands, with the error bound of each output -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

lattice() runs alpha and beta of one utterance over the anti-diagonals t + u with numpy (full or banded lattice), so
T ~ 1000 frames against 1023 labels takes seconds.  simple_z() is the simple joint's normalizer as max + log-sum-exp of
am[t] + lm[u] directly, not factored.  The bounds (u = 2^-24, f32 unit roundoff, so one ulp is at most 2 u relative;
CUDA's expf and tanhf are within 2 ulp, 4 u, and logf within 1 ulp, 2 u) are first-order sums of the relative errors
each kernel's arithmetic can make; each function says which arithmetic it covers.  tests/test_gpu_rnnt_kernels.py
prints every measured error as a ratio to its bound.
"""
import math

import numpy as np

U = 2.0 ** -24          # f32 unit roundoff
U64 = 2.0 ** -53        # f64 unit roundoff
NINF = -np.inf


# ------------------------------------------------------------------------------------------------ the lattice
def band_keep(T, U1, s=None, S=None):
    """[T, U1] bool: the nodes that exist (every node, or s_t <= u < s_t + S)."""
    if s is None:
        return np.ones((T, U1), dtype=bool)
    u = np.arange(U1)[None, :]
    st = np.asarray(s, dtype=np.int64)[:, None]
    return (u >= st) & (u < st + S)


def lattice(lpb, lpy, s=None, S=None):
    """One utterance of T frames and U labels: lpb [T, U + 1] log p(blank), lpy [T, >= U] log p(y_{u+1}) (float64), the
    band s [T] of width S or None -> dict(alpha, beta [T, U + 1] (-inf at missing nodes), logp, gb, gy [T, U + 1]) with
    gb, gy = exp(alpha + lp + beta(next) - logp), the posterior of each arc (the nll's gradient is -gb, -gy); all zero
    when no alignment exists (logp = -inf)."""
    lpb = np.asarray(lpb, dtype=np.float64)
    T, U1 = lpb.shape
    Ul = U1 - 1
    ly = np.full((T, U1), NINF)
    ly[:, :Ul] = np.asarray(lpy, dtype=np.float64)[:, :Ul]
    keep = band_keep(T, U1, s, S)
    alpha = np.full((T, U1), NINF)
    beta = np.full((T, U1), NINF)
    with np.errstate(invalid='ignore'):
        for d in range(T + Ul):
            u = np.arange(max(0, d - T + 1), min(d, Ul) + 1)
            t = d - u
            a = np.where(d == 0, 0.0, NINF) * np.ones(len(u))
            tb = t > 0
            a[tb] = alpha[t[tb] - 1, u[tb]] + lpb[t[tb] - 1, u[tb]]
            uy = u > 0
            a[uy] = np.logaddexp(a[uy], alpha[t[uy], u[uy] - 1] + ly[t[uy], u[uy] - 1])
            alpha[t, u] = np.where(keep[t, u], a, NINF)
        for d in range(T + Ul - 1, -1, -1):
            u = np.arange(max(0, d - T + 1), min(d, Ul) + 1)
            t = d - u
            bt = np.full(len(u), NINF)
            nt = t + 1 < T
            bt[nt] = beta[t[nt] + 1, u[nt]]
            bt[(t == T - 1) & (u == Ul)] = 0.0
            bu = np.full(len(u), NINF)
            nu = u < Ul
            bu[nu] = beta[t[nu], u[nu] + 1]
            b = np.logaddexp(bt + lpb[t, u], bu + ly[t, u])
            beta[t, u] = np.where(keep[t, u], b, NINF)
        logp = alpha[T - 1, Ul] + lpb[T - 1, Ul]
        nxt_b = np.full((T, U1), NINF)
        nxt_b[:-1] = beta[1:]
        nxt_b[T - 1, Ul] = 0.0
        nxt_y = np.full((T, U1), NINF)
        nxt_y[:, :-1] = beta[:, 1:]
        if logp == NINF:
            gb = gy = np.zeros((T, U1))
        else:
            gb = np.where(keep, np.exp(alpha + lpb + nxt_b - logp), 0.0)
            gy = np.where(keep, np.exp(alpha + ly + nxt_y - logp), 0.0)
    return dict(alpha=alpha, beta=beta, logp=logp, gb=np.nan_to_num(gb), gy=np.nan_to_num(gy))


def loss_bound(lat, T, Ul):
    """otb_rnnt_loss: the recursion in fp64 (each of the T + U steps one logadd: exp, log1p, two adds, within 4 f64
    roundings of its magnitude; the restatement's the same), then one f32 rounding of -logp.  -> the bound on |nll - want|
    and the relative bound on each node gradient -gs exp(e): exp(e) in fp64 from the same fp64 terms, one f32 rounding, the
    f32 scale gs = (grad_scale * scale_dev) / B (two roundings) and the product (one): 4 u, plus the fp64 error of e."""
    fin = np.isfinite(lat['alpha'])
    mag = 1.0 + (np.abs(lat['alpha'][fin]).max() if fin.any() else 0.0) + (
        np.abs(lat['beta'][np.isfinite(lat['beta'])]).max() if np.isfinite(lat['beta']).any() else 0.0)
    e64 = 8.0 * (T + Ul + 2) * U64 * mag
    nll = U * abs(lat['logp']) + e64 if np.isfinite(lat['logp']) else 0.0
    return nll, 4 * U + 2 * e64


# ------------------------------------------------------------------------------------------------ per-row log-probs
def row_lse(x):
    """x [rows, V] float64 -> (m, s, lse, the mean gap m - E_p[x] with p = softmax(x))."""
    m = x.max(-1)
    e = np.exp(x - m[:, None])
    s = e.sum(-1)
    gap = m - (e * x).sum(-1) / s if x.shape[0] else m
    return m, s, m + np.log(s), gap


def row_lse_rel(V, gap):
    """Relative error bound of warp_row_lse's s, in u: every term passes through one expf (4 u), at most R = ceil(V / 512)
    + 1 + 5 rescales of its lane's sum (expf 4 u and a product 1 u each; the rounded arguments m - m' telescope into the
    term's own gap x - m, u |x - m| first order, whose p-weighted mean is `gap`) and at most 4 ceil(V / 512) + 8
    additions of the float4 chains plus 5 of the xor tree."""
    it = -(-V // 512)
    R = it + 6
    return 4 + 5 * R + 4 * it + 13 + gap


def logprob_bound(x64, y_cols):
    """otb_rnnt_logprob on f32 rows x64 [rows, V] (as float64), y_cols [rows] the label column or -1 -> (want [rows, 3],
    bound [rows, 3]): lse = m + logf(s) (the s error, logf 2 u |log s|, the add: u |lse|); log p(k) = (x_k - m) - logf(s)
    (u |x_k - m|, the same, u |log p|)."""
    m, s, lse, gap = row_lse(x64)
    rel = row_lse_rel(x64.shape[1], gap)
    ls = np.log(s)
    r = np.arange(x64.shape[0])
    xy = np.where(y_cols >= 0, x64[r, np.maximum(y_cols, 0)], NINF)
    want = np.stack([lse, x64[:, 0] - lse, xy - lse], 1)
    base = rel + 2 * np.abs(ls)
    with np.errstate(invalid='ignore'):
        bound = U * np.stack([base + np.abs(lse),
                              base + np.abs(x64[:, 0] - m) + np.abs(want[:, 1]),
                              np.where(y_cols >= 0, base + np.abs(xy - m) + np.abs(want[:, 2]), 0.0)], 1)
    return want, bound


def dlogits_bound(x64, lse, a, c, y_cols):
    """otb_rnnt_dlogits: dz_k = [k = 0] a + [k = y] c - exp(x_k - lse) (a + c) from the kernel's own f32 lse and (a, c)
    -> (want, abs_tol): a + c (u), x_k - lse (u |x_k - lse|, into the exponential), expf (4 u), the product (u), the two
    sums (u |a| + u |c| and u |dz|), before the bf16 rounding; an exponential below 2^-126 is within 2^-149, so the
    product within 2^-149 |a + c|."""
    rows, V = x64.shape
    ac = a + c
    p = np.exp(x64 - lse[:, None])
    want = -p * ac[:, None]
    want[:, 0] += a
    r = np.nonzero(y_cols >= 0)[0]
    want[r, y_cols[r]] += c[r]
    tol = U * (np.abs(p * ac[:, None]) * (7 + np.abs(x64 - lse[:, None])) + 2 * (np.abs(a) + np.abs(c))[:, None]
               + np.abs(want)) + 2.0 ** -149 * np.abs(ac)[:, None]
    return want, tol


# ------------------------------------------------------------------------------------------------ the joint
def joint(ep, pp):
    """tanh(ep + pp) in float64, ep [..., D] and pp [..., D] the bf16 operands -> (want, abs_tol): the f32 sum (u |e + p|,
    through tanh' <= 1) and tanhf (4 u |tanh|), before the bf16 rounding."""
    z = ep + pp
    want = np.tanh(z)
    return want, U * (np.abs(z) * (1 - want ** 2) + 4 * np.abs(want))


def joint_bwd_bound(g, n):
    """One output column: the n terms g_k (1 - y_k^2) of dZ summed in ascending order in f32: each term within 3 u |g_k|
    (y^2, 1 - y^2 and the product, |y| <= 1), and n - 1 additions at most (n - 1) u sum |g_k| -> the abs_tol of the f32
    sum before the bf16 rounding, from sum_k |g_k| (float64)."""
    return U * (n + 3) * g


# ------------------------------------------------------------------------------------------------ the simple joint
def simple_z(am, lm):
    """Z [T, U1] = logsumexp_v (am[t, v] + lm[u, v]) in float64 directly (am [T, V], lm [U1, V]), with the p-weighted mean
    of (m_t - am[t, v]) + (m_u - lm[u, v]) and of |am + lm|, chunked over t."""
    T, U1 = am.shape[0], lm.shape[0]
    Z = np.empty((T, U1))
    gap = np.empty((T, U1))
    mx = np.empty((T, U1))
    mt, mu = am.max(1), lm.max(1)
    step = max(1, int(4e6 // max(1, U1 * am.shape[1])))
    for t0 in range(0, T, step):
        x = am[t0:t0 + step, None, :] + lm[None, :, :]
        m = x.max(-1)
        e = np.exp(x - m[..., None])
        s = e.sum(-1)
        Z[t0:t0 + step] = m + np.log(s)
        gap[t0:t0 + step] = mt[t0:t0 + step, None] + mu[None, :] - (e * x).sum(-1) / s
        mx[t0:t0 + step] = np.abs(x).max(-1)
    return Z, gap, mx


def simple_lse_bound(am, lm, Z, gap, mx):
    """otb_rnnt_simple_lse's Z, either path.  Factored: exp(x - m) of each operand (4 u each, and the rounded argument:
    u (m_t - am) + u (m_u - lm), p-weighted = gap), the V-term fmaf sum (V u), logf (2 u |log acc|), the two adds
    (u |m_t + m_u| + u |Z|).  Direct: am + lm (u |am + lm| <= u mx), the argument and expf, V additions, logf, one add.
    Both are within u (V + 10 + gap + |m_t + m_u| + 2 |Z - m_t - m_u| + |Z| + mx), plus the subnormal terms of the
    factored sum: within 2^-149 each, V 2^-149 against acc >= 2^-100, V 2^-49 in Z."""
    mt, mu = am.max(1)[:, None], lm.max(1)[None, :]
    V = am.shape[1]
    return U * (V + 10 + gap + np.abs(mt + mu) + 2 * np.abs(Z - mt - mu) + np.abs(Z) + mx) + V * 2.0 ** -49


def simple_bwd(am, lm, Z, ga, gc, labels, Ub, sc):
    """d am [T, V] and d lm [U1, V] of one utterance (T = T_b frames, U1 = U_b + 1 positions) from the kernel's own f32
    operands: am, lm, its Z [T, U1] and node gradients (a, c) [T, U1], scale sc (float64) ->
    (d_am, d_lm, tol_am, tol_lm), tol the abs_tol before the bf16 rounding.
      d am[t,v] = sum_u sc ([v = 0] a + [v = y_{u+1}] c) - sum_u sc (a + c) exp(am[t,v] + lm[u,v] - Z[t,u]), lm the same.
    The f32 arithmetic: w = sc (a + c) (2 u), exp(m_t + m_u - Z) (argument u (|m_t + m_u| + |gap|), expf 4 u, product u),
    each exp(x - m) (4 u, argument u (m - x)), the reduction's fmaf sum over n rows (n u), the final product and difference
    (2 u): each |term| within u (n + 18 + K), K the largest |m_t + m_u| + |m_t + m_u - Z| + (m_t - am) + (m_u - lm) over
    the live entries; the one-hot part's n-term ascending sum (n u of its |terms|); the exact terms of the nodes whose Z
    came directly (am + lm, the argument, expf, product, sum: within the same).  An exponential factor below 2^-126 is
    within 2^-149 absolute, so each product P exp(x - m) exp(y - m') within 2^-148 |P| (both factors <= 1), with
    |P| <= |w| 2^100 for the factored nodes; each exact term w exp(x + y - Z) within 2^-149 |w|."""
    T, V = am.shape
    U1 = lm.shape[0]
    w = sc * (ga + gc)
    mt, mu = am.max(1), lm.max(1)
    ea, el = np.exp(am - mt[:, None]), np.exp(lm - mu[:, None])
    E = np.exp(mt[:, None] + mu[None, :] - Z)
    P = w * E
    Pa = np.abs(w) * E
    D_am = np.zeros((T, V))
    D_lm = np.zeros((U1, V))
    Da_abs = np.zeros((T, V))
    Dl_abs = np.zeros((U1, V))
    D_am[:, 0] += sc * ga.sum(1)
    Da_abs[:, 0] += np.abs(sc * ga).sum(1)
    D_lm[:, 0] += sc * ga.sum(0)
    Dl_abs[:, 0] += np.abs(sc * ga).sum(0)
    for u in range(Ub):
        y = int(labels[u])
        if 1 <= y < V:
            D_am[:, y] += sc * gc[:, u]
            Da_abs[:, y] += np.abs(sc * gc[:, u])
            D_lm[u, y] += sc * gc[:, u].sum()
            Dl_abs[u, y] += np.abs(sc * gc[:, u]).sum()
    d_am = D_am - ea * (P @ el)
    d_lm = D_lm - el * (P.T @ ea)
    K = (np.abs(mt[:, None] + mu[None, :]) + np.abs(mt[:, None] + mu[None, :] - Z)).max() + (
        (mt[:, None] - am).max() + (mu[:, None] - lm).max())
    Pf = np.abs(w) * np.where(E <= 2.0 ** 101, E, 1.0)        # the factored nodes (with a margin at the threshold)
    tol_am = U * ((U1 + 18 + K) * ea * (Pa @ el) + (U1 + 1) * Da_abs + np.abs(d_am)) + 2.0 ** -148 * Pf.sum(1)[:, None]
    tol_lm = U * ((T + 18 + K) * el * (Pa.T @ ea) + (T + 1) * Dl_abs + np.abs(d_lm)) + 2.0 ** -148 * Pf.sum(0)[:, None]
    return d_am, d_lm, tol_am, tol_lm


# ------------------------------------------------------------------------------------------------ bf16
def bf16_ulp(want):
    """Spacing of bf16 numbers at |want| (float64 array): 2^(e - 8) for |want| in [2^(e-1), 2^e), and 2^-133 (the
    subnormal spacing) below 2^-126."""
    _, e = np.frexp(np.maximum(np.abs(want), 2.0 ** -126))
    return np.ldexp(1.0, e - 8)


def round_bf16(x):
    """float64 -> the nearest bf16 value (ties to even), as float64."""
    f = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    f = (f + 0x7FFF + ((f >> 16) & 1)) & 0xFFFF0000
    return f.astype(np.uint32).view(np.float32).astype(np.float64)


def ratio_bf16(got, want, abs_tol):
    """max |got - want| / (one bf16 ulp of want + abs_tol) (NaN in got counts as infinite)."""
    err = np.abs(np.asarray(got, dtype=np.float64) - want)
    err = np.where(np.isnan(err), np.inf, err)
    return float((err / (bf16_ulp(want) + abs_tol)).max()) if err.size else 0.0


def ratio_f32(got, want, bound):
    """max |got - want| / bound over the finite entries of want; the non-finite ones must match exactly (else inf)."""
    got = np.asarray(got, dtype=np.float64)
    fin = np.isfinite(want)
    if not np.array_equal(fin, np.isfinite(got)) or not np.array_equal(got[~fin], want[~fin]):
        return math.inf
    if not fin.any():
        return 0.0
    b = np.broadcast_to(bound, want.shape)[fin]
    return float((np.abs(got[fin] - want[fin]) / np.maximum(b, 1e-300)).max())
