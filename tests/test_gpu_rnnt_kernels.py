"""The transducer's training kernels (csrc/rnnt.cu, csrc/rnnt_pruned.cu) at every configuration their launchers accept,
against the float64 restatements of tests/rnnt_kernels_ref.py on the same f32 / bf16 operands:
  * otb_rnnt_joint and otb_rnnt_joint_bwd: D at the edges of the 8-column vectors and of the 2 x 128-column loop, long
    sums, lengths past the padded sizes, T_b = 0, bands of width 2 and wider than the transcript;
  * otb_rnnt_logprob: V at the float4 body, its second 512-column pass and the V % 4 tail, row pitches wider than V,
    chunks that cut utterances, labels that are blank or >= V, equal and 1e4-sized logits;
  * otb_rnnt_loss: U + 1 from 1 to 1024, T up to 1000 against 1023 labels, empty and negative lengths, underflowing arcs,
    both gradient scales, bands with no path and bands as wide as the transcript;
  * otb_rnnt_dlogits, otb_rnnt_simple_lse (logit scales sigma = 1 .. 64), otb_rnnt_simple_bwd, otb_rnnt_prune_ranges;
  * every refusal of the launchers and the ops wrappers.
A bf16 output is within one bf16 ulp of the float64 value plus the error of the f32 arithmetic before the rounding; an
f32 output is within the bound rnnt_kernels_ref derives from the kernel's arithmetic.  Every case prints its error as a
ratio to its bound (<= 1 passes), outputs the caller supplies sit inside NaN canaries, and every run is repeated and must
be bit-identical.  Run with -m gpu on an H100."""
import numpy as np
import pytest
import torch

from opentransformer_b200 import _lib, ops
from tests import rnnt_kernels_ref as ref
from tests import rnnt_pruned_ref as prr

pytestmark = pytest.mark.gpu
DEV = 'cuda'
BF = torch.bfloat16
NAN = float('nan')
U = ref.U


def _lens(t, u):
    return torch.tensor(t, dtype=torch.int32, device=DEV), torch.tensor(u, dtype=torch.int32, device=DEV)


def _report(name, ratio):
    print(f'{name}: error / bound {ratio:.3f}')
    assert ratio <= 1.0, f'{name}: error {ratio:.3f} times its bound'


def _np(t):
    return t.detach().cpu().double().numpy()


def _nodes(B, T, U1, t_len, u_len, s=None, S=None):
    """-> (b, t, u, valid) of every stored node [B T W] (W = U1, or S with the band s [B, T])."""
    W = U1 if s is None else S
    b, t, k = np.meshgrid(np.arange(B), np.arange(T), np.arange(W), indexing='ij')
    u = k if s is None else k + np.asarray(s)[b, t]
    Tb = np.minimum(np.asarray(t_len), T)[b]
    Ub = np.minimum(np.asarray(u_len), U1 - 1)[b]
    valid = (u < U1) & (t < Tb) & (u <= Ub)
    return b.ravel(), t.ravel(), u.ravel(), valid.ravel()


def _label_cols(labels, b, u, u_len, U1, V):
    """The label column of each node (rnnt_label): -1 at u >= U_b and for blank or out-of-range labels."""
    Ub = np.minimum(np.asarray(u_len), U1 - 1)[b]
    y = np.where(u < Ub, labels[b, np.minimum(u, labels.shape[1] - 1)], -1)
    return np.where((y >= 1) & (y < V), y, -1)


def _band(B, T, U1, seed):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, U1, (B, T)).astype(np.int32))


# ------------------------------------------------------------------------------------------------ the joint
JOINT_CASES = [  # B, T, U1, t_len, u_len, S (None: full lattice)
    (3, 5, 7, [5, 2, 9], [6, 0, 10], None),
    (2, 3, 4, None, None, None),
    (3, 5, 7, [5, 2, 9], [6, 0, 10], 2),
    (2, 4, 5, [4, 3], [4, 2], 9),
]


@pytest.mark.parametrize('D', [8, 16, 264, 1024])
@pytest.mark.parametrize('case', range(len(JOINT_CASES)))
def test_joint(D, case):
    B, T, U1, t_len, u_len, S = JOINT_CASES[case]
    g = torch.Generator().manual_seed(D + case)
    ep = (1.5 * torch.randn(B * T, D, generator=g)).to(BF)
    pp = (1.5 * torch.randn(B * U1, D, generator=g)).to(BF)
    tl, ul = _lens(t_len, u_len) if t_len else (None, None)
    s = _band(B, T, U1, D) if S else None
    band = dict(s_begin=s.to(DEV), S=S) if S else {}
    W = S or U1
    rows = B * T * W
    canvas = torch.full((rows + 3, D), NAN, dtype=BF, device=DEV)
    out = ops.rnnt_joint(ep.to(DEV), pp.to(DEV), B, T, U1, tl, ul, out=canvas[:rows], **band)
    again = ops.rnnt_joint(ep.to(DEV), pp.to(DEV), B, T, U1, tl, ul, **band)
    assert torch.equal(out, again)
    assert bool(torch.isnan(canvas[rows:].float()).all()), 'wrote past the lattice'
    b, t, u, valid = _nodes(B, T, U1, t_len or [T] * B, u_len or [U1 - 1] * B, s.numpy() if S else None, S)
    got = _np(out)
    assert not got[~valid].any(), 'a missing node is not zero'
    want, tol = ref.joint(_np(ep)[b * T + t][valid], _np(pp)[b * U1 + np.minimum(u, U1 - 1)][valid])
    _report(f'joint D={D} case {case}', ref.ratio_bf16(got[valid], want, tol))


JOINT_BWD_CASES = [  # B, T, U1, t_len, u_len, S
    (2, 4, 5, [4, 9], [4, 7], None),            # lengths past the padded sizes
    (3, 3, 4, [0, 3, 2], [3, 3, 0], None),      # T_b = 0: its dPp rows are zero
    (3, 5, 7, [5, 2, 6], [6, 0, 9], 2),
    (2, 4, 5, [4, 3], [4, 2], 8),
]


def _joint_bwd_check(name, B, T, U1, D, t_len, u_len, S, seed):
    g = torch.Generator().manual_seed(seed)
    s = _band(B, T, U1, seed) if S else None
    band = dict(s_begin=s.to(DEV), S=S) if S else {}
    W = S or U1
    h = torch.tanh(torch.randn(B * T * W, D, generator=g)).to(BF)
    dh = torch.randn(B * T * W, D, generator=g).to(BF)
    tl, ul = _lens(t_len, u_len)
    dep, dpp = ops.rnnt_joint_bwd(dh.to(DEV), h.to(DEV), B, T, U1, tl, ul, **band)
    again = ops.rnnt_joint_bwd(dh.to(DEV), h.to(DEV), B, T, U1, tl, ul, **band)
    assert torch.equal(dep, again[0]) and torch.equal(dpp, again[1])
    b, t, u, valid = _nodes(B, T, U1, t_len, u_len, s.numpy() if S else None, S)
    hv, gv = _np(h), _np(dh)
    dz = np.where(valid[:, None], gv * (1 - hv * hv), 0.0)
    ga = np.where(valid[:, None], np.abs(gv), 0.0)
    want_e = dz.reshape(B * T, W, D).sum(1)
    gabs_e = ga.reshape(B * T, W, D).sum(1)
    r = (b * U1 + np.minimum(u, U1 - 1))[valid]
    if S:
        want_p = np.zeros((B * U1, D))
        gabs_p = np.zeros((B * U1, D))
        np.add.at(want_p, r, dz[valid])
        np.add.at(gabs_p, r, ga[valid])
    else:
        want_p = dz.reshape(B, T, U1, D).sum(1).reshape(B * U1, D)
        gabs_p = ga.reshape(B, T, U1, D).sum(1).reshape(B * U1, D)
    _report(f'{name} dEp', ref.ratio_bf16(_np(dep), want_e, ref.joint_bwd_bound(gabs_e, W)))
    _report(f'{name} dPp', ref.ratio_bf16(_np(dpp), want_p, ref.joint_bwd_bound(gabs_p, T)))
    live_p = np.zeros(B * U1, dtype=bool)
    live_p[r] = True
    assert not _np(dpp)[~live_p].any() and not _np(dep)[~valid.reshape(B * T, W).any(1)].any()


@pytest.mark.parametrize('D', [2, 6, 254, 256, 258, 520, 1024])
@pytest.mark.parametrize('case', range(len(JOINT_BWD_CASES)))
def test_joint_bwd(D, case):
    B, T, U1, t_len, u_len, S = JOINT_BWD_CASES[case]
    _joint_bwd_check(f'joint_bwd D={D} case {case}', B, T, U1, D, t_len, u_len, S, D * 10 + case)


@pytest.mark.parametrize('D', [2, 6])
def test_joint_bwd_long_sums(D):
    """U + 1 = 1024 terms into each dEp row, 500 into each dPp row."""
    _joint_bwd_check(f'joint_bwd long D={D}', 1, 500, 1024, D, [500], [1023], None, D)


# ------------------------------------------------------------------------------------------------ lattice log-probs
LP_V = [2, 3, 5, 31, 32, 33, 127, 128, 129, 511, 512, 513, 4234, 5000]


def _logits(rows, V, seed, special=True):
    """f32 [rows, ld] with ld > V a multiple of 4 and NaN past V; row 1 all equal, row 2 of magnitude 1e4."""
    g = torch.Generator().manual_seed(seed)
    ld = (V + 3) // 4 * 4 + 4
    x = torch.full((rows, ld), NAN)
    x[:, :V] = 3 * torch.randn(rows, V, generator=g)
    if special:
        x[1, :V] = 0.625
        x[2, :V] = 1e4 + 2 * torch.randn(V, generator=g)
    return x


def _labels(B, n, V, seed):
    """i32 [B, n] with labels in [1, V), one blank and one >= V when there is room."""
    g = torch.Generator().manual_seed(seed)
    y = torch.randint(1, V, (B, n), generator=g, dtype=torch.int32)
    if n >= 3:
        y[0, 1] = 0
        y[-1, 2] = V + 3
    return y


@pytest.mark.parametrize('banded', [False, True], ids=['full', 'band'])
@pytest.mark.parametrize('V', LP_V)
def test_logprob(V, banded):
    B, T, U1 = 2, 3, 5
    t_len, u_len = [3, 7], [4, 9]
    S = 3 if banded else None
    s = _band(B, T, U1, V) if banded else None
    band = dict(s_begin=s.to(DEV), S=S) if banded else {}
    W = S or U1
    rows = B * T * W
    x = _logits(rows, V, V)
    labels = _labels(B, U1 + 1, V, V)
    tl, ul = _lens(t_len, u_len)
    canvas = torch.full((rows + 2, 3), NAN, device=DEV)
    lp = canvas[:rows]
    xd, yd = x.to(DEV), labels.to(DEV)
    ops.rnnt_logprob(xd[:0], 0, V, B, T, U1, tl, ul, yd, lp, **band)         # rows = 0: nothing written
    assert bool(torch.isnan(canvas).all())
    for r0 in range(0, rows, 7):                    # chunks that cut utterances and frames
        ops.rnnt_logprob(xd[r0:r0 + 7], r0, V, B, T, U1, tl, ul, yd, lp, **band)
    again = torch.full_like(lp, NAN)
    ops.rnnt_logprob(xd, 0, V, B, T, U1, tl, ul, yd, again, **band)
    assert torch.equal(lp, again), 'chunked and whole runs differ'
    assert bool(torch.isnan(canvas[rows:]).all()), 'wrote past the lattice'
    b, t, u, valid = _nodes(B, T, U1, t_len, u_len, s.numpy() if banded else None, S)
    got = _np(lp)
    assert not got[~valid].any()
    y = _label_cols(labels.numpy(), b, u, u_len, U1, V)
    want, bound = ref.logprob_bound(x[:, :V].double().numpy()[valid], y[valid])
    _report(f'logprob V={V} {"band" if banded else "full"}', ref.ratio_f32(got[valid], want, bound))


# ------------------------------------------------------------------------------------------------ the loss
def _lp_tensor(B, T, W, seed, tiny=False):
    """Node log-probs [B T W, 3]: log p(blank), log p(label) of two random probabilities each; tiny: some at -1e4."""
    rng = np.random.default_rng(seed)
    lp = np.zeros((B * T * W, 3), dtype=np.float32)
    lp[:, 1] = np.log(rng.uniform(0.05, 0.6, B * T * W))
    lp[:, 2] = np.log(rng.uniform(0.05, 0.4, B * T * W))
    if tiny:
        pick = rng.random((B * T * W, 2)) < 0.3
        lp[:, 1:][pick] = -1e4 + rng.normal(size=int(pick.sum()))
    return torch.from_numpy(lp)


def _loss_check(name, B, T, U1, t_len, u_len, seed, S=None, s=None, tiny=False, grad_scale=1.0, scale_dev=None):
    W = S or U1
    band = dict(s_begin=s.to(DEV), S=S) if S else {}
    lp = _lp_tensor(B, T, W, seed, tiny)
    tl, ul = _lens(t_len, u_len)
    sd = torch.tensor([scale_dev], device=DEV) if scale_dev is not None else None
    loss, nll, grad = ops.rnnt_loss(lp.to(DEV), B, T, U1, tl, ul, grad_scale=grad_scale, scale_dev=sd, **band)
    loss2, nll2, grad2 = ops.rnnt_loss(lp.to(DEV), B, T, U1, tl, ul, grad_scale=grad_scale, scale_dev=sd, **band)
    assert torch.equal(nll, nll2) and torch.equal(grad, grad2) and torch.equal(loss, loss2)
    gs = float(np.float32(grad_scale)) * (scale_dev if scale_dev is not None else 1.0) / B     # the kernel's f32 scale
    got_n, got_g = _np(nll), _np(grad).reshape(B, T, W, 2)
    lpn = lp.double().numpy().reshape(B, T, W, 3)
    worst_n = worst_g = 0.0
    for bi in range(B):
        Tb, Ub = min(t_len[bi], T), min(u_len[bi], U1 - 1)
        if Tb < 1 or Ub < 0:
            assert got_n[bi] == np.inf and not got_g[bi].any(), f'{name}: utterance {bi} without nodes'
            continue
        sb = s[bi, :Tb].numpy().astype(np.int64) if S else np.zeros(Tb, dtype=np.int64)
        tt, kk = np.meshgrid(np.arange(Tb), np.arange(W), indexing='ij')
        uu = sb[:, None] + kk
        on = uu <= Ub
        lpb = np.full((Tb, Ub + 1), -np.inf)
        lpy = np.full((Tb, Ub + 1), -np.inf)
        lpb[tt[on], uu[on]] = lpn[bi, :Tb, :, 1][on]
        lpy[tt[on], uu[on]] = lpn[bi, :Tb, :, 2][on]
        lat = ref.lattice(lpb, lpy, sb if S else None, S)
        nb, rel = ref.loss_bound(lat, Tb, Ub)
        if not np.isfinite(lat['logp']):
            assert got_n[bi] == np.inf and not got_g[bi].any(), f'{name}: utterance {bi} with no path'
            continue
        worst_n = max(worst_n, abs(got_n[bi] + lat['logp']) / nb)
        want = np.zeros((T, W, 2))
        want[tt[on], kk[on], 0] = -gs * lat['gb'][tt[on], uu[on]]
        want[tt[on], kk[on], 1] = -gs * lat['gy'][tt[on], uu[on]]
        bound = rel * np.abs(want) + 2 * abs(gs) * 2.0 ** -149
        worst_g = max(worst_g, float((np.abs(got_g[bi] - want) / bound).max()))
    _report(f'{name} nll', worst_n)
    _report(f'{name} grad', worst_g)
    if np.isfinite(got_n).all():
        _report(f'{name} loss', abs(float(loss) - got_n.sum() / B) / (U * (B + 1) * np.abs(got_n).sum() / B + 1e-30))
    else:
        assert float(loss) == np.inf
    return nll, grad


@pytest.mark.parametrize('U1', [1, 2, 31, 32, 33, 1023, 1024])
def test_loss_transcript_lengths(U1):
    B, T = 4, 6
    u_len = [U1 - 1, 0, max(U1 - 3, 0), U1 + 3]        # U_b = 0 and u_len past the padded U
    t_len = [6, 4, 0, 9]                                # T_b = 0 and t_len past the padded T
    _loss_check(f'loss U1={U1}', B, T, U1, t_len, u_len, U1, grad_scale=0.7, scale_dev=3.0)


@pytest.mark.parametrize('T', [1, 2, 1000])
def test_loss_frames(T):
    U1 = 1024 if T == 1000 else 33                      # T ~ 1000 against 1023 labels: alpha in the thousands
    _loss_check(f'loss T={T}', 1, T, U1, [T], [U1 - 1], T)


def test_loss_underflowing_arcs_and_scales():
    _loss_check('loss tiny arcs', 2, 7, 9, [7, 5], [8, 6], 3, tiny=True)
    _, g1 = _loss_check('loss scale', 2, 5, 6, [5, 4], [5, 3], 4, grad_scale=0.5, scale_dev=3.0)
    _, g2 = _loss_check('loss scale host', 2, 5, 6, [5, 4], [5, 3], 4, grad_scale=1.5)
    assert torch.equal(g1, g2)


def test_loss_negative_lengths():
    """A negative length leaves the utterance without nodes: nll +inf, zero gradients, the others unchanged."""
    B, T, U1 = 4, 5, 6
    nll, grad = _loss_check('loss negative lengths', B, T, U1, [5, 3, -2, 4], [5, -1, 2, -7], 5)
    assert np.isfinite(_np(nll)[[0]]).all()


@pytest.mark.parametrize('case', ['ragged', 'no_path'])
def test_banded_loss(case):
    if case == 'ragged':
        B, T, U1, S, t_len, u_len = 3, 10, 9, 3, [10, 1, 6], [8, 0, 5]
    else:                                               # utterance 1: U_b > T_b (S - 1)
        B, T, U1, S, t_len, u_len = 2, 6, 10, 2, [6, 4], [5, 9]
    s = torch.zeros(B, T, dtype=torch.int32)
    rng = np.random.default_rng(U1)
    for b in range(B):
        occ = rng.random((t_len[b], u_len[b] + 1)).astype(np.float32)
        s[b, :t_len[b]] = torch.from_numpy(prr.prune_ranges(occ, t_len[b], u_len[b], S).astype(np.int32))
    nll, _ = _loss_check(f'banded loss {case}', B, T, U1, t_len, u_len, S, S=S, s=s)
    if case == 'no_path':
        assert float(nll[1]) == np.inf


@pytest.mark.parametrize('extra', [0, 3])
def test_wide_band_is_the_full_lattice(extra):
    """S >= U + 1 with every band at 0 runs the same recursion as the full lattice, bit for bit."""
    B, T, U1 = 2, 7, 6
    S = U1 + extra
    t_len, u_len = [7, 4], [5, 2]
    tl, ul = _lens(t_len, u_len)
    lp = _lp_tensor(B, T, U1, 11)
    lpb = torch.zeros(B * T * S, 3)
    lpb.view(B, T, S, 3)[:, :, :U1] = lp.view(B, T, U1, 3)
    s = torch.zeros(B, T, dtype=torch.int32, device=DEV)
    _, nf, gf = ops.rnnt_loss(lp.to(DEV), B, T, U1, tl, ul)
    _, nb, gb = ops.rnnt_loss(lpb.to(DEV), B, T, U1, tl, ul, s_begin=s, S=S)
    assert torch.equal(nf, nb)
    assert torch.equal(gb.view(B, T, S, 2)[:, :, :U1], gf.view(B, T, U1, 2))
    assert not gb.view(B, T, S, 2)[:, :, U1:].any()


# ------------------------------------------------------------------------------------------------ dlogits
@pytest.mark.parametrize('V,ldd,banded', [(33, 34, False), (129, 130, True), (32, 32, False), (31, 48, False),
                                          (513, 528, True), (4234, 4234, False)])
def test_dlogits(V, ldd, banded):
    B, T, U1 = 2, 3, 5
    t_len, u_len = [3, 5], [4, 7]
    S = 2 if banded else None
    s = _band(B, T, U1, V) if banded else None
    band = dict(s_begin=s.to(DEV), S=S) if banded else {}
    W = S or U1
    rows = B * T * W
    x = _logits(rows, V, V + 1, special=False)
    labels = _labels(B, U1 + 1, V, V + 1)
    tl, ul = _lens(t_len, u_len)
    xd, yd = x.to(DEV), labels.to(DEV)
    lp = torch.empty(rows, 3, device=DEV)
    ops.rnnt_logprob(xd, 0, V, B, T, U1, tl, ul, yd, lp, **band)
    grad = 0.3 * torch.randn(rows, 2, generator=torch.Generator().manual_seed(V))
    grad[::4] = 0.0                                      # a = c = 0: an exactly zero row
    grad = grad.to(DEV)
    canvas = torch.full((rows + 2, ldd), NAN, dtype=BF, device=DEV)
    out = canvas[:rows]
    for r0 in range(0, rows, 5):
        ops.rnnt_dlogits(xd[r0:r0 + 5], r0, V, B, T, U1, tl, ul, yd, lp, grad, out=out[r0:r0 + 5], **band)
    again = torch.full((rows, ldd), NAN, dtype=BF, device=DEV)
    ops.rnnt_dlogits(xd, 0, V, B, T, U1, tl, ul, yd, lp, grad, out=again, **band)
    assert torch.equal(out, again)
    assert bool(torch.isnan(canvas[rows:].float()).all()), 'wrote past the rows'
    b, t, u, valid = _nodes(B, T, U1, t_len, u_len, s.numpy() if banded else None, S)
    got = _np(out)
    assert not got[:, V:].any(), 'columns past V are not zero'
    live = valid & (_np(grad) != 0).any(1)
    assert not got[~live].any(), 'a missing node or one with a = c = 0 is not zero'
    y = _label_cols(labels.numpy(), b, u, u_len, U1, V)
    g = _np(grad)
    want, tol = ref.dlogits_bound(x[:, :V].double().numpy()[live], _np(lp)[live, 0], g[live, 0], g[live, 1], y[live])
    _report(f'dlogits V={V} ldd={ldd} {"band" if banded else "full"}', ref.ratio_bf16(got[live, :V], want, tol))


# ------------------------------------------------------------------------------------------------ the simple joint
def _simple_operands(B, T, U1, V, sigma, seed):
    g = torch.Generator().manual_seed(seed)
    lda, ldl = V + 3, V + 9
    am = torch.full((B * T, lda), NAN)
    lm = torch.full((B * U1, ldl), NAN)
    am[:, :V] = sigma * torch.randn(B * T, V, generator=g)
    lm[:, :V] = sigma * torch.randn(B * U1, V, generator=g)
    return am, lm


def _simple_case(T, U1, V, sigma, seed, scale_dev=None, ldd=None):
    B = 4                                                   # T_b = 0; t_len and u_len past T and U; U_b = 0
    t_len, u_len = [T, 0, T + 4, T], [U1 - 1, 2, U1 + 2, 0]
    am, lm = _simple_operands(B, T, U1, V, sigma, seed)
    labels = _labels(B, U1 + 1, V, seed)
    tl, ul = _lens(t_len, u_len)
    ad, ld_, yd = am.to(DEV), lm.to(DEV), labels.to(DEV)
    lp, m_am, m_lm = ops.rnnt_simple_lse(ad, ld_, V, B, T, U1, tl, ul, yd)
    again = ops.rnnt_simple_lse(ad, ld_, V, B, T, U1, tl, ul, yd)
    assert all(torch.equal(x, y) for x, y in zip((lp, m_am, m_lm), again))
    name = f'T={T} U1={U1} V={V} sigma={sigma}'
    a64, l64 = am[:, :V].double().numpy(), lm[:, :V].double().numpy()
    lpn = _np(lp).reshape(B, T, U1, 3)
    worst = [0.0, 0.0, 0.0]
    for b in range(B):
        Tb, Ub = min(t_len[b], T), min(u_len[b], U1 - 1)
        live_t = Tb if Tb > 0 else 0
        live_u = Ub + 1 if Tb > 0 else 0
        ma = _np(m_am)[b * T:(b + 1) * T]
        ml = _np(m_lm)[b * U1:(b + 1) * U1]
        assert np.array_equal(ma[:live_t], a64[b * T:b * T + live_t].max(1)) and not ma[live_t:].any(), f'{name}: m_am'
        assert np.array_equal(ml[:live_u], l64[b * U1:b * U1 + live_u].max(1)) and not ml[live_u:].any(), f'{name}: m_lm'
        dead = np.ones((T, U1), dtype=bool)
        dead[:live_t, :live_u] = False
        assert not lpn[b][dead].any(), f'{name}: a missing node is not zero'
        if not live_t or not live_u:
            continue
        A, L = a64[b * T:b * T + Tb], l64[b * U1:b * U1 + Ub + 1]
        Z, gap, mx = ref.simple_z(A, L)
        zb = ref.simple_lse_bound(A, L, Z, gap, mx)
        x0 = A[:, None, 0] + L[None, :, 0]
        yc = np.array([int(labels[b, u]) if u < Ub and 1 <= int(labels[b, u]) < V else -1 for u in range(Ub + 1)])
        xy = np.where(yc >= 0, A[:, np.maximum(yc, 0)] + L[np.arange(Ub + 1), np.maximum(yc, 0)][None, :], -np.inf)
        got = lpn[b, :Tb, :Ub + 1]
        worst[0] = max(worst[0], ref.ratio_f32(got[..., 0], Z, zb))
        worst[1] = max(worst[1], ref.ratio_f32(got[..., 1], x0 - Z, zb + U * (np.abs(x0) + np.abs(x0 - Z))))
        with np.errstate(invalid='ignore'):
            worst[2] = max(worst[2], ref.ratio_f32(got[..., 2], xy - Z,
                                                   np.where(np.isfinite(xy), zb + U * (np.abs(xy) + np.abs(xy - Z)), 0.0)))
    for k, what in enumerate(('Z', 'log p(blank)', 'log p(label)')):
        _report(f'simple_lse {name} {what}', worst[k])

    _, _, grad = ops.rnnt_loss(lp, B, T, U1, tl, ul)
    assert bool(torch.isfinite(grad).all()), f'{name}: non-finite node gradients'
    sd = torch.tensor([scale_dev], device=DEV) if scale_dev is not None else None
    d_am, d_lm = ops.rnnt_simple_bwd(ad, ld_, V, B, T, U1, tl, ul, yd, lp, m_am, m_lm, grad, 0.5, sd, ldd=ldd)
    again = ops.rnnt_simple_bwd(ad, ld_, V, B, T, U1, tl, ul, yd, lp, m_am, m_lm, grad, 0.5, sd, ldd=ldd)
    assert torch.equal(d_am, again[0]) and torch.equal(d_lm, again[1])
    sc = 0.5 * (scale_dev if scale_dev is not None else 1.0)
    gn = _np(grad).reshape(B, T, U1, 2)
    da, dl = _np(d_am), _np(d_lm)
    assert not da[:, V:].any() and not dl[:, V:].any(), f'{name}: gradient columns past V'
    wa = wl = 0.0
    for b in range(B):
        Tb, Ub = min(t_len[b], T), min(u_len[b], U1 - 1)
        live_u = Ub + 1 if Tb > 0 else 0
        assert not da[b * T + max(Tb, 0):(b + 1) * T].any() and not dl[b * U1 + live_u:(b + 1) * U1].any()
        if Tb < 1:
            continue
        A, L = a64[b * T:b * T + Tb], l64[b * U1:b * U1 + Ub + 1]
        want_a, want_l, tol_a, tol_l = ref.simple_bwd(A, L, lpn[b, :Tb, :Ub + 1, 0], gn[b, :Tb, :Ub + 1, 0],
                                                      gn[b, :Tb, :Ub + 1, 1], labels[b].numpy(), Ub, sc)
        wa = max(wa, ref.ratio_bf16(da[b * T:b * T + Tb, :V], want_a, tol_a))
        wl = max(wl, ref.ratio_bf16(dl[b * U1:b * U1 + Ub + 1, :V], want_l, tol_l))
    _report(f'simple_bwd {name} ldd={d_am.shape[1]} d am', wa)
    _report(f'simple_bwd {name} ldd={d_am.shape[1]} d lm', wl)


@pytest.mark.parametrize('V', [2, 31, 32, 33, 4234])
@pytest.mark.parametrize('T,U1', [(1, 1), (31, 33), (32, 32), (33, 65), (65, 31)])
def test_simple_joint_shapes(T, U1, V):
    _simple_case(T, U1, V, 2.0, T * 1000 + U1 * 10 + V, scale_dev=3.0 if V % 2 else None, ldd=V if V % 2 == 0 else V + 13)


@pytest.mark.parametrize('V', [50, 4234])
@pytest.mark.parametrize('sigma', [1.0, 8.0, 16.0, 32.0, 48.0, 64.0])
def test_simple_joint_logit_scale(sigma, V):
    """Above sigma ~ 24 the factorized sum of some nodes leaves the normal fp32 range; their Z and gradients must stay
    within the same bounds."""
    _simple_case(33, 33, V, sigma, int(sigma) + V, scale_dev=2.0)


# ------------------------------------------------------------------------------------------------ prune ranges
@pytest.mark.parametrize('S', [2, 39, 40, 1024])
def test_prune_ranges(S):
    B, T, U1 = 4, 300, 40                       # T > 256: the thread-stride loop
    t_len, u_len = [300, 400, 0, 120], [39, 20, 5, 0]
    rng = np.random.default_rng(S)
    g = np.zeros((B * T * U1, 2), dtype=np.float32)
    g[:, 0] = -rng.integers(0, 3, B * T * U1).astype(np.float32)            # integer occupancies: exact ties
    g[:, 1] = -(rng.integers(0, 2, B * T * U1) * 0.5).astype(np.float32)
    tl, ul = _lens(t_len, u_len)
    gd = torch.from_numpy(g).to(DEV)
    s = ops.rnnt_prune_ranges(gd, B, T, U1, tl, ul, S).cpu().numpy()
    assert np.array_equal(s, ops.rnnt_prune_ranges(gd, B, T, U1, tl, ul, S).cpu().numpy())
    occ = (-(g[:, 0] + g[:, 1])).astype(np.float32).reshape(B, T, U1)
    for b in range(B):
        Tb, Ub = min(t_len[b], T), min(u_len[b], U1 - 1)
        want = prr.prune_ranges(occ[b, :Tb, :Ub + 1], Tb, Ub, S)
        assert s[b, :Tb].tolist() == want.tolist(), f'S={S} utterance {b}'
        assert not s[b, Tb:].any()
    print(f'prune_ranges S={S}: equal integer for integer')


# ------------------------------------------------------------------------------------------------ refusals
def _refused(fn, what, exc=RuntimeError):
    with pytest.raises(exc, match=what):
        fn()
    torch.cuda.synchronize()


def test_refusals():
    B, T, U1, V = 1, 2, 3, 8
    tl, ul = _lens([2], [2])
    e = lambda *s: torch.zeros(*s, dtype=BF, device=DEV)               # noqa: E731
    f = lambda *s: torch.zeros(*s, device=DEV)                         # noqa: E731
    y = torch.ones(B, U1 - 1, dtype=torch.int32, device=DEV)
    y1 = torch.ones(B, 1, dtype=torch.int32, device=DEV)            # ldy = 1 < U
    s = torch.zeros(B, T, dtype=torch.int32, device=DEV)
    lp = f(B * T * U1, 3)
    # joint and its backward
    _refused(lambda: ops.rnnt_joint(e(B * T, 12), e(B * U1, 12), B, T, U1), 'positive multiple of 8')
    _refused(lambda: ops.rnnt_joint_bwd(e(B * T * U1, 3), e(B * T * U1, 3), B, T, U1, tl, ul), 'positive even number')
    _refused(lambda: ops.rnnt_joint(e(B * T, 8), e(B * U1, 8), B, T, U1, s_begin=s, S=2), 'needs t_len and u_len')
    _refused(lambda: ops.rnnt_joint(e(B * T, 8), e(B * U1, 8), B, T, U1, tl, ul, s_begin=s, S=1025), r'\[2, 1024\]')
    _refused(lambda: ops.rnnt_joint(e(B * T, 8), e(B * U1, 8), B, T, U1, tl, ul, s_begin=s, S=1), 'int >= 2', ValueError)
    # logits rows
    x = f(B * T * U1, 12)
    _refused(lambda: ops.rnnt_logprob(x[:, :6].contiguous(), 0, 5, B, T, U1, tl, ul, y, lp), '16-byte aligned')
    _refused(lambda: ops.rnnt_logprob(x[:, 1:9], 0, 5, B, T, U1, tl, ul, y, lp), '16-byte aligned')
    _refused(lambda: ops.rnnt_logprob(x, 0, 1, B, T, U1, tl, ul, y, lp), 'V >= 2')
    _refused(lambda: ops.rnnt_logprob(x, 0, 13, B, T, U1, tl, ul, y, lp), 'ld >= V')
    _refused(lambda: ops.rnnt_logprob(x, 0, V, B, T, U1, tl, ul, y1, lp), 'labels narrower')
    _refused(lambda: ops.rnnt_logprob(x, 0, V, B, T, U1, tl, ul, y, lp, s_begin=s, S=1025), r'\[2, 1024\]')
    g2 = f(B * T * U1, 2)
    _refused(lambda: ops.rnnt_dlogits(x, 0, V, B, T, U1, tl, ul, y, lp, g2, out=e(B * T * U1, 7)), 'even ldd >= V')
    _refused(lambda: ops.rnnt_dlogits(x, 0, 9, B, T, U1, tl, ul, y, lp, g2, out=e(B * T * U1, 8)), 'even ldd >= V')
    _refused(lambda: ops.rnnt_dlogits(x[:, 1:9], 0, V, B, T, U1, tl, ul, y, lp, g2), '16-byte aligned')
    # the loss: the wrapper and the launcher refuse more than 1023 labels
    big = 1025
    tb, ub = _lens([2], [1024])
    _refused(lambda: ops.rnnt_loss(f(B * T * big, 3), B, T, big, tb, ub), 'at most 1023', ValueError)
    alpha = torch.empty(B * T * big, dtype=torch.float64, device=DEV)
    nll, loss, gr = f(B), f(1), f(B * T * big, 2)
    _refused(lambda: _lib.check(_lib.lib().otb_rnnt_loss(ops._p(f(B * T * big, 3)), B, T, big, ops._p(tb), ops._p(ub),
                                                         ops._p(alpha), ops._p(nll), ops._p(loss), ops._p(gr), 1.0, None,
                                                         None, 0, ops._stream()), 'otb_rnnt_loss'), '1023 labels')
    _refused(lambda: ops.rnnt_loss(lp, B, T, U1, tl, ul, s_begin=s, S=1025), r'\[2, 1024\]')
    # the simple joint and the prune ranges
    am, lm = f(B * T, V), f(B * U1, V)
    _refused(lambda: ops.rnnt_simple_lse(am, lm, 1, B, T, U1, tl, ul, y), 'V >= 2')
    _refused(lambda: ops.rnnt_simple_lse(am, lm, V + 1, B, T, U1, tl, ul, y), 'row strides >= V')
    _refused(lambda: ops.rnnt_simple_lse(am, lm, V, B, T, U1, tl, ul, y1), 'labels narrower')
    _refused(lambda: ops.rnnt_simple_lse(f(B * T, V), f(B * big, V), V, B, T, big, tb, ub,
                                         torch.ones(B, big, dtype=torch.int32, device=DEV)), 'at most 1023')
    lps, m_am, m_lm = ops.rnnt_simple_lse(am, lm, V, B, T, U1, tl, ul, y)
    _refused(lambda: ops.rnnt_simple_bwd(am, lm, V, B, T, U1, tl, ul, y, lps, m_am, m_lm, g2, ldd=V - 1), 'narrower than V')
    _refused(lambda: ops.rnnt_prune_ranges(g2, B, T, U1, tl, ul, 1), r'\[2, 1024\]')
    _refused(lambda: ops.rnnt_prune_ranges(g2, B, T, U1, tl, ul, 1025), r'\[2, 1024\]')
