"""The float64 restatements of tests/rnnt_kernels_ref.py against the definitions they restate: the anti-diagonal lattice
against rnnt_ref's autograd and enumeration and rnnt_pruned_ref's banded loss, the direct simple-joint normalizer against
torch.logsumexp, the simple backward against autograd, and the bf16 helpers.  CPU only."""
import time

import numpy as np
import pytest
import torch

from tests import rnnt_kernels_ref as ref
from tests import rnnt_pruned_ref as prr
from tests import rnnt_ref


def _lp(T, U, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    x = scale * torch.randn(T, U + 1, 7, generator=g, dtype=torch.float64)
    labels = torch.randint(1, 7, (U,), generator=g)
    return rnnt_ref.node_logprobs(x, labels)


def _autograd(lpb, lpy, nll_fn):
    a = lpb.clone().requires_grad_(True)
    c = lpy.clone().requires_grad_(True)
    nll = nll_fn(a, c)
    if torch.isfinite(nll):
        nll.backward()
    gb = -a.grad if a.grad is not None else torch.zeros_like(lpb)
    gy = -c.grad if c.grad is not None else torch.zeros_like(lpy)
    return float(nll.detach()), gb.numpy(), gy.numpy()


@pytest.mark.parametrize('T,U', [(1, 0), (1, 3), (4, 0), (3, 2), (5, 4), (9, 17), (30, 12)])
def test_lattice_matches_autograd(T, U):
    lpb, lpy = _lp(T, U, seed=T * 100 + U)
    lat = ref.lattice(lpb.numpy(), lpy.numpy())
    nll, gb, gy = _autograd(lpb, lpy, rnnt_ref.lattice_nll)
    assert abs(-lat['logp'] - nll) <= 1e-12 * max(1.0, abs(nll))
    assert np.abs(lat['gb'] - gb).max() < 1e-12
    assert np.abs(lat['gy'][:, :U] - gy).max(initial=0) < 1e-12
    assert not lat['gy'][:, U].any()
    if T + U <= 9:
        assert abs(-lat['logp'] - float(rnnt_ref.enumerate_nll(lpb, lpy))) <= 1e-12 * max(1.0, abs(nll))
    # every alignment passes once through some arc of each anti-diagonal: the posteriors of a diagonal sum to 1
    for d in range(T + U):
        u = np.arange(max(0, d - T + 1), min(d, U) + 1)
        assert abs(lat['gb'][d - u, u].sum() + lat['gy'][d - u, u].sum() - 1) < 1e-12


@pytest.mark.parametrize('T,U,S,seed', [(6, 5, 2, 0), (8, 7, 3, 1), (5, 9, 2, 2), (7, 4, 5, 3), (4, 3, 6, 4)])
def test_banded_lattice_matches_band_nll(T, U, S, seed):
    lpb, lpy = _lp(T, U, seed=seed)
    occ = np.random.default_rng(seed).random((T, U + 1)).astype(np.float32)
    s = prr.prune_ranges(occ, T, U, S)
    lat = ref.lattice(lpb.numpy(), lpy.numpy(), s, S)
    nll, gb, gy = _autograd(lpb, lpy, lambda a, c: prr.band_nll(a, c, s.tolist(), S))
    assert prr.has_complete_path(s, T, U, S) == np.isfinite(lat['logp'])
    if not np.isfinite(nll):
        assert lat['logp'] == -np.inf and not lat['gb'].any() and not lat['gy'].any()
        return
    assert abs(-lat['logp'] - nll) <= 1e-12 * max(1.0, abs(nll))
    assert np.abs(lat['gb'] - gb).max() < 1e-12 and np.abs(lat['gy'][:, :U] - gy).max(initial=0) < 1e-12
    keep = ref.band_keep(T, U + 1, s, S)
    assert not lat['gb'][~keep].any() and not lat['gy'][~keep].any()
    if S >= U + 1:      # a band as wide as the transcript is the full lattice
        full = ref.lattice(lpb.numpy(), lpy.numpy())
        assert lat['logp'] == full['logp'] and np.array_equal(lat['gb'], full['gb'])


def test_lattice_is_fast_at_the_largest_lattice():
    """T = 1000 frames, U = 1023 labels: alpha reaches thousands, and the restatement takes seconds."""
    rng = np.random.default_rng(0)
    T, U = 1000, 1023
    lpb = np.log(rng.uniform(0.001, 0.01, (T, U + 1)))
    lpy = np.log(rng.uniform(0.001, 0.01, (T, U)))
    t0 = time.time()
    lat = ref.lattice(lpb, lpy)
    assert time.time() - t0 < 30
    assert np.isfinite(lat['logp']) and np.abs(lat['alpha']).max() > 1000
    for d in (0, 700, T + U - 1):
        u = np.arange(max(0, d - T + 1), min(d, U) + 1)
        assert abs(lat['gb'][d - u, u].sum() + lat['gy'][d - u, u].sum() - 1) < 1e-9


@pytest.mark.parametrize('sigma', [1.0, 16.0, 64.0])
def test_simple_z_is_logsumexp(sigma):
    g = torch.Generator().manual_seed(int(sigma))
    am = sigma * torch.randn(5, 33, generator=g, dtype=torch.float64)
    lm = sigma * torch.randn(4, 33, generator=g, dtype=torch.float64)
    Z, gap, mx = ref.simple_z(am.numpy(), lm.numpy())
    want = torch.logsumexp(am[:, None] + lm[None], -1).numpy()
    assert np.abs(Z - want).max() <= 1e-13 * np.abs(want).max()
    assert (gap >= 0).all() and (mx >= 0).all()
    # the p-weighted gap: m_t + m_u - E_p[am + lm]
    x = (am[:, None] + lm[None]).numpy()
    p = np.exp(x - want[..., None])
    assert np.allclose(gap, am.max(1).values.numpy()[:, None] + lm.max(1).values.numpy()[None] - (p * x).sum(-1))


def test_simple_bwd_matches_autograd():
    T, U, V = 6, 4, 11
    g = torch.Generator().manual_seed(3)
    am = 3 * torch.randn(T, V, generator=g, dtype=torch.float64)
    lm = 3 * torch.randn(U + 1, V, generator=g, dtype=torch.float64)
    labels = torch.randint(1, V, (U,), generator=g)
    a, l = am.clone().requires_grad_(True), lm.clone().requires_grad_(True)
    lpb, lpy = prr.simple_logprobs(a, l, labels)
    (0.75 * rnnt_ref.lattice_nll(lpb, lpy)).backward()
    lpb, lpy = prr.simple_logprobs(am, lm, labels)
    lat = ref.lattice(lpb.numpy(), lpy.numpy())
    Z, _, _ = ref.simple_z(am.numpy(), lm.numpy())
    d_am, d_lm, tol_am, tol_lm = ref.simple_bwd(am.numpy(), lm.numpy(), Z, -lat['gb'], -lat['gy'], labels.numpy(), U, 0.75)
    assert np.abs(d_am - a.grad.numpy()).max() < 1e-12 and np.abs(d_lm - l.grad.numpy()).max() < 1e-12
    assert (tol_am > 0).all() and (tol_lm > 0).all()


def test_bf16_helpers():
    x = torch.randn(1000, dtype=torch.float64) * torch.logspace(-30, 30, 1000, dtype=torch.float64)
    assert np.array_equal(ref.round_bf16(x.numpy()), x.to(torch.bfloat16).double().numpy())
    ulp = ref.bf16_ulp(x.numpy())
    up = (x.to(torch.bfloat16).double() + torch.from_numpy(ulp)).to(torch.bfloat16).double()
    assert ((up - x.to(torch.bfloat16).double()).abs().numpy() <= ulp).all()
    assert ref.bf16_ulp(np.array([1.0, 1.5, 0.75]))[0] == 2.0 ** -7 and ref.bf16_ulp(np.array([0.75]))[0] == 2.0 ** -8
    assert ref.bf16_ulp(np.array([2.0 ** -130, 0.0]))[1] == 2.0 ** -133 == float(torch.tensor(2.0 ** -133).to(torch.bfloat16))


def test_logprob_want_and_f32_ratio():
    x = np.random.default_rng(1).normal(size=(4, 9)) * 3
    want, bound = ref.logprob_bound(x, np.array([3, -1, 8, 1]))
    lse = np.log(np.exp(x).sum(1))
    assert np.allclose(want[:, 0], lse) and np.allclose(want[:, 1], x[:, 0] - lse)
    assert want[1, 2] == -np.inf and bound[1, 2] == 0 and (bound[:, :2] > 0).all()
    assert ref.ratio_f32(want.astype(np.float32), want, bound) <= 1
    got = want.copy()
    got[1, 2] = 0.0
    assert ref.ratio_f32(got, want, bound) == np.inf
