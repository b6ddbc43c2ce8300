"""Pins the float64 restatements of tests/simt_kernels_ref.py, which tests/test_gpu_simt_kernels.py checks the SIMT kernels
against, to torch.nn.functional (and the oracle's label-smoothing loss with autograd) in float64.  CPU only."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import speech_model as om
from tests import simt_kernels_ref as ref

F64 = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


@pytest.mark.parametrize('N', [8, 264, 1024])
def test_layernorm_matches_torch(N):
    g = _g(1)
    x = torch.randn(7, N, generator=g, dtype=F64) * 3 + 2
    g1, b1, g2, b2 = (torch.randn(N, generator=g, dtype=F64) for _ in range(4))
    y1 = F.layer_norm(x, (N,), g1, b1, 1e-5)
    assert torch.allclose(ref.layernorm(x, g1, b1), y1, rtol=1e-12, atol=1e-12)
    got = ref.layernorm(x, g1, b1, g2, b2, eps=1e-12)
    assert torch.allclose(got, F.layer_norm(F.layer_norm(x, (N,), g1, b1, 1e-12), (N,), g2, b2, 1e-12), rtol=1e-12, atol=1e-12)
    const = torch.full((1, N), 0.75, dtype=F64)                          # variance 0: exactly beta
    assert torch.equal(ref.layernorm(const, g1, b1), b1[None])


def test_log_softmax_matches_torch():
    x = torch.randn(5, 257, generator=_g(2), dtype=F64) * 4
    x[1, ::3] = -math.inf
    x[2, 1:] = -math.inf                                                 # one finite entry: 0 there
    x[3] = -math.inf                                                     # no finite entry: NaN, as torch
    x[4, 0], x[4, 1] = 1e30, -1e30
    got, want = ref.log_softmax(x), F.log_softmax(x, -1)
    assert torch.equal(torch.isnan(got), torch.isnan(want)) and bool(torch.isnan(got[3]).all())
    ok = ~torch.isnan(want)
    assert torch.allclose(got[ok], want[ok], rtol=1e-13, atol=1e-13)
    assert got[2, 0] == 0 and bool(torch.isneginf(got[2, 1:]).all())
    lm = F.log_softmax(torch.randn(5, 257, generator=_g(3), dtype=F64), -1)
    assert torch.allclose(ref.fused_logp(x[:3], lm[:3], 0.3), F.log_softmax(x[:3], -1) + 0.3 * lm[:3], equal_nan=True)


def test_stable_topk_breaks_ties_by_lower_index():
    v = torch.tensor([[0.5, 2.0, 1.0, 2.0, -math.inf, 2.0, 1.0, -math.inf],
                      [-math.inf] * 6 + [3.0, -math.inf]], dtype=F64)
    vals, ids = ref.stable_topk(v, 6)
    assert ids[0].tolist() == [1, 3, 5, 2, 6, 0]
    assert vals[0].tolist() == [2.0, 2.0, 2.0, 1.0, 1.0, 0.5]
    assert ids[1].tolist() == [6, 0, 1, 2, 3, 4]                         # -inf entries in index order after the finite one
    x = torch.randn(3, 1000, generator=_g(4), dtype=F64)
    vals, ids = ref.stable_topk(x, 16)
    tv, ti = torch.topk(x, 16, -1)                                       # no ties: torch.topk agrees
    assert torch.equal(vals, tv) and torch.equal(ids, ti)
    big = torch.zeros(1, 40000, dtype=F64)                               # all tied: ids 0..k-1
    assert ref.stable_topk(big, 16)[1][0].tolist() == list(range(16))


@pytest.mark.parametrize('smoothing', [0.0, 0.1, 1.0])
def test_ls_ce_matches_oracle_loss_and_autograd(smoothing):
    """pad_id 0 and in-range targets: the oracle's LabelSmoothingLoss, loss and gradient."""
    rows, V = 37, 50
    g = _g(5)
    x = (torch.randn(rows, V, generator=g, dtype=F64) * 3).requires_grad_(True)
    tgt = torch.randint(1, V, (rows,), generator=g)
    tgt[::5] = 0
    want = om.label_smoothing_loss(x.unsqueeze(0), tgt.unsqueeze(0), smoothing)
    want.backward()
    loss, per_tok, n, grad = ref.ls_ce(x.detach(), tgt, V, smoothing, 0)
    assert n == int((tgt != 0).sum())
    assert abs(float(loss) - want.item()) < 1e-12 * max(1.0, abs(want.item()))
    assert torch.allclose(per_tok.sum() / n, want.detach(), rtol=1e-12, atol=1e-12)
    assert torch.allclose(grad, x.grad, rtol=1e-12, atol=1e-14)
    assert bool((per_tok[tgt == 0] == 0).all())


def test_ls_ce_out_of_range_targets_are_pad():
    """A non-zero pad_id, and targets outside [0, V): scored and counted like PAD; the rest as with those rows removed."""
    rows, V, pad = 12, 9, 4
    x = torch.randn(rows, V + 3, generator=_g(6), dtype=F64)
    tgt = torch.tensor([0, pad, 3, -3, V, V - 1, pad, 2, 7, -1, 1, 0])
    loss, per_tok, n, grad = ref.ls_ce(x, tgt, V, 0.1, pad)
    keep = (tgt != pad) & (tgt >= 0) & (tgt < V)
    assert n == int(keep.sum()) == 7
    l2, p2, n2, g2 = ref.ls_ce(x[keep], tgt[keep], V, 0.1, pad)
    assert n2 == n and torch.allclose(loss, l2) and torch.equal(per_tok[keep], p2) and torch.equal(grad[keep], g2)
    assert bool((per_tok[~keep] == 0).all()) and bool((grad[~keep] == 0).all())
    allpad = ref.ls_ce(x, torch.full((rows,), pad), V, 0.1, pad)
    assert float(allpad[0]) == 0.0 and allpad[2] == 0 and bool((allpad[3] == 0).all())


def test_embed_posenc_all_position_modes():
    V, d, N = 11, 16, 9
    g = _g(7)
    emb = torch.randn(V, d, generator=g, dtype=F64)
    table = torch.randn(20, d, generator=g, dtype=F64)
    tok = torch.tensor([[3, 99], [-1, 0], [V, 5], [10, 0], [0, 0], [4, 0], [7, 0], [2, 0], [1, 0]])
    ids = [3, 0, 0, 10, 0, 4, 7, 2, 1]
    rp = torch.tensor([5, -1, 0, 19, 3, 3, 2, 1, 0])
    for kw, pos in (({'period': 4}, [n % 4 for n in range(N)]), ({'step': 13}, [13] * N),
                    ({'row_pos': rp}, [max(p, 0) for p in rp.tolist()])):
        got = ref.embed_posenc(tok, emb, table, d, tok_stride=2, **kw)
        want = torch.stack([emb[ids[n]] * math.sqrt(d) + table[pos[n]] for n in range(N)])
        assert torch.allclose(got, want, rtol=1e-14, atol=1e-14), kw


def test_scale_add_table():
    x = torch.randn(7, 5, generator=_g(8), dtype=F64)
    t = torch.randn(3, 5, generator=_g(9), dtype=F64)
    want = torch.stack([x[r] * 2.5 + t[r % 3] for r in range(7)])
    assert torch.allclose(ref.scale_add_table(x, 2.5, t, 3), want)
    assert torch.equal(ref.scale_add_table(x, 2.5), x * 2.5)


@pytest.mark.parametrize('k,T', [(1, 5), (3, 2), (15, 14), (31, 40)])
def test_dwconv_swish_matches_conv1d_batchnorm(k, T):
    B, d = 3, 8
    g = _g(10)
    x = torch.randn(B, T, d, generator=g, dtype=F64)
    w = torch.randn(d, 1, k, generator=g, dtype=F64)
    b = torch.randn(d, generator=g, dtype=F64)
    mean, var = torch.randn(d, generator=g, dtype=F64), torch.rand(d, generator=g, dtype=F64) + 0.5
    gam, bet = torch.randn(d, generator=g, dtype=F64), torch.randn(d, generator=g, dtype=F64)
    y = F.conv1d(x.transpose(1, 2), w, b, padding=(k - 1) // 2, groups=d)
    y = F.batch_norm(y, mean, var, gam, bet, training=False, eps=1e-5)
    want = F.silu(y).transpose(1, 2).reshape(B * T, d)
    s = gam / torch.sqrt(var + 1e-5)
    got = ref.dwconv_swish(x.reshape(B * T, d), (w[:, 0, :] * s[:, None]).t(), (b - mean) * s + bet, B, T)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)


def _attend_loop(q, ks, vs, H):
    """One row, one head at a time, with F.softmax: q [d], ks / vs [L, d] -> [d]."""
    d = q.shape[0]
    dk = d // H
    out = torch.empty(d, dtype=F64)
    for h in range(H):
        sl = slice(h * dk, (h + 1) * dk)
        p = F.softmax(ks[:, sl] @ q[sl] / math.sqrt(dk), -1)
        out[sl] = p @ vs[:, sl]
    return out


@pytest.mark.parametrize('dk,H', [(64, 2), (96, 3)])
def test_decode_self_attn_both_cache_layouts(dk, H):
    """The ancestry gather against a hand-built loop over rows and positions."""
    N, Lmax = 5, 9
    d = H * dk
    g = _g(11)
    qkv = torch.randn(N, 3 * d, generator=g, dtype=F64)
    kc, vc = torch.randn(Lmax, N, d, generator=g, dtype=F64), torch.randn(Lmax, N, d, generator=g, dtype=F64)
    anc = torch.randint(0, N, (2, N, Lmax), generator=g, dtype=torch.int32)
    for step in (0, 1, 6):
        got = ref.decode_self_attn(qkv, kc, vc, anc, H, step=step)
        for n in range(N):
            ks = torch.stack([kc[s, anc[step & 1, n, s]] for s in range(step)] + [qkv[n, d:2 * d]])
            vs = torch.stack([vc[s, anc[step & 1, n, s]] for s in range(step)] + [qkv[n, 2 * d:]])
            assert torch.allclose(got[n], _attend_loop(qkv[n, :d], ks, vs, H), rtol=1e-12, atol=1e-12)
    rows = 17
    kr, vr = torch.randn(rows, d, generator=g, dtype=F64), torch.randn(rows, d, generator=g, dtype=F64)
    anc_r = torch.randint(0, rows, (N, Lmax), generator=g, dtype=torch.int32)
    row_pos = torch.tensor([3, -1, 0, 8, 3], dtype=torch.int32)
    got = ref.decode_self_attn(qkv, kr, vr, anc_r, H, row_pos=row_pos)
    for n in range(N):
        p = int(row_pos[n])
        if p < 0:
            assert bool((got[n] == 0).all())
            continue
        ks = torch.stack([kr[anc_r[n, s]] for s in range(p)] + [qkv[n, d:2 * d]])
        vs = torch.stack([vr[anc_r[n, s]] for s in range(p)] + [qkv[n, 2 * d:]])
        assert torch.allclose(got[n], _attend_loop(qkv[n, :d], ks, vs, H), rtol=1e-12, atol=1e-12)
