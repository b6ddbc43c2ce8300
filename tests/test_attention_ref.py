"""The float64 attention restatement (tests/attention_ref.py) without a GPU:
  * its forward and backward equal torch autograd in float64, the band and kv_len 0 rows included;
  * a CPU emulation of the kernels' arithmetic stays inside the bounds on every case of tests/test_gpu_attention.py,
    and each plausible kernel mistake, computed in float64 and rounded like a kernel output, falls outside them;
  * the case table reaches every instantiation and branch of attn_tc.cu / attn_bwd.cu;
  * ops.attention / attention_train / attention_bwd and otb_attention refuse the shapes the kernels cannot take before
    any device work."""
import ctypes
import math

import pytest
import torch

from tests import attention_ref as ar


def _autograd(q, k, v, B, H, Tq, Tk, lens, causal, bd, dk, dout):
    """softmax((QK^T + BD) / sqrt(dk)) V written the plain way, differentiated by autograd."""
    q, k, v = (t.clone().requires_grad_() for t in (q, k, v))
    s = q @ k.transpose(-1, -2)
    bdg = None
    if bd is not None:
        bdg = bd.clone().requires_grad_()
        idx = torch.arange(Tk)[None, :] - torch.arange(Tq)[:, None] + Tq - 1
        s = s + torch.gather(bdg, 3, idx.expand(B, H, Tq, Tk))
    vis = torch.arange(Tk)[None, None, :] < torch.tensor(lens)[:, None, None].clamp(max=Tk)
    if causal:
        vis = vis & (torch.arange(Tk)[None, :] <= torch.arange(Tq)[:, None])
    z = (s / math.sqrt(dk)).masked_fill(~vis[:, None], float('-inf'))
    lse = torch.logsumexp(z, -1) / math.log(2.0)
    o = torch.softmax(z, -1).nan_to_num(0.0) @ v
    (o * dout).sum().backward()
    return o, lse, q.grad, k.grad, v.grad, (bdg.grad if bdg is not None else None)


@pytest.mark.parametrize('B,H,Tq,Tk,lens,causal,band,dk', [
    (3, 2, 9, 9, [9, 4, 0], False, True, 64),
    (3, 2, 7, 11, [11, 0, 5], True, False, 64),
    (2, 2, 12, 5, [5, 2], True, False, 64),
    (2, 2, 6, 6, [6, 3], False, True, 96),
])
def test_restatement_matches_autograd(B, H, Tq, Tk, lens, causal, band, dk):
    g = torch.Generator().manual_seed(Tq * Tk)
    d = H * dk
    qm = torch.randn(B * Tq, d, generator=g, dtype=torch.float64)
    km = torch.randn(B * Tk, 2 * d, generator=g, dtype=torch.float64)
    dout = torch.randn(B * Tq, d, generator=g, dtype=torch.float64)
    resid = torch.randn(B * Tq, d, generator=g, dtype=torch.float64)
    bd = 3 * torch.randn(H, B * Tq, 2 * Tq + 2, generator=g, dtype=torch.float64) if band else None
    kv = torch.tensor(lens, dtype=torch.int32)
    F = ar.forward(qm, km, km, B, H, Tq, Tk, kv, causal, (0, 0, d), bd, resid, dk)
    G = ar.backward(F, dout)
    q4, k4, v4 = ar.heads(qm, 0, B, H, Tq, dk), ar.heads(km, 0, B, H, Tk, dk), ar.heads(km, d, B, H, Tk, dk)
    bd4 = bd[:, :, :2 * Tq - 1].reshape(H, B, Tq, -1).transpose(0, 1) if band else None
    o, lse, dq, dk_, dv, dbd = _autograd(q4, k4, v4, B, H, Tq, Tk, lens, causal, bd4, dk, ar.heads(dout, 0, B, H, Tq, dk))
    torch.testing.assert_close(F['out'], ar.flat(o) + resid, rtol=1e-12, atol=1e-12)
    assert torch.equal(torch.isinf(F['lse']), torch.isinf(lse))
    torch.testing.assert_close(F['lse'][torch.isfinite(lse)], lse[torch.isfinite(lse)], rtol=1e-12, atol=1e-12)
    for got, want in ((G['dq'], ar.flat(dq)), (G['dk'], ar.flat(dk_)), (G['dv'], ar.flat(dv))):
        torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    if band:
        got, written = ar.band_layout(G['dS'], F['vis'], B, H, Tq, bd.shape[-1])
        want = dbd.transpose(0, 1).reshape(H, B * Tq, -1)
        torch.testing.assert_close(got[..., :2 * Tq - 1], want, rtol=1e-12, atol=1e-12)
        assert not written[..., 2 * Tq - 1:].any()
    dead = [b for b, L in enumerate(lens) if L == 0]
    for b in dead:   # no visible key: zero output (resid passes through) and zero gradients, as the kernels write them
        assert torch.equal(F['out'][b * Tq:(b + 1) * Tq], resid[b * Tq:(b + 1) * Tq])
        assert float(G['dq'][b * Tq:(b + 1) * Tq].abs().max()) == 0.0
        assert float(G['dk'][b * Tk:(b + 1) * Tk].abs().max()) == 0.0 and float(G['dv'][b * Tk:(b + 1) * Tk].abs().max()) == 0.0


def reference_and_bounds(c, X, mutate=None):
    """(F, G, bounds) of case c in float64 on the CPU; bounds are those of a kernel given `out` as its bf16 output."""
    F = ar.run_reference(c, X, 'cpu', mutate)
    FB = ar.forward_bounds(F)
    G = ar.backward(F, X['dout'].double(), mutate) if c[10] else None
    return F, FB, G


def check_all(c, X, F, FB, G, got):
    """Check a kernel-like result `got` (dict of out, lse and, for training cases, dq, dk, dv, dS, dsum) against the
    true reference; returns the worst err/bound."""
    name, dk, B, H, Tq, Tk = c[:6]
    w = [ar.check('out', got['out'], F['out'], FB['out']), ar.check('lse', got['lse'], F['lse'], FB['lse'])]
    if G is not None:
        BB = ar.backward_bounds(F, G, FB, got['out'])
        D, eD = ar.dsum_ref(got['out'], X['dout'], B, H, Tq)
        w.append(ar.check('dsum', got['dsum'], D, eD))
        for n in ('dq', 'dk', 'dv'):
            w.append(ar.check(n, got[n], G[n], BB[n]))
        vis = F['vis'].expand(B, H, Tq, Tk)
        w.append(ar.check('dS', got['dS'][vis], G['dS'][vis], BB['dS'][vis]))
    return max(w)


@pytest.mark.parametrize('name', ar.NAMES)
def test_emulation_within_bounds(name):
    """The kernels' arithmetic, emulated, stays inside every bound.  Where an output has one term (a row with one visible
    key, a key seen by one query) the bf16 rounding of P and that of the output can both reach 2^-8, the two terms the
    bound holds for them, so the worst ratio comes near 1 by construction there, as the GEMM's bf16 outputs do."""
    c = ar.CASE[name]
    X = ar.make_inputs(c)
    F, FB, G = reference_and_bounds(c, X)
    print(f'{name}:')
    worst = check_all(c, X, F, FB, G, ar.emulate(c, X))
    print(f'{name}: worst err/bound of the emulation {worst:.3f}')
    assert worst < 1.0


def _rounded(c, X, F, G):
    """A float64 result rounded the way the kernels store it: bf16 out / dq / dk / dv / dS, fp32 lse and D."""
    R = dict(out=F['out'].to(torch.bfloat16), lse=F['lse'].float())
    if G is not None:
        B, H, Tq = c[2], c[3], c[4]
        R['dsum'] = ar.dsum_ref(R['out'], X['dout'], B, H, Tq)[0].float()
        R.update(dq=G['dq'].to(torch.bfloat16), dk=G['dk'].to(torch.bfloat16), dv=G['dv'].to(torch.bfloat16),
                 dS=G['dS'].to(torch.bfloat16))
    return R


MUTATIONS = {   # mistake: the case it is planted in
    'drop_last_key': 'kv_edges', 'drop_key_127': 'kv_edges', 'drop_key_128': 'kv_edges',
    'causal_excl_diag': 'causal_300', 'causal_plus_one': 'causal_300', 'band_shift': 'band64_train',
    'scale_64': 'dk96_causal', 'lse_natural': 'kv_edges', 'ds_no_scale': 'causal_q_gt_k', 'D_from_dOV': 'band64_7',
    'dk_zero_tail_row': 'band64_train', 'dq_zero_wg1_row': 'causal_300',
}


@pytest.mark.parametrize('mutation', list(MUTATIONS))
def test_mutations_fail(mutation):
    c = ar.CASE[MUTATIONS[mutation]]
    X = ar.make_inputs(c)
    F, FB, G = reference_and_bounds(c, X)
    print('unmutated:')
    check_all(c, X, F, FB, G, _rounded(c, X, F, G))      # the true result, rounded, passes
    Fm, _, Gm = reference_and_bounds(c, X, mutation)
    got = _rounded(c, X, Fm, Gm)
    Tk = c[5]
    if mutation == 'dk_zero_tail_row':        # the last key row of the tail tile of batch 0 (visible there)
        assert Tk % 128 and c[6][0] >= Tk
        got['dk'][Tk - 1] = 0
    elif mutation == 'dq_zero_wg1_row':       # query row 197 = tile 1, second warpgroup
        got['dq'][197] = 0
    print(f'{mutation}:')
    with pytest.raises(AssertionError, match='out of bound'):
        check_all(c, X, F, FB, G, got)


def test_cases_reach_every_configuration():
    reached = set().union(*(ar.cells(c) for c in ar.CASES))
    outside = {c[0]: ar.cells(c) - ar.REACHABLE for c in ar.CASES if ar.cells(c) - ar.REACHABLE}
    assert not outside, f'cases outside what the kernels can run: {outside}'
    missing = ar.REACHABLE - reached
    assert not missing, f'configurations no case reaches: {sorted(missing, key=str)}'
    # the classifier sees what the host refuses: a band with a causal mask, lse at d_k 96, resid in training
    bad = ('x', 96, 2, 2, 8, 8, None, True, True, False, True, 'relpos', 0, 1.0, ())
    assert ar.cells(bad) - ar.REACHABLE >= {('fwd', 96, 'band_needs_self_noncausal'), ('fwd', 96, 'lse')}
    assert ('bwd', 'resid') in ar.cells(('x', 64, 2, 2, 8, 8, None, False, False, True, True, 'qkv', 0, 1.0, ()))


def test_planted_rows_aim_at_every_edge_key():
    """Each edge key (0, 127, 128, kv_len - 1, the causal diagonal) has a query row aimed at it: P above 0.3, mostly 0.6-0.9."""
    for name in ('kv_edges', 'causal_300', 'band64_train', 'dk96_cross'):
        c = ar.CASE[name]
        X = ar.make_inputs(c)
        F = ar.run_reference(c, X, 'cpu')
        lims = [min(x, c[5]) for x in (ar.kv_list(c) or [c[5]] * c[2])]
        for b, L in enumerate(lims):
            keys = {j for bb, _, j in X['planted'] if bb == b}
            assert set(ar.edge_keys(L, c[5])) <= keys, (name, b)
        p = torch.stack([F['P'][b, :, i, j] for b, i, j in X['planted']])
        assert float(p.min()) > 0.3 and float(p.median()) > 0.6, (name, float(p.min()))


# ------------------------------------------------------------------------------------------------ refusals
class Fake:
    """Claims to be a CUDA tensor so the device checks pass; the shape checks then run on the wrapped CPU tensor."""

    def __init__(self, t):
        self.t = t
        self.is_cuda, self.dtype, self.shape, self.device = True, t.dtype, t.shape, 'cuda'

    def is_contiguous(self):
        return self.t.is_contiguous()

    def dim(self):
        return self.t.dim()

    def stride(self, i):
        return self.t.stride(i)

    def numel(self):
        return self.t.numel()


def _z(*shape, dtype=torch.bfloat16):
    return Fake(torch.zeros(*shape, dtype=dtype))


@pytest.fixture
def no_library(monkeypatch):
    from opentransformer_b200 import _lib

    def stub():
        raise AssertionError('the library was reached')
    monkeypatch.setattr(_lib, 'lib', stub)


def test_attention_refuses_before_device_work(no_library):
    from opentransformer_b200 import ops
    B, H, T = 2, 2, 8
    qkv = _z(B * T, 3 * H * 64)
    kw = dict(q_col0=0, k_col0=128, v_col0=256)
    with pytest.raises(ValueError, match=r'v must be a matrix with columns \[264, 392\)'):
        ops.attention(qkv, qkv, qkv, B, H, T, T, q_col0=0, k_col0=128, v_col0=264)
    with pytest.raises(ValueError, match=r'q must be a matrix'):
        ops.attention(_z(B * T, 96), qkv, qkv, B, H, T, T, **kw)
    with pytest.raises(ValueError, match=r'q must be a matrix with columns \[0, 192\)'):
        ops.attention(_z(B * T, 190), qkv, qkv, B, H, T, T, q_col0=0, k_col0=0, v_col0=0, d_k=96)
    with pytest.raises(ValueError, match=r'out must have at least 16 rows and 128 columns'):
        ops.attention(qkv, qkv, qkv, B, H, T, T, out=_z(B * T - 1, 128), **kw)
    with pytest.raises(ValueError, match=r'out must have at least 16 rows and 128 columns'):
        ops.attention(qkv, qkv, qkv, B, H, T, T, out=_z(B * T, 120), **kw)
    with pytest.raises(TypeError, match='out must be a 2-D torch.bfloat16'):
        ops.attention(qkv, qkv, qkv, B, H, T, T, out=_z(B * T, 128, dtype=torch.float32), **kw)
    with pytest.raises(ValueError, match=r'resid must have at least 16 rows'):
        ops.attention(qkv, qkv, qkv, B, H, T, T, resid=_z(B * T - 8, 128), **kw)
    with pytest.raises(ValueError, match=r'resid must have at least 16 rows and 128 columns'):
        ops.attention(qkv, qkv, qkv, B, H, T, T, resid=_z(B * T, 120), **kw)
    with pytest.raises(TypeError, match='resid must be a 2-D torch.bfloat16'):
        ops.attention(qkv, qkv, qkv, B, H, T, T, resid=_z(B * T, 128, dtype=torch.float32), **kw)
    with pytest.raises(TypeError, match='int32'):
        ops.attention(qkv, qkv, qkv, B, H, T, T, kv_len=_z(B, dtype=torch.int64), **kw)
    with pytest.raises(ValueError, match='one length per batch entry'):
        ops.attention(qkv, qkv, qkv, B, H, T, T, kv_len=_z(B - 1, dtype=torch.int32), **kw)
    bd = _z(H, B * T, 2 * T, dtype=torch.float32)
    with pytest.raises(TypeError, match='float32'):
        ops.attention(qkv, qkv, qkv, B, H, T, T, bd=_z(H, B * T, 2 * T), **kw)
    with pytest.raises(ValueError, match='rel-pos band'):
        ops.attention(qkv, qkv, qkv, B, H, T, T, bd=bd, causal=True, **kw)
    with pytest.raises(ValueError, match='rel-pos band'):
        ops.attention(qkv, qkv, qkv, B, H, T, T - 1, bd=bd, **kw)
    with pytest.raises(ValueError, match=r'bd must have 32 rows of at least 15 columns'):
        ops.attention(qkv, qkv, qkv, B, H, T, T, bd=_z(H, B * T, 2 * T - 2, dtype=torch.float32), **kw)
    with pytest.raises(ValueError, match=r'bd must have 32 rows'):
        ops.attention(qkv, qkv, qkv, B, H, T, T, bd=_z(H, B * T - 1, 2 * T, dtype=torch.float32), **kw)
    with pytest.raises(ValueError, match=r'q must be a matrix'):
        ops.attention_train(_z(B * T, 100), qkv, qkv, B, H, T, T, **kw)
    with pytest.raises(ValueError, match='one length per batch entry'):
        ops.attention_train(qkv, qkv, qkv, B, H, T, T, kv_len=_z(1, dtype=torch.int32), **kw)
    with pytest.raises(ValueError, match=r'lse must be \[2, 2, 8\]'):
        ops.attention_train(qkv, qkv, qkv, B, H, T, T, lse=_z(B, H, T + 1, dtype=torch.float32), **kw)
    with pytest.raises(TypeError, match='lse must be torch.float32'):
        ops.attention_train(qkv, qkv, qkv, B, H, T, T, lse=_z(B, H, T), **kw)
    with pytest.raises(ValueError, match=r'out must have at least 16 rows'):
        ops.attention_train(qkv, qkv, qkv, B, H, T, T, out=_z(B * T - 1, 128), **kw)


def test_attention_bwd_refuses_before_device_work(no_library):
    from opentransformer_b200 import ops
    B, H, T = 2, 2, 8
    M, d = B * T, H * 64
    qkv, o, do, dqkv = _z(M, 3 * d), _z(M, d), _z(M, d), _z(M, 3 * d)
    lse = _z(B, H, T, dtype=torch.float32)
    kw = dict(q_col0=0, k_col0=d, v_col0=2 * d, dq_col0=0, dk_col0=d, dv_col0=2 * d)

    def call(**over):
        a = dict(q=qkv, k=qkv, v=qkv, out=o, dout=do, lse=lse, B=B, H=H, Tq=T, Tk=T, dq=dqkv, dk=dqkv, dv=dqkv, **kw)
        a.update(over)
        ops.attention_bwd(**a)
    with pytest.raises(ValueError, match=r'v must be a matrix with columns \[288, 416\)'):
        call(v_col0=2 * d + 32)
    with pytest.raises(ValueError, match=r'q must be a matrix with columns \[0, 128\)'):
        call(q=_z(M, 96), k=_z(M, 96), v=_z(M, 96), q_col0=0, k_col0=0, v_col0=0)
    with pytest.raises(ValueError, match=r'dv must be a matrix'):
        call(dv_col0=2 * d + 8)
    with pytest.raises(ValueError, match=r'out must have at least 16 rows and 128 columns'):
        call(out=_z(M, d - 64))
    with pytest.raises(ValueError, match=r'dout must have at least 16 rows'):
        call(dout=_z(M - 1, d))
    with pytest.raises(ValueError, match=r'dq must have at least 16 rows'):
        call(dq=_z(M - 1, 3 * d))
    with pytest.raises(ValueError, match=r'dk must have at least 24 rows'):
        call(Tk=12, k=_z(B * 12, 3 * d), v=_z(B * 12, 3 * d))
    with pytest.raises(TypeError, match='float32'):
        call(lse=_z(B, H, T))
    with pytest.raises(ValueError, match=r'lse must be \[2, 2, 8\]'):
        call(lse=_z(B, H, T - 1, dtype=torch.float32))
    with pytest.raises(ValueError, match=r'dsum must be \[2, 2, 8\]'):
        call(dsum=_z(B * H * T, dtype=torch.float32))
    with pytest.raises(TypeError, match='dsum must be torch.float32'):
        call(dsum=_z(B, H, T))
    with pytest.raises(ValueError, match='one length per batch entry'):
        call(kv_len=_z(1, dtype=torch.int32))
    bd, dbd = _z(H, M, 2 * T, dtype=torch.float32), _z(H, M, ops.rel_band_ld(T))
    with pytest.raises(ValueError, match='both be given'):
        call(bd=bd)
    with pytest.raises(ValueError, match='rel-pos band'):
        call(bd=bd, dbd=dbd, causal=True)
    with pytest.raises(ValueError, match=r'dbd must have 32 rows'):
        call(bd=bd, dbd=_z(H, M - 1, ops.rel_band_ld(T)))
    with pytest.raises(ValueError, match=r'dbd must have 32 rows of at least 15 columns'):
        call(bd=bd, dbd=_z(H, M, 2 * T - 2))
    with pytest.raises(TypeError, match='dbd must be torch.bfloat16'):
        call(bd=bd, dbd=_z(H, M, ops.rel_band_ld(T), dtype=torch.float32))
    with pytest.raises(TypeError, match='bd must be torch.float32'):
        call(bd=_z(H, M, 2 * T), dbd=dbd)
    with pytest.raises(ValueError, match=r'bd must have 32 rows of at least 15 columns'):
        call(bd=_z(H, M, 2 * T - 2, dtype=torch.float32), dbd=dbd)


@pytest.mark.skipif(torch.cuda.is_available(), reason='host-only check: it hands the entry point placeholder pointers')
def test_otb_attention_refuses_bad_bands():
    """The C entry point refuses a band it cannot index before any device work.  The pointers are placeholders, so this
    runs only where no GPU is visible: there a check that failed to refuse would end in a clean error (no CUDA driver or
    device), never in a launch."""
    from opentransformer_b200 import _lib
    lib = _lib.lib()
    p = ctypes.c_void_p(256)
    B, H, T, d = 2, 2, 8, 128

    def call(Tq, Tk, causal, ldbd):
        st = lib.otb_attention(p, 3 * d, B * Tq, p, 3 * d, B * Tk, p, 3 * d, p, d, B, H, Tq, Tk, None, causal, 0, d, 2 * d,
                               ctypes.cast(p, ctypes.POINTER(ctypes.c_float)), ldbd, None, 0, None, 64, None)
        return st, lib.otb_last_error().decode()
    for args, msg in (((T, T, 1, 2 * T), 'non-causal'), ((T, T + 1, 0, 2 * T + 2), 'Tq == Tk'),
                      ((T, T, 0, 2 * T - 2), 'must hold 2 Tq - 1 columns')):
        st, err = call(*args)
        assert st != 0 and msg in err, (args, err)
