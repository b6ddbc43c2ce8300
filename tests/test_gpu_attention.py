"""The tensor-core attention forward (attn_tc_kernel, otb_attention) and backward (attn_bwd_dq_kernel /
attn_bwd_dkv_kernel, otb_attention_bwd) against the float64 restatement of tests/attention_ref.py, element by element,
at every configuration they accept: the cases of attention_ref.CASES reach every cell of attention_ref.REACHABLE
(tests/test_attention_ref.py checks that on the CPU, and that the bounds hold for an emulation of the kernels and fail for
plausible mistakes).  The bounds are derived in attention_ref's docstring; the float64 references run on the device.

Every operand lives in a matrix with NaN in its pitch padding; out, dq, dk and dv are column windows of NaN-filled
buffers with wider pitches and extra rows, lse and dsum NaN-filled, dBD NaN-filled rather than zeroed: what the kernels
do not write must stay NaN, and exactly the visible (i, j) entries of dBD are written.  q, k and v have rows past B*T,
and dout NaN rows past B*Tq: the backward reads dO at rows [0, B*Tq) only (its last query tile takes TMA zero fill past
them), and a NaN read there would reach dV through 0 * NaN.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, the worst err/bound over all cases: O 0.93 (band96_resid),
lse 0.048, dsum 0.023, dQ 0.26, dK 0.40, dV 0.88 (dec_self_bench), dBD 0.41; the 29 cases take 11 s.  Before the
backward sized dO's tensor map by B*Tq, it read dout rows past B*Tq up to q's row count, and enc_bench, cross_bench and
band64_7 failed here with NaN in dV (every key row whose query loop reached the last tile).  O and dV come near 1
where an output has a single term (a row with one visible key, a key seen by one query): there the bf16 rounding of P and
that of the output can both reach 2^-8, which is exactly what the bound allows them, as the GEMM's bf16 outputs do."""
import pytest
import torch

from tests import attention_ref as ar

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops
    DEV = torch.device('cuda:0')
BF = torch.bfloat16
NAN = float('nan')
ROWS_PAST = 5


def _window(rows, cols, col0, dtype=BF, extra=3):
    """(NaN buffer with `extra` more rows and a pitch of col0 + cols + 24, its [rows, cols] window at column col0)."""
    buf = torch.full((rows + extra, col0 + cols + 24), NAN, dtype=dtype, device=DEV)
    return buf, buf[:rows, col0:col0 + cols]


def _outside_nan(buf, rows, c0, c1, what):
    keep = torch.ones(buf.shape, dtype=torch.bool, device=DEV)
    keep[:rows, c0:c1] = False
    assert bool(torch.isnan(buf[keep].float()).all()), f'{what} was written outside its window'


@pytest.mark.parametrize('name', ar.NAMES)
def test_attention_matches_float64(name):
    c = ar.CASE[name]
    _, dk, B, H, Tq, Tk, _, causal, _, _, train = c[:11]
    d = H * dk
    X = ar.make_inputs(c)
    moved = {}

    def dev(t, extra_rows=0):
        if t is None:
            return None
        if id(t) not in moved:
            moved[id(t)] = torch.cat([t, t.new_zeros(extra_rows, t.shape[1])]).to(DEV) if extra_rows else t.to(DEV)
        return moved[id(t)]
    # q, k and v carry 5 rows past B*T: the backward must not size dO's reads by q's rows (dout below has NaN after B*Tq)
    q, k, v = (dev(X[n], ROWS_PAST) for n in ('q', 'k', 'v'))
    kv_len, bd, resid = (dev(X[n]) for n in ('kv_len', 'bd', 'resid'))
    qc, kc, vc = X['col0s']
    cols = dict(q_col0=qc, k_col0=kc, v_col0=vc)
    obuf, out = _window(B * Tq, d, 16)
    if train:
        lse = torch.full((B, H, Tq), NAN, device=DEV)
        ops.attention_train(q, k, v, B, H, Tq, Tk, kv_len=kv_len, causal=causal, bd=bd, out=out, lse=lse, **cols)
        plain = ops.attention(q, k, v, B, H, Tq, Tk, kv_len=kv_len, causal=causal, bd=bd, **cols)
        assert torch.equal(out, plain), 'attention_train must compute what attention computes, bit for bit'
    else:
        ops.attention(q, k, v, B, H, Tq, Tk, kv_len=kv_len, causal=causal, bd=bd, resid=resid, d_k=dk, out=out, **cols)
    torch.cuda.synchronize()
    _outside_nan(obuf, B * Tq, 16, 16 + d, 'out')

    F = ar.forward(q, k, v, B, H, Tq, Tk, kv_len, causal, X['col0s'], bd, resid, dk)
    FB = ar.forward_bounds(F)
    print(f'{name}:')
    ar.check('out', out, F['out'], FB['out'])
    lims = [min(x, Tk) for x in (ar.kv_list(c) or [Tk] * B)]
    dead = [b for b, L in enumerate(lims) if L == 0]
    for b in dead:   # no visible key: the output is the residual (zero without one)
        want = resid[b * Tq:(b + 1) * Tq, :d] if resid is not None else torch.zeros_like(out[b * Tq:(b + 1) * Tq])
        assert torch.equal(out[b * Tq:(b + 1) * Tq], want)
    if not train:
        return

    # lse: log2 units, +inf exactly on the rows without a visible key
    assert torch.equal(torch.isinf(lse) & (lse > 0), torch.isinf(F['lse'])), 'lse must be +inf exactly on rows without keys'
    ar.check('lse', lse, F['lse'], FB['lse'])

    dbuf, dout = _window(B * Tq, d, 0, extra=2 * ROWS_PAST)
    dout.copy_(X['dout'])
    qbuf, dq = _window(B * Tq, d, 16)
    kvbuf, _ = _window(B * Tk, 2 * d, 8)
    dsum = torch.full((B, H, Tq), NAN, device=DEV)
    dbd = None
    if bd is not None:
        dbd = torch.full((H, B * Tq, ops.rel_band_ld(Tq)), NAN, dtype=BF, device=DEV)
    ops.attention_bwd(q, k, v, out, dout, lse, B, H, Tq, Tk, qbuf, kvbuf, kvbuf, kv_len=kv_len, causal=causal,
                      dq_col0=16, dk_col0=8, dv_col0=8 + d, bd=bd, dbd=dbd, dsum=dsum, **cols)
    torch.cuda.synchronize()
    _outside_nan(qbuf, B * Tq, 16, 16 + d, 'dq')
    _outside_nan(kvbuf, B * Tk, 8, 8 + 2 * d, 'dk / dv')
    dk_, dv = kvbuf[:B * Tk, 8:8 + d], kvbuf[:B * Tk, 8 + d:8 + 2 * d]

    G = ar.backward(F, dout)
    BB = ar.backward_bounds(F, G, FB, out)
    D, eD = ar.dsum_ref(out, dout, B, H, Tq)
    ar.check('dsum', dsum, D, eD)
    ar.check('dq', dq, G['dq'], BB['dq'])
    ar.check('dk', dk_, G['dk'], BB['dk'])
    ar.check('dv', dv, G['dv'], BB['dv'])
    if dbd is not None:
        ref, written = ar.band_layout(G['dS'], F['vis'], B, H, Tq, dbd.shape[-1])
        bound, _ = ar.band_layout(BB['dS'], F['vis'], B, H, Tq, dbd.shape[-1])
        assert bool(torch.isnan(dbd[~written].float()).all()), 'dBD must be written exactly at the visible (i, j)'
        ar.check('dbd', dbd[written], ref[written], bound[written])
    for b in dead:   # zero gradients on a batch entry without keys
        for t, T in ((dq, Tq), (dk_, Tk), (dv, Tk)):
            assert float(t[b * T:(b + 1) * T].float().abs().max()) == 0.0
