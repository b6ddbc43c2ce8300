"""The LSTM recurrence kernels (csrc/lstm.cu, through ops.lstm_fwd / ops.lstm_bwd / ops.embedding) one call at a time against
the float64 restatement of tests/lstm_kernel_ref.py, at every hidden-size, batch and sequence edge they take.

Teacher forcing: each step of the restatement is fed the kernel's own inputs of that step -- its bf16 y_{t-1} (or h_0 rounded
to bf16, as the kernel stages it) and fp32 c_{t-1} in the forward, its bf16 dG_{t+1} in the backward, with dc carried in
float64 -- so the comparison sees one step's arithmetic however long the sequence, and the bounds follow from it (u = 2^-24):
  * The recurrent contraction is fp32: each warp runs ceil(K / 128) m16n8k16 steps (K = ceil16(H) forward, 4H backward),
    then the 8 warp partials and G_x (dy) are added one at a time.  The bound is C_DOT u S with S = |G_x| + |h||W_hh|^T
    (|dy| + |dG||W_hh|) and C_DOT = 4 ceil(K / 128) + 2 x 9: 4u per tensor-core step (it may truncate rather than round),
    2u per fp32 add.  C_DOT is 50 at H = 1024 forward and 146 at H = 1024 backward.
  * s(a) = 1 / (1 + __expf(-a)).  __expf(x) is within 2 + 1.173|x| ulps of e^x (CUDA C++ Programming Guide, intrinsic
    functions), a relative error d_e <= (2 + 1.173|a|) 2^-23, and ds / s = -(1 - s) de / e, so
    |ds| <= s(1 - s)(E_a + d_e) + 2u s (the add and the IEEE division).  tanhf is within 2 ulps: 4u relative.
  * Every other fp32 operation: u relative to the magnitude of its operands.
  * bf16 outputs (y, dG): one bf16 ulp of the float64 value plus the fp32 bound above (round to nearest takes half an ulp;
    the fp32 bound matters only where cancellation leaves the value far below its terms).
Free-running, the whole sequence against the float64 restatement that rounds h (dG) to bf16 at the same points: relative
L2, which catches an error that compounds over time.  Exact invariants are compared bit for bit.

Each test prints its worst error as a fraction of the bound it asserts (run with -s to see it).  Run with -m gpu on an H100."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops
    DEV = torch.device('cuda:0')

from tests import lstm_kernel_ref as kr

BF = torch.bfloat16
U = 2.0 ** -24
LSTM_WARPS = 8
FREE_REL = 2e-3          # free-running relative L2 (see test_lstm_layer)

# (H, B, L, initial state).  H: 8 is one CTA; 24, 72 and 1000 are not multiples of 16 (the forward's kp > H path); 1056
# fills 132 SMs.  B: the forward works in chunks of 32 rows, the backward in chunks of 16; 320 = 32 utterances x beam 10 is
# the shallow-fusion / LM-rescoring step with a carried (h, c).  Each edge of each axis meets large values of the others.
CASES = [
    (8, 65, 300, 'h0c0'),
    (16, 33, 300, 'h0'),
    (24, 17, 64, 'c0'),
    (24, 15, 2, 'h0c0'),
    (72, 31, 300, 'none'),
    (72, 1, 1, 'none'),
    (256, 1, 300, 'h0c0'),
    (256, 15, 64, 'h0'),
    (256, 16, 64, 'c0'),
    (1000, 33, 64, 'h0c0'),
    (1000, 17, 64, 'none'),
    (1024, 16, 300, 'none'),
    (1024, 32, 64, 'c0'),
    (1024, 65, 2, 'h0'),
    (1024, 320, 1, 'h0c0'),
    (1056, 31, 300, 'h0c0'),
    (1056, 65, 64, 'c0'),
    (1056, 16, 1, 'h0'),
]


def _need_sms(H):
    if H > 8 * ops.num_sms():
        pytest.skip(f'H = {H} needs {H // 8} SMs at 8 units per CTA; this device has {ops.num_sms()}')


def _case(H, B, L, init, seed=0):
    """W_hh ~ U(-1/sqrt(H), 1/sqrt(H)) (nn.LSTM's initialisation) in bf16, G_x ~ N(0, 0.8^2), h_0 ~ N(0, 0.5^2),
    c_0 ~ N(0, 1), dy ~ N(0, 0.5^2) in bf16."""
    g = torch.Generator().manual_seed(seed * 7919 + H + 31 * B + 977 * L)
    w = ((torch.rand(4 * H, H, generator=g) * 2 - 1) * H ** -0.5).to(BF)
    gx = 0.8 * torch.randn(L * B, 4 * H, generator=g)
    h0 = 0.5 * torch.randn(B, H, generator=g) if 'h0' in init else None
    c0 = torch.randn(B, H, generator=g) if 'c0' in init else None
    dy = (0.5 * torch.randn(L * B, H, generator=g)).to(BF)
    dev = lambda t: None if t is None else t.to(DEV)
    return dev(w), dev(gx), dev(h0), dev(c0), dev(dy)


def _bf(t):
    """Round a float64 value to bf16 the way the kernels do: fp32 first, then round to nearest even."""
    return t.float().to(BF).double()


def _ulp_bf16(x):
    """Spacing of bf16 numbers at |x| (x float64)."""
    _, e = torch.frexp(x)
    return torch.ldexp(torch.ones_like(x), e - 8)


def _c_dot(K):
    return 4 * math.ceil(K / (16 * LSTM_WARPS)) + 2 * (LSTM_WARPS + 1)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _worst(err, bound):
    return float((err / bound).max())


def _state(t, B, H):
    return t.double() if t is not None else torch.zeros(B, H, dtype=torch.float64, device=DEV)


def _sig_bound(s, a, e_a):
    return s * (1 - s) * (e_a + (2 + 1.173 * a.abs()) * 2.0 ** -23) + 2 * U * s


def check_forward_step(w, gx, h0, c0, y, hn, gates, c_all, L, B, H):
    """Teacher-forced forward: the kernel's gates, c_t, y_t and h_n against one float64 step from the kernel's own inputs.
    Returns the worst error of each as a fraction of its bound (y also in bf16 ulps)."""
    W = w.double()
    gx64 = gx.double().view(L, B, 4 * H)
    Y = y.double().view(L, B, H)
    C = c_all.double().view(L, B, H)
    h_in = torch.cat([_bf(_state(h0, B, H))[None], Y[:-1]])
    c_in = torch.cat([_state(c0, B, H)[None], C[:-1]])
    g64, c64, h64 = kr.fwd_step(gx64, h_in, c_in, W)
    a = gx64 + h_in @ W.t()
    e_a = _c_dot((H + 15) // 16 * 16) * U * (gx64.abs() + h_in.abs() @ W.abs().t())
    del gx64
    i, f, g, o = g64.chunk(4, -1)
    ai, af, ag, ao = a.chunk(4, -1)
    ei, ef, eg, eo = e_a.chunk(4, -1)
    e_i, e_f, e_o = _sig_bound(i, ai, ei), _sig_bound(f, af, ef), _sig_bound(o, ao, eo)
    e_g = (1 - g * g) * eg + 4 * U * g.abs()
    del a, e_a, ai, af, ag, ao, ei, ef, eg, eo
    r_gates = _worst((gates.double().view(L, B, 4 * H) - g64).abs(), torch.cat([e_i, e_f, e_g, e_o], -1))
    e_c = c_in.abs() * e_f + g.abs() * e_i + i * e_g + e_i * e_g + 2 * U * ((f * c_in).abs() + (i * g).abs())
    r_c = _worst((C - c64).abs(), e_c)
    tc = torch.tanh(c64)
    e_h = tc.abs() * e_o + o * e_c + e_o * e_c + 4 * U * o * tc.abs() + U * h64.abs()
    r_hn = _worst((hn.double() - h64[-1]).abs(), e_h[-1])
    ulp = _ulp_bf16(h64)
    r_y = _worst((Y - h64).abs(), ulp + e_h)
    y_ulps = float(((Y - h64).abs() / ulp).max())
    return r_gates, r_c, r_hn, r_y, y_ulps


def check_backward_step(w, dy, gates, c_all, c0, dg, L, B, H):
    """Teacher-forced backward: every dG_t against the float64 step from the kernel's own dG_{t+1}, dc carried in float64
    with its error bound carried beside it.  Returns the worst error as a fraction of (1 bf16 ulp + bound), and in ulps."""
    W = w.double()
    DY = dy.double().view(L, B, H)
    G = gates.double().view(L, B, 4 * H)
    C = c_all.double().view(L, B, H)
    DG = dg.double().view(L, B, 4 * H)
    nxt = torch.cat([DG[1:], torch.zeros_like(DG[:1])])
    dh_all = DY + nxt @ W
    e_dh_all = _c_dot(4 * H) * U * (DY.abs() + nxt.abs() @ W.abs())
    c_prev = torch.cat([_state(c0, B, H)[None], C[:-1]])
    carry = torch.zeros(B, H, dtype=torch.float64, device=DEV)
    e_carry = torch.zeros_like(carry)
    r_worst, ulp_worst = 0.0, 0.0
    for t in range(L - 1, -1, -1):
        ref, carry_next = kr.bwd_step(DY[t], nxt[t] if t + 1 < L else None, W, G[t], C[t], c_prev[t], carry)
        i, f, g, o = G[t].chunk(4, -1)
        dh, e_dh, cp = dh_all[t], e_dh_all[t], c_prev[t]
        tc = torch.tanh(C[t])
        A = o * (1 - tc * tc)
        dc = carry + dh * A
        e_dc = e_carry + dh.abs() * 10 * U * o * (1 + tc * tc) + A * e_dh + 2 * U * (carry.abs() + (dh * A).abs())
        ri, rf, rg, ro = ref.abs().chunk(4, -1)
        e = torch.cat([e_dc * (g * i * (1 - i)).abs() + 6 * U * ri,
                       e_dc * (cp * f * (1 - f)).abs() + 6 * U * rf,
                       e_dc * i * (1 - g * g) + dc.abs() * i * 2 * U * (1 + g * g) + 6 * U * rg,
                       e_dh * (tc * o * (1 - o)).abs() + dh.abs() * o * (1 - o) * 4 * U * tc.abs() + 6 * U * ro], -1)
        err, ulp = (DG[t] - ref).abs(), _ulp_bf16(ref)
        r_worst = max(r_worst, _worst(err, ulp + e))
        ulp_worst = max(ulp_worst, float((err / ulp).max()))
        e_carry = f * e_dc + U * (dc * f).abs()
        carry = carry_next
    return r_worst, ulp_worst


def _fwd(w, gx, L, B, h0, c0, train=True):
    return ops.lstm_fwd(gx.clone(), w, L, B, h0, c0, train=train)


@pytest.mark.parametrize('H,B,L,init', CASES, ids=[f'H{H}-B{B}-L{L}-{i}' for H, B, L, i in CASES])
def test_lstm_layer(H, B, L, init):
    """Forward and backward of one layer: teacher-forced step bounds, free-running relative L2, exact invariants.

    Free-running, the kernel and the restatement see the same bf16 rounding points, so what separates them is the odd h
    (dG) that falls on the other side of a bf16 rounding boundary, one bf16 ulp (2^-8 relative) on one element, which
    the recurrence then damps: FREE_REL = 2e-3 relative L2 over the sequence."""
    _need_sms(H)
    w, gx, h0, c0, dy = _case(H, B, L, init)
    y, hn, cn, gates, c_all = out = ops.lstm_fwd(gxk := gx.clone(), w, L, B, h0, c0, train=True)
    assert gates is gxk                                     # training mode records the gates over G_x
    r_gates, r_c, r_hn, r_y, y_ulps = check_forward_step(w, gx, h0, c0, y, hn, gates, c_all, L, B, H)
    assert max(r_gates, r_c, r_hn, r_y) <= 1.0, (r_gates, r_c, r_hn, r_y)

    # exact invariants
    assert torch.equal(hn.to(BF), y[(L - 1) * B:]) and torch.equal(cn, c_all[(L - 1) * B:])
    for a, b in zip(out, _fwd(w, gx, L, B, h0, c0)):
        assert torch.equal(a, b), 'two identical calls differ'
    yi, hni, cni, gi, ci = _fwd(w, gx, L, B, h0, c0, train=False)
    assert gi is None and ci is None
    assert torch.equal(yi, y) and torch.equal(hni, hn) and torch.equal(cni, cn), 'inference mode differs from training mode'

    # free-running forward
    g64, c64, y64, hn64, cn64 = kr.forward(gx.double().view(L, B, 4 * H), w.double(), None if h0 is None else h0.double(),
                                           None if c0 is None else c0.double(), round_h=_bf)
    free = [_rel(y, y64.view(L * B, H)), _rel(c_all, c64.view(L * B, H)), _rel(gates, g64.view(L * B, 4 * H)),
            _rel(hn, hn64), _rel(cn, cn64)]
    del g64, c64, y64
    assert max(free) < FREE_REL, free

    # backward
    dg = ops.lstm_bwd(dy, w, gates, c_all, L, B, c0)
    assert torch.equal(dg, ops.lstm_bwd(dy, w, gates, c_all, L, B, c0)), 'two identical calls differ'
    r_dg, dg_ulps = check_backward_step(w, dy, gates, c_all, c0, dg, L, B, H)
    assert r_dg <= 1.0, r_dg
    dg64 = kr.backward(dy.double().view(L, B, H), w.double(), gates.double().view(L, B, 4 * H), c_all.double().view(L, B, H),
                       None if c0 is None else c0.double(), round_dg=_bf)
    free_dg = _rel(dg, dg64.view(L * B, 4 * H))
    assert free_dg < FREE_REL, free_dg
    print(f'\nH{H} B{B} L{L} {init}: forward step, worst error / bound: gates {r_gates:.3f}, c {r_c:.3f}, h_n {r_hn:.3f}, '
          f'y {r_y:.3f} ({y_ulps:.3f} bf16 ulp); free-running rel L2 y {free[0]:.2e} c {free[1]:.2e} gates {free[2]:.2e} '
          f'h_n {free[3]:.2e} c_n {free[4]:.2e} (< {FREE_REL:.0e}) | backward step dG {r_dg:.3f} of (1 ulp + bound) '
          f'({dg_ulps:.3f} bf16 ulp); free-running rel L2 {free_dg:.2e}')


# ------------------------------------------------------------------------------------------------ the grid barrier
def _calls(specs):
    """One closure per (kind, H, B, L, init): the forward (training mode) or the backward of a prepared layer."""
    calls = []
    for k, (kind, H, B, L, init) in enumerate(specs):
        w, gx, h0, c0, dy = _case(H, B, L, init, seed=100 + k)
        if kind == 'fwd':
            calls.append((L, lambda w=w, gx=gx, h0=h0, c0=c0, L=L, B=B: _fwd(w, gx, L, B, h0, c0)))
        else:
            _, _, _, gates, c_all = _fwd(w, gx, L, B, h0, c0)
            calls.append((L, lambda w=w, dy=dy, g=gates, ca=c_all, c0=c0, L=L, B=B: (ops.lstm_bwd(dy, w, g, ca, L, B, c0),)))
    torch.cuda.synchronize()
    return calls


def test_barrier_shared_across_grid_sizes():
    """Forward and backward launches of different H (grids of 1 to 132 CTAs) back to back on one stream's barrier: each
    result equals the same call made alone, and the barrier's generation advanced by exactly one per step boundary."""
    big = 1056 if ops.num_sms() >= 132 else 8 * ops.num_sms()
    specs = [('fwd', 1024, 17, 9, 'h0c0'), ('bwd', 8, 5, 12, 'c0'), ('fwd', big, 33, 6, 'none'), ('fwd', 72, 3, 20, 'h0'),
             ('bwd', big, 16, 7, 'h0c0'), ('bwd', 256, 40, 5, 'none'), ('fwd', 8, 2, 30, 'c0'), ('bwd', 1024, 31, 8, 'c0'),
             ('fwd', 24, 65, 3, 'none')]
    calls = _calls(specs)
    alone = []
    for _, call in calls:
        alone.append(call())
        torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        bar = ops._lstm_barrier(DEV)
        gen0 = bar.clone()
        together = [call() for _, call in calls]
        assert ops._lstm_barrier(DEV) is bar
    torch.cuda.synchronize()
    for spec, a, b in zip(specs, alone, together):
        for x, y in zip(a, b):
            assert torch.equal(x, y), f'{spec}: differs from the same call made alone'
    steps = sum(L - 1 for L, _ in calls)
    assert int(bar[0]) == 0 and (int(bar[1]) - int(gen0[1])) % 2 ** 32 == steps, (bar.tolist(), gen0.tolist(), steps)
    print(f'\n{len(calls)} launches on one barrier, {steps} grid barriers: each bit-identical to the call made alone')


def test_barrier_per_stream_concurrent():
    """One small forward (16 and 8 CTAs, so both grids fit the device together) on each of two streams, each with its own
    barrier: each equals its serial result."""
    specs = [('fwd', 128, 33, 64, 'h0c0'), ('fwd', 64, 17, 64, 'none')]
    calls = _calls(specs)
    serial = []
    for _, call in calls:
        serial.append(call())
        torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    assert streams[0].cuda_stream != streams[1].cuda_stream
    bars, outs = [], []
    for st, (_, call) in zip(streams, calls):
        with torch.cuda.stream(st):
            bars.append(ops._lstm_barrier(DEV))
            outs.append(call())
    assert bars[0] is not bars[1]
    torch.cuda.synchronize()
    for spec, a, b in zip(specs, serial, outs):
        for x, y in zip(a, b):
            assert torch.equal(x, y), f'{spec}: the concurrent call differs from the serial one'
    print('\ntwo concurrent forwards on two streams: each bit-identical to its serial result')


# ------------------------------------------------------------------------------------------------ embedding
@pytest.mark.parametrize('d', [8, 256, 264, 1024])
def test_embedding(d):
    """A gather, bit for bit: repeated ids, and ids out of range (-1, V and beyond) read row 0."""
    V = 50
    g = torch.Generator().manual_seed(d)
    emb = torch.randn(V, d, generator=g).to(BF).to(DEV)
    fixed = torch.tensor([3, 3, 0, V - 1, -1, V, 7, 3, 12, V - 1, -1, 10 ** 6, 5])
    tok = torch.cat([fixed, torch.randint(-3, V + 3, (1003,), generator=g)])
    ref = emb.cpu()[torch.where((tok >= 0) & (tok < V), tok, torch.zeros_like(tok))]
    for t in (fixed, tok, tok[:1]):
        out = ops.embedding(t.to(DEV), emb)
        assert torch.equal(out.cpu(), ref[:t.numel()]), t.numel()
    out = torch.full((tok.numel(), d), 7.0, dtype=BF, device=DEV)
    assert ops.embedding(tok.view(8, -1).to(DEV), emb, out=out) is out and torch.equal(out.cpu(), ref)
