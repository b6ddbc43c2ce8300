"""Without a GPU: the float64 LSTM restatement of tests/lstm_kernel_ref.py against nn.LSTM and autograd, and the launch plan
of the recurrence kernels (otb_lstm_config, host only) over every hidden size up to 2048 on both H100 variants."""
import pytest
import torch

from tests import lstm_kernel_ref as kr

INITS = ['none', 'h0', 'c0', 'h0c0']
SMEM_OPTIN = 232448                   # H100 opt-in shared memory per block
LSTM_WARPS = 8
BWD_ROWS = 16


def _problem(I, H, L, B, init, seed):
    torch.manual_seed(seed)
    lstm = torch.nn.LSTM(I, H).double()
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(L, B, I, generator=g, dtype=torch.float64)
    h0 = 0.5 * torch.randn(B, H, generator=g, dtype=torch.float64) if 'h0' in init else None
    c0 = torch.randn(B, H, generator=g, dtype=torch.float64) if 'c0' in init else None
    return lstm, x, h0, c0


def _gx(lstm, x):
    return x @ lstm.weight_ih_l0.detach().t() + lstm.bias_ih_l0.detach() + lstm.bias_hh_l0.detach()


def _nn_state(t, B, H):
    return (t if t is not None else torch.zeros(B, H, dtype=torch.float64))[None]


@pytest.mark.parametrize('init', INITS)
def test_forward_matches_nn_lstm(init):
    I, H, L, B = 12, 24, 9, 5
    lstm, x, h0, c0 = _problem(I, H, L, B, init, seed=3)
    with torch.no_grad():
        y_ref, (hn_ref, cn_ref) = lstm(x, (_nn_state(h0, B, H), _nn_state(c0, B, H)))
        gates, c_all, y, hn, cn = kr.forward(_gx(lstm, x), lstm.weight_hh_l0, h0, c0)
    assert gates.shape == (L, B, 4 * H) and c_all.shape == (L, B, H)
    assert torch.allclose(y, y_ref, rtol=0, atol=1e-12)
    assert torch.allclose(hn, hn_ref[0], rtol=0, atol=1e-12) and torch.allclose(cn, cn_ref[0], rtol=0, atol=1e-12)
    assert torch.equal(c_all[-1], cn) and torch.equal(y[-1], hn)
    i, f, g, o = gates.chunk(4, -1)
    assert bool(((i > 0) & (i < 1) & (f > 0) & (f < 1) & (o > 0) & (o < 1) & (g.abs() < 1)).all())


@pytest.mark.parametrize('init', INITS)
def test_backward_matches_autograd(init):
    """dG_t against autograd's gradient of sum(y * dy) with respect to the pre-activation gates of a hand-written float64
    cell; sum_t dG_t^T y_{t-1} (y_{-1} = h_0), sum_t dG_t^T x_t and sum_t dG_t against nn.LSTM's weight_hh / weight_ih /
    bias gradients."""
    I, H, L, B = 10, 16, 8, 4
    lstm, x, h0, c0 = _problem(I, H, L, B, init, seed=11)
    dy = torch.randn(L, B, H, generator=torch.Generator().manual_seed(12), dtype=torch.float64)
    w_hh = lstm.weight_hh_l0.detach()
    gx = _gx(lstm, x).detach()

    zero = torch.zeros(B, H, dtype=torch.float64)
    w_leaf = w_hh.clone().requires_grad_(True)             # so that every a_t is a non-leaf whose gradient autograd keeps
    h, c, pre, ys = (h0 if h0 is not None else zero), (c0 if c0 is not None else zero), [], []
    for t in range(L):
        a = gx[t] + h @ w_leaf.t()
        a.retain_grad()
        pre.append(a)
        ai, af, ag, ao = a.chunk(4, -1)
        c = torch.sigmoid(af) * c + torch.sigmoid(ai) * torch.tanh(ag)
        h = torch.sigmoid(ao) * torch.tanh(c)
        ys.append(h)
    (torch.stack(ys) * dy).sum().backward()
    dg_auto = torch.stack([a.grad for a in pre])

    with torch.no_grad():
        gates, c_all, y, _, _ = kr.forward(gx, w_hh, h0, c0)
        dg = kr.backward(dy, w_hh, gates, c_all, c0)
    assert torch.allclose(dg, dg_auto, rtol=0, atol=1e-12)

    y_ref, _ = lstm(x, (_nn_state(h0, B, H), _nn_state(c0, B, H)))
    (y_ref * dy).sum().backward()
    y_prev = torch.cat([(h0 if h0 is not None else zero)[None], y[:-1]])
    assert torch.allclose(torch.einsum('tbg,tbh->gh', dg, y_prev), lstm.weight_hh_l0.grad, rtol=0, atol=1e-10)
    assert torch.allclose(torch.einsum('tbg,tbi->gi', dg, x), lstm.weight_ih_l0.grad, rtol=0, atol=1e-10)
    assert torch.allclose(dg.sum((0, 1)), lstm.bias_hh_l0.grad, rtol=0, atol=1e-10)


def test_rounding_points():
    """round_h is applied to h_0 and to each y_t the next step reads, not to h_n; round_dg to each dG_t the step before
    reads."""
    H, L, B = 8, 4, 3
    g = torch.Generator().manual_seed(5)
    gx = torch.randn(L, B, 4 * H, generator=g, dtype=torch.float64)
    w = 0.3 * torch.randn(4 * H, H, generator=g, dtype=torch.float64)
    h0, c0 = torch.randn(B, H, generator=g, dtype=torch.float64), torch.randn(B, H, generator=g, dtype=torch.float64)
    bf = lambda t: t.to(torch.bfloat16).double()
    gates, c_all, y, hn, cn = kr.forward(gx, w, h0, c0, round_h=bf)
    assert torch.equal(y, bf(y)) and not torch.equal(hn, bf(hn)) and torch.equal(bf(hn), y[-1])
    h_prev = torch.cat([bf(h0)[None], y[:-1]])
    c_prev = torch.cat([c0[None], c_all[:-1]])
    g1, c1, h1 = kr.fwd_step(gx, h_prev, c_prev, w)          # one step over the whole teacher-forced stack
    close = lambda a, b: torch.allclose(a, b, rtol=0, atol=1e-14)       # one batched matmul vs L small ones
    assert close(g1, gates) and close(c1, c_all) and torch.equal(bf(h1), y)
    dy = torch.randn(L, B, H, generator=g, dtype=torch.float64)
    dg = kr.backward(dy, w, gates, c_all, c0, round_dg=bf)
    assert torch.equal(dg, bf(dg))
    assert not torch.equal(dg, bf(kr.backward(dy, w, gates, c_all, c0)))


# ------------------------------------------------------------------------------------------------ launch plan
def _fwd_smem(u, H):
    """lstm_fwd_kernel<u / 4>: W_hh rows of the 4u gate rows and BC = 256 / u staged h rows, both [.][ceil16(H) + 8] bf16,
    then the cross-warp partial sums [warps][BC][4u + 1] fp32."""
    bc, ld = 256 // u, (H + 15) // 16 * 16 + 8
    return (4 * u + bc) * ld * 2 + LSTM_WARPS * bc * (4 * u + 1) * 4


def _bwd_smem(u, H):
    """lstm_bwd_kernel<u>: W_hh columns of the u units and 16 staged dG rows, both [.][4H + 8] bf16, then [warps][16][17] fp32."""
    return (u + BWD_ROWS) * (4 * H + 8) * 2 + LSTM_WARPS * BWD_ROWS * 17 * 4


@pytest.fixture(scope='module')
def ops():
    from opentransformer_b200 import build
    build.build()
    from opentransformer_b200 import ops
    return ops


@pytest.mark.parametrize('sms', [132, 114])           # H100 SXM, H100 PCIe
def test_plan_table(ops, sms):
    """Every accepted H runs 8 units per CTA on H / 8 <= SMs CTAs, with the shared memory of the layout above; the first
    refused H is 8 x SMs + 8.  Above 8 x SMs the plan asks for 16 units, and the 16-unit backward needs
    32 x (4H + 8) x 2 + 8704 B > 232448 B for every H > 872, so no H ever gets 16 units on an H100."""
    accepted = []
    for H in range(8, 2049, 8):
        try:
            u, f, b = ops.lstm_config(H, sms, SMEM_OPTIN)
        except NotImplementedError as e:
            assert 'does not fit' in str(e), (H, str(e))
            continue
        accepted.append(H)
        assert u == 8 and H // u <= sms, (H, u)
        assert (f, b) == (_fwd_smem(8, H), _bwd_smem(8, H)), H
        assert f <= SMEM_OPTIN and b <= SMEM_OPTIN
    assert accepted == list(range(8, 8 * sms + 1, 8))
    assert max(H for H in range(8, 2049, 8) if _bwd_smem(16, H) <= SMEM_OPTIN) == 872 < 8 * 114
    assert ops.lstm_config(1024, 132, SMEM_OPTIN)[0] == 8
    with pytest.raises(NotImplementedError, match='does not fit'):
        ops.lstm_config(1024, 114, SMEM_OPTIN)      # rnnlm.yaml's H = 1024 on a 114-SM H100
    for H in (0, 4, 1020, 2047):
        with pytest.raises(NotImplementedError, match='multiple of 8'):
            ops.lstm_config(H, sms, SMEM_OPTIN)
