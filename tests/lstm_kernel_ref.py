"""One LSTM layer in float64, step by step, as csrc/lstm.cu computes it -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

nn.LSTM semantics, gates in the order i, f, g, o: a = G_x + h_{t-1} W_hh^T (G_x already holds both biases),
c_t = s(f) c_{t-1} + s(i) tanh(g), h_t = s(o) tanh(c_t).  The backward step is the one lstm_bwd_kernel takes: it gets the
recorded post-activation gates and c_t, forms dh_t = dy_t + dG_{t+1} W_hh and carries dc_t f_t to the step before.

Every function works on any leading batch shape, so a test can hand one step a whole [L, B, .] stack of teacher-forced
inputs.  The free-running drivers take a `round_h` / `round_dg` callable applied where the kernels store bf16 (h_{t-1} as it
is staged, including h_0; dG_{t+1} as it is read back); None keeps everything float64.  tests/test_lstm_kernel_ref.py pins
this restatement to nn.LSTM and autograd.
"""
import torch


def fwd_step(gx, h_prev, c_prev, w_hh):
    """gx [..., 4H], h_prev / c_prev [..., H], w_hh [4H, H] -> (post-activation gates [..., 4H] (i, f, g, o), c_t, h_t)."""
    i, f, g, o = (gx + h_prev @ w_hh.t()).chunk(4, dim=-1)
    i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
    c = f * c_prev + i * g
    h = o * torch.tanh(c)
    return torch.cat([i, f, g, o], -1), c, h


def bwd_step(dy, dg_next, w_hh, gates, c, c_prev, dc_carry):
    """dy [..., H]; dg_next [..., 4H] = dG_{t+1} or None at the last step; gates [..., 4H] and c = c_t, c_prev = c_{t-1} of the
    forward; dc_carry = dc_{t+1} f_{t+1} (zero at the last step) -> (dG_t [..., 4H] pre-activation gradients (i, f, g, o),
    the dc_t f_t to carry to step t - 1)."""
    dh = dy if dg_next is None else dy + dg_next @ w_hh
    i, f, g, o = gates.chunk(4, dim=-1)
    tc = torch.tanh(c)
    dc = dc_carry + dh * o * (1 - tc * tc)
    dg = torch.cat([dc * g * i * (1 - i), dc * c_prev * f * (1 - f), dc * i * (1 - g * g), dh * tc * o * (1 - o)], -1)
    return dg, dc * f


def forward(gx, w_hh, h0=None, c0=None, round_h=None):
    """gx [L, B, 4H] -> (gates [L, B, 4H], c_all [L, B, H], y [L, B, H], h_n, c_n [B, H]).  With round_h, y_t = round_h(h_t) is
    what the next step reads (and h_0 is rounded the same way); h_n is h_{L-1} unrounded, as otb_lstm_fwd returns it."""
    L, B, H4 = gx.shape
    rnd = round_h or (lambda t: t)
    zero = gx.new_zeros(B, H4 // 4)
    h = rnd(h0) if h0 is not None else zero
    c = c0 if c0 is not None else zero
    gates, cs, ys = [], [], []
    for t in range(L):
        gt, c, hf = fwd_step(gx[t], h, c, w_hh)
        h = rnd(hf)
        gates.append(gt)
        cs.append(c)
        ys.append(h)
    return torch.stack(gates), torch.stack(cs), torch.stack(ys), hf, c


def backward(dy, w_hh, gates, c_all, c0=None, round_dg=None):
    """Backward through time of forward(): dy [L, B, H], gates [L, B, 4H], c_all [L, B, H] -> dG [L, B, 4H].  With round_dg,
    dG_t = round_dg(dG_t) is what step t - 1 reads."""
    L = dy.shape[0]
    rnd = round_dg or (lambda t: t)
    carry = torch.zeros_like(dy[0])
    c0 = c0 if c0 is not None else torch.zeros_like(dy[0])
    dgs, nxt = [None] * L, None
    for t in range(L - 1, -1, -1):
        dg, carry = bwd_step(dy[t], nxt, w_hh, gates[t], c_all[t], c_all[t - 1] if t > 0 else c0, carry)
        nxt = dgs[t] = rnd(dg)
    return torch.stack(dgs)
