"""The SIMT kernels of the training step in float64 -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Plain restatements of what csrc/backward.cu (LayerNorm backward, GLU, dropout backward, dropout_add, embedding backward,
the clipped Adam step with its schedule, SpecAugment) and csrc/conformer_train.cu (the Conformer convolution module in
training mode) compute, written from the module semantics the kernels cite, with no fusion.  Each function takes the
operands as the kernel receives them (bf16 or f32 tensors, upcast here) and returns float64.  Dropout keep masks are
explicit operands: the counter hash that draws them is checked bit for bit against ops.dropout_mask, not restated.
tests/test_simt_train_kernels_ref.py pins each one to torch autograd, torch.optim.Adam and nn.BatchNorm1d in float64.
"""
import math

import torch

F64 = torch.float64


def layernorm_bwd(dy, z, gamma, eps=1e-5):
    """Backward of y = LayerNorm(z) * gamma + beta over the last dim (biased variance), statistics recomputed from z.
    -> (dz [M, N], dgamma [N], dbeta [N])."""
    z, dy, gamma = z.to(F64), dy.to(F64), gamma.to(F64)
    mean = z.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((z - mean) ** 2).mean(-1, keepdim=True) + eps)
    xh = (z - mean) * rstd
    g = dy * gamma
    dz = rstd * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
    return dz, (dy * xh).sum(0), dy.sum(0)


def glu(u):
    """F.glu over the last dim: u = [a | g] -> a * sigmoid(g)."""
    a, g = u.to(F64).chunk(2, -1)
    return a * torch.sigmoid(g)


def glu_bwd(dh, u):
    """Gradient of glu with respect to u = [a | g]: [dh * s | dh * a * s * (1 - s)], s = sigmoid(g)."""
    a, g = u.to(F64).chunk(2, -1)
    dh = dh.to(F64)
    s = torch.sigmoid(g)
    return torch.cat([dh * s, dh * a * s * (1 - s)], -1)


def dropout_scale(p, p2=0.0):
    """1 / ((1 - p) (1 - p2)) of the rates as the kernel receives them (f32), in float64."""
    p, p2 = float(torch.tensor(p, dtype=torch.float32)), float(torch.tensor(p2, dtype=torch.float32))
    return 1.0 / ((1.0 - p) * (1.0 - p2))


def dropout_bwd(dy, keep, p, p2=0.0):
    """dy * keep / ((1 - p) (1 - p2)); keep is the product of the masks of both sites."""
    return dy.to(F64) * keep.to(F64) * dropout_scale(p, p2)


def row_live(M, row_len=None, row_period=0, device=None):
    """Rows with row % row_period < row_len[row // row_period] (all rows without row_len) -> bool [M]."""
    if row_len is None:
        return torch.ones(M, dtype=torch.bool, device=device)
    r = torch.arange(M, device=row_len.device)
    return r % row_period < row_len.long()[r // row_period]


def dropout_add(x, resid, keep, p, alpha=1.0, row_len=None, row_period=0):
    """resid + alpha * dropout_p(rowmask(x)); resid None: no residual.  keep None: every element kept (p = 0)."""
    x = x.to(F64)
    kept = row_live(x.shape[0], row_len, row_period, x.device)[:, None].to(F64)
    if keep is not None:
        kept = kept * keep.to(F64)
    y = alpha * x * kept * dropout_scale(p)
    return y if resid is None else resid.to(F64) + y


def embed_bwd(tok, dx, dE, scale):
    """dE + scatter-add of scale * dx[n] into row tok[n]; ids outside [0, V) add nothing."""
    out = dE.to(F64).clone()
    tok = tok.reshape(-1).long()
    ok = (tok >= 0) & (tok < dE.shape[0])
    out.index_add_(0, tok[ok], dx.to(F64)[ok] * scale)
    return out


def transformer_lr(step, model_size, warmup, factor):
    """TransformerScheduler.get_step_lr: factor * model_size^-0.5 * min(step^-0.5, step * warmup^-1.5)."""
    return factor * model_size ** -0.5 * min(step ** -0.5, step * warmup ** -1.5)


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def adam_step(p, g, m, v, sumsq, counters, max_norm, base_lr, model_size, warmup, factor, b1, b2, eps, wd):
    """One step of clip_grad_norm_(max_norm) + torch.optim.Adam (L2 weight decay) with the TransformerScheduler learning
    rate, given sumsq = sum g^2 as the kernel reads it.  max_norm 0: no clip; warmup <= 0: lr = base_lr.  A non-finite
    norm skips the step: p, m, v unchanged and only the skip count counters[2] advances.  The scalar hyper-parameters are
    the f32 values the kernel receives.  -> (p, m, v, counters [3] list, hyper [4] = (lr, 1 - b1^t, 1 - b2^t, applied))."""
    p, g, m, v = (t.to(F64) for t in (p, g, m, v))
    max_norm, base_lr, model_size, warmup, factor, b1, b2, eps, wd = (
        _f32(x) for x in (max_norm, base_lr, model_size, warmup, factor, b1, b2, eps, wd))
    steps, gstep, skipped = (int(c) for c in counters)
    total = math.sqrt(sumsq) if sumsq >= 0 else math.nan
    if not math.isfinite(total):
        return p, m, v, [steps, gstep, skipped + 1], None
    t, s = steps + 1, gstep + 1
    lr = transformer_lr(s, model_size, warmup, factor) if warmup > 0 else base_lr
    bc1, bc2 = 1.0 - b1 ** t, 1.0 - b2 ** t
    coef = min(1.0, max_norm / (total + 1e-6)) if max_norm > 0 else 1.0
    gd = g * coef + wd * p
    m = b1 * m + (1 - b1) * gd
    v = b2 * v + (1 - b2) * gd * gd
    p = p - lr / bc1 * m / (torch.sqrt(v) / math.sqrt(bc2) + eps)
    return p, m, v, [t, s, skipped], [lr, bc1, bc2, 1.0]


def spec_augment(x, bands, nf, nt):
    """x [B, T, F] with, per utterance, frequency bins [f0, f0 + f) of its nf bands and frames [t0, t0 + t) of its nt
    bands set to zero; bands [B, 2 (nf + nt)] = (f0, f) * nf, (t0, t) * nt.  A band may be empty, overlap another or reach
    past the edge."""
    x = x.to(F64).clone()
    for b, row in enumerate(bands.tolist()):
        for j in range(nf):
            f0, f = row[2 * j], row[2 * j + 1]
            if f > 0:
                x[b, :, max(f0, 0):max(f0 + f, 0)] = 0.0
        for j in range(nt):
            t0, t = row[2 * (nf + j)], row[2 * (nf + j) + 1]
            if t > 0:
                x[b, max(t0, 0):max(t0 + t, 0)] = 0.0
    return x


# ------------------------------------------------------------------------------------------------ Conformer conv module
def frame_mask(lens, B, T):
    """Valid frames [B, T]: t < min(len[b], T) (a length above T means every frame is valid)."""
    return torch.arange(T, device=lens.device)[None, :] < lens.long().clamp(max=T)[:, None]


def _dwconv(x, w, B, T):
    """Depthwise conv over time inside each utterance, zero padding (k - 1) / 2: x [B, T, d], w [d, k] -> [B, T, d]."""
    d, k = w.shape
    pad = (k - 1) // 2
    xp = torch.nn.functional.pad(x, (0, 0, pad, pad))
    out = torch.zeros(B, T, d, dtype=F64, device=x.device)
    for tap in range(k):
        out = out + xp[:, tap:tap + T] * w[:, tap]
    return out


def conv_module_train(x, lens, w, wb, gamma, beta, running_mean, running_var, num_batches, B, T, momentum=0.1, eps=1e-5):
    """The middle of the Conformer convolution module in train(): c = depthwise_conv(mask(x)) + wb; BatchNorm1d with the
    batch statistics of all B*T positions (biased variance); out = mask(swish(BN(c))).  The running buffers follow
    nn.BatchNorm1d: (1 - momentum) * old + momentum * batch, running_var with the unbiased variance (the biased one when
    B*T = 1), num_batches_tracked + 1.  x [B*T, d], w [d, k], wb [d] or None.
    -> dict(out, c [B*T, d], mean, invstd, running_mean, running_var [d], num_batches)."""
    d = x.shape[1]
    M = B * T
    mask = frame_mask(lens, B, T)
    xm = x.to(F64).view(B, T, d) * mask[..., None]
    c = _dwconv(xm, w.to(F64), B, T).view(M, d)
    if wb is not None:
        c = c + wb.to(F64)
    mean = c.mean(0)
    var = ((c - mean) ** 2).mean(0)
    invstd = 1.0 / torch.sqrt(var + eps)
    a = (c - mean) * invstd * gamma.to(F64) + beta.to(F64)
    out = a * torch.sigmoid(a) * mask.view(M, 1)
    mo = _f32(momentum)
    res = dict(out=out, c=c, mean=mean, invstd=invstd, num_batches=None)
    unbiased = var * M / (M - 1) if M > 1 else var
    res['running_mean'] = None if running_mean is None else (1 - mo) * running_mean.to(F64) + mo * mean
    res['running_var'] = None if running_var is None else (1 - mo) * running_var.to(F64) + mo * unbiased
    if num_batches is not None:
        res['num_batches'] = int(num_batches) + 1
    return res


def conv_module_bwd(dy, x, lens, w, gamma, beta, B, T, c=None, mean=None, invstd=None, wb=None, eps=1e-5):
    """Backward of conv_module_train for the gradient dy of out.  The batch statistics and c are the forward's: pass the
    forward kernel's c, mean and invstd (the backward kernel's own operands), or leave them None to recompute them from x
    (and wb).  -> dict(dx [B*T, d] (zero on padded frames), dw [d, k], dwb [d], dgamma [d], dbeta [d], and the
    intermediates da, xh, dc [B*T, d])."""
    d, k = w.shape
    M = B * T
    pad = (k - 1) // 2
    mask = frame_mask(lens, B, T)
    m = mask.reshape(M, 1).to(F64)
    xm = x.to(F64).view(B, T, d) * mask[..., None]
    if c is None:
        c = _dwconv(xm, w.to(F64), B, T).view(M, d)
        if wb is not None:
            c = c + wb.to(F64)
        mean = c.mean(0)
        invstd = 1.0 / torch.sqrt(((c - mean) ** 2).mean(0) + eps)
    c, mean, invstd, gamma = c.to(F64), mean.to(F64), invstd.to(F64), gamma.to(F64)
    xh = (c - mean) * invstd
    a = xh * gamma + beta.to(F64)
    s = torch.sigmoid(a)
    da = dy.to(F64) * m * s * (1 + a * (1 - s))
    dbeta, dgamma = da.sum(0), (da * xh).sum(0)
    dc = gamma * invstd * (da - dbeta / M - xh * dgamma / M)
    # dx[t] = mask[t] * sum_tap w[tap] * dc[t - tap + pad] over the conv's output frames [0, T): the transposed conv
    dcp = torch.nn.functional.pad(dc.view(B, T, d), (0, 0, pad, pad))
    dx = torch.zeros(B, T, d, dtype=F64, device=dc.device)
    w64 = w.to(F64)
    for tap in range(k):
        dx = dx + dcp[:, 2 * pad - tap:2 * pad - tap + T] * w64[:, tap]
    dx = dx * mask[..., None]
    # dw[ch, tap] = sum_t dc[t] * mask(x)[t + tap - pad]
    xp = torch.nn.functional.pad(xm, (0, 0, pad, pad))
    dw = torch.stack([(dc.view(B, T, d) * xp[:, tap:tap + T]).sum((0, 1)) for tap in range(k)], 1)
    return dict(dx=dx.view(M, d), dw=dw, dwb=dc.sum(0), dgamma=dgamma, dbeta=dbeta, da=da, xh=xh, dc=dc)
