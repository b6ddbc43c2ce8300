"""The SIMT inference and loss kernels in float64 -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Plain restatements of what csrc/ops_simt.cu, csrc/loss.cu and logsoftmax_topk_kernel (csrc/beam.cu) compute, written the
obvious way with no fusion: each function takes the operands exactly as the kernel receives them (bf16-rounded or f32
tensors, converted here to float64) and returns float64.  Every function runs on whichever device its inputs live on.
tests/test_simt_kernels_ref.py pins each one to torch.nn.functional (and the oracle's label-smoothing loss) in float64.
"""
import math

import torch

F64 = torch.float64


def layernorm(x, g1, b1, g2=None, b2=None, eps=1e-5):
    """nn.LayerNorm over the last dim (biased variance), optionally a second one applied to the first one's output."""
    def one(v, g, b):
        mean = v.mean(-1, keepdim=True)
        var = ((v - mean) ** 2).mean(-1, keepdim=True)
        return (v - mean) / torch.sqrt(var + eps) * g.to(F64) + b.to(F64)
    y = one(x.to(F64), g1, b1)
    return y if g2 is None else one(y, g2, b2)


def log_softmax(x):
    """Row log-softmax x - (max + log sum exp(x - max)); a row of -inf gives NaN, as torch does."""
    x = x.to(F64)
    m = x.amax(-1, keepdim=True)
    return x - (m + torch.log(torch.exp(x - m).sum(-1, keepdim=True)))


def fused_logp(x, lm=None, lm_weight=0.0):
    """log_softmax(x) + lm_weight * lm: the scores logsoftmax_topk ranks."""
    lp = log_softmax(x)
    return lp if lm is None else lp + lm_weight * lm.to(F64)


def stable_topk(v, k):
    """Per-row top-k in the order (value descending, index ascending) -> (values, ids int64).  A stable descending sort on
    the CPU keeps equal values in index order; torch.topk on CUDA promises no tie order."""
    vals, ids = torch.sort(v.to(F64).cpu(), dim=-1, descending=True, stable=True)
    return vals[..., :k].to(v.device), ids[..., :k].to(v.device)


def ls_ce(logits, tgt, V, smoothing, pad_id):
    """LabelSmoothingLoss with a PAD id: per-token KL(conf || softmax) with xlogy semantics (0 log 0 = 0), conf = 1 - smoothing
    on the target and smoothing / (V - 1) elsewhere.  A row whose target is PAD or outside [0, V) is not scored: loss 0,
    gradient 0, and it does not count.  logits [rows, >= V] -> (mean loss, per-token loss [rows], n_valid, d(mean)/dlogits
    [rows, V])."""
    x = logits[:, :V].to(F64)
    tgt = tgt.to(x.device)
    valid = (tgt != pad_id) & (tgt >= 0) & (tgt < V)
    conf = torch.full_like(x, smoothing / (V - 1))
    rows = torch.nonzero(valid).view(-1)
    conf[rows, tgt[rows]] = 1.0 - smoothing
    logp = log_softmax(x)
    per_tok = (torch.xlogy(conf, conf) - conf * logp).sum(-1) * valid
    n = int(valid.sum())
    denom = max(n, 1)
    grad = (torch.exp(logp) - conf) * valid[:, None] / denom
    return per_tok.sum() / denom, per_tok, n, grad


def embed_posenc(tok, emb, table, d, tok_stride=1, period=None, step=None, row_pos=None):
    """out[n] = emb[tok[n * tok_stride]] * sqrt(d) + table[pos], an id outside [0, vocab) reading row 0, and pos =
    max(row_pos[n], 0) (row_pos given), else step (given), else n % period."""
    t = tok.reshape(-1)[::tok_stride].long()
    N = t.numel()
    t = torch.where((t >= 0) & (t < emb.shape[0]), t, torch.zeros_like(t))
    if row_pos is not None:
        pos = row_pos.long().clamp(min=0)
    elif step is not None:
        pos = torch.full((N,), int(step), dtype=torch.long, device=t.device)
    else:
        pos = torch.arange(N, device=t.device) % period
    return emb.to(F64)[t] * math.sqrt(d) + table.to(F64)[pos]


def scale_add_table(x, alpha, table=None, period=1):
    """x * alpha + table[row % period] (table None: x * alpha)."""
    y = x.to(F64) * alpha
    if table is not None:
        y = y + table.to(F64)[torch.arange(x.shape[0], device=x.device) % period]
    return y


def dwconv_swish(x, w, b, B, T):
    """Depthwise Conv1d over time with zero padding (k - 1) / 2 inside each utterance, the BatchNorm folded into w f32 [k, d]
    and b f32 [d], then swish.  x [B*T, d] -> [B*T, d]."""
    k, d = w.shape
    pad = (k - 1) // 2
    xp = torch.nn.functional.pad(x.to(F64).view(B, T, d), (0, 0, pad, pad))
    acc = b.to(F64).expand(B, T, d).clone()
    for tap in range(k):
        acc = acc + xp[:, tap:tap + T] * w[tap].to(F64)
    return (acc * torch.sigmoid(acc)).view(B * T, d)


def _attend(q, ks, vs, scale):
    """q [N, H, dk], ks / vs [N, L, H, dk] -> softmax(q . k * scale) . v  [N, H, dk]."""
    s = torch.einsum('nhd,nlhd->nhl', q, ks) * scale
    return torch.einsum('nhl,nlhd->nhd', torch.softmax(s, -1), vs)


def decode_self_attn(qkv, kc, vc, anc, H, step=None, row_pos=None):
    """One query per row over its cached prefix and its own newest K/V.  qkv [N, 3d] (Q | K | V of the newest token).
    step: kc / vc [Lmax, N, d], anc [2, N, Lmax]; position s < step of row n is kc[s, anc[step & 1, n, s]].
    row_pos [N]: kc / vc [rows, d], anc [N, Lmax]; position s < row_pos[n] of row n is kc[anc[n, s]], and a row at -1 gets
    zeros.  The newest position's K/V come from qkv.  Scale 1 / sqrt(d_k).  Returns float64 [N, d]."""
    N, d3 = qkv.shape
    d = d3 // 3
    dk = d // H
    scale = 1.0 / math.sqrt(dk)
    qkv = qkv.to(F64)
    q = qkv[:, :d].view(N, H, dk)
    knew, vnew = qkv[:, d:2 * d], qkv[:, 2 * d:]
    if row_pos is None:
        cur = anc[step & 1, :, :step].long()                                   # [N, step]
        pos = torch.arange(step, device=cur.device)[None, :].expand(N, step)
        ks = torch.cat([kc[pos, cur].to(F64), knew[:, None]], 1).view(N, step + 1, H, dk)
        vs = torch.cat([vc[pos, cur].to(F64), vnew[:, None]], 1).view(N, step + 1, H, dk)
        return _attend(q, ks, vs, scale).reshape(N, d)
    out = torch.zeros(N, d, dtype=F64, device=qkv.device)
    for p in sorted(set(int(v) for v in row_pos.tolist()) - {-1}):            # rows at the same position in one batch
        rows = torch.nonzero(row_pos == p).view(-1)
        cur = anc[rows, :p].long()                                             # [n, p]
        ks = torch.cat([kc[cur].to(F64), knew[rows, None]], 1).view(len(rows), p + 1, H, dk)
        vs = torch.cat([vc[cur].to(F64), vnew[rows, None]], 1).view(len(rows), p + 1, H, dk)
        out[rows] = _attend(q[rows], ks, vs, scale).reshape(len(rows), d)
    return out
