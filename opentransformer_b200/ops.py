"""torch.Tensor-level wrappers around the C ABI (include/otb200.h).

PyTorch is plumbing here: it owns device memory and the current CUDA stream; all compute is in
libotb200.so.  Every wrapper launches on ``torch.cuda.current_stream()`` so the calls can be
captured into a CUDA graph (recognize.BeamDecoder captures a decode step, train.FusedTrainer a training micro-step).
"""
import ctypes
import math
import operator

import torch

from . import _lib
from ._lib import check

EPI_BIAS, EPI_RELU, EPI_GLU, EPI_TABLE, EPI_RESID, EPI_RESID_LN, EPI_SWISH, EPI_GELU, EPI_TANH = range(9)
ACT_EPILOGUE = {'relu': EPI_RELU, 'glu': EPI_GLU, 'swish': EPI_SWISH, 'gelu': EPI_GELU, 'tanh': EPI_TANH}
# the activations act_fwd / act_bwd take (training runs ReLU fused into the GEMM and GLU through glu_fwd / glu_bwd)
TRAIN_ACT = {k: ACT_EPILOGUE[k] for k in ('gelu', 'tanh', 'swish')}
BF16 = torch.bfloat16


# ---- instrumentation (bench.py): kernel-launch counter and optional per-launch CUDA-event timing ----
COUNTERS = {'launches': 0}
PROFILE = None          # set to a list to collect (kind, algorithmic_flops, start_event, end_event) per GEMM launch


def _count(n=1):
    COUNTERS['launches'] += n


class _Timed:
    """Record CUDA events around one launch on the current stream when PROFILE is enabled."""

    def __init__(self, kind, flops, tag=None):
        self.kind, self.flops, self.tag = kind, flops, tag

    def __enter__(self):
        if PROFILE is not None and not torch.cuda.is_current_stream_capturing():
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        else:
            self.e0 = None

    def __exit__(self, *exc):
        if self.e0 is not None:
            self.e1.record()
            PROFILE.append((self.kind, self.flops, self.e0, self.e1, self.tag))


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _need(t, dtype, name):
    if not t.is_cuda:
        raise RuntimeError(f'{name} must be a CUDA tensor: the CUDA hot path has no CPU fallback')
    if t.dtype != dtype:
        raise TypeError(f'{name} must be {dtype}, got {t.dtype}')
    if not t.is_contiguous():
        raise ValueError(f'{name} must be contiguous')
    return t


def _mat(t, name, dtype=BF16):
    """A matrix operand: 2-D CUDA tensor of `dtype` (a GEMM's bf16 by default) with unit column stride (row-strided views
    such as one head's columns of a wider matrix are fine: the TMA map takes the row pitch)."""
    if not t.is_cuda:
        raise RuntimeError(f'{name} must be a CUDA tensor: the CUDA hot path has no CPU fallback')
    if t.dtype != dtype or t.dim() != 2 or t.stride(1) != 1:
        raise TypeError(f'{name} must be a 2-D {dtype} tensor with unit column stride')
    return t


def set_decode_barrier(kind):
    """'cluster', 'software' or 'default': group barrier of the persistent decode kernel (otb_set_decode_barrier)."""
    check(_lib.lib().otb_set_decode_barrier({'default': -1, 'software': 0, 'cluster': 1}[kind]), 'otb_set_decode_barrier')


def set_tile_policy(policy):
    """'latency' (default) or 'throughput': tiling of the small decode-step GEMMs (otb_set_tile_policy).  Takes effect for
    launches / graph captures made afterwards."""
    check(_lib.lib().otb_set_tile_policy({'latency': 0, 'throughput': 1}[policy]), 'otb_set_tile_policy')


def num_sms():
    return int(_lib.lib().otb_num_sms())


# (kt1, kf1, st1, sf1, kt2, kf2, st2, sf2) of the shipped conv front end: two 3x3 convolutions at stride 2
CONV_SHIPPED = (3, 3, 2, 2, 3, 3, 2, 2)


def conv_sizes(T, F, geom=CONV_SHIPPED):
    """otb_conv_geometry -> (T1, F1, T2, F2, T1p, F1p): the two layers' output sizes and the conv1 activation buffer's rows
    and columns.  The front end's own geometry (modules.conv_frontend_geometry) is what callers size their outputs by."""
    out = (ctypes.c_int * 6)()
    check(_lib.lib().otb_conv_geometry(T, F, *geom, out), 'otb_conv_geometry')
    return tuple(out)


def conv_geometry(T, F):
    """(T1, F1, T2, F2) of the shipped conv front end."""
    return conv_sizes(T, F)[:4]


def conv1_relu(x, w, bias, out=None, geom=CONV_SHIPPED):
    """x f32 [B,T,F]; w f32 [C1,1,kt1,kf1] -> bf16 NHWC [B, T1p, F1p, C1] (conv_sizes; [B, 2*(T2+1), 2*F2, C1] shipped)."""
    _need(x, torch.float32, 'x'); _need(w, torch.float32, 'w'); _need(bias, torch.float32, 'bias')
    B, T, F = x.shape
    C1 = w.shape[0]
    T1p, F1p = conv_sizes(T, F, geom)[4:]
    if out is None:
        out = torch.empty(B, T1p, F1p, C1, dtype=BF16, device=x.device)
    check(_lib.lib().otb_conv1_relu(_p(x), _p(w), _p(bias), _p(out), B, T, F, C1, *geom, _stream()), 'otb_conv1_relu')
    _count()
    return out


def conv2_relu(h1, w, bias, B, T, F, out=None, geom=CONV_SHIPPED):
    """h1 = conv1 buffer; w bf16 [C2, kt2*kf2*C1] (kh,kw,c order) -> bf16 [B*T2, F2*C2] (feature = f*C2 + c)."""
    _need(h1, BF16, 'h1'); _need(w, BF16, 'w'); _need(bias, torch.float32, 'bias')
    C2, K = w.shape
    C1 = K // (geom[4] * geom[5])
    _, _, T2, F2, _, _ = conv_sizes(T, F, geom)
    if out is None:
        out = torch.empty(B * T2, F2 * C2, dtype=BF16, device=h1.device)
    with _Timed('conv2_gemm', 2.0 * B * T2 * F2 * C2 * K):
        check(_lib.lib().otb_conv2_relu(_p(h1), _p(w), _p(bias), _p(out), B, T, F, C1, C2, *geom, _stream()),
              'otb_conv2_relu')
    _count()
    return out


def linear(a, w, bias=None, epilogue=EPI_BIAS, out=None, out_f32=False, resid=None, gamma=None, beta=None,
           eps=1e-5, alpha=1.0, table=None, period=0, row_len=None, row_period=0, n_out=None):
    """out[M,N] = epi(a[M,K] @ w[N(,2N),K]^T + bias).  a, w: see _mat."""
    _mat(a, 'a'); _mat(w, 'w')
    M, K = a.shape
    N = w.shape[0] // 2 if epilogue == EPI_GLU else w.shape[0]
    if w.shape[1] != K:
        raise ValueError(f'linear: K mismatch {w.shape} vs {a.shape}')
    if out is None:
        ldc = n_out if n_out is not None else N
        out = torch.empty(M, ldc, dtype=torch.float32 if out_f32 else BF16, device=a.device)
    ldc = out.stride(0)
    with _Timed('gemm', 2.0 * M * w.shape[0] * K, (epilogue, M, w.shape[0], K, out.dtype == torch.float32)):
        check(_lib.lib().otb_linear(_p(a), a.stride(0), _p(w), w.stride(0), _p(bias), _p(out), ldc, M, N, K, epilogue,
                                    1 if out.dtype == torch.float32 else 0, _p(resid),
                                    resid.stride(0) if resid is not None else 0, _p(gamma), _p(beta), eps, alpha,
                                    _p(table), period, _p(row_len), row_period, _stream()), 'otb_linear')
    _count()
    return out


def gemm_config(M, N, epilogue=EPI_BIAS, out_f32=False):
    """N tile width (64, 128 or 256) linear() launches for an M x N output under the current tile policy
    (otb_gemm_config: host only, no GPU needed); raises RuntimeError where linear() would refuse the combination."""
    bn = ctypes.c_int()
    check(_lib.lib().otb_gemm_config(M, N, epilogue, 1 if out_f32 else 0, bn), 'otb_gemm_config')
    return bn.value


def linear_dropout_resid(a, w, bias, resid, p, seed, site, alpha=1.0, out=None, p2=0.0, site2=0):
    """out = resid + alpha * dropout_p(a @ w^T + bias): training-mode residual connection (otb_linear_dropout_resid).
    seed: int32/uint32 device tensor [1] (read at run time), site: dropout site id.  (p2, site2): a second independent
    mask on the same tensor (the attention's output dropout): out = resid + alpha * dropout_p(dropout_p2(a @ w^T + bias))."""
    _mat(a, 'a'); _mat(w, 'w'); _mat(resid, 'resid')
    M, K = a.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty(M, N, dtype=BF16, device=a.device)
    check(_lib.lib().otb_linear_dropout_resid(_p(a), a.stride(0), _p(w), w.stride(0), _p(bias), _p(out), out.stride(0), M, N, K,
                                              _p(resid), resid.stride(0), alpha, float(p), _p(seed), int(site), float(p2), int(site2),
                                              _stream()),
          'otb_linear_dropout_resid')
    _count()
    return out


def dropout_bwd(dy, p, seed, site, p2=0.0, site2=0):
    """dy * keep / (1 - p) with the mask of dropout site `site` replayed from (seed, site); with p2 > 0 also the mask of
    site2, as linear_dropout_resid drew them: dy * keep * keep2 / ((1 - p) (1 - p2))."""
    _need(dy, BF16, 'dy')
    M, N = dy.shape
    out = torch.empty_like(dy)
    check(_lib.lib().otb_dropout_bwd(_p(dy), dy.stride(0), _p(out), out.stride(0), None, M, N, float(p), _p(seed), int(site),
                                     float(p2), int(site2), _stream()), 'otb_dropout_bwd')
    _count()
    return out


def dropout_add(x, resid, p=0.0, seed=None, site=0, alpha=1.0, row_len=None, row_period=0, out=None):
    """out = resid + alpha * dropout_p(x) with the mask of (seed, site) (otb_dropout_add); resid None: alpha * dropout_p(x),
    also the backward of such a site.  row_len / row_period: rows past their utterance's length read x as zero."""
    _mat(x, 'x')
    if resid is not None:
        _mat(resid, 'resid')
    if row_len is not None:
        _need(row_len, torch.int32, 'row_len')
    M, N = x.shape
    if out is None:
        out = torch.empty(M, N, dtype=BF16, device=x.device)
    check(_lib.lib().otb_dropout_add(_p(x), x.stride(0), _p(resid), resid.stride(0) if resid is not None else 0, _p(out), out.stride(0),
                                     M, N, float(alpha), float(p), _p(seed), int(site), _p(row_len), int(row_period), _stream()),
          'otb_dropout_add')
    _count()
    return out


def dropout_mask(M, N, p, seed, site, p2=0.0, site2=0):
    """u8 [M,N] keep mask of a dropout site (parity tests replay it in the oracle) -- any site, the attention-output sites
    (train.ATTN_SITE + ...) included; with p2 > 0 the product of the masks of site and site2, as dropout_bwd applies it."""
    mask = torch.empty(M, N, dtype=torch.uint8, device=seed.device)
    check(_lib.lib().otb_dropout_bwd(None, 0, None, 0, _p(mask), M, N, float(p), _p(seed), int(site), float(p2), int(site2),
                                     _stream()), 'otb_dropout_bwd')
    _count()
    return mask


HEAD_DIMS = (64, 96)   # head widths the attention kernels are built for


def check_head_dim(d_k):
    if d_k not in HEAD_DIMS:
        raise NotImplementedError(f'the sm_90a attention kernels support head widths d_k in {HEAD_DIMS}, got {d_k}')


def _head_cols(op, t, col0, width, name):
    """Heads read or write columns [col0, col0 + width) of matrix t."""
    if t.dim() != 2 or col0 < 0 or col0 + width > t.shape[1]:
        raise ValueError(f'{op}: {name} must be a matrix with columns [{col0}, {col0 + width}) for the heads, got {tuple(t.shape)}')


def _rows_cols(op, t, rows, cols, name):
    """A matrix the kernel reads or writes at rows [0, rows) and columns [0, cols)."""
    if t.shape[0] < rows or t.shape[1] < cols:
        raise ValueError(f'{op}: {name} must have at least {rows} rows and {cols} columns, got {tuple(t.shape)}')


def _kv_len(op, kv_len, B):
    if kv_len is not None:
        _need(kv_len, torch.int32, 'kv_len')
        if kv_len.numel() < B:
            raise ValueError(f'{op}: kv_len must hold one length per batch entry ({B}), got {kv_len.numel()}')


def _band(op, bd, B, H, Tq, Tk, causal, dtype, name):
    """The rel-pos band (or its gradient): H*B*Tq rows of at least 2 Tq - 1 columns, for non-causal self-attention."""
    _need(bd, dtype, name)
    if Tq != Tk or causal:
        raise ValueError(f'{op}: the rel-pos band is for non-causal self-attention (Tq == Tk)')
    if bd.dim() < 2 or bd.shape[-1] < 2 * Tq - 1 or bd.numel() // bd.shape[-1] < H * B * Tq:
        raise ValueError(f'{op}: {name} must have {H * B * Tq} rows of at least {2 * Tq - 1} columns, got {tuple(bd.shape)}')


def _attention(q, k, v, B, H, Tq, Tk, kv_len, causal, q_col0, k_col0, v_col0, out=None, bd=None, resid=None, d_k=64,
               with_lse=False, lse=None):
    """otb_attention -> (out bf16 [B*Tq, H*d_k], lse f32 [B,H,Tq] (written into lse when given) if with_lse else None)."""
    for t, n in ((q, 'q'), (k, 'k'), (v, 'v')):
        _need(t, BF16, n)
    check_head_dim(d_k)
    for t, c0, n in ((q, q_col0, 'q'), (k, k_col0, 'k'), (v, v_col0, 'v')):
        _head_cols('attention', t, c0, H * d_k, n)
    if out is not None:
        _rows_cols('attention', _mat(out, 'out'), B * Tq, H * d_k, 'out')
    if resid is not None:
        _rows_cols('attention', _mat(resid, 'resid'), B * Tq, H * d_k, 'resid')
    if bd is not None:
        _band('attention', bd, B, H, Tq, Tk, causal, torch.float32, 'bd')
    _kv_len('attention', kv_len, B)
    if with_lse and lse is not None:
        _need(lse, torch.float32, 'lse')
        if tuple(lse.shape) != (B, H, Tq):
            raise ValueError(f'attention: lse must be [{B}, {H}, {Tq}], got {tuple(lse.shape)}')
    if out is None:
        out = torch.empty(B * Tq, H * d_k, dtype=BF16, device=q.device)
    if not with_lse:
        lse = None
    elif lse is None:
        lse = torch.empty(B, H, Tq, dtype=torch.float32, device=q.device)
    check(_lib.lib().otb_attention(_p(q), q.stride(0), q.shape[0], _p(k), k.stride(0), k.shape[0], _p(v), v.stride(0), _p(out),
                                   out.stride(0), B, H, Tq, Tk, _p(kv_len), 1 if causal else 0, q_col0, k_col0, v_col0, _p(bd),
                                   bd.shape[-1] if bd is not None else 0, _p(resid), resid.stride(0) if resid is not None else 0,
                                   _p(lse), d_k, _stream()), 'otb_attention')
    _count()
    return out, lse


def attention(q, k, v, B, H, Tq, Tk, kv_len=None, causal=False, q_col0=0, k_col0=0, v_col0=0, out=None, bd=None,
              resid=None, d_k=64):
    """q/k/v: bf16 2-D matrices (may be the same [M,3d] buffer with different column offsets); head h of each starts
    at column col0 + d_k*h.  Returns bf16 [B*Tq, H*d_k]."""
    return _attention(q, k, v, B, H, Tq, Tk, kv_len, causal, q_col0, k_col0, v_col0, out, bd, resid, d_k)[0]


def attention_probs(q, k, B, H, Tq, Tk, kv_len=None, causal=False, q_col0=0, k_col0=0, bd=None, d_k=64, out=None):
    """The attention weights of attention() over the same q / k operands, column offsets, mask and band
    (otb_attention_probs) -> f32 [B, H, Tq, Tk]: masked entries 0, batch entries with kv_len 0 all NaN."""
    for t, n in ((q, 'q'), (k, 'k')):
        _need(t, BF16, n)
    check_head_dim(d_k)
    if kv_len is not None:
        _need(kv_len, torch.int32, 'kv_len')
    if bd is not None:
        _need(bd, torch.float32, 'bd')
        if Tq != Tk or causal:
            raise ValueError('attention_probs: the rel-pos band is for non-causal self-attention (Tq == Tk)')
    if out is None:
        out = torch.empty(B, H, Tq, Tk, dtype=torch.float32, device=q.device)
    else:
        _need(out, torch.float32, 'out')
        if tuple(out.shape) != (B, H, Tq, Tk):
            raise ValueError(f'attention_probs: out must be [{B}, {H}, {Tq}, {Tk}], got {tuple(out.shape)}')
    check(_lib.lib().otb_attention_probs(_p(q), q.stride(0), q.shape[0], _p(k), k.stride(0), k.shape[0], _p(out), B, H, Tq, Tk,
                                         _p(kv_len), 1 if causal else 0, q_col0, k_col0, _p(bd),
                                         bd.shape[-1] if bd is not None else 0, d_k, _stream()), 'otb_attention_probs')
    _count()
    return out


def dwconv_swish(x, w, b, B, T, out=None):
    """depthwise conv over time + folded BatchNorm + swish; x bf16 [B*T, d], w f32 [k, d], b f32 [d]."""
    _need(x, BF16, 'x'); _need(w, torch.float32, 'w'); _need(b, torch.float32, 'b')
    d = x.shape[1]
    if out is None:
        out = torch.empty_like(x)
    check(_lib.lib().otb_dwconv_swish(_p(x), _p(w), _p(b), _p(out), B, T, d, w.shape[0], _stream()),
          'otb_dwconv_swish')
    _count()
    return out


def layernorm(x, g1, b1, g2=None, b2=None, eps=1e-5, out=None, out_f32=False):
    _need(x, BF16, 'x')
    M, N = x.shape
    if out is None:
        out = torch.empty(M, N, dtype=torch.float32 if out_f32 else BF16, device=x.device)
    check(_lib.lib().otb_layernorm(_p(x), x.stride(0), _p(out), out.stride(0), 1 if out.dtype == torch.float32 else 0,
                                   _p(g1), _p(b1), _p(g2), _p(b2), eps, M, N, _stream()), 'otb_layernorm')
    _count()
    return out


def scale_add_table(x, alpha=1.0, table=None, period=1, out=None, scale_dev=None):
    """bf16 out = x * alpha + table[row % period]; x f32 or bf16 2-D.  scale_dev: an f32 device scalar alpha is multiplied
    by on the device (a loss-gradient scale that never goes to the host)."""
    M, N = x.shape
    if out is None:
        out = torch.empty(M, N, dtype=BF16, device=x.device)
    if scale_dev is not None:
        _need(scale_dev, torch.float32, 'scale_dev')
    check(_lib.lib().otb_scale_add_table(_p(x), x.stride(0), 1 if x.dtype == torch.float32 else 0, _p(out),
                                         out.stride(0), alpha, _p(table), period, M, N, _p(scale_dev), _stream()),
          'otb_scale_add_table')
    _count()
    return out


_TABLES = {}


def sinusoid_table(n_pos, d, first_pos=0, device=None):
    """Cached f32 [n_pos, d] sinusoid table (module/pos.py:30-42), computed once on the device."""
    device = torch.device(device if device is not None else torch.cuda.current_device())
    key = (n_pos, d, first_pos, device.index if device.index is not None else torch.cuda.current_device())
    t = _TABLES.get(key)
    if t is None:
        t = torch.empty(n_pos, d, dtype=torch.float32, device=device)
        check(_lib.lib().otb_sinusoid_table(_p(t), n_pos, d, first_pos, _stream()), 'otb_sinusoid_table')
        _count()
        _TABLES[key] = t
    return t


def embed_posenc(tok, emb, table, N, d, period=1, tok_stride=1, step_ptr=None, out=None, row_pos=None):
    """row_pos i32 [N]: a position per row (-1 reads position 0), instead of step_ptr's or period's."""
    _need(emb, BF16, 'emb')
    if row_pos is not None:
        _need(row_pos, torch.int32, 'row_pos')
    if out is None:
        out = torch.empty(N, d, dtype=BF16, device=emb.device)
    check(_lib.lib().otb_embed_posenc(_p(tok), tok_stride, _p(emb), _p(table), _p(out), N, d, period, _p(step_ptr),
                                      _p(row_pos), emb.shape[0], _stream()), 'otb_embed_posenc')
    _count()
    return out


def log_softmax(x, V, out=None):
    _need(x, torch.float32, 'x')
    rows = x.shape[0]
    if out is None:
        out = torch.empty(rows, V, dtype=torch.float32, device=x.device)
    check(_lib.lib().otb_log_softmax(_p(x), x.stride(0), _p(out), out.stride(0), rows, V, _stream()),
          'otb_log_softmax')
    _count()
    return out


def logsoftmax_topk(logits, V, k, lm_logp=None, lm_weight=0.0, out_val=None, out_idx=None, out_logp=None, lm_beta=0.0,
                    lm_exempt=-1):
    """Fused log-softmax (+ LM shallow fusion) + per-row top-k.  logits f32 [rows, ld].  lm_exempt >= 0 (the transducer's
    fusion): that column (blank) gets no LM term, every other one gets + (lm_weight * lm_logp + lm_beta), and out_logp keeps
    the plain log-probs; the defaults are the attention decoder's fusion."""
    _need(logits, torch.float32, 'logits')
    rows = logits.shape[0]
    if out_val is None:
        out_val = torch.empty(rows, k, dtype=torch.float32, device=logits.device)
    if out_idx is None:
        out_idx = torch.empty(rows, k, dtype=torch.int32, device=logits.device)
    check(_lib.lib().otb_logsoftmax_topk(_p(logits), logits.stride(0), V, _p(lm_logp),
                                         lm_logp.stride(0) if lm_logp is not None else 0, lm_weight, lm_beta, lm_exempt, k, rows,
                                         _p(out_val), _p(out_idx), _p(out_logp),
                                         out_logp.stride(0) if out_logp is not None else 0, _stream()),
          'otb_logsoftmax_topk')
    _count()
    return out_val, out_idx


def _ls_ce(logits, targets, V, smoothing, pad_id, grad_dtype):
    """otb_ls_ce -> (loss f32 scalar tensor, dlogits or None): no gradient for grad_dtype None, f32 [rows, V] for float32,
    bf16 [rows, ld] with ld = logits.stride(0) and zero pad columns for bfloat16."""
    _need(logits, torch.float32, 'logits')
    rows = logits.shape[0]
    targets = targets.contiguous().view(-1)
    dev = logits.device
    tok = torch.empty(rows, dtype=torch.float32, device=dev)
    loss = torch.empty(1, dtype=torch.float32, device=dev)
    nv = torch.empty(1, dtype=torch.int32, device=dev)
    ldd = {None: 0, torch.float32: V, BF16: logits.stride(0)}[grad_dtype]
    dl = torch.empty(rows, ldd, dtype=grad_dtype, device=dev) if grad_dtype is not None else None
    check(_lib.lib().otb_ls_ce(_p(logits), logits.stride(0), _p(targets), rows, V, smoothing, pad_id, _p(tok), _p(loss),
                               _p(nv), _p(dl), ldd, 1 if grad_dtype == BF16 else 0, _stream()), 'otb_ls_ce')
    _count(3)
    return loss[0], dl


def ls_cross_entropy(logits, targets, V, smoothing=0.1, pad_id=0, want_grad=False):
    """Label-smoothed CE (module/loss.py:21-48).  logits f32 [rows, ld]; targets i64 [rows].
    Returns (loss f32 scalar tensor, dlogits f32 [rows, V] or None)."""
    return _ls_ce(logits, targets, V, smoothing, pad_id, torch.float32 if want_grad else None)


DECODE_MAX_LEN = 1023   # cached positions of otb_decode_self_attn: the longest KV-cached beam search (max_len)


def decode_self_attn(qkv, kc, vc, anc, step_ptr, N, H, Lmax, out=None, row_pos=None):
    """kc/vc bf16 [Lmax, N, d]: the head width d_k = d // H is taken from the cache.
    row_pos i32 [N]: a query position per row (-1: zeros) in place of step_ptr, which is then ignored; kc/vc bf16
    [cache rows, d] and anc i32 [N, Lmax] the cache row of each position of each row, the newest included."""
    d = kc.shape[-1]
    if d % H:
        raise ValueError(f'decode_self_attn: cache width {d} is not a multiple of H = {H}')
    d_k = d // H
    check_head_dim(d_k)
    if out is None:
        out = torch.empty(N, d, dtype=BF16, device=qkv.device)
    if row_pos is not None:
        _need(row_pos, torch.int32, 'row_pos'); _need(anc, torch.int32, 'anc')
        if anc.shape != (N, Lmax):
            raise ValueError(f'decode_self_attn: with row_pos, anc must be [N = {N}, Lmax = {Lmax}], got {tuple(anc.shape)}')
        step_ptr = None
    check(_lib.lib().otb_decode_self_attn(_p(qkv), _p(kc), _p(vc), _p(anc), _p(step_ptr), _p(row_pos), _p(out), N, H, Lmax, d_k,
                                          _stream()), 'otb_decode_self_attn')
    _count()
    return out


class BeamState:
    """Device-resident beam-search state (otb_beam_state)."""

    def __init__(self, batch, beam, max_len, device):
        self.B, self.beam, self.Lmax = batch, beam, max_len
        self.N = N = batch * beam
        kw = dict(device=device)
        self.tok_hist = torch.zeros(max_len, N, dtype=torch.int32, **kw)
        self.par_hist = torch.zeros(max_len, N, dtype=torch.int32, **kw)
        self.last_tok = torch.ones(N, dtype=torch.int64, **kw)
        self.scores = torch.zeros(N, dtype=torch.float32, **kw)
        self.flag = torch.zeros(N, dtype=torch.uint8, **kw)
        self.anc = torch.zeros(2, N, max_len, dtype=torch.int32, **kw)
        self.ctrl = torch.zeros(4, dtype=torch.int32, **kw)
        self.c = _lib.BeamStateC(self.tok_hist.data_ptr(), self.par_hist.data_ptr(), self.last_tok.data_ptr(),
                                 self.scores.data_ptr(), self.flag.data_ptr(), self.anc.data_ptr(),
                                 self.ctrl.data_ptr(), N, beam, max_len)

    @property
    def step_ptr(self):
        return self.ctrl  # ctrl[0] is the step counter

    def init(self):
        check(_lib.lib().otb_beam_init(ctypes.byref(self.c), _stream()), 'otb_beam_init')
        _count()

    def step(self, logp, V, lm_logp=None, lm_weight=0.0, dbg_ktok=None, dbg_offs=None):
        _need(logp, torch.float32, 'logp')
        check(_lib.lib().otb_beam_step(_p(logp), logp.stride(0), V, _p(lm_logp),
                                       lm_logp.stride(0) if lm_logp is not None else 0, lm_weight, None, None,
                                       ctypes.byref(self.c), _p(dbg_ktok), _p(dbg_offs), _stream()), 'otb_beam_step')
        _count()

    def step_topk(self, topk_val, topk_idx, dbg_ktok=None, dbg_offs=None):
        """The beam step on a per-hypothesis top-k (logsoftmax_topk with k = beam) instead of log-prob rows."""
        check(_lib.lib().otb_beam_step(None, 0, 0, None, 0, 0.0, _p(topk_val), _p(topk_idx), ctypes.byref(self.c),
                                       _p(dbg_ktok), _p(dbg_offs), _stream()), 'otb_beam_step')
        _count()

    def reconstruct(self, steps):
        preds = torch.empty(self.N, steps + 1, dtype=torch.int64, device=self.scores.device)
        check(_lib.lib().otb_beam_reconstruct(ctypes.byref(self.c), _p(preds), steps + 1, steps, _stream()),
              'otb_beam_reconstruct')
        _count()
        return preds

    def finalize(self, penalty, lamda, nbest):
        k = min(nbest, self.beam)
        out_preds = torch.empty(self.B, k, self.Lmax, dtype=torch.int64, device=self.scores.device)
        out_scores = torch.empty(self.B, k, dtype=torch.float32, device=self.scores.device)
        check(_lib.lib().otb_beam_finalize(ctypes.byref(self.c), float(penalty), float(lamda), k, _p(out_preds),
                                           _p(out_scores), _stream()), 'otb_beam_finalize')
        _count()
        return out_preds, out_scores


SAMPLE_MAX_VOCAB = 48 * 1024


def sample_step(logits, V, state, seed):
    """One step of ancestral sampling on a BeamState (otb_sample_step, DESIGN.md 4.11): every live row draws its next token
    from softmax(logits[n, :V]) by the Gumbel-max trick on the counter hash of (seed, step, row, token), adds the token's
    log-prob to its score and ends on <S/E>; rows are never reordered.  logits f32 [N, ld]; seed i32 device tensor [1],
    read at run time (a captured step draws fresh samples when the seed or the step counter changes)."""
    _mat(logits, 'logits', torch.float32)
    _need(seed, torch.int32, 'seed')
    if logits.shape[0] != state.N or not 1 <= V <= min(SAMPLE_MAX_VOCAB, logits.shape[1]):
        raise ValueError(f'sample_step: need logits [N = {state.N}, >= V] and 1 <= V <= {SAMPLE_MAX_VOCAB}, got '
                         f'{tuple(logits.shape)} and V = {V}')
    check(_lib.lib().otb_sample_step(_p(logits), logits.stride(0), V, ctypes.byref(state.c), _p(seed), _stream()),
          'otb_sample_step')
    _count()


def decode_persistent_workspace(N, n_layers, Lmax, B, beam, vocab, device):
    n = int(_lib.lib().otb_decode_persistent_workspace(N, n_layers, Lmax, B, beam, vocab))
    if n < 0:
        raise ValueError('otb_decode_persistent_workspace: bad geometry')
    return torch.zeros(n, dtype=torch.uint8, device=device)


def decode_persistent(model_c, kvx, mem_len, kc, vc, state, B, T, max_steps, workspace, dbg_logp=None, dbg_scores=None):
    """The whole beam-search decode loop in one persistent kernel (otb_decode_persistent, csrc/decode_group.cu)."""
    _need(kvx, BF16, 'kvx'); _need(kc, BF16, 'kc'); _need(vc, BF16, 'vc'); _need(mem_len, torch.int32, 'mem_len')
    check(_lib.lib().otb_decode_persistent(ctypes.byref(model_c), _p(kvx), _p(mem_len), _p(kc), _p(vc), ctypes.byref(state.c),
                                           B, T, max_steps, _p(workspace), workspace.numel(), _p(dbg_logp), _p(dbg_scores),
                                           _stream()), 'otb_decode_persistent')
    _count()


# ------------------------------------------------------------------------------------------------
# training step: backward kernels (include/otb200.h "Training step")
# ------------------------------------------------------------------------------------------------
def attention_train(q, k, v, B, H, Tq, Tk, kv_len=None, causal=False, q_col0=0, k_col0=0, v_col0=0, bd=None, out=None,
                    lse=None):
    """attention (d_k 64, the width of the backward) + the per-row log-sum-exp the backward needs
    -> (out bf16 [B*Tq, H*64], lse f32 [B,H,Tq]), written into out / lse when given.  bd: the rel-pos band, as for
    attention()."""
    return _attention(q, k, v, B, H, Tq, Tk, kv_len, causal, q_col0, k_col0, v_col0, out=out, bd=bd, with_lse=True, lse=lse)


def rel_band_ld(T):
    """Row pitch of the bf16 band gradient dBD: 2T - 1 columns rounded up to 8 (a TMA operand of the band GEMMs)."""
    return (2 * T - 1 + 7) // 8 * 8


def attention_bwd(q, k, v, out, dout, lse, B, H, Tq, Tk, dq, dk, dv, kv_len=None, causal=False, q_col0=0, k_col0=0,
                  v_col0=0, dq_col0=0, dk_col0=0, dv_col0=0, bd=None, dbd=None, dsum=None):
    """Gradients of otb_attention written into dq/dk/dv (bf16 matrices, column offsets d*_col0).  With the rel-pos band bd
    f32 [H, B*Tq, ld] of the forward, its gradient is written into dbd bf16 [H, B*Tq, rel_band_ld(Tq)], which the caller
    zeroes.  Returns D = rowsum(dout * out) f32 [B,H,Tq], written into dsum when given."""
    for t, n in ((q, 'q'), (k, 'k'), (v, 'v'), (out, 'out'), (dout, 'dout'), (dq, 'dq'), (dk, 'dk'), (dv, 'dv')):
        _mat(t, n)
    d = H * 64    # the backward is 64-wide
    for t, c0, n in ((q, q_col0, 'q'), (k, k_col0, 'k'), (v, v_col0, 'v'), (dq, dq_col0, 'dq'), (dk, dk_col0, 'dk'),
                     (dv, dv_col0, 'dv')):
        _head_cols('attention_bwd', t, c0, d, n)
    for t, n in ((out, 'out'), (dout, 'dout')):
        _rows_cols('attention_bwd', t, B * Tq, d, n)
    for t, rows, n in ((dq, B * Tq, 'dq'), (dk, B * Tk, 'dk'), (dv, B * Tk, 'dv')):
        _rows_cols('attention_bwd', t, rows, 0, n)
    _need(lse, torch.float32, 'lse')
    if tuple(lse.shape) != (B, H, Tq):
        raise ValueError(f'attention_bwd: lse must be [{B}, {H}, {Tq}], got {tuple(lse.shape)}')
    if dsum is not None:
        _need(dsum, torch.float32, 'dsum')
        if tuple(dsum.shape) != (B, H, Tq):
            raise ValueError(f'attention_bwd: dsum must be [{B}, {H}, {Tq}], got {tuple(dsum.shape)}')
    _kv_len('attention_bwd', kv_len, B)
    ldbd = lddbd = 0
    if (bd is None) != (dbd is None):
        raise ValueError('attention_bwd: bd and dbd must both be given or both be None')
    if bd is not None:
        _band('attention_bwd', bd, B, H, Tq, Tk, causal, torch.float32, 'bd')
        _band('attention_bwd', dbd, B, H, Tq, Tk, causal, BF16, 'dbd')
        ldbd, lddbd = bd.shape[-1], dbd.shape[-1]
    if dsum is None:
        dsum = torch.empty(B, H, Tq, dtype=torch.float32, device=q.device)
    check(_lib.lib().otb_attention_bwd(_p(q), q.stride(0), q.shape[0], _p(k), k.stride(0), k.shape[0], _p(v), v.stride(0), _p(out),
                                       out.stride(0), _p(dout), dout.stride(0), _p(lse), _p(dsum), _p(dq), dq.stride(0), dq_col0,
                                       _p(dk), dk.stride(0), dk_col0, _p(dv), dv.stride(0), dv_col0, B, H, Tq, Tk, _p(kv_len),
                                       1 if causal else 0, q_col0, k_col0, v_col0, _p(bd), ldbd, _p(dbd), lddbd, _stream()),
          'otb_attention_bwd')
    _count(2)
    return dsum


def conformer_conv_train(x, lengths, w, wb, gamma, beta, running_mean, running_var, num_batches, B, T, momentum=0.1, eps=1e-5):
    """Training-mode middle of the Conformer convolution module (otb_conformer_conv_train): x bf16 [B*T, d] GLU output,
    w f32 [d, k] depthwise weight, wb f32 [d] or None; BatchNorm over batch statistics, running buffers updated in place.
    -> (out bf16 [B*T, d] = swish(BN(conv(x))) zero on padded frames, c f32 [B*T, d] conv output, stats f32 [2, d])."""
    _need(x, BF16, 'x'); _need(lengths, torch.int32, 'lengths'); _need(w, torch.float32, 'w')
    _need(gamma, torch.float32, 'gamma'); _need(beta, torch.float32, 'beta')
    M, d = x.shape
    c = torch.empty(M, d, dtype=torch.float32, device=x.device)
    stats = torch.empty(2, d, dtype=torch.float32, device=x.device)
    out = torch.empty_like(x)
    check(_lib.lib().otb_conformer_conv_train(_p(x), _p(lengths), _p(w), _p(wb), _p(gamma), _p(beta), _p(running_mean), _p(running_var),
                                              _p(num_batches), float(momentum), float(eps), _p(c), _p(stats), _p(out), B, T, d,
                                              w.shape[-1], _stream()), 'otb_conformer_conv_train')
    _count(4)
    return out, c, stats


def conformer_conv_bwd(dy, x, lengths, w, gamma, beta, c, stats, B, T, dw=None, dwb=None, dgamma=None, dbeta=None, accumulate=False,
                       has_bias=True):
    """Backward of conformer_conv_train -> (dx bf16 [B*T, d], dw f32 [d, k], dwb f32 [d] or None, dgamma, dbeta); with accumulate
    the given gradient tensors are added to."""
    _need(dy, BF16, 'dy'); _need(x, BF16, 'x')
    M, d = x.shape
    dev = x.device
    f32 = dict(dtype=torch.float32, device=dev)
    dw = dw if dw is not None else torch.empty(d, w.shape[-1], **f32)
    dwb = (dwb if dwb is not None else torch.empty(d, **f32)) if has_bias else None
    dgamma = dgamma if dgamma is not None else torch.empty(d, **f32)
    dbeta = dbeta if dbeta is not None else torch.empty(d, **f32)
    red = torch.empty(2, d, **f32)
    dc = torch.empty(M, d, **f32)
    dx = torch.empty_like(x)
    check(_lib.lib().otb_conformer_conv_bwd(_p(dy), _p(x), _p(lengths), _p(w), _p(gamma), _p(beta), _p(c), _p(stats), _p(red), _p(dc),
                                            _p(dx), _p(dw), _p(dwb), _p(dgamma), _p(dbeta), 1 if accumulate else 0, B, T, d, w.shape[-1],
                                            _stream()), 'otb_conformer_conv_bwd')
    _count(4)
    return dx, dw, dwb, dgamma, dbeta


def linear_wgrad(dy, x, out=None, accumulate=False):
    """dW f32 [N,K] (+)= dy[M,N]^T x[M,K]  (bf16 2-D, unit column stride)."""
    _mat(dy, 'dy'); _mat(x, 'x')
    M, N = dy.shape
    K = x.shape[1]
    if x.shape[0] != M:
        raise ValueError('linear_wgrad: row mismatch')
    if out is None:
        out = torch.empty(N, K, dtype=torch.float32, device=dy.device)
    with _Timed('wgrad', 2.0 * M * N * K, (M, N, K)):
        check(_lib.lib().otb_linear_wgrad(_p(dy), dy.stride(0), _p(x), x.stride(0), _p(out), out.stride(0), M, N, K,
                                          1 if accumulate else 0, _stream()), 'otb_linear_wgrad')
    _count(2)
    return out


def colsum(x, out=None, accumulate=False):
    M, N = x.shape
    if out is None:
        out = torch.empty(N, dtype=torch.float32, device=x.device)
    check(_lib.lib().otb_colsum(_p(x), x.stride(0), _p(out), M, N, 1 if accumulate else 0, _stream()), 'otb_colsum')
    _count()
    return out


def layernorm_bwd(dy, z, gamma, eps=1e-5, dgamma=None, dbeta=None, accumulate=False):
    """-> (dz bf16 [M,N], dgamma f32 [N], dbeta f32 [N]); with accumulate the given dgamma / dbeta are added to."""
    _need(dy, BF16, 'dy'); _need(z, BF16, 'z')
    M, N = z.shape
    dz = torch.empty(M, N, dtype=BF16, device=z.device)
    dg = dgamma if dgamma is not None else torch.empty(N, dtype=torch.float32, device=z.device)
    db = dbeta if dbeta is not None else torch.empty(N, dtype=torch.float32, device=z.device)
    check(_lib.lib().otb_layernorm_bwd(_p(dy), dy.stride(0), _p(z), z.stride(0), _p(gamma), _p(dz), dz.stride(0), _p(dg),
                                       _p(db), eps, M, N, 1 if accumulate else 0, _stream()), 'otb_layernorm_bwd')
    _count()
    return dz, dg, db


def glu_fwd(u):
    _need(u, BF16, 'u')
    M, F2 = u.shape
    h = torch.empty(M, F2 // 2, dtype=BF16, device=u.device)
    check(_lib.lib().otb_glu_fwd(_p(u), _p(h), M, F2 // 2, _stream()), 'otb_glu_fwd')
    _count()
    return h


def glu_bwd(dh, u):
    _need(u, BF16, 'u'); _need(dh, BF16, 'dh')
    M, F2 = u.shape
    du = torch.empty(M, F2, dtype=BF16, device=u.device)
    check(_lib.lib().otb_glu_bwd(_p(dh), _p(u), _p(du), M, F2 // 2, _stream()), 'otb_glu_bwd')
    _count()
    return du


def act_fwd(u, act):
    """h = act(u) for act in 'gelu' (erf form), 'tanh', 'swish' (otb_act_fwd): the training feed-forward's activation,
    un-fused from the w_1 GEMM so that u stays for the backward.  u bf16 [M, N] contiguous -> h bf16 [M, N]."""
    _need(u, BF16, 'u')
    M, N = u.shape
    h = torch.empty_like(u)
    check(_lib.lib().otb_act_fwd(_p(u), _p(h), M, N, TRAIN_ACT[act], _stream()), 'otb_act_fwd')
    _count()
    return h


def act_bwd(dh, u, act):
    """du = dh * act'(u) (otb_act_bwd), the backward of act_fwd."""
    _need(u, BF16, 'u'); _need(dh, BF16, 'dh')
    if dh.shape != u.shape:
        raise ValueError(f'act_bwd: dh {tuple(dh.shape)} and u {tuple(u.shape)} differ')
    M, N = u.shape
    du = torch.empty_like(u)
    check(_lib.lib().otb_act_bwd(_p(dh), _p(u), _p(du), M, N, TRAIN_ACT[act], _stream()), 'otb_act_bwd')
    _count()
    return du


def relu_bwd(dy, y, out=None):
    _need(dy, BF16, 'dy'); _need(y, BF16, 'y')
    if out is None:
        out = torch.empty_like(dy)
    check(_lib.lib().otb_relu_bwd(_p(dy), _p(y), _p(out), dy.numel(), _stream()), 'otb_relu_bwd')
    _count()
    return out


def embed_bwd(tok, dx, dE, scale):
    """dE[tok[n]] += scale * dx[n]   (dE f32 [V,d], accumulated in place)."""
    _need(dx, BF16, 'dx'); _need(dE, torch.float32, 'dE')
    tok = tok.contiguous().view(-1)
    check(_lib.lib().otb_embed_bwd(_p(tok), _p(dx), _p(dE), tok.numel(), dx.shape[1], dE.shape[0], scale, _stream()),
          'otb_embed_bwd')
    _count()


def ls_cross_entropy_train(logits, targets, V, smoothing=0.1, pad_id=0):
    """-> (loss f32 scalar tensor, dlogits bf16 [rows, ld] with ld = logits.stride(0); pad columns zero)."""
    return _ls_ce(logits, targets, V, smoothing, pad_id, BF16)


def sumsq(g, out, zero_first=True):
    check(_lib.lib().otb_sumsq(_p(g), g.numel(), _p(out), 1 if zero_first else 0, _stream()), 'otb_sumsq')
    _count()


def adam_step_sched(p, g, m, v, sumsq_buf, max_norm, base_lr, model_size, warmup_steps, factor, betas, eps, weight_decay,
                    counters, hyper, noise_std=0.0, noise_seed=None, noise_mask=None):
    """clip + Adam with the step counters / Noam schedule evaluated on the device (otb_adam_step_sched).  noise_std > 0:
    gradient noise noise_std * N(0, 1) after the clip on the elements whose bit is set in noise_mask (u8 [(n + 7) // 8],
    noise_bitmask), drawn from the i32 device scalar noise_seed and the step count."""
    for t, n in ((p, 'p'), (g, 'g'), (m, 'm'), (v, 'v'), (hyper, 'hyper')):
        _need(t, torch.float32, n)
    _need(counters, torch.int32, 'counters')
    if noise_std < 0:
        raise ValueError('adam_step_sched: noise_std must be >= 0')
    if noise_std > 0:
        _need(noise_seed, torch.int32, 'noise_seed'); _need(noise_mask, torch.uint8, 'noise_mask')
        if noise_mask.numel() < (p.numel() + 7) // 8:
            raise ValueError('adam_step_sched: noise_mask needs (n + 7) // 8 bytes')
    check(_lib.lib().otb_adam_step_sched(_p(p), _p(g), _p(m), _p(v), p.numel(), _p(sumsq_buf), max_norm, base_lr,
                                         float(model_size), float(warmup_steps or 0), factor, betas[0], betas[1], eps,
                                         weight_decay, _p(counters), _p(hyper), float(noise_std),
                                         _p(noise_seed) if noise_std > 0 else None, _p(noise_mask) if noise_std > 0 else None,
                                         _stream()), 'otb_adam_step_sched')
    _count(2)


def noise_bitmask(n, spans):
    """The noise_mask of adam_step_sched: u8 [(n + 7) // 8] with bit i & 7 of byte i >> 3 set for every i in one of the
    [offset, offset + count) spans (the parameters of a flat buffer), little bit order.  Built on the host."""
    bits = torch.zeros((n + 7) // 8 * 8, dtype=torch.bool)
    for o, k in spans:
        bits[o:o + k] = True
    weights = torch.tensor([1 << j for j in range(8)], dtype=torch.int32)
    return (bits.view(-1, 8).to(torch.int32) * weights).sum(1).to(torch.uint8)


def mixspeech(x, mask, seed, step, scale, lam_out):
    """MixSpeech's input (otb_mixspeech): x f32 [B, T, F], mask bool [B, T], B >= 2 -> (x_mix f32 [B // 2, T, F], mask_mix
    bool [B // 2, T]); lambda is drawn on the device from the i32 device scalars seed / step, and lam_out f32 [3] receives
    {lambda, lambda * scale, (1 - lambda) * scale}."""
    _need(x, torch.float32, 'x'); _need(mask, torch.bool, 'mask'); _need(lam_out, torch.float32, 'lam_out')
    _need(seed, torch.int32, 'seed'); _need(step, torch.int32, 'step')
    if x.dim() != 3 or mask.shape != x.shape[:2]:
        raise ValueError(f'mixspeech: x [B, T, F] and mask [B, T], got {tuple(x.shape)} and {tuple(mask.shape)}')
    B, T, F = x.shape
    if B < 2:
        raise ValueError('MixSpeech mixes pairs of utterances: it needs a batch of at least 2')
    x_out = torch.empty(B // 2, T, F, dtype=torch.float32, device=x.device)
    m_out = torch.empty(B // 2, T, dtype=torch.bool, device=x.device)
    check(_lib.lib().otb_mixspeech(_p(x), _p(mask), B, T, F, _p(seed), _p(step), float(scale), _p(lam_out), _p(x_out), _p(m_out),
                                   _stream()), 'otb_mixspeech')
    _count()
    return x_out, m_out


def frame_stack(x, n, s, T2, alpha=1.0, table=None, out=None):
    """Low-frame-rate stacking of the concat front ends (otb_frame_stack): x f32 [B, T, F] -> bf16 [B*T2, W], W = n*F
    rounded up to 8; row b*T2 + i = x[b, i*s : i*s + n] flattened frame-major, frames at or past T zero, columns n*F .. W - 1
    zero.  table f32 [T2, n*F] (optional): y * alpha + table[i] on the n*F columns.  out: a bf16 [B*T2, >= W] matrix with
    unit column stride; its columns past W are left as they are."""
    _need(x, torch.float32, 'x')
    if x.dim() != 3:
        raise ValueError(f'frame_stack: x must be [B, T, F], got {tuple(x.shape)}')
    B, T, F = x.shape
    W = (n * F + 7) // 8 * 8
    if table is not None:
        _need(table, torch.float32, 'table')
        if tuple(table.shape) != (T2, n * F):
            raise ValueError(f'frame_stack: table must be [{T2}, {n * F}], got {tuple(table.shape)}')
    if out is None:
        out = torch.empty(B * T2, W, dtype=BF16, device=x.device)
    else:
        _mat(out, 'out')
        if out.shape[0] != B * T2 or out.shape[1] < W:
            raise ValueError(f'frame_stack: out must be [{B * T2}, >= {W}], got {tuple(out.shape)}')
    check(_lib.lib().otb_frame_stack(_p(x), B, T, F, n, s, T2, _p(out), out.stride(0), float(alpha), _p(table), _stream()),
          'otb_frame_stack')
    _count()
    return out


CTC_LOSS_MAX_LABELS = 1023   # padded target width of otb_ctc_loss


INT32_MAX = 2 ** 31 - 1


def resample_rates(freq, B, name):
    """A rate argument of resample(): an int or B of them (a sequence or a tensor, read on the host) -> list of B ints,
    each a positive integer.  Raises ValueError otherwise."""
    if isinstance(freq, torch.Tensor):
        if freq.dim() == 0:
            freq = freq.item()
        else:
            if freq.is_floating_point() or freq.is_complex() or freq.dtype == torch.bool:
                raise ValueError(f'{name} must hold integer rates, got a {freq.dtype} tensor')
            freq = freq.tolist()
    if isinstance(freq, (list, tuple)):
        if len(freq) != B:
            raise ValueError(f'{name} must be one rate or {B} of them, got {len(freq)}')
        rates = list(freq)
    else:
        rates = [freq] * B
    out = []
    for r in rates:
        if isinstance(r, float) and r.is_integer():
            r = int(r)
        try:
            if isinstance(r, bool):
                raise TypeError
            r = operator.index(r)
        except TypeError:
            raise ValueError(f'{name}: sample rates must be integers, got {r!r}') from None
        if not 0 < r <= INT32_MAX:
            raise ValueError(f'{name}: sample rates must be positive int32 integers, got {r}')
        out.append(r)
    return out


def resample_width(N, orig, new):
    """Columns resample() writes for a [B, N] input: the longest row's ceil(new N / orig), from host rates."""
    return max(1, max(-(-n * N // o) for o, n in zip(orig, new)))


def resample(x, lengths, orig_freq, new_freq, width=None):
    """Band-limited resampling, one rate pair per row (otb_resample): x f32 [B, N] (row b's first lengths[b] samples; the
    padding is never read), lengths i32 [B] on the device -> (out f32 [B, width], out_lengths i32 [B] on the device), row b of
    out equal to torchaudio.functional.resample(x[b, :lengths[b]], orig[b], new[b]) at its defaults (sinc_interp_hann,
    lowpass_filter_width 6, rolloff 0.99) and zero past out_lengths[b] = ceil(new N_b / orig).  Rows with orig == new are
    copied bit for bit.

    orig_freq / new_freq: an int, or one per row as a sequence or an integer tensor; they are checked on the host and
    width = max over rows of ceil(new N / orig) is computed there, so nothing waits for the device.  Rates already held as
    CUDA int32 [B] tensors are passed on as they are when ``width`` (at least every row's output length) is given, which
    is how FbankExtractor passes speeds drawn on the device; a row with a rate <= 0 then comes out empty."""
    on_device = width is not None and all(isinstance(f, torch.Tensor) and f.is_cuda for f in (orig_freq, new_freq))
    if x.dim() != 2:
        raise ValueError(f'resample: x must be [B, N], got {tuple(x.shape)}')
    B, N = x.shape
    if not on_device:
        orig = resample_rates(orig_freq, B, 'orig_freq')
        new = resample_rates(new_freq, B, 'new_freq')
        need = resample_width(N, orig, new)
        width = need if width is None else int(width)
        if width < need:
            raise ValueError(f'resample: width {width} is shorter than the longest output, {need}')
    if not 1 <= width <= INT32_MAX:
        raise ValueError(f'resample: {width} output samples per row is past int32')
    _need(x, torch.float32, 'x')
    _need(lengths, torch.int32, 'lengths')
    if on_device:
        rates = torch.stack([_need(orig_freq, torch.int32, 'orig_freq'), _need(new_freq, torch.int32, 'new_freq')])
    else:
        rates = torch.tensor([orig, new], dtype=torch.int32).to(x.device)
    if rates.shape != (2, B) or lengths.shape != (B,):
        raise ValueError(f'resample: rates and lengths must be [B] = [{B}]')
    out = torch.empty(B, width, dtype=torch.float32, device=x.device)
    out_len = torch.empty(B, dtype=torch.int32, device=x.device)
    check(_lib.lib().otb_resample(_p(x), x.stride(0), _p(lengths), _p(rates[0]), _p(rates[1]), _p(out), width, _p(out_len), B,
                                  width, _stream()), 'otb_resample')
    _count()
    return out, out_len


def ctc_loss(logits, B, T, V, in_len, targets, tgt_len, blank=0, want_grad=False, grad_scale=1.0, scale_dev=None):
    """nn.CTCLoss(blank, 'mean', zero_infinity=True) on logits f32 [B*T, ld] (model/ctc.py:48-52).
    -> (loss 0-d, nll f32 [B], dlogits bf16 [B*T, ld] or None).  The gradient is scaled by grad_scale, times the f32 device
    scalar scale_dev when one is given (read on the device).  targets [B, L] takes L <= 1023 (padded width); the scratch
    is f32 [B, T, 2 L + 1] (262 MB at B 32, T 1000, L 1023)."""
    if targets.shape[1] > CTC_LOSS_MAX_LABELS:
        raise ValueError(f'ctc_loss: targets are {targets.shape[1]} labels wide; at most {CTC_LOSS_MAX_LABELS} are supported')
    _need(logits, torch.float32, 'logits'); _need(in_len, torch.int32, 'in_len'); _need(tgt_len, torch.int32, 'tgt_len')
    if scale_dev is not None:
        _need(scale_dev, torch.float32, 'scale_dev')
    targets = targets.contiguous()
    dev = logits.device
    ld = logits.stride(0)
    logp = torch.empty(B * T, ld, dtype=torch.float32, device=dev)
    check(_lib.lib().otb_log_softmax(_p(logits), ld, _p(logp), ld, B * T, V, _stream()), 'otb_log_softmax')
    max_tgt = targets.shape[1]
    nll = torch.empty(B, dtype=torch.float32, device=dev)
    loss = torch.empty(1, dtype=torch.float32, device=dev)
    ws = torch.empty(B, T, 2 * max_tgt + 1, dtype=torch.float32, device=dev)
    dl = torch.empty(B * T, ld, dtype=BF16, device=dev) if want_grad else None
    check(_lib.lib().otb_ctc_loss(_p(logp), ld, B, T, V, _p(in_len), _p(targets), targets.stride(0), _p(tgt_len), max_tgt, blank,
                                  _p(nll), _p(loss), _p(ws), _p(dl), ld if want_grad else 0, float(grad_scale),
                                  _p(scale_dev), _stream()),
          'otb_ctc_loss')
    _count(4 if want_grad else 3)
    return loss[0], nll, dl


def ctc_frame_topk(logits, B, T, V, in_len, K):
    """Per frame of logits f32 [B*T, ld]: the K best tokens' log-probs (log-softmax over V) and ids, best first, ties to the
    lower id (otb_ctc_frame_topk).  -> (top_lp f32 [B*T, K], top_id i32 [B*T, K]); frames at or past in_len: -inf / -1."""
    if logits.dim() != 2 or logits.shape[0] != B * T or logits.shape[1] < V:
        raise ValueError(f'ctc_frame_topk: logits must be [B*T = {B * T}, >= V = {V}], got {tuple(logits.shape)}')
    _ctc_lengths(in_len, B)
    _need(logits, torch.float32, 'logits'); _need(in_len, torch.int32, 'in_len')
    dev = logits.device
    lp = torch.empty(B * T, K, dtype=torch.float32, device=dev)
    ids = torch.empty(B * T, K, dtype=torch.int32, device=dev)
    check(_lib.lib().otb_ctc_frame_topk(_p(logits), logits.stride(0), B, T, V, _p(in_len), K, _p(lp), _p(ids), _stream()),
          'otb_ctc_frame_topk')
    _count()
    return lp, ids


def _ctc_lengths(in_len, B):
    if in_len.dim() != 1 or in_len.shape[0] != B:
        raise ValueError(f'in_len must be [B = {B}], got {tuple(in_len.shape)}')


def _ctc_topk_pair(top_lp, top_id, B, T, in_len):
    """top_lp / top_id: the [B*T, K] pair of ctc_frame_topk."""
    if top_id.dim() != 2 or top_id.shape[0] != B * T or top_lp.shape != top_id.shape:
        raise ValueError(f'top_lp and top_id must both be [B*T = {B * T}, K], got {tuple(top_lp.shape)} and {tuple(top_id.shape)}')
    _ctc_lengths(in_len, B)
    _need(top_lp, torch.float32, 'top_lp'); _need(top_id, torch.int32, 'top_id'); _need(in_len, torch.int32, 'in_len')


def ctc_greedy(top_lp, top_id, B, T, in_len, blank=0):
    """Greedy CTC collapse of the best token per frame (otb_ctc_greedy).  -> (ids i32 [B, T], lengths i32 [B], scores f32 [B])."""
    _ctc_topk_pair(top_lp, top_id, B, T, in_len)
    dev = top_lp.device
    ids = torch.empty(B, T, dtype=torch.int32, device=dev)
    lengths = torch.empty(B, dtype=torch.int32, device=dev)
    scores = torch.empty(B, dtype=torch.float32, device=dev)
    check(_lib.lib().otb_ctc_greedy(_p(top_lp), _p(top_id), top_id.shape[1], B, T, _p(in_len), blank, _p(ids), _p(lengths),
                                    _p(scores), _stream()), 'otb_ctc_greedy')
    _count()
    return ids, lengths, scores


def ctc_prefix_beam(top_lp, top_id, B, T, in_len, beam, blank=0):
    """CTC prefix beam search over each frame's top-K tokens (otb_ctc_prefix_beam), one launch for the batch.
    -> (ids i32 [B, beam, T] best first, lengths i32 [B, beam], scores f32 [B, beam])."""
    _ctc_topk_pair(top_lp, top_id, B, T, in_len)
    dev = top_lp.device
    nodes = torch.empty(B, 1 + T * beam, 2, dtype=torch.int32, device=dev)
    ids = torch.empty(B, beam, T, dtype=torch.int32, device=dev)
    lengths = torch.empty(B, beam, dtype=torch.int32, device=dev)
    scores = torch.empty(B, beam, dtype=torch.float32, device=dev)
    check(_lib.lib().otb_ctc_prefix_beam(_p(top_lp), _p(top_id), top_id.shape[1], B, T, _p(in_len), blank, beam, _p(nodes), _p(ids),
                                         _p(lengths), _p(scores), _stream()), 'otb_ctc_prefix_beam')
    _count()
    return ids, lengths, scores


def ctc_prefix_beam_slots(B, device):
    """The slot state of otb_ctc_prefix_beam_step for B utterances (uint8 bytes)."""
    return torch.zeros(int(_lib.lib().otb_ctc_prefix_beam_slots_bytes(B)), dtype=torch.uint8, device=device)


def ctc_prefix_beam_step(top_lp, top_id, B, T, in_len, beam, blank, lm, lm_weight, beta, slots, ctl, nodes, src, tok, ext,
                         ids, lengths, scores, anc=None, anc_tmp=None, pos=None):
    """One frame of the LM-fused CTC prefix beam search (otb_ctc_prefix_beam_step, DESIGN.md 4.19) on preallocated
    buffers: lm f32 [B*beam, V] the LM rows of the slots; ctl i32 [2] (frame, 0) before frame 0; nodes i32
    [B, 1 + T*beam, 2]; src / ext i32 and tok i64 [B*beam] written; ids / lengths / scores as ctc_prefix_beam, written at
    frame T - 1.  Transformer LM: anc / anc_tmp i32 [B*beam, Lpos], pos i32 [B*beam]."""
    Lpos = anc.shape[1] if anc is not None else 0
    check(_lib.lib().otb_ctc_prefix_beam_step(_p(top_lp), _p(top_id), top_id.shape[1], B, T, _p(in_len), blank, beam, _p(lm),
                                              lm.stride(0), float(lm_weight), float(beta), _p(slots), _p(ctl), _p(nodes),
                                              _p(src), _p(tok), _p(ext), _p(anc), _p(anc_tmp), _p(pos), Lpos, _p(ids),
                                              _p(lengths), _p(scores), _stream()), 'otb_ctc_prefix_beam_step')
    _count()


def ctc_lm_carry(dst, b, idx=None, ext=None, a=None):
    """Rows of 4-byte elements (otb_ctc_lm_carry): dst[n] = a[n] where ext[n] (dst[n] kept when a is None), else
    b[idx[n]] (b[n] without idx)."""
    rows, width = dst.shape[0], dst[0].numel()
    for t in (dst, a, b):
        if t is not None and (t.element_size() != 4 or t.stride(-1) != 1 or t[0].numel() != width):
            raise ValueError('ctc_lm_carry: rows of equal width of 4-byte elements')
    ld = lambda t: t.stride(0) if t is not None else 0
    check(_lib.lib().otb_ctc_lm_carry(_p(dst), ld(dst), _p(a), ld(a), _p(b), ld(b), _p(idx), _p(ext), rows, width, _stream()),
          'otb_ctc_lm_carry')
    _count()
    return dst


CTC_ALIGN_MAX_TOKENS = 1023


def ctc_align(rows, in_len, targets, tgt_len, lse=None, blank=0):
    """CTC forced alignment (otb_ctc_align): the best path of each utterance through the CTC trellis of its target, blank =
    `blank`.  rows f32 [B, T', V] with unit column stride (any row pitch, e.g. rows[:, :, :V] of a padded head output):
    log-probs, or logits when lse f32 [B, T'] gives each frame's log-sum-exp.  in_len i32 [B] valid frames; targets int
    [B, Lmax] (Lmax <= 1023), of which the first tgt_len[b] (i32 [B]) count.
    -> (labels i32 [B, T'] the token of each frame, blank included, -1 at or past in_len; frame_scores f32 [B, T'] its
    log-prob (-inf where the label is -1); spans i32 [B, Lmax, 2] [start, end) of each target token in frames of `rows`,
    -1 past tgt_len; path_score f32 [B]).  An utterance without an alignment (fewer frames than tokens plus adjacent
    repeats, a blank or out-of-range token, no frames for a non-empty target) gets path_score -inf and labels / spans -1.
    Ties prefer staying in a state, then one state back, then two; the end prefers the last token's blank."""
    if rows.dim() != 3 or rows.stride(2) != 1 or rows.stride(0) != rows.shape[1] * rows.stride(1):
        raise ValueError(f'ctc_align: rows must be [B, T, V] with unit column stride and evenly pitched rows, got '
                         f'{tuple(rows.shape)} strides {rows.stride()}')
    B, T, V = rows.shape
    if targets.dim() != 2 or targets.shape[0] != B:
        raise ValueError(f'ctc_align: targets must be [B = {B}, Lmax], got {tuple(targets.shape)}')
    if targets.shape[1] > CTC_ALIGN_MAX_TOKENS:
        raise ValueError(f'ctc_align: targets of up to {CTC_ALIGN_MAX_TOKENS} tokens are supported, got {targets.shape[1]}')
    _ctc_lengths(in_len, B)
    _ctc_lengths(tgt_len, B)
    if lse is not None and tuple(lse.shape) != (B, T):
        raise ValueError(f'ctc_align: lse must be [B = {B}, T = {T}], got {tuple(lse.shape)}')
    if not rows.is_cuda:
        raise RuntimeError('rows must be a CUDA tensor: the CUDA hot path has no CPU fallback')
    if rows.dtype != torch.float32:
        raise TypeError(f'rows must be torch.float32, got {rows.dtype}')
    _need(in_len, torch.int32, 'in_len'); _need(tgt_len, torch.int32, 'tgt_len')
    if lse is not None:
        _need(lse, torch.float32, 'lse')
    targets = targets.to(device=rows.device, dtype=torch.int64).contiguous()
    Lmax, dev = targets.shape[1], rows.device
    bp = torch.empty(B, T, 2 * Lmax + 1, dtype=torch.uint8, device=dev)
    labels = torch.empty(B, T, dtype=torch.int32, device=dev)
    scores = torch.empty(B, T, dtype=torch.float32, device=dev)
    spans = torch.empty(B, Lmax, 2, dtype=torch.int32, device=dev)
    path = torch.empty(B, dtype=torch.float32, device=dev)
    check(_lib.lib().otb_ctc_align(_p(rows), rows.stride(1), B, T, V, _p(lse), _p(in_len), _p(targets) if Lmax else None,
                                   max(Lmax, 1), _p(tgt_len), Lmax, blank, _p(bp), _p(labels), _p(scores),
                                   _p(spans) if Lmax else None, _p(path), _stream()), 'otb_ctc_align')
    _count()
    return labels, scores, spans, path


CTC_PREFIX_MAX_CANDIDATES = 16      # KMAX of csrc/beam_common.cuh


class CTCPrefixState:
    """Device buffers of CTC prefix scoring (csrc/ctc_prefix.cu) for one search of N = batch * beam hypotheses over
    log-probs lp f32 [batch * T, V] with P candidates per hypothesis: gamma f32 [2, N, T, 2] and psi f32 [2, N] of the
    hypotheses (ping-pong on the step counter's parity), gamma_cand f32 [N, P, T, 2], psi_cand f32 [N, P] and the
    candidates cand_val f32 / cand_id i32 [N, P] of one step."""

    def __init__(self, batch, beam, T, V, P, device, blank=0):
        if not beam <= P <= CTC_PREFIX_MAX_CANDIDATES:
            raise ValueError(f'CTC prefix scoring takes beam <= P <= {CTC_PREFIX_MAX_CANDIDATES} candidates, got beam {beam}, P {P}')
        self.B, self.beam, self.T, self.V, self.P, self.blank = batch, beam, T, V, P, blank
        N = batch * beam
        f32 = dict(dtype=torch.float32, device=device)
        self.lp = torch.zeros(batch * T, V, **f32)
        self.gamma = torch.zeros(2, N, T, 2, **f32)
        self.psi = torch.zeros(2, N, **f32)
        self.gamma_cand = torch.zeros(N, P, T, 2, **f32)
        self.psi_cand = torch.zeros(N, P, **f32)
        self.cand_val = torch.zeros(N, P, **f32)
        self.cand_id = torch.zeros(N, P, dtype=torch.int32, device=device)

    def init(self, in_len):
        """gamma / psi of the empty prefix from self.lp (otb_ctc_prefix_init); in_len i32 [batch] valid frames."""
        _ctc_lengths(in_len, self.B)
        _need(in_len, torch.int32, 'in_len')
        check(_lib.lib().otb_ctc_prefix_init(_p(self.lp), self.lp.stride(0), self.B, self.T, _p(in_len), self.blank, self.beam,
                                             _p(self.gamma), _p(self.psi), _stream()), 'otb_ctc_prefix_init')
        _count()

    def score(self, state, in_len, ctc_weight, out_val, out_idx, lm_logp=None, lm_weight=0.0):
        """otb_ctc_prefix_score on self.cand_val / self.cand_id (logsoftmax_topk with k = P of this step): fills gamma_cand /
        psi_cand and writes each hypothesis' `beam` best candidates by the joint score to out_val f32 / out_idx i32
        [N, beam], what BeamState.step_topk takes."""
        check(_lib.lib().otb_ctc_prefix_score(_p(self.lp), self.lp.stride(0), self.T, self.V, _p(in_len), self.blank,
                                              _p(self.gamma), _p(self.psi), _p(self.cand_val), _p(self.cand_id), self.P,
                                              _p(lm_logp), lm_logp.stride(0) if lm_logp is not None else 0, lm_weight,
                                              ctc_weight, ctypes.byref(state.c), _p(self.gamma_cand), _p(self.psi_cand),
                                              _p(out_val), _p(out_idx), _stream()), 'otb_ctc_prefix_score')
        _count()

    def advance(self, state, in_len):
        """otb_ctc_prefix_advance, after state.step_topk: the surviving hypotheses take their candidates' gamma / psi."""
        check(_lib.lib().otb_ctc_prefix_advance(ctypes.byref(state.c), _p(self.cand_id), self.P, self.T, _p(in_len),
                                                _p(self.gamma_cand), _p(self.psi_cand), _p(self.gamma), _p(self.psi), _stream()),
              'otb_ctc_prefix_advance')
        _count()


CTC_SCORE_MAX_LABELS = 1024      # max_len 1023 tokens and the closing <S/E>


def ctc_nbest_score(logp, B, T, in_len, targets, blank=0):
    """log p_ctc(targets[b, k] | utterance b) of K label rows per utterance (otb_ctc_nbest_score, DESIGN.md 4.18): the
    blank-extended forward recursion in fp32 over the utterance's log-probs, no copy of them per row and no workspace.
    logp f32 [B*T, V] (any row pitch, unit column stride) the head's log-softmax; in_len i32 [B] valid frames; targets i32
    [B, K, Lp] (Lp <= 1024), a row's labels being its entries before the first negative one (second_pass_rows' y <S/E>
    -1...).  -> f32 [B, K]; -inf where no alignment exists (a blank or out-of-range label, in_len 0, too few frames)."""
    if logp.dim() != 2 or logp.shape[0] != B * T or logp.stride(1) != 1:
        raise ValueError(f'ctc_nbest_score: logp must be [B*T = {B * T}, V] with unit column stride, got {tuple(logp.shape)}')
    if targets.dim() != 3 or targets.shape[0] != B:
        raise ValueError(f'ctc_nbest_score: targets must be [B = {B}, K, Lp], got {tuple(targets.shape)}')
    _, K, Lp = targets.shape
    if K < 1 or not 1 <= Lp <= CTC_SCORE_MAX_LABELS:
        raise ValueError(f'ctc_nbest_score: targets must have K >= 1 rows of 1..{CTC_SCORE_MAX_LABELS} labels, got '
                         f'{tuple(targets.shape)}')
    _ctc_lengths(in_len, B)
    for t, name, dtype in ((logp, 'logp', torch.float32), (targets, 'targets', torch.int32), (in_len, 'in_len', torch.int32)):
        if t.dtype != dtype:
            raise TypeError(f'ctc_nbest_score: {name} must be {dtype}, got {t.dtype}')
    if not logp.is_cuda:
        raise RuntimeError('logp must be a CUDA tensor: the CUDA hot path has no CPU fallback')
    _need(targets, torch.int32, 'targets'); _need(in_len, torch.int32, 'in_len')
    out = torch.empty(B, K, dtype=torch.float32, device=logp.device)
    check(_lib.lib().otb_ctc_nbest_score(_p(logp), logp.stride(0), B, T, logp.shape[1], _p(in_len), _p(targets), K, Lp, blank,
                                         _p(out), _stream()), 'otb_ctc_nbest_score')
    _count()
    return out


def token_logprob(logits, V, target):
    """out f32 [rows] = log_softmax(logits[r, :V])[target[r]], 0 where target[r] < 0 (otb_token_logprob): each row is read
    once and no [rows, V] log-softmax is written.  logits f32 [rows, ld] with ld % 4 == 0; target i32 [rows]."""
    _mat(logits, 'logits', torch.float32)
    rows = logits.shape[0]
    if target.shape != (rows,):
        raise ValueError(f'token_logprob: target must be [rows = {rows}], got {tuple(target.shape)}')
    _need(target, torch.int32, 'target')
    out = torch.empty(rows, dtype=torch.float32, device=logits.device)
    check(_lib.lib().otb_token_logprob(_p(logits), logits.stride(0), rows, V, _p(target), _p(out), _stream()), 'otb_token_logprob')
    _count()
    return out


def nbest_rescore(tgt, lengths, s1, tok_lp, weight, nbest, width, pad_id):
    """Re-rank each utterance's K first-pass hypotheses by s = s1 + weight * (sum of their second-pass token log-probs)
    (otb_nbest_rescore, DESIGN.md 4.10).  tgt i32 [B, K, Lp] the scored tokens y <S/E> (-1 after), lengths i32 [B, K] the
    length of y, s1 f32 [B, K], tok_lp f32 [M, B, K, Lp] the token log-probs of M models.  -> (ids i64 [B, nbest, width]
    y then pad_id, lengths i32 [B, nbest], scores f32 [B, nbest]); duplicates of a better first-pass hypothesis rank last
    with score -inf, length 0 and pad_id throughout."""
    B, K, Lp = tgt.shape
    if lengths.shape != (B, K) or s1.shape != (B, K) or tok_lp.dim() != 4 or tuple(tok_lp.shape[1:]) != (B, K, Lp):
        raise ValueError(f'nbest_rescore: need lengths / s1 [B, K] = [{B}, {K}] and tok_lp [M, {B}, {K}, {Lp}], got '
                         f'{tuple(lengths.shape)}, {tuple(s1.shape)}, {tuple(tok_lp.shape)}')
    _need(tgt, torch.int32, 'tgt'); _need(lengths, torch.int32, 'lengths'); _need(s1, torch.float32, 's1')
    _need(tok_lp, torch.float32, 'tok_lp')
    dev = tgt.device
    ids = torch.empty(B, nbest, width, dtype=torch.int64, device=dev)
    out_len = torch.empty(B, nbest, dtype=torch.int32, device=dev)
    scores = torch.empty(B, nbest, dtype=torch.float32, device=dev)
    check(_lib.lib().otb_nbest_rescore(_p(tgt), Lp, _p(lengths), _p(s1), _p(tok_lp), tok_lp.shape[0], B, K, float(weight), nbest,
                                       width, int(pad_id), _p(ids), _p(out_len), _p(scores), _stream()), 'otb_nbest_rescore')
    _count()
    return ids, out_len, scores


EDIT_DISTANCE_MAX_TOKENS = 1023


def edit_distance(hyp, hyp_len, ref, ref_len, K=1):
    """Levenshtein distances (unit costs) of hypothesis rows against reference rows (otb_edit_distance): hyp int [N, Lh] of
    which the first hyp_len[i] (i32 [N]) count, ref int [ceil(N / K), Lr] with ref_len i32 [ceil(N / K)]; hypothesis i is
    compared with reference i // K.  Lh, Lr <= 1023.  -> i32 [N], exact."""
    if hyp.dim() != 2 or ref.dim() != 2:
        raise ValueError(f'edit_distance: hyp and ref must be 2-D, got {tuple(hyp.shape)} and {tuple(ref.shape)}')
    N, Lh = hyp.shape
    Lr = ref.shape[1]
    if max(Lh, Lr) > EDIT_DISTANCE_MAX_TOKENS:
        raise ValueError(f'edit_distance: sequences of up to {EDIT_DISTANCE_MAX_TOKENS} tokens are supported, got rows of {Lh} '
                         f'and {Lr}')
    if K < 1 or ref.shape[0] != -(-N // K) or hyp_len.shape != (N,) or ref_len.shape != (ref.shape[0],):
        raise ValueError(f'edit_distance: need K >= 1, ref [ceil(N / K)] rows and lengths [N] / [ceil(N / K)], got K {K}, hyp '
                         f'{tuple(hyp.shape)}, ref {tuple(ref.shape)}, lengths {tuple(hyp_len.shape)}, {tuple(ref_len.shape)}')
    hyp = hyp.to(torch.int32).contiguous()
    ref = ref.to(torch.int32).contiguous()
    for t, n in ((hyp, 'hyp'), (ref, 'ref'), (hyp_len, 'hyp_len'), (ref_len, 'ref_len')):
        _need(t, torch.int32, n)
    out = torch.empty(N, dtype=torch.int32, device=hyp.device)
    check(_lib.lib().otb_edit_distance(_p(hyp), max(Lh, 1), _p(hyp_len), _p(ref), max(Lr, 1), _p(ref_len), N, K, Lh, Lr, _p(out),
                                       _stream()), 'otb_edit_distance')
    _count()
    return out


def mwer_coeff(tgt, lengths, err, tok_lp, grad_scale=1.0, scale_dev=None):
    """The expected-risk term of each utterance's K hypotheses (otb_mwer_coeff, DESIGN.md 4.11).  tgt i32 [B, K, Lp] the scored
    tokens y <S/E> (-1 after), lengths i32 [B, K] the length of y, err i32 [B, K] the edit distances, tok_lp f32 [B, K, Lp].
    -> (loss f32 [B] = sum_k P_k (W_k - mean W) over the kept hypotheses, coeff f32 [B, K] = dloss/dl_k * grad_scale (times
    the f32 device scalar scale_dev when given); 0 for a duplicate of a better-ranked hypothesis)."""
    B, K, Lp = tgt.shape
    if lengths.shape != (B, K) or err.shape != (B, K) or tok_lp.shape != (B, K, Lp):
        raise ValueError(f'mwer_coeff: need lengths / err [B, K] = [{B}, {K}] and tok_lp [{B}, {K}, {Lp}], got '
                         f'{tuple(lengths.shape)}, {tuple(err.shape)}, {tuple(tok_lp.shape)}')
    _need(tgt, torch.int32, 'tgt'); _need(lengths, torch.int32, 'lengths'); _need(err, torch.int32, 'err')
    _need(tok_lp, torch.float32, 'tok_lp')
    if scale_dev is not None:
        _need(scale_dev, torch.float32, 'scale_dev')
    coeff = torch.empty(B, K, dtype=torch.float32, device=tgt.device)
    loss = torch.empty(B, dtype=torch.float32, device=tgt.device)
    check(_lib.lib().otb_mwer_coeff(_p(lengths), _p(err), _p(tok_lp), Lp, _p(tgt), B, K, float(grad_scale), _p(scale_dev), _p(coeff),
                                    _p(loss), _stream()), 'otb_mwer_coeff')
    _count()
    return loss, coeff


def mwer_sample_coeff(err, grad_scale=1.0, scale_dev=None):
    """The sampled estimator's coefficients (otb_mwer_sample_coeff, DESIGN.md 4.11): err i32 [B, K] the edit distances of
    K samples per utterance, drawn with replacement.  -> (loss f32 [B] = mean_k W_k, coeff f32 [B, K] = (W_k - mean W) / K *
    grad_scale (times the f32 device scalar scale_dev when given)), exactly 0 when an utterance's W are all equal."""
    if err.dim() != 2:
        raise ValueError(f'mwer_sample_coeff: err must be [B, K], got {tuple(err.shape)}')
    _need(err, torch.int32, 'err')
    if scale_dev is not None:
        _need(scale_dev, torch.float32, 'scale_dev')
    B, K = err.shape
    coeff = torch.empty(B, K, dtype=torch.float32, device=err.device)
    loss = torch.empty(B, dtype=torch.float32, device=err.device)
    check(_lib.lib().otb_mwer_sample_coeff(_p(err), B, K, float(grad_scale), _p(scale_dev), _p(coeff), _p(loss), _stream()),
          'otb_mwer_sample_coeff')
    _count()
    return loss, coeff


def mwer_grad(logits, V, target, tok_lp, coeff):
    """bf16 dlogits [rows, ld] = coeff[r // Lp] * (onehot(target[r]) - softmax(logits[r, :V])) (otb_mwer_grad): logits f32
    [rows, ld] (ld % 4 == 0), target i32 [rows] (-1: a zero row), tok_lp f32 [rows] = token_logprob(logits, V, target),
    coeff f32 [rows // Lp] (the hypotheses of Lp rows each); padding columns are zero."""
    _mat(logits, 'logits', torch.float32)
    rows, ld = logits.shape[0], logits.stride(0)
    coeff = coeff.reshape(-1)
    if target.shape != (rows,) or tok_lp.shape != (rows,) or coeff.numel() < 1 or rows % coeff.numel():
        raise ValueError(f'mwer_grad: need target / tok_lp [rows = {rows}] and coeff dividing the rows, got {tuple(target.shape)}, '
                         f'{tuple(tok_lp.shape)}, {tuple(coeff.shape)}')
    _need(target, torch.int32, 'target'); _need(tok_lp, torch.float32, 'tok_lp'); _need(coeff, torch.float32, 'coeff')
    out = torch.empty(rows, ld, dtype=BF16, device=logits.device)
    check(_lib.lib().otb_mwer_grad(_p(logits), ld, rows, V, _p(target), _p(tok_lp), _p(coeff), rows // coeff.numel(), _p(out),
                                   _stream()), 'otb_mwer_grad')
    _count()
    return out


def conv_im2col(h1, B, T, F, C1, geom=CONV_SHIPPED):
    _, _, T2, F2, _, _ = conv_sizes(T, F, geom)
    col = torch.empty(B * T2 * F2, geom[4] * geom[5] * C1, dtype=BF16, device=h1.device)
    check(_lib.lib().otb_conv_im2col(_p(h1), _p(col), B, T, F, C1, *geom, _stream()), 'otb_conv_im2col')
    _count()
    return col


def conv_col2im_relu(dcol, h1, B, T, F, C1, geom=CONV_SHIPPED):
    dpre1 = torch.empty_like(h1)
    check(_lib.lib().otb_conv_col2im_relu(_p(dcol), _p(h1), _p(dpre1), B, T, F, C1, *geom, _stream()), 'otb_conv_col2im_relu')
    _count()
    return dpre1


def conv1_wgrad(dpre1, x, B, T, F, C1, geom=CONV_SHIPPED):
    """-> f32 [C1, kt1*kf1 + 1]: conv1's tap gradients, then its bias gradient."""
    out = torch.empty(C1, geom[0] * geom[1] + 1, dtype=torch.float32, device=x.device)
    check(_lib.lib().otb_conv1_wgrad(_p(dpre1), _p(x), _p(out), B, T, F, C1, *geom, _stream()), 'otb_conv1_wgrad')
    _count()
    return out



# ------------------------------------------------------------------------------------------------
# recurrent language model: LSTM recurrence (include/otb200.h "Recurrent language model")
# ------------------------------------------------------------------------------------------------
def lstm_config(H, sms, smem_optin):
    """-> (hidden units per CTA, forward / backward dynamic shared memory) of the LSTM recurrence kernels for hidden size H on
    a device with `sms` SMs and `smem_optin` bytes of opt-in shared memory per block (otb_lstm_config: host only).  Raises
    NotImplementedError where otb_lstm_fwd / otb_lstm_bwd refuse H."""
    u, f, b = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    if _lib.lib().otb_lstm_config(int(H), int(sms), int(smem_optin), u, f, b) != 0:
        raise NotImplementedError(_lib.lib().otb_last_error().decode('utf-8', 'replace'))
    return u.value, f.value, b.value


_LSTM_BARRIERS = {}


def _lstm_barrier(device):
    """The grid-barrier counter of the LSTM kernels, one per stream: launches on one stream run one after another, and the
    counter's generation scheme needs no reset between them."""
    stream = torch.cuda.current_stream(device)
    key = (stream.device.index, stream.cuda_stream)
    bar = _LSTM_BARRIERS.get(key)
    if bar is None:
        bar = _LSTM_BARRIERS[key] = torch.zeros(2, dtype=torch.int32, device=device)
    return bar


def lstm_fwd(gx, w_hh, L, B, h0=None, c0=None, train=False, barrier=None):
    """One LSTM layer over gx f32 [L*B, 4H] (time-major input projection incl. both biases), w_hh bf16 [4H, H], h0 / c0 f32
    [B, H] or None -> (y bf16 [L*B, H], h_n f32 [B, H], c_n f32 [B, H], gates, c_all); with train the post-activation gates
    (written over gx) and c_t f32 [L*B, H] for lstm_bwd, else None.  barrier: an i32 [2] zero-initialised grid-barrier
    counter owned by the caller (a captured CUDA graph must not allocate one), else the current stream's."""
    _need(gx, torch.float32, 'gx'); _need(w_hh, BF16, 'w_hh')
    H = w_hh.shape[1]
    for t, n in ((h0, 'h0'), (c0, 'c0')):
        if t is not None:
            _need(t, torch.float32, n)
    dev = gx.device
    y = torch.empty(L * B, H, dtype=BF16, device=dev)
    h_n = torch.empty(B, H, dtype=torch.float32, device=dev)
    c_n = torch.empty(B, H, dtype=torch.float32, device=dev)
    gates = gx if train else None
    c_all = torch.empty(L * B, H, dtype=torch.float32, device=dev) if train else None
    check(_lib.lib().otb_lstm_fwd(_p(gx), _p(w_hh), _p(h0), _p(c0), _p(y), _p(h_n), _p(c_n), _p(gates), _p(c_all),
                                  _p(barrier if barrier is not None else _lstm_barrier(dev)), L, B, H, _stream()), 'otb_lstm_fwd')
    _count()
    return y, h_n, c_n, gates, c_all


def lstm_bwd(dy, w_hh, gates, c_all, L, B, c0=None):
    """Backward through time of lstm_fwd(train=True): dy bf16 [L*B, H] -> dG bf16 [L*B, 4H] (pre-activation gates)."""
    _need(dy, BF16, 'dy'); _need(w_hh, BF16, 'w_hh'); _need(gates, torch.float32, 'gates'); _need(c_all, torch.float32, 'c_all')
    H = w_hh.shape[1]
    dev = dy.device
    dg = torch.empty(L * B, 4 * H, dtype=BF16, device=dev)
    dc = torch.empty(B, H, dtype=torch.float32, device=dev)
    check(_lib.lib().otb_lstm_bwd(_p(dy), _p(w_hh), _p(gates), _p(c_all), _p(c0), _p(dg), _p(dc), _p(_lstm_barrier(dev)), L, B, H,
                                  _stream()), 'otb_lstm_bwd')
    _count()
    return dg


def embedding(tok, emb, out=None):
    """nn.Embedding lookup: tok i64 [N] -> bf16 [N, d] = emb[tok] (no scale)."""
    _need(emb, BF16, 'emb')
    tok = tok.contiguous().view(-1)
    N, d = tok.numel(), emb.shape[1]
    if out is None:
        out = torch.empty(N, d, dtype=BF16, device=emb.device)
    check(_lib.lib().otb_embedding(_p(tok), _p(emb), _p(out), N, d, emb.shape[0], _stream()), 'otb_embedding')
    _count()
    return out


# ------------------------------------------------------------------------------------------------
# transducer (RNN-T) model: joint network, lattice log-probs, loss and greedy step (include/otb200.h "Transducer")
# ------------------------------------------------------------------------------------------------
RNNT_MAX_LABELS = 1023


def _rnnt_lengths(t_len, u_len):
    _need(t_len, torch.int32, 't_len'); _need(u_len, torch.int32, 'u_len')
    return t_len, u_len


def _rnnt_band(s_begin, S, B, T, U1):
    """-> (row width of the stored lattice, S as the kernels take it): (U1, 0) for the full lattice, (S, S) for the band
    s_begin i32 [B, T] of width S (pruned RNN-T)."""
    if s_begin is None:
        return U1, 0
    _need(s_begin, torch.int32, 's_begin')
    if s_begin.numel() != B * T:
        raise ValueError(f's_begin must be [B, T] = [{B}, {T}], got {tuple(s_begin.shape)}')
    if not isinstance(S, int) or S < 2:
        raise ValueError(f'the band width S must be an int >= 2, got {S!r}')
    return S, S


def rnnt_joint(ep, pp, B, T, U1, t_len=None, u_len=None, out=None, s_begin=None, S=None):
    """Hj bf16 [B*T*U1, D] = tanh(ep[b*T + t] + pp[b*U1 + u]) over the padded lattice, u fastest (otb_rnnt_joint); ep bf16
    [B*T, D], pp bf16 [B*U1, D].  Nodes with t >= t_len[b] or u > u_len[b] (i32 [B]) are zero; without lengths every node
    is valid.  With s_begin i32 [B, T] (pruned RNN-T): [B*T*S, D], row (b*T + t)*S + k holding u = s_begin[b, t] + k."""
    _need(ep, BF16, 'ep'); _need(pp, BF16, 'pp')
    D = ep.shape[1]
    if ep.shape[0] != B * T or tuple(pp.shape) != (B * U1, D):
        raise ValueError(f'rnnt_joint: ep must be [B*T, D] = [{B * T}, D] and pp [B*U1, D] = [{B * U1}, {D}], got '
                         f'{tuple(ep.shape)} and {tuple(pp.shape)}')
    if (t_len is None) != (u_len is None):
        raise ValueError('rnnt_joint: t_len and u_len are given together')
    if t_len is not None:
        _rnnt_lengths(t_len, u_len)
    W, Sk = _rnnt_band(s_begin, S, B, T, U1)
    if out is None:
        out = torch.empty(B * T * W, D, dtype=BF16, device=ep.device)
    check(_lib.lib().otb_rnnt_joint(_p(ep), _p(pp), B, T, U1, D, _p(t_len), _p(u_len), _p(out), _p(s_begin), Sk, _stream()),
          'otb_rnnt_joint')
    _count()
    return out


def rnnt_joint_bwd(dh, h, B, T, U1, t_len, u_len, s_begin=None, S=None):
    """Backward of rnnt_joint from dh = dHj bf16 [B*T*U1, D] and its output h -> (dEp bf16 [B*T, D], dPp bf16 [B*U1, D]):
    dZ = dh (1 - h^2) summed over u and over t, in a fixed order (otb_rnnt_joint_bwd).  s_begin, S: as rnnt_joint."""
    _need(dh, BF16, 'dh'); _need(h, BF16, 'h'); _rnnt_lengths(t_len, u_len)
    _, Sk = _rnnt_band(s_begin, S, B, T, U1)
    D = h.shape[1]
    dep = torch.empty(B * T, D, dtype=BF16, device=h.device)
    dpp = torch.empty(B * U1, D, dtype=BF16, device=h.device)
    check(_lib.lib().otb_rnnt_joint_bwd(_p(dh), _p(h), B, T, U1, D, _p(t_len), _p(u_len), _p(dep), _p(dpp), _p(s_begin), Sk,
                                        _stream()), 'otb_rnnt_joint_bwd')
    _count()
    return dep, dpp


def rnnt_logprob(logits, row0, V, B, T, U1, t_len, u_len, labels, lp, s_begin=None, S=None):
    """Lattice rows [row0, row0 + rows) of logits f32 [rows, ld] -> lp f32 [B*T*U1, 3] rows row0.. = (logsumexp, log p(blank),
    log p(labels[b, u])) (otb_rnnt_logprob); labels i32 [B, >= U1 - 1].  s_begin, S: as rnnt_joint (lp [B*T*S, 3])."""
    _mat(logits, 'logits', torch.float32); _rnnt_lengths(t_len, u_len); _need(labels, torch.int32, 'labels')
    _need(lp, torch.float32, 'lp')
    _, Sk = _rnnt_band(s_begin, S, B, T, U1)
    check(_lib.lib().otb_rnnt_logprob(_p(logits), logits.stride(0), logits.shape[0], row0, V, B, T, U1, _p(t_len), _p(u_len),
                                      _p(labels), labels.stride(0), _p(lp), _p(s_begin), Sk, _stream()), 'otb_rnnt_logprob')
    _count()
    return lp


def rnnt_loss(lp, B, T, U1, t_len, u_len, grad_scale=1.0, scale_dev=None, s_begin=None, S=None):
    """The RNN-T loss over the lattice log-probs lp (rnnt_logprob) -> (loss 0-d = mean_b nll_b, nll f32 [B], grad f32
    [B*T*U1, 2] = grad_scale (x the f32 device scalar scale_dev) / B * d nll_b / d (log p(blank), log p(label)))
    (otb_rnnt_loss).  s_begin, S: the alignments restricted to the bands (as rnnt_joint; lp and grad [B*T*S, .]); an
    utterance with no alignment inside them has nll +inf and zero gradients."""
    _need(lp, torch.float32, 'lp'); _rnnt_lengths(t_len, u_len)
    if U1 - 1 > RNNT_MAX_LABELS:
        raise ValueError(f'rnnt_loss: transcripts of {U1 - 1} labels; at most {RNNT_MAX_LABELS} are supported')
    if scale_dev is not None:
        _need(scale_dev, torch.float32, 'scale_dev')
    W, Sk = _rnnt_band(s_begin, S, B, T, U1)
    dev = lp.device
    alpha = torch.empty(B * T * W, dtype=torch.float64, device=dev)
    nll = torch.empty(B, dtype=torch.float32, device=dev)
    loss = torch.empty(1, dtype=torch.float32, device=dev)
    grad = torch.empty(B * T * W, 2, dtype=torch.float32, device=dev)
    check(_lib.lib().otb_rnnt_loss(_p(lp), B, T, U1, _p(t_len), _p(u_len), _p(alpha), _p(nll), _p(loss), _p(grad), float(grad_scale),
                                   _p(scale_dev), _p(s_begin), Sk, _stream()), 'otb_rnnt_loss')
    _count(2)
    return loss[0], nll, grad


def rnnt_dlogits(logits, row0, V, B, T, U1, t_len, u_len, labels, lp, grad, out=None, s_begin=None, S=None):
    """dz bf16 [rows, ld] = [k = blank] a + [k = label] c - softmax_k (a + c) of the lattice rows [row0, row0 + rows) in
    logits f32 [rows, ld], with lp's logsumexp and (a, c) = grad of the node (otb_rnnt_dlogits); columns >= V are zero.
    s_begin, S: as rnnt_joint."""
    _mat(logits, 'logits', torch.float32); _rnnt_lengths(t_len, u_len); _need(labels, torch.int32, 'labels')
    _need(lp, torch.float32, 'lp'); _need(grad, torch.float32, 'grad')
    _, Sk = _rnnt_band(s_begin, S, B, T, U1)
    rows, ld = logits.shape[0], logits.shape[1]
    if out is None:
        out = torch.empty(rows, ld, dtype=BF16, device=logits.device)
    check(_lib.lib().otb_rnnt_dlogits(_p(logits), logits.stride(0), rows, row0, V, B, T, U1, _p(t_len), _p(u_len), _p(labels),
                                      labels.stride(0), _p(lp), _p(grad), _p(out), out.stride(0), _p(s_begin), Sk, _stream()),
          'otb_rnnt_dlogits')
    _count()
    return out


def rnnt_simple_lse(am, lm, V, B, T, U1, t_len, u_len, labels):
    """The simple joint of pruned RNN-T (otb_rnnt_simple_lse): logits am[b*T + t] + lm[b*U1 + u] of am f32 [B*T, >= V] and
    lm f32 [B*U1, >= V] -> (lp f32 [B*T*U1, 3] as rnnt_logprob's, m_am f32 [B*T], m_lm f32 [B*U1] the row maxima)."""
    _mat(am, 'am', torch.float32); _mat(lm, 'lm', torch.float32); _rnnt_lengths(t_len, u_len); _need(labels, torch.int32, 'labels')
    if am.shape[0] != B * T or lm.shape[0] != B * U1:
        raise ValueError(f'rnnt_simple_lse: am must have B*T = {B * T} rows and lm B*U1 = {B * U1}, got {am.shape[0]} and '
                         f'{lm.shape[0]}')
    dev = am.device
    lp = torch.empty(B * T * U1, 3, dtype=torch.float32, device=dev)
    m_am = torch.empty(B * T, dtype=torch.float32, device=dev)
    m_lm = torch.empty(B * U1, dtype=torch.float32, device=dev)
    check(_lib.lib().otb_rnnt_simple_lse(_p(am), am.stride(0), _p(lm), lm.stride(0), V, B, T, U1, _p(t_len), _p(u_len), _p(labels),
                                         labels.stride(0), _p(lp), _p(m_am), _p(m_lm), _stream()), 'otb_rnnt_simple_lse')
    _count()
    return lp, m_am, m_lm


def rnnt_simple_bwd(am, lm, V, B, T, U1, t_len, u_len, labels, lp, m_am, m_lm, grad, scale=1.0, scale_dev=None, ldd=None):
    """Backward of the simple joint (otb_rnnt_simple_bwd) from grad = rnnt_loss's over rnnt_simple_lse's lp, times scale (x
    the f32 device scalar scale_dev) -> (d am bf16 [B*T, ldd], d lm bf16 [B*U1, ldd]), columns >= V zero."""
    _mat(am, 'am', torch.float32); _mat(lm, 'lm', torch.float32); _rnnt_lengths(t_len, u_len); _need(labels, torch.int32, 'labels')
    _need(grad, torch.float32, 'grad')
    if scale_dev is not None:
        _need(scale_dev, torch.float32, 'scale_dev')
    ldd = ldd or (V + 7) // 8 * 8
    d_am = torch.empty(B * T, ldd, dtype=BF16, device=am.device)
    d_lm = torch.empty(B * U1, ldd, dtype=BF16, device=am.device)
    check(_lib.lib().otb_rnnt_simple_bwd(_p(am), am.stride(0), _p(lm), lm.stride(0), V, B, T, U1, _p(t_len), _p(u_len), _p(labels),
                                         labels.stride(0), _p(lp), _p(m_am), _p(m_lm), _p(grad), float(scale), _p(scale_dev),
                                         _p(d_am), _p(d_lm), ldd, _stream()), 'otb_rnnt_simple_bwd')
    _count()
    return d_am, d_lm


def rnnt_prune_ranges(grad, B, T, U1, t_len, u_len, S):
    """The band of each frame for pruned RNN-T (otb_rnnt_prune_ranges): s_begin i32 [B, T] from the simple loss's node
    gradients grad f32 [B*T*U1, 2] (rnnt_loss), by the range rule of DESIGN.md 4.22."""
    _need(grad, torch.float32, 'grad'); _rnnt_lengths(t_len, u_len)
    s_begin = torch.empty(B, T, dtype=torch.int32, device=grad.device)
    check(_lib.lib().otb_rnnt_prune_ranges(_p(grad), B, T, U1, _p(t_len), _p(u_len), int(S), _p(s_begin), _stream()),
          'otb_rnnt_prune_ranges')
    _count()
    return s_begin


def rnnt_greedy_step(idx, logp, h_new, c_new, pp_new, h, c, pp, ep, T, ep_cur, t_len, frame, n_sym, n_out, ids, max_sym, score,
                     active, val=None, emit=None, lm_pos=None):
    """One step of batched greedy transducer search (otb_rnnt_greedy_step): the decision of every row from the arg-max idx
    i32 [B] and log-probs logp f32 [B, ld] of the joint, the predictor state (h, c f32 [layers, B, H], pp bf16 [B, D]) moved
    forward from (h_new, c_new, pp_new) where a row emitted, and the frame state (ep_cur, frame, n_sym, n_out, ids i32
    [B, max_len], score, active) updated in place.  LM fusion: val f32 [B] the arg-max's fused value, which an emitted label
    adds to the score; emit i32 [B] <- 1 where the row emitted; lm_pos i32 [B] <- the label's LM position n_out, else -1."""
    for t, name in ((val, 'val'), (emit, 'emit'), (lm_pos, 'lm_pos')):
        if t is not None:
            _need(t, torch.float32 if name == 'val' else torch.int32, name)
    layers, B, H = h.shape
    D = pp.shape[1]
    check(_lib.lib().otb_rnnt_greedy_step(_p(idx), _p(logp), logp.stride(0), _p(h_new), _p(c_new), _p(pp_new), _p(h), _p(c), _p(pp),
                                          layers, B, H, D, _p(ep), T, _p(ep_cur), _p(t_len), _p(frame), _p(n_sym), _p(n_out),
                                          _p(ids), ids.shape[1], max_sym, _p(score), _p(active), _p(val), _p(emit), _p(lm_pos),
                                          _stream()), 'otb_rnnt_greedy_step')
    _count()


RNNT_BEAM_MAX = 15          # beam width: K + 1 log-probs per slot from logsoftmax_topk, whose k is at most 16


def rnnt_beam_step(logp, val, idx, V, T, t_len, state, out, beta=0.0, lm=None):
    """One step of the transducer's ALSD beam search (otb_rnnt_beam_step) for every utterance not yet ended, from the
    joint's log-probs at each slot: logp f32 [B*K, ld] and the top min(K + 1, V) (val f32, idx i32 [B*K, k1]) of
    logsoftmax_topk.  state: dict of the search's device arrays, updated in place -- the slots (score f32, u, frame, node i32
    [B*K]), the step's actions (par i32, tok i64 [B*K]), the node table (node_par, node_tok i32 [B, n_cap], n_nodes i32 [B]),
    the n-best so far (f_score f32, f_node, f_u i32 [B, W], f_n i32 [B]), done i32 [B] and active i32 [1].  out: (ids i32
    [B, W, max_len], lengths i32 [B, W], scores f32 [B, W]), written for each utterance when it ends.
    LM fusion (val holds the fused label values): beta > 0 loosens the end bound by beta per label still to come; lm, a dict
    of i32 outputs for the LM carry: src and ext [B*K], and for the Transformer LM anc / anc_tmp [B*K, Lpos] and pos [B*K]."""
    s = state
    lm = lm or {}
    for k in ('src', 'ext', 'anc', 'anc_tmp', 'pos'):
        if lm.get(k) is not None:
            _need(lm[k], torch.int32, k)
    anc = lm.get('anc')
    _need(logp, torch.float32, 'logp'); _need(val, torch.float32, 'val'); _need(idx, torch.int32, 'idx')
    B, W = s['f_score'].shape
    K = s['score'].numel() // B
    ids, lengths, scores = out
    check(_lib.lib().otb_rnnt_beam_step(_p(logp), logp.stride(0), _p(val), _p(idx), idx.shape[1], B, K, W, V, T, ids.shape[2],
                                        _p(t_len), _p(s['score']), _p(s['u']), _p(s['frame']), _p(s['node']), _p(s['par']),
                                        _p(s['tok']), _p(s['node_par']), _p(s['node_tok']), s['node_par'].shape[1],
                                        _p(s['n_nodes']), _p(s['f_score']), _p(s['f_node']), _p(s['f_u']), _p(s['f_n']),
                                        _p(s['done']), _p(s['active']), _p(ids), _p(lengths), _p(scores), float(beta),
                                        _p(lm.get('src')), _p(lm.get('ext')), _p(anc), _p(lm.get('anc_tmp')), _p(lm.get('pos')),
                                        anc.shape[1] if anc is not None else 0, _stream()),
          'otb_rnnt_beam_step')
    _count()


def rnnt_beam_gather(par, frame, K, h, c, pp, ep, T, hg, cg, ppg, ep_cur):
    """Each slot row r of utterance b = r // K takes the predictor state of row b*K + par[r]: (h, c) f32 [layers, B*K, H]
    and pp bf16 [B*K, D] -> (hg, cg, ppg) row r; and its frame's encoder projection, ep bf16 [B*T, D] row b*T + frame[r]
    -> ep_cur bf16 [B*K, D] row r (otb_rnnt_beam_gather)."""
    layers, BK, H = h.shape
    D = pp.shape[1]
    check(_lib.lib().otb_rnnt_beam_gather(_p(par), _p(frame), BK // K, K, layers, H, D, T, _p(h), _p(c), _p(pp), _p(ep), _p(hg),
                                          _p(cg), _p(ppg), _p(ep_cur), _stream()), 'otb_rnnt_beam_gather')
    _count()


def rnnt_beam_commit(tok, hg, cg, ppg, hn, cn, ppn, h, c, pp):
    """(h, c, pp) row r = the predictor's output (hn, cn, ppn) row r where tok[r] (i64) is a label, else the gathered
    (hg, cg, ppg) row r (otb_rnnt_beam_commit)."""
    layers, BK, H = h.shape
    check(_lib.lib().otb_rnnt_beam_commit(_p(tok), BK, layers, H, pp.shape[1], _p(hg), _p(cg), _p(ppg), _p(hn), _p(cn), _p(ppn),
                                          _p(h), _p(c), _p(pp), _stream()), 'otb_rnnt_beam_commit')
    _count()
