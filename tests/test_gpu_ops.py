"""GPU parity of every C-ABI op against a plain fp32 torch restatement of the same op (the checker),
on bf16-rounded operands so that only accumulation order / output rounding differ.  Integer results
(beam search) are compared bit-exactly against oracle/.  Run with -m gpu on an H100."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops
    DEV = torch.device('cuda:0')
BF = torch.bfloat16
torch.backends.cudnn.allow_tf32 = False        # the fp32 checker must not silently run in TF32
torch.backends.cuda.matmul.allow_tf32 = False


def _rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def _report(name, got, ref, tol_rel, tol_abs=0.0):
    got, ref = got.float(), ref.float()
    diff = (got - ref).abs()
    denom = ref.abs().max().item() + 1e-12
    rel_l2 = ((got - ref).norm() / (ref.norm() + 1e-12)).item()
    worst = diff.max().item()
    bad = torch.isnan(got).sum().item()
    msg = f'{name}: rel_l2={rel_l2:.3e} max_abs={worst:.3e} (ref max {denom:.3e}) nan={bad} shape={tuple(got.shape)}'
    if not (rel_l2 <= tol_rel and bad == 0 and worst <= tol_abs + 8 * tol_rel * denom):
        idx = torch.nonzero(diff > tol_abs + 8 * tol_rel * denom)[:8].tolist()
        rows = torch.nonzero(diff.reshape(diff.shape[0], -1).amax(1) > tol_abs + 8 * tol_rel * denom).view(-1)[:16].tolist()
        raise AssertionError(msg + f'\n first bad idx {idx}\n bad rows {rows}\n got {got.flatten()[:8].tolist()}\n ref {ref.flatten()[:8].tolist()}')
    return msg


# ------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize('M,N,K', [(128, 256, 64), (128, 256, 256), (300, 768, 256), (7968, 768, 256),
                                   (320, 4234, 256), (1000, 256, 2560), (77, 64, 128), (513, 520, 192)])
def test_linear_bias_fp32_out(M, N, K):
    a = _rnd(M, K, seed=1).to(BF)
    w = _rnd(N, K, scale=K ** -0.5, seed=2).to(BF)
    b = _rnd(N, seed=3)
    ld = (N + 7) // 8 * 8
    out = ops.linear(a, w, b, ops.EPI_BIAS, out_f32=True, n_out=ld)
    ref = a.float() @ w.float().t() + b
    print(_report(f'linear[{M},{N},{K}]', out[:, :N], ref, 2e-5, 1e-4))
    if ld > N:
        assert True  # padding columns are unspecified


@pytest.mark.parametrize('epi', ['relu', 'swish', 'gelu', 'tanh'])
def test_linear_activations_bf16_out(epi):
    M, N, K = 777, 384, 256
    a = _rnd(M, K, seed=1).to(BF)
    w = _rnd(N, K, scale=K ** -0.5, seed=2).to(BF)
    b = _rnd(N, seed=3)
    out = ops.linear(a, w, b, ops.ACT_EPILOGUE[epi])
    v = a.float() @ w.float().t() + b
    ref = {'relu': torch.relu, 'swish': lambda x: x * torch.sigmoid(x), 'gelu': F.gelu, 'tanh': torch.tanh}[epi](v)
    print(_report(f'linear+{epi}', out, ref, 4e-3))


@pytest.mark.parametrize('M,Nh,K', [(7968, 2048, 256), (300, 768, 256), (130, 256, 256), (64, 96, 64)])
def test_linear_glu(M, Nh, K):
    a = _rnd(M, K, seed=1).to(BF)
    w = _rnd(2 * Nh, K, scale=K ** -0.5, seed=2).to(BF)
    b = _rnd(2 * Nh, seed=3)
    out = ops.linear(a, w, b, ops.EPI_GLU)
    assert out.shape == (M, Nh)
    ref = F.glu(a.float() @ w.float().t() + b, dim=-1)
    print(_report(f'linear+glu[{M},{Nh},{K}]', out, ref, 4e-3))


@pytest.mark.parametrize('M,N,K', [(7968, 256, 256), (7968, 256, 2048), (333, 256, 256), (100, 128, 64), (50, 64, 64)])
def test_linear_residual_layernorm(M, N, K):
    a = _rnd(M, K, seed=1).to(BF)
    w = _rnd(N, K, scale=K ** -0.5, seed=2).to(BF)
    b = _rnd(N, seed=3)
    res = _rnd(M, N, seed=4).to(BF)
    g = 1 + 0.2 * _rnd(N, seed=5)
    be = 0.2 * _rnd(N, seed=6)
    out = ops.linear(a, w, b, ops.EPI_RESID_LN, resid=res, gamma=g, beta=be)
    ref = F.layer_norm(res.float() + a.float() @ w.float().t() + b, (N,), g, be, 1e-5)
    print(_report(f'linear+resid+ln[{M},{N},{K}]', out, ref, 4e-3))


def test_linear_residual_scale_and_row_mask():
    B, T, N, K = 5, 61, 256, 128
    M = B * T
    a = _rnd(M, K, seed=1).to(BF)
    w = _rnd(N, K, scale=K ** -0.5, seed=2).to(BF)
    b = _rnd(N, seed=3)
    res = _rnd(M, N, seed=4).to(BF)
    lens = torch.tensor([61, 40, 1, 17, 60], dtype=torch.int32, device=DEV)
    out = ops.linear(a, w, b, ops.EPI_RESID, resid=res, alpha=0.5, row_len=lens, row_period=T)
    live = (torch.arange(T, device=DEV)[None] < lens[:, None]).reshape(M, 1)
    ref = res.float() + 0.5 * torch.where(live, a.float() @ w.float().t() + b, torch.zeros((), device=DEV))
    print(_report('linear+resid*0.5+mask', out, ref, 4e-3))


def test_linear_table_epilogue_is_posenc():
    B, T, N, K = 3, 249, 256, 2560
    a = _rnd(B * T, K, seed=1).to(BF)
    w = _rnd(N, K, scale=K ** -0.5, seed=2).to(BF)
    b = _rnd(N, seed=3)
    table = ops.sinusoid_table(T, N, 0, DEV)
    out = ops.linear(a, w, b, ops.EPI_TABLE, alpha=math.sqrt(N), table=table, period=T, out_f32=True)
    ref = (a.float() @ w.float().t() + b) * math.sqrt(N) + table.repeat(B, 1)
    print(_report('linear+posenc', out, ref, 2e-5, 1e-3))


def test_sinusoid_table_matches_torch_cpu_formula():
    for n, d, first in [(249, 256, 0), (497, 256, -248), (61, 32, 0)]:
        t = ops.sinusoid_table(n, d, first, DEV).cpu()
        pos = torch.arange(first, first + n)
        div = torch.exp(torch.arange(0, d, 2, dtype=torch.float32) * -(math.log(10000.0) / d))
        ref = torch.zeros(n, d)
        ref[:, 0::2] = torch.sin(pos.float().unsqueeze(-1) * div)
        ref[:, 1::2] = torch.cos(pos.float().unsqueeze(-1) * div)
        print(_report(f'sinusoid[{n},{d},{first}]', t, ref, 1e-5, 2e-5))


# ------------------------------------------------------------------------------------------------ conv front end
@pytest.mark.parametrize('B,T,Fdim,C1,C2', [(2, 200, 80, 64, 128), (3, 1000, 80, 64, 128), (2, 91, 40, 64, 128),
                                            (1, 77, 83, 64, 64), (2, 64, 20, 128, 256)])
@pytest.mark.parametrize('policy', ['latency', 'throughput'])
def test_conv_subsampling(B, T, Fdim, C1, C2, policy):
    """conv1 + conv2's implicit GEMM.  Under the throughput policy the two shapes with at most 4 row blocks (T 91 and 64)
    take 128-wide tiles where the latency policy takes 64-wide ones."""
    ops.set_tile_policy(policy)
    try:
        _conv_subsampling(B, T, Fdim, C1, C2)
    finally:
        ops.set_tile_policy('latency')


def _conv_subsampling(B, T, Fdim, C1, C2):
    x = _rnd(B, T, Fdim, seed=1)
    w1 = _rnd(C1, 1, 3, 3, scale=0.3, seed=2)
    b1 = _rnd(C1, scale=0.1, seed=3)
    w2 = _rnd(C2, C1, 3, 3, scale=(9 * C1) ** -0.5, seed=4)
    b2 = _rnd(C2, scale=0.1, seed=5)
    T1, F1, T2, F2 = ops.conv_geometry(T, Fdim)
    h1 = ops.conv1_relu(x, w1, b1)
    r1 = torch.relu(F.conv2d(x.unsqueeze(1), w1, b1, stride=2, padding=(0, 1)))          # [B,C1,T1,F1]
    assert r1.shape[2:] == (T1, F1)
    got1 = h1[:, :T1, :F1, :].permute(0, 3, 1, 2)
    print(_report('conv1', got1, r1, 4e-3))
    if 2 * F2 > F1:
        assert float(h1[:, :T1, F1:, :].float().abs().max()) == 0.0     # right frequency padding is zero
    w2p = w2.permute(0, 2, 3, 1).reshape(C2, 9 * C1).to(BF).contiguous()
    h2 = ops.conv2_relu(h1, w2p, b2, B, T, Fdim)
    r1b = torch.zeros(B, C1, T1, F1, device=DEV)
    r1b.copy_(got1.float())
    r2 = torch.relu(F.conv2d(r1b, w2.to(BF).float(), b2, stride=2, padding=(0, 1)))      # [B,C2,T2,F2]
    assert r2.shape[2:] == (T2, F2)
    got2 = h2.view(B, T2, F2, C2).permute(0, 3, 1, 2)
    print(_report('conv2', got2, r2, 4e-3))


# ------------------------------------------------------------------------------------------------ attention
def _attn_ref(q, k, v, B, H, Tq, Tk, kv_len, causal):
    qh = q.float().view(B, Tq, H, 64).transpose(1, 2)
    kh = k.float().view(B, Tk, H, 64).transpose(1, 2)
    vh = v.float().view(B, Tk, H, 64).transpose(1, 2)
    s = qh @ kh.transpose(2, 3) / 8.0
    mask = torch.arange(Tk, device=DEV)[None, :] < kv_len[:, None].long()           # [B,Tk]
    mask = mask[:, None, None, :].expand(B, H, Tq, Tk)
    if causal:
        mask = mask & torch.tril(torch.ones(Tq, Tk, dtype=torch.bool, device=DEV))[None, None]
    s = s.masked_fill(~mask, float('-inf'))
    p = torch.softmax(s, dim=-1)
    return (p @ vh).transpose(1, 2).reshape(B * Tq, H * 64)


@pytest.mark.parametrize('B,H,T,lens', [(2, 4, 249, [249, 200]), (3, 4, 128, [128, 1, 77]), (2, 2, 300, [300, 129]),
                                        (1, 4, 64, [64]), (32, 4, 249, None)])
def test_self_attention_padding_mask(B, H, T, lens):
    d = H * 64
    qkv = _rnd(B * T, 3 * d, seed=1).to(BF)
    if lens is None:
        g = torch.Generator().manual_seed(5)
        lens = torch.randint(150, T + 1, (B,), generator=g).tolist()
        lens[0] = T
    kv_len = torch.tensor(lens, dtype=torch.int32, device=DEV)
    out = ops.attention(qkv, qkv, qkv, B, H, T, T, kv_len=kv_len, q_col0=0, k_col0=d, v_col0=2 * d)
    ref = _attn_ref(qkv[:, :d].contiguous(), qkv[:, d:2 * d].contiguous(), qkv[:, 2 * d:].contiguous(), B, H, T, T,
                    kv_len, False)
    print(_report(f'self-attn[{B},{H},{T}]', out, ref, 6e-3))


@pytest.mark.parametrize('B,H,L', [(3, 4, 30), (2, 4, 130), (1, 4, 1)])
def test_causal_attention(B, H, L):
    d = H * 64
    qkv = _rnd(B * L, 3 * d, seed=2).to(BF)
    out = ops.attention(qkv, qkv, qkv, B, H, L, L, causal=True, q_col0=0, k_col0=d, v_col0=2 * d)
    ref = _attn_ref(qkv[:, :d].contiguous(), qkv[:, d:2 * d].contiguous(), qkv[:, 2 * d:].contiguous(), B, H, L, L,
                    torch.full((B,), L, dtype=torch.int32, device=DEV), True)
    print(_report(f'causal-attn[{B},{H},{L}]', out, ref, 6e-3))


@pytest.mark.parametrize('B,H,Tq,Tk', [(4, 4, 10, 249), (3, 4, 30, 249), (2, 4, 1, 17)])
def test_cross_attention(B, H, Tq, Tk):
    d = H * 64
    q = _rnd(B * Tq, d, seed=3).to(BF)
    kv = _rnd(B * Tk, 2 * d, seed=4).to(BF)
    g = torch.Generator().manual_seed(9)
    kv_len = torch.randint(1, Tk + 1, (B,), generator=g).to(torch.int32).to(DEV)
    out = ops.attention(q, kv, kv, B, H, Tq, Tk, kv_len=kv_len, k_col0=0, v_col0=d)
    ref = _attn_ref(q, kv[:, :d].contiguous(), kv[:, d:].contiguous(), B, H, Tq, Tk, kv_len, False)
    print(_report(f'cross-attn[{B},{H},{Tq},{Tk}]', out, ref, 6e-3))


def test_relpos_bias_and_residual_attention():
    """scores = (q k^T + BD[i, j-i+T-1]) / 8, output added to a residual (attention.py:196-253 without out-proj)."""
    B, H, T = 3, 4, 150
    d = H * 64
    qkv = _rnd(B * T, 3 * d, seed=1).to(BF)
    ld = (2 * T - 1 + 3) // 4 * 4
    bd = _rnd(H, B * T, ld, scale=2.0, seed=2)
    res = _rnd(B * T, d, seed=3).to(BF)
    lens = torch.tensor([150, 90, 129], dtype=torch.int32, device=DEV)
    out = ops.attention(qkv, qkv, qkv, B, H, T, T, kv_len=lens, q_col0=0, k_col0=d, v_col0=2 * d, bd=bd, resid=res)
    qh = qkv[:, :d].float().view(B, T, H, 64).transpose(1, 2)
    kh = qkv[:, d:2 * d].float().view(B, T, H, 64).transpose(1, 2)
    vh = qkv[:, 2 * d:].float().view(B, T, H, 64).transpose(1, 2)
    idx = (torch.arange(T, device=DEV)[None, :] - torch.arange(T, device=DEV)[:, None]) + (T - 1)
    full = bd.view(H, B, T, ld).permute(1, 0, 2, 3)[..., :2 * T - 1]
    band = torch.gather(full, 3, idx.view(1, 1, T, T).expand(B, H, T, T))
    s = (qh @ kh.transpose(2, 3) + band) / 8.0
    mask = (torch.arange(T, device=DEV)[None, :] < lens[:, None].long())[:, None, None, :]
    p = torch.softmax(s.masked_fill(~mask, float('-inf')), -1)
    ref = (p @ vh).transpose(1, 2).reshape(B * T, d) + res.float()
    print(_report('relpos-attn+resid', out, ref, 6e-3))


@pytest.mark.parametrize('B,T,d,k', [(3, 249, 256, 5), (2, 17, 384, 15), (1, 3, 64, 7)])
def test_depthwise_conv_bn_swish(B, T, d, k):
    x = _rnd(B * T, d, seed=1).to(BF)
    w = _rnd(d, 1, k, scale=0.5, seed=2)
    b = _rnd(d, scale=0.2, seed=3)
    mean, var = _rnd(d, scale=0.3, seed=4), 1 + 0.5 * torch.rand(d, device=DEV)
    gam, bet = 1 + 0.2 * _rnd(d, seed=5), 0.2 * _rnd(d, seed=6)
    s = gam / torch.sqrt(var + 1e-5)
    out = ops.dwconv_swish(x, (w[:, 0, :] * s[:, None]).t().contiguous(), ((b - mean) * s + bet).contiguous(), B, T)
    y = F.conv1d(x.float().view(B, T, d).transpose(1, 2), w, b, padding=(k - 1) // 2, groups=d)
    y = F.batch_norm(y, mean, var, gam, bet, False, 0.0, 1e-5)
    ref = (y * torch.sigmoid(y)).transpose(1, 2).reshape(B * T, d)
    print(_report(f'dwconv+bn+swish[{B},{T},{d},{k}]', out, ref, 4e-3))


def test_linear_on_strided_head_views():
    """BD_full[h] = (q+v)_h P_h^T: A and W are 64-column views of wider matrices (row-strided TMA maps)."""
    M, d, R = 500, 256, 497
    ext = _rnd(M, 4 * d, seed=1).to(BF)
    pp = _rnd(R, d, seed=2).to(BF)
    out = torch.empty(M, 500, device=DEV)
    for h in range(4):
        ops.linear(ext[:, d + 64 * h: d + 64 * (h + 1)], pp[:, 64 * h: 64 * (h + 1)], out=out)
        ref = ext[:, d + 64 * h: d + 64 * (h + 1)].float() @ pp[:, 64 * h: 64 * (h + 1)].float().t()
        print(_report(f'head-view gemm h={h}', out[:, :R], ref, 2e-5, 1e-4))


# ------------------------------------------------------------------------------------------------ small SIMT ops
@pytest.mark.parametrize('M,N', [(1000, 256), (33, 384), (7, 1024), (5, 64)])
def test_layernorm_single_and_double(M, N):
    x = _rnd(M, N, scale=3.0, seed=1).to(BF)
    g1, b1 = 1 + 0.3 * _rnd(N, seed=2), 0.3 * _rnd(N, seed=3)
    g2, b2 = 1 + 0.3 * _rnd(N, seed=4), 0.3 * _rnd(N, seed=5)
    out = ops.layernorm(x, g1, b1, out_f32=True)
    ref = F.layer_norm(x.float(), (N,), g1, b1, 1e-5)
    print(_report('layernorm', out, ref, 1e-5, 1e-5))
    out2 = ops.layernorm(x, g1, b1, g2, b2, out_f32=True)
    print(_report('layernorm x2', out2, F.layer_norm(ref, (N,), g2, b2, 1e-5), 1e-5, 1e-5))
    out3 = ops.layernorm(x, g1, b1)
    print(_report('layernorm bf16', out3, ref, 4e-3))


def test_embed_posenc_and_scale_add_table():
    V, d, B, L = 500, 256, 4, 31
    emb = _rnd(V, d, seed=1).to(BF)
    g = torch.Generator().manual_seed(2)
    tok = torch.randint(0, V, (B, L), generator=g).to(DEV)
    table = ops.sinusoid_table(L, d, 0, DEV)
    out = ops.embed_posenc(tok, emb, table, B * L, d, period=L)
    ref = emb.float()[tok.view(-1)] * math.sqrt(d) + table.repeat(B, 1)
    print(_report('embed+posenc', out, ref, 4e-3))
    step = torch.tensor([7, 0, 0, 0], dtype=torch.int32, device=DEV)
    out = ops.embed_posenc(tok[:, 0].contiguous(), emb, table, B, d, step_ptr=step)
    ref = emb.float()[tok[:, 0]] * math.sqrt(d) + table[7]
    print(_report('embed+posenc(step)', out, ref, 4e-3))
    x = _rnd(B * L, d, seed=3)
    out = ops.scale_add_table(x, 16.0, table, L)
    print(_report('scale_add_table', out, x * 16.0 + table.repeat(B, 1), 4e-3))


def test_log_softmax_rows():
    x = _rnd(320, 4240, scale=4.0, seed=1)
    out = ops.log_softmax(x, 4234)
    ref = torch.log_softmax(x[:, :4234], dim=-1)
    print(_report('log_softmax', out, ref, 1e-6, 2e-5))


@pytest.mark.parametrize('rows,V,k,lm', [(320, 4234, 10, False), (7, 100, 5, True), (3, 40, 16, False), (5, 9000, 1, True)])
def test_logsoftmax_topk_fused(rows, V, k, lm):
    ld = (V + 7) // 8 * 8
    x = _rnd(rows, ld, scale=4.0, seed=1)
    lm_lp = torch.log_softmax(_rnd(rows, V, seed=2), -1) if lm else None
    lp = torch.empty(rows, V, device=DEV)
    val, idx = ops.logsoftmax_topk(x, V, k, lm_lp, 0.3, out_logp=lp)
    ref = torch.log_softmax(x[:, :V], -1) + (0.3 * lm_lp if lm else 0)
    print(_report('fused log-probs', lp, ref, 1e-6, 3e-5))
    tv, ti = torch.topk(lp, k, dim=-1)                   # top-k over the kernel's own log-probs must be identical
    assert torch.equal(idx.long(), ti), 'fused top-k ids differ from topk(log_probs)'
    assert torch.equal(val, tv)
    val2, idx2 = ops.logsoftmax_topk(x, V, k, lm_lp, 0.3)          # without materialising log-probs
    assert torch.equal(idx2, idx) and torch.equal(val2, val)


@pytest.mark.parametrize('smoothing', [0.1, 0.0, 1.0])
def test_label_smoothing_cross_entropy_forward_and_grad(smoothing):
    """smoothing 0 / 1: the constant sum_v conf_v log conf_v has 0*log(0) terms, which F.kl_div (xlogy) treats as 0
    (otrans/module/loss.py:43); the loss must stay finite."""
    from oracle import speech_model as om
    rows, V = 93, 4234
    g = torch.Generator().manual_seed(5)
    logits = (torch.randn(rows, 4240, generator=g) * 3).to(DEV)
    tgt = torch.randint(1, V, (rows,), generator=g)
    tgt[::7] = 0                                                   # PAD rows
    loss, dl = ops.ls_cross_entropy(logits, tgt.to(DEV), V, smoothing, want_grad=True)
    x = logits[:, :V].detach().cpu().double().requires_grad_(True)
    ref = om.label_smoothing_loss(x.unsqueeze(0), tgt.unsqueeze(0), smoothing)
    ref.backward()
    assert math.isfinite(float(loss))
    assert abs(float(loss) - float(ref)) < 2e-5 * max(1.0, abs(float(ref))), (float(loss), float(ref))
    print(_report('ls-ce dlogits', dl.cpu(), x.grad.float(), 1e-5, 1e-7))


def test_decode_self_attention_with_ancestry_cache():
    N, H, Lmax, step = 12, 4, 60, 45
    d = H * 64
    qkv = _rnd(N, 3 * d, seed=1).to(BF)
    kc = _rnd(Lmax, N, d, seed=2).to(BF)
    vc = _rnd(Lmax, N, d, seed=3).to(BF)
    g = torch.Generator().manual_seed(4)
    anc = torch.randint(0, N, (2, N, Lmax), generator=g).to(torch.int32).to(DEV)
    ctrl = torch.tensor([step, 0, 0, 0], dtype=torch.int32, device=DEV)
    kc0, vc0 = kc.clone(), vc.clone()
    out = ops.decode_self_attn(qkv, kc, vc, anc, ctrl, N, H, Lmax)
    cur = anc[step & 1].long()                                              # [N, Lmax]
    ks = torch.stack([kc0[s, cur[:, s]] for s in range(step)] + [qkv[:, d:2 * d]], 1).float()   # [N, step+1, d]
    vs = torch.stack([vc0[s, cur[:, s]] for s in range(step)] + [qkv[:, 2 * d:]], 1).float()
    q = qkv[:, :d].float().view(N, H, 1, 64)
    s = (q @ ks.view(N, step + 1, H, 64).transpose(1, 2).transpose(2, 3)) / 8.0
    ref = (torch.softmax(s, -1) @ vs.view(N, step + 1, H, 64).transpose(1, 2)).reshape(N, d)
    print(_report('decode self-attn', out, ref, 6e-3))
    assert torch.equal(kc[step], qkv[:, d:2 * d]) and torch.equal(vc[step], qkv[:, 2 * d:])   # appended to the cache
    assert torch.equal(kc[:step], kc0[:step])


# ------------------------------------------------------------------------------------------------ beam search kernels
def _run_beam_step(case):
    from oracle import beam_search as obs
    beam = case['beam']
    lp = case['log_probs'].to(DEV).contiguous()
    n, v = lp.shape
    st = ops.BeamState(n // beam, beam, 4, DEV)
    st.init()
    st.scores.copy_(case['scores'].view(-1).to(DEV))
    st.flag.copy_(case['flag'].view(-1).to(torch.uint8).to(DEV))
    ktok = torch.zeros(n, beam, dtype=torch.int64, device=DEV)
    offs = torch.zeros(n, dtype=torch.int32, device=DEV)
    st.step(lp, v, dbg_ktok=ktok, dbg_offs=offs)
    trace = []
    p, s, f = obs.beam_step(case['log_probs'], case['preds'], case['scores'], case['flag'], beam, trace=trace)
    tr = trace[0]
    live = ~case['flag'].view(-1)
    assert torch.equal(ktok.cpu()[live], tr['k_tok'][live]), 'per-hypothesis top-k token ids differ'
    assert torch.equal(offs.cpu().long().view(-1, beam), tr['offs']), 'beam^2 top-k offsets differ'
    assert torch.equal(st.par_hist[0].cpu().long(), tr['parent'])
    assert torch.equal(st.tok_hist[0].cpu().long(), tr['tok'])
    assert torch.equal(st.scores.cpu(), s.view(-1)), 'scores must be bit-identical (same fp32 adds)'
    assert torch.equal(st.flag.cpu().bool(), f.view(-1))
    assert int(st.ctrl[0]) == 1
    new_preds = torch.cat((case['preds'].to(DEV).index_select(0, st.par_hist[0].long()),
                           st.tok_hist[0].long().view(-1, 1)), 1)
    assert torch.equal(new_preds.cpu(), p)
    # the fused path (top-k computed by otb_logsoftmax_topk from logits == log-probs up to the constant lse)
    st2 = ops.BeamState(n // beam, beam, 4, DEV)
    st2.init()
    st2.scores.copy_(case['scores'].view(-1).to(DEV))
    st2.flag.copy_(case['flag'].view(-1).to(torch.uint8).to(DEV))
    tv, ti = torch.topk(lp, beam, dim=-1)
    st2.step_topk(tv.contiguous(), ti.to(torch.int32).contiguous())
    assert torch.equal(st2.tok_hist[0], st.tok_hist[0]) and torch.equal(st2.par_hist[0], st.par_hist[0])
    assert torch.equal(st2.scores, st.scores) and torch.equal(st2.flag, st.flag)
    return st


def test_beam_step_matches_reference_golden_cases(golden_dir):
    cases = torch.load(os.path.join(golden_dir, 'beam_step_cases.pt'), weights_only=False)
    for c in cases:
        _run_beam_step(c)
        assert torch.equal(c['new_preds'], c['new_preds'])


@pytest.mark.parametrize('b,beam,v', [(32, 10, 4234), (7, 5, 100), (3, 16, 600), (5, 1, 50), (2, 2, 33)])
def test_beam_step_random_bit_exact(b, beam, v):
    g = torch.Generator().manual_seed(b * 100 + beam)
    n = b * beam
    case = {'beam': beam, 'log_probs': torch.log_softmax(torch.randn(n, v, generator=g) * 2, -1),
            'preds': torch.randint(2, v, (n, 6), generator=g), 'scores': -torch.rand(n, 1, generator=g) * 9,
            'flag': torch.rand(n, 1, generator=g) < 0.25}
    _run_beam_step(case)


def test_beam_multi_step_reconstruct_and_finalize():
    """Several steps on random log-probs: back-pointer reconstruction == cat(preds[parent], tok) chain,
    early-stop bookkeeping and finalisation == oracle.beam_finalize."""
    from oracle import beam_search as obs
    b, beam, v, steps = 4, 3, 23, 7
    g = torch.Generator().manual_seed(3)
    st = ops.BeamState(b, beam, steps, DEV)
    st.init()
    n = b * beam
    preds = torch.full((n, 1), 1, dtype=torch.long)
    scores = torch.tensor([0.0] + [float('-inf')] * (beam - 1)).repeat(b).unsqueeze(1)
    flag = torch.zeros_like(scores, dtype=torch.bool)
    for s in range(steps):
        lp = torch.log_softmax(torch.randn(n, v, generator=g) * 2, -1)
        lp[:, 1] += 1.5                                   # make EOS likely so hypotheses finish
        lp = torch.log_softmax(lp, -1)
        st.step(lp.to(DEV), v)
        preds, scores, flag = obs.beam_step(lp, preds, scores, flag, beam)
        assert torch.equal(st.reconstruct(s + 1).cpu(), preds)
        assert torch.equal(st.scores.cpu(), scores.view(-1))
        if bool(flag.all()):                                  # reference breaks here (speech2text.py:66-67)
            assert int(st.ctrl[1]) == 1
            st.step(lp.to(DEV), v)                            # a step launched after the end must be a no-op
            assert int(st.ctrl[0]) == s + 1 and torch.equal(st.scores.cpu(), scores.view(-1))
            steps = s + 1
            break
        assert int(st.ctrl[1]) == 0
    nb, ns = obs.beam_finalize(preds, scores, beam, 2, 0.6, 5)
    got_p, got_s = st.finalize(0.6, 5, 2)
    assert torch.equal(got_p[:, :, :steps].cpu(), nb)
    torch.testing.assert_close(got_s.cpu(), ns, rtol=1e-6, atol=1e-6)

