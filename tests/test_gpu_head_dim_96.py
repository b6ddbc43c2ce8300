"""96-wide attention heads on the GPU (d_model 384 / 4 heads: the shipped Conformer configuration).

Kernels against fp32 torch on bf16-rounded operands (the tolerances of tests/test_gpu_ops.py), then the drop-in modules
against the oracle at the shipped widths: Conformer encoder states, decoder logits, KV-cached decoding, beam search in
lock-step, the whole conformer_baseline model through SpeechToTextRecognizer, and the port on the reference's own d_k = 96
fixture (tests/golden/live_ref_dk96.pt)."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops
    from opentransformer_b200.model import SpeechToText
    from opentransformer_b200.recognize import SpeechToTextRecognizer, BeamDecoder
    DEV = torch.device('cuda:0')

from oracle import beam_search as obs
from oracle import speech_model as om
from tests.test_gpu_ops import _rnd, _report
from tests.test_gpu_model import _batch, _rel, _valid, REL_L2_STATES, REL_L2_LOGITS, MAX_ABS_FRAC
from tests.test_gpu_bench_config import _lockstep
from tests.test_head_dim_96 import CONFORMER_BASELINE, load_case

BF = torch.bfloat16
DK = 96
torch.backends.cuda.matmul.allow_tf32 = False


# ------------------------------------------------------------------------------------------------ attention kernel
def _attn_ref(q, k, v, B, H, Tq, Tk, kv_len, causal, bd=None, resid=None):
    """fp32 softmax(q k^T / sqrt(96) (+ rel-pos band)) v (+ resid) on [B*T, H*96] matrices."""
    qh = q.float().view(B, Tq, H, DK).transpose(1, 2)
    kh = k.float().view(B, Tk, H, DK).transpose(1, 2)
    vh = v.float().view(B, Tk, H, DK).transpose(1, 2)
    s = qh @ kh.transpose(2, 3)
    if bd is not None:
        T = Tq
        idx = (torch.arange(T, device=DEV)[None, :] - torch.arange(T, device=DEV)[:, None]) + (T - 1)
        full = bd.view(H, B, T, bd.shape[-1]).permute(1, 0, 2, 3)[..., :2 * T - 1]
        s = s + torch.gather(full, 3, idx.view(1, 1, T, T).expand(B, H, T, T))
    s = s / DK ** 0.5
    mask = (torch.arange(Tk, device=DEV)[None, :] < kv_len[:, None].long())[:, None, None, :]
    if causal:
        mask = mask & (torch.arange(Tk, device=DEV)[None, :] <= torch.arange(Tq, device=DEV)[:, None])[None, None]
    out = (torch.softmax(s.masked_fill(~mask, float('-inf')), -1) @ vh).transpose(1, 2).reshape(B * Tq, H * DK)
    return out + resid.float() if resid is not None else out


@pytest.mark.parametrize('B,H,T,lens', [(2, 4, 249, [249, 200]), (3, 4, 128, [128, 1, 77]), (2, 2, 300, [300, 129])])
def test_self_attention_96_ragged_lengths(B, H, T, lens):
    d = H * DK
    qkv = _rnd(B * T, 3 * d, seed=1).to(BF)
    kv_len = torch.tensor(lens, dtype=torch.int32, device=DEV)
    out = ops.attention(qkv, qkv, qkv, B, H, T, T, kv_len=kv_len, q_col0=0, k_col0=d, v_col0=2 * d, d_k=DK)
    assert out.shape == (B * T, d)
    ref = _attn_ref(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], B, H, T, T, kv_len, False)
    print(_report(f'self-attn d_k 96 [{B},{H},{T}]', out, ref, 6e-3))


@pytest.mark.parametrize('B,H,L', [(3, 4, 30), (2, 4, 130), (1, 4, 1)])
def test_causal_attention_96(B, H, L):
    d = H * DK
    qkv = _rnd(B * L, 3 * d, seed=2).to(BF)
    out = ops.attention(qkv, qkv, qkv, B, H, L, L, causal=True, q_col0=0, k_col0=d, v_col0=2 * d, d_k=DK)
    ref = _attn_ref(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], B, H, L, L, torch.full((B,), L, dtype=torch.int32, device=DEV), True)
    print(_report(f'causal-attn d_k 96 [{B},{H},{L}]', out, ref, 6e-3))


@pytest.mark.parametrize('B,H,Tq,Tk', [(4, 4, 10, 249), (3, 4, 30, 249), (2, 4, 1, 17)])
def test_cross_attention_96(B, H, Tq, Tk):
    """Tq = 10 is the decode-step cross-attention shape (beam 10 hypotheses of one utterance)."""
    d = H * DK
    q = _rnd(B * Tq, d, seed=3).to(BF)
    kv = _rnd(B * Tk, 2 * d, seed=4).to(BF)
    g = torch.Generator().manual_seed(9)
    kv_len = torch.randint(1, Tk + 1, (B,), generator=g).to(torch.int32).to(DEV)
    out = ops.attention(q, kv, kv, B, H, Tq, Tk, kv_len=kv_len, k_col0=0, v_col0=d, d_k=DK)
    ref = _attn_ref(q, kv[:, :d], kv[:, d:], B, H, Tq, Tk, kv_len, False)
    print(_report(f'cross-attn d_k 96 [{B},{H},{Tq},{Tk}]', out, ref, 6e-3))


def test_relpos_band_and_residual_attention_96():
    """The Conformer's attention: [q+u | q+v | k | v] in one [M, 4d] matrix, rel-pos band, residual, no output projection.
    The last head's V is the right edge of the matrix: the upper 32 columns of its second box are TMA zero-fill."""
    B, H, T = 3, 4, 150
    d = H * DK
    ext = _rnd(B * T, 4 * d, seed=1).to(BF)
    ld = (2 * T - 1 + 3) // 4 * 4
    bd = _rnd(H, B * T, ld, scale=2.0, seed=2)
    res = _rnd(B * T, d, seed=3).to(BF)
    lens = torch.tensor([150, 90, 129], dtype=torch.int32, device=DEV)
    out = ops.attention(ext, ext, ext, B, H, T, T, kv_len=lens, q_col0=0, k_col0=2 * d, v_col0=3 * d, bd=bd, resid=res, d_k=DK)
    ref = _attn_ref(ext[:, :d], ext[:, 2 * d:3 * d], ext[:, 3 * d:], B, H, T, T, lens, False, bd=bd, resid=res)
    print(_report('relpos-attn+resid d_k 96', out, ref, 6e-3))


@pytest.mark.parametrize('width', [3, 4])
def test_last_head_at_the_right_matrix_edge_96(width):
    """Q, K and V of the last head end at the last column of an [M, 3d] / [M, 4d] matrix, and the output is written into a
    wider buffer whose other columns must stay untouched."""
    B, H, T = 2, 4, 77
    d = H * DK
    m = _rnd(B * T, width * d, seed=5).to(BF)
    c0 = (width - 3) * d
    lens = torch.tensor([77, 50], dtype=torch.int32, device=DEV)
    out = torch.full((B * T, d + 64), 7.0, dtype=BF, device=DEV)
    ops.attention(m, m, m, B, H, T, T, kv_len=lens, q_col0=c0, k_col0=c0 + d, v_col0=c0 + 2 * d, out=out, d_k=DK)
    ref = _attn_ref(m[:, c0:c0 + d], m[:, c0 + d:c0 + 2 * d], m[:, c0 + 2 * d:], B, H, T, T, lens, False)
    print(_report(f'right-edge attn d_k 96 [M,{width}d]', out[:, :d], ref, 6e-3))
    assert bool((out[:, d:] == 7.0).all()), 'columns past H*96 were written'


def test_attention_and_decode_entry_points_refuse_other_head_widths():
    qkv = torch.zeros(8, 3 * 320, dtype=BF, device=DEV)
    with pytest.raises(NotImplementedError, match=r'\(64, 96\)'):
        ops.attention(qkv, qkv, qkv, 1, 4, 8, 8, k_col0=320, v_col0=640, d_k=80)
    from opentransformer_b200 import _lib
    lib = _lib.lib()
    st = ops._stream()
    assert lib.otb_attention(ops._p(qkv), qkv.stride(0), 8, ops._p(qkv), qkv.stride(0), 8, ops._p(qkv), qkv.stride(0),
                             ops._p(qkv), qkv.stride(0), 1, 4, 8, 8, None, 0, 0, 320, 640, None, 0, None, 0, None, 80, st) != 0
    assert b'64 or 96' in lib.otb_last_error()
    assert lib.otb_decode_self_attn(ops._p(qkv), ops._p(qkv), ops._p(qkv), ops._p(qkv), ops._p(qkv), None, ops._p(qkv), 1, 4, 8,
                                    80, st) != 0
    assert b'64 or 96' in lib.otb_last_error()
    # the log-sum-exp feeds the 64-wide backward: a 96-wide forward that asks for it is refused (valid operands throughout)
    q96, out96 = torch.zeros(8, 3 * 384, dtype=BF, device=DEV), torch.empty(8, 384, dtype=BF, device=DEV)
    lse = torch.empty(1, 4, 8, device=DEV)
    assert lib.otb_attention(ops._p(q96), q96.stride(0), 8, ops._p(q96), q96.stride(0), 8, ops._p(q96), q96.stride(0),
                             ops._p(out96), out96.stride(0), 1, 4, 8, 8, None, 0, 0, 384, 768, None, 0, None, 0, ops._p(lse), 96,
                             st) != 0
    assert b'd_k = 64' in lib.otb_last_error()


def test_linear_on_96_wide_strided_head_views():
    """The rel-pos band GEMM at d_k 96: K = 96 is not a multiple of the 64-wide k-block, so the second k-block's upper 32
    columns come from TMA zero-fill (the map's width is K) and not from the next head's columns."""
    M, d, R = 500, 384, 497
    ext = _rnd(M, 4 * d, seed=1).to(BF)
    pp = _rnd(R, d, seed=2).to(BF)
    out = torch.empty(M, 500, device=DEV)
    for h in range(4):
        ops.linear(ext[:, d + DK * h: d + DK * (h + 1)], pp[:, DK * h: DK * (h + 1)], out=out)
        ref = ext[:, d + DK * h: d + DK * (h + 1)].float() @ pp[:, DK * h: DK * (h + 1)].float().t()
        print(_report(f'head-view gemm K=96 h={h}', out[:, :R], ref, 2e-5, 1e-4))


# ------------------------------------------------------------------------------------------------ KV-cache decode attention
@pytest.mark.parametrize('step', [0, 1, 63, 127])
def test_decode_self_attention_96_with_shuffled_ancestry(step):
    N, H, Lmax = 12, 4, 128
    d = H * DK
    qkv = _rnd(N, 3 * d, seed=1).to(BF)
    kc = _rnd(Lmax, N, d, seed=2).to(BF)
    vc = _rnd(Lmax, N, d, seed=3).to(BF)
    g = torch.Generator().manual_seed(4)
    anc = torch.stack([torch.stack([torch.randperm(N, generator=g) for _ in range(Lmax)], 1) for _ in range(2)])  # [2, N, Lmax]
    anc = anc.to(torch.int32).to(DEV)
    ctrl = torch.tensor([step, 0, 0, 0], dtype=torch.int32, device=DEV)
    kc0, vc0 = kc.clone(), vc.clone()
    out = ops.decode_self_attn(qkv, kc, vc, anc, ctrl, N, H, Lmax)
    assert out.shape == (N, d)
    cur = anc[step & 1].long()
    ks = torch.stack([kc0[s, cur[:, s]] for s in range(step)] + [qkv[:, d:2 * d]], 1).float()   # [N, step+1, d]
    vs = torch.stack([vc0[s, cur[:, s]] for s in range(step)] + [qkv[:, 2 * d:]], 1).float()
    q = qkv[:, :d].float().view(N, H, 1, DK)
    s = (q @ ks.view(N, step + 1, H, DK).transpose(1, 2).transpose(2, 3)) / DK ** 0.5
    ref = (torch.softmax(s, -1) @ vs.view(N, step + 1, H, DK).transpose(1, 2)).reshape(N, d)
    print(_report(f'decode self-attn d_k 96 step {step}', out, ref, 6e-3))
    assert torch.equal(kc[step], qkv[:, d:2 * d]) and torch.equal(vc[step], qkv[:, 2 * d:])   # appended to the cache
    assert torch.equal(kc[:step], kc0[:step]) and torch.equal(kc[step + 1:], kc0[step + 1:])
    assert torch.equal(vc[:step], vc0[:step]) and torch.equal(vc[step + 1:], vc0[step + 1:])


# ------------------------------------------------------------------------------------------------ modules at the shipped widths
def _conformer_params(n_enc=12, n_dec=6):
    p = copy.deepcopy(CONFORMER_BASELINE)
    p['encoder']['nblocks'] = n_enc
    p['decoder']['n_blocks'] = n_dec
    return p


def _build(params, seed=1234):
    """Random init with perturbed LayerNorm / biases, non-trivial BatchNorm statistics and the decoder EOS bias at -1e4
    (every step of the search runs), as bench.py builds its models."""
    torch.manual_seed(seed)
    model = SpeechToText(params).eval()
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if 'norm' in n:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif n.endswith('.bias'):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
        for n, b in model.named_buffers():
            if n.endswith('running_mean'):
                b.copy_(0.3 * torch.randn(b.shape, generator=g))
            if n.endswith('running_var'):
                b.copy_(1.0 + 0.5 * torch.rand(b.shape, generator=g))
        model.decoder.output_layer.bias[1] = -1e4
    sd = {}
    for part in ('frontend', 'encoder', 'decoder'):
        for k, v in getattr(model, part).state_dict().items():
            sd[f'{part}.{k}'] = v.detach().clone().float() if v.dtype.is_floating_point else v.clone()
    return model.to(DEV), sd


@pytest.mark.parametrize('n_enc,B,T,lens', [(2, 3, 400, [400, 300, 255]), (12, 2, 1000, [1000, 777])])
def test_conformer_encoder_at_shipped_widths_matches_oracle(n_enc, B, T, lens):
    params = _conformer_params(n_enc=n_enc, n_dec=1)
    model, sd = _build(params)
    x, mask = _batch(B, T, 80, lens)
    mem_ref, mmask = om.encode(x, mask, sd, params)
    with torch.no_grad():
        fe, fmask = model.frontend(x.to(DEV), mask.to(DEV))
        mem, _, _ = model.encoder(fe, fmask)
        fused, flens, B2, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
    r1 = _rel(_valid(mem.cpu(), mmask), _valid(mem_ref, mmask))
    r2 = _rel(_valid(fused.float().view(B2, T2, -1).cpu(), mmask), _valid(mem_ref, mmask))
    print(f'conformer d 384 / 4 heads, {n_enc} blocks, {B} x {T} frames: encoder rel_l2 module-API={r1:.3e} fused={r2:.3e}')
    assert flens.cpu().tolist() == mmask.sum(1).tolist()
    assert r1 < REL_L2_STATES and r2 < REL_L2_STATES


@pytest.fixture(scope='module')
def dec_model():
    params = _conformer_params(n_enc=1, n_dec=2)
    model, sd = _build(params)
    x, mask = _batch(3, 300, 80, [300, 211, 250])
    mem_ref, mmask = om.encode(x, mask, sd, params)
    return params, model, sd, x, mask, mem_ref, mmask


def test_decoder_384_teacher_forced_logits_and_cached_seam(dec_model):
    params, model, sd, x, mask, mem_ref, mmask = dec_model
    g = torch.Generator().manual_seed(5)
    tgt = torch.randint(3, 4234, (3, 31), generator=g)
    tgt[:, 0] = 1
    kw = om.decoder_kwargs(params)
    logits_ref = om.transformer_decoder(tgt[:, :-1], mem_ref, mmask, sd, 'decoder.', **kw)
    keep = [i for i in range(4234) if i != 1]            # column 1 (EOS) carries the -1e4 bias
    with torch.no_grad():
        logits, _ = model.decoder(tgt[:, :-1].to(DEV), mem_ref.to(DEV), mmask.to(DEV))
        r = _rel(logits.cpu()[..., keep], logits_ref[..., keep])
        d_abs = float((logits.cpu()[..., keep] - logits_ref[..., keep]).abs().max())
        lim = MAX_ABS_FRAC * float(logits_ref[..., keep].abs().max())
        print(f'decoder d 384 teacher-forced logits rel_l2={r:.3e} max_abs={d_abs:.3e} (limit {lim:.3e})')
        assert r < REL_L2_LOGITS and d_abs <= lim
        # KV cache through the reference seam (one token per call, every row continues itself) vs full-prefix recompute
        dc = model.decoder.init_cache(mem_ref.to(DEV), mmask.to(DEV), 12)
        worst = 0.0
        for s in range(12):
            lp, dc, _ = model.decoder.inference(tgt[:, :s + 1].to(DEV), mem_ref.to(DEV), mmask.to(DEV), dc)
            dc.advance_without_reorder()
            lp_ref = om.decoder_inference(tgt[:, :s + 1], mem_ref, mmask, sd, 'decoder.', **kw)
            rr = _rel(lp.cpu()[:, keep], lp_ref[:, keep])
            worst = max(worst, rr)
            assert rr < REL_L2_LOGITS, (s, rr)
            assert float((lp.cpu()[:, keep] - lp_ref[:, keep]).abs().max()) <= MAX_ABS_FRAC * float(lp_ref[:, keep].abs().max())
        print(f'decoder d 384 KV-cached log-probs vs oracle full-prefix recompute over 12 steps: worst rel_l2={worst:.3e}')


def test_decoder_384_beam_search_lockstep(dec_model):
    """Beam 10 for 24 steps on the graph path: the oracle's beam_step is fed the CUDA decoder's log-probs; ids, parents and
    fp32 scores must be bit-exact at every step, the KV-cached log-probs must match the oracle's full-prefix recompute."""
    params, model, sd, x, mask, _, _ = dec_model
    B, beam, max_len = 3, 10, 24
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
        bd = BeamDecoder(model.decoder, B, beam, T2, max_len, DEV, use_graph=True, keep_logp=True)
        assert not bd.persistent, 'd_model 384 takes the per-step graph path'
        bd.setup(mem, lens)
        preds, scores, flag, steps, worst, worst_rel, scale = _lockstep(bd, model, sd, params, mem, lens, B, beam, max_len, T2,
                                                                        bd.step, check_every=3)
        assert bd.graph is not None
    print(f'decoder d 384, beam {beam}: {steps} steps bit-exact (ids, parents, scores); cached log-probs vs oracle '
          f'rel_l2<={worst_rel:.3e} max_abs={worst:.3e} (|ref|_inf {scale:.3e})')
    assert steps == max_len
    assert worst_rel < REL_L2_LOGITS and worst < MAX_ABS_FRAC * scale


def test_conformer_baseline_whole_model_recognize_matches_bf16_oracle():
    """The full conformer_baseline model (12 Conformer blocks, 6 decoder blocks, d 384, 4 heads), 4 x 1000 frames, beam 10:
    every 1-best of SpeechToTextRecognizer.recognize_ids equals oracle.recognize(policy='bf16')."""
    params = _conformer_params()
    model, sd = _build(params)
    lens = [1000, 873, 640, 999]
    beam, max_len = 10, 30
    x, mask = _batch(4, 1000, 80, lens)
    nb_ref, ns_ref, _, _ = obs.recognize(x, mask, sd, params, beam=beam, nbest=beam, max_len=max_len, penalty=0.6, lamda=5,
                                         policy='bf16')
    rec = SpeechToTextRecognizer(model, beam_width=beam, nbest=beam, max_len=max_len, penalty=0.6, lamda=5, ngpu=1)
    p, s, n = rec.recognize_ids(x.to(DEV), mask.to(DEV))
    assert not next(iter(rec._decoders.values())).persistent
    best_same = sum(int(torch.equal(p[b, 0].cpu(), nb_ref[b, 0])) for b in range(4))
    print(f'conformer_baseline recognize: 1-best identical to the bf16-policy oracle for {best_same}/4 utterances; '
          f'scores gpu {s[:, 0].tolist()} oracle {ns_ref[:, 0].tolist()}')
    assert n == max_len
    assert best_same == 4
    torch.testing.assert_close(s[:, 0].cpu(), ns_ref[:, 0], rtol=3e-2, atol=0.3)


def test_live_reference_dk96_fixture_on_gpu():
    """The port on the reference's own d_k = 96 model: encoder states within rel-L2 2e-2; recognize ids reported."""
    c = load_case('dk96')
    params, sd, x, mask, beam, max_len = c['params'], c['sd'], c['x'], c['mask'], c['beam'], c['max_len']
    model = SpeechToText(params).eval()
    for part in ('frontend', 'encoder', 'decoder'):
        m = getattr(model, part)
        m.load_state_dict({k[len(part) + 1:]: v for k, v in sd.items() if k.startswith(part + '.')})
    model = model.to(DEV)
    with torch.no_grad():
        mem, lens, B, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
    mm = c['mm_ref']
    assert lens.cpu().tolist() == mm.sum(1).tolist()
    r = _rel(_valid(mem.float().view(B, T2, -1).cpu(), mm), _valid(c['mem_ref'], mm))
    rec = SpeechToTextRecognizer(model, beam_width=beam, nbest=beam, max_len=max_len, penalty=0.6, lamda=5, ngpu=1)
    p, s, n = rec.recognize_ids(x.to(DEV), mask.to(DEV))
    same = 0
    for b in range(B):
        port = [int(t) for t in p[b, 0].tolist()]
        port = port[:port.index(1)] if 1 in port else port
        want = [int(t) for t in c['hyps'][b][0].split()] if c['hyps'][b][0] else []
        same += int(port == want)
        print(f'utterance {b}: port 1-best {port} reference {want}')
    print(f'live reference d_k 96: encoder rel_l2={r:.3e}; 1-best identical for {same}/{B} utterances')
    assert r < REL_L2_STATES
