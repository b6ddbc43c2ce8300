"""Attention weights on the GPU (otb_attention_probs, csrc/attn_probs.cu, and the modules' return_attn_weights switch).

  * the kernel against a float64 softmax of the same bf16 Q/K (and fp32 band): max abs error 1e-5, rows summing to 1 within
    1e-5, masked and causal entries exactly 0, NaN rows exactly where kv_len is 0, nothing written outside the output;
  * P V in fp32 against otb_attention's context (the attention tolerance, rel-L2 6e-3);
  * every block's map of the modules against the policy='bf16' oracle on the fixture's models (rel-L2 2e-2 on valid rows),
    and the recognizer's maps against model.encoder.forward's;
  * the switch changes no output bit, costs one launch per attention site, and works inside a CUDA graph."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops
    from opentransformer_b200.model import SpeechToText
    from opentransformer_b200.modules import rel_pos_band
    from opentransformer_b200.recognize import SpeechToTextRecognizer
    DEV = torch.device('cuda:0')

from tests.attn_weights_ref import CASES, load_cases, oracle_maps
from tests.test_gpu_model import _rel

BF = torch.bfloat16
REL_L2_MAPS = 2e-2      # the encoder-state tolerance (DESIGN.md section 2)
CANARY = -12345.0


def _probs_ref(q, k, B, H, Tq, Tk, dk, kv_len, causal, q_col0, k_col0, bd=None):
    """float64 softmax(Q K^T (+ BD) / sqrt(dk) + mask) of the bf16 operands -> [B, H, Tq, Tk] on the CPU."""
    qh = q[:, q_col0:q_col0 + H * dk].double().cpu().view(B, Tq, H, dk).transpose(1, 2)
    kh = k[:, k_col0:k_col0 + H * dk].double().cpu().view(B, Tk, H, dk).transpose(1, 2)
    s = qh @ kh.transpose(2, 3)
    if bd is not None:
        idx = torch.arange(Tk)[None, :] - torch.arange(Tq)[:, None] + (Tq - 1)
        full = bd.double().cpu().view(H, B, Tq, bd.shape[-1]).permute(1, 0, 2, 3)
        s = s + torch.gather(full, 3, idx.view(1, 1, Tq, Tk).expand(B, H, Tq, Tk))
    s = s / math.sqrt(dk)
    lens = kv_len.cpu().long() if kv_len is not None else torch.full((B,), Tk)
    mask = (torch.arange(Tk)[None, :] < lens[:, None])[:, None, None, :]
    if causal:
        mask = mask & (torch.arange(Tk)[None, :] <= torch.arange(Tq)[:, None])[None, None]
    return torch.softmax(s.masked_fill(~mask, float('-inf')), -1), mask.expand(B, H, Tq, Tk)


def _canary_out(B, H, Tq, Tk, pad):
    """A [B, H, Tq, Tk] view starting `pad` floats into a canary-filled buffer, with `pad` canary floats after it."""
    n = B * H * Tq * Tk
    buf = torch.full((n + 2 * pad,), CANARY, dtype=torch.float32, device=DEV)
    return buf, buf[pad:pad + n].view(B, H, Tq, Tk)


def _check_probs(got, ref, mask, nan_rows, label):
    got = got.cpu().double()
    assert torch.equal(torch.isnan(got), nan_rows[:, None, None, None].expand_as(got)), f'{label}: NaN rows'
    ok = ~nan_rows
    g, r, m = got[ok], ref[ok], mask[ok]
    err = (g - r).abs().max().item() if g.numel() else 0.0
    row_err = (g.sum(-1) - 1).abs().max().item() if g.numel() else 0.0
    print(f'{label}: max_abs={err:.2e} row_sum_err={row_err:.2e}')
    assert err <= 1e-5 and row_err <= 1e-5, label
    assert torch.all(g[~m] == 0), f'{label}: masked entries must be exactly 0'


def _kv_len(B, Tk):
    lens = [max(1, Tk - (b * Tk) // 3) for b in range(B)]
    return torch.tensor(lens, dtype=torch.int32, device=DEV)


# (mode, d_k, Tq, Tk): self = [M, 3d] QKV with ragged lengths, causal = the decoder's self-attention, cross = a separate q
# and [M, 2d] K|V, relpos = the [M, 4d] [q+u | q+v | k | v] layout with the band and ragged lengths
KERNEL_CASES = ([('self', dk, t, t) for dk in (64, 96) for t in (1, 7, 127, 128, 129, 249, 513)] +
                [('causal', dk, t, t) for dk in (64, 96) for t in (1, 7, 128, 129, 249)] +
                [('relpos', dk, t, t) for dk in (64, 96) for t in (1, 7, 129, 249)] +
                [('cross', dk, tq, tk) for dk in (64, 96) for tq, tk in ((1, 249), (7, 513), (129, 7), (249, 127), (513, 1))])


@pytest.mark.parametrize('mode,dk,Tq,Tk', KERNEL_CASES)
def test_probs_kernel_against_float64(mode, dk, Tq, Tk):
    B, H = 3, 2
    d = H * dk
    g = torch.Generator().manual_seed(Tq * 1000 + Tk + dk)
    rnd = lambda *s: (1.5 * torch.randn(*s, generator=g)).to(BF).to(DEV)     # noqa: E731
    kv_len, causal, bd = None, False, None
    if mode == 'self':
        q = k = rnd(B * Tq, 3 * d)
        q_col0, k_col0, kv_len = 0, d, _kv_len(B, Tk)
    elif mode == 'causal':
        q = k = rnd(B * Tq, 3 * d)
        q_col0, k_col0, causal = 0, d, True
    elif mode == 'cross':
        q, k = rnd(B * Tq, d), rnd(B * Tk, 2 * d)
        q_col0, k_col0, kv_len = 0, 0, _kv_len(B, Tk)
    else:
        q = k = rnd(B * Tq, 4 * d)
        q_col0, k_col0, kv_len = 0, 2 * d, _kv_len(B, Tk)
        pproj = rnd(2 * Tq - 1, d)
        bd = rel_pos_band(q, pproj, H, B, Tq)
    pad = 5 if Tk % 2 else 64          # an output that starts off 16-byte alignment, and one that does not
    buf, out = _canary_out(B, H, Tq, Tk, pad)
    ops.attention_probs(q, k, B, H, Tq, Tk, kv_len=kv_len, causal=causal, q_col0=q_col0, k_col0=k_col0, bd=bd, d_k=dk, out=out)
    torch.cuda.synchronize()
    assert torch.all(buf[:pad] == CANARY) and torch.all(buf[-pad:] == CANARY), 'written outside the output'
    ref, mask = _probs_ref(q, k, B, H, Tq, Tk, dk, kv_len, causal, q_col0, k_col0, bd)
    _check_probs(out, ref, mask, torch.zeros(B, dtype=torch.bool), f'{mode} d_k {dk} Tq {Tq} Tk {Tk}')


@pytest.mark.parametrize('dk', [64, 96])
def test_probs_kernel_nan_rows_where_no_key_is_visible(dk):
    B, H, T = 3, 2, 129
    d = H * dk
    g = torch.Generator().manual_seed(3)
    qkv = torch.randn(B * T, 3 * d, generator=g).to(BF).to(DEV)
    kv_len = torch.tensor([T, 0, 40], dtype=torch.int32, device=DEV)
    out = ops.attention_probs(qkv, qkv, B, H, T, T, kv_len=kv_len, q_col0=0, k_col0=d, d_k=dk)
    ref, mask = _probs_ref(qkv, qkv, B, H, T, T, dk, kv_len, False, 0, d)
    _check_probs(out, ref, mask, torch.tensor([False, True, False]), f'kv_len 0 d_k {dk}')


@pytest.mark.parametrize('dk', [64, 96])
def test_probs_times_v_matches_fused_attention(dk):
    """P V in fp32 is the context otb_attention computes, within the attention tolerance."""
    B, H = 2, 4
    d = H * dk
    g = torch.Generator().manual_seed(11)
    for label, T, causal, lens, relpos in (('self', 249, False, [249, 130], False), ('causal', 129, True, None, False),
                                           ('relpos', 200, False, [200, 77], True)):
        m = torch.randn(B * T, (4 if relpos else 3) * d, generator=g).to(BF).to(DEV)
        kv_len = torch.tensor(lens, dtype=torch.int32, device=DEV) if lens else None
        k0, v0 = (2 * d, 3 * d) if relpos else (d, 2 * d)
        bd = rel_pos_band(m, torch.randn(2 * T - 1, d, generator=g).to(BF).to(DEV), H, B, T) if relpos else None
        ctx = ops.attention(m, m, m, B, H, T, T, kv_len=kv_len, causal=causal, q_col0=0, k_col0=k0, v_col0=v0, bd=bd, d_k=dk)
        p = ops.attention_probs(m, m, B, H, T, T, kv_len=kv_len, causal=causal, q_col0=0, k_col0=k0, bd=bd, d_k=dk)
        v = m[:, v0:v0 + d].float().view(B, T, H, dk).transpose(1, 2)
        pv = (p @ v).transpose(1, 2).reshape(B * T, d)
        r = _rel(ctx, pv)
        print(f'{label} d_k {dk}: P V vs otb_attention rel_l2={r:.3e}')
        assert r < 6e-3, label


# ------------------------------------------------------------------------------------------------ modules
@pytest.fixture(scope='module')
def cases():
    return load_cases()


def _model(c):
    model = SpeechToText(c['params']).eval()
    for part in ('frontend', 'encoder', 'decoder'):
        getattr(model, part).load_state_dict({k[len(part) + 1:]: v for k, v in c['sd'].items() if k.startswith(part + '.')})
    return model.to(DEV)


def _run(model, c, on):
    """encoder.forward and decoder.forward with the switch set to `on` -> (enc out, enc maps, logits, dec maps, launches)."""
    model.encoder.return_attn_weights = model.decoder.return_attn_weights = on
    x, mask = c['x'].to(DEV), c['mask'].to(DEV)
    with torch.no_grad():
        fx, fm = model.frontend(x, mask)
        n0 = ops.COUNTERS['launches']
        y, _, enc_w = model.encoder(fx, fm)
        n_enc = ops.COUNTERS['launches'] - n0
        n0 = ops.COUNTERS['launches']
        logits, dec_w = model.decoder(c['tgt'].to(DEV), c['mem_ref'].to(DEV), c['mm_ref'].to(DEV))
        n_dec = ops.COUNTERS['launches'] - n0
    return y, enc_w, logits, dec_w, (n_enc, n_dec)


@pytest.mark.parametrize('name', CASES)
def test_module_maps_against_bf16_oracle(cases, name):
    c = cases[name]
    model = _model(c)
    _, enc_w, _, dec_w, _ = _run(model, c, True)
    enc_ref, dec_ref = oracle_maps(c, policy='bf16')
    lens = c['mm_ref'].sum(1).tolist()
    worst = 0.0
    for i, want in enumerate(enc_ref):
        got = enc_w['enc_block_%d' % i]['slf_attn_weights'].cpu()
        assert got.shape == want.shape
        for b, n in enumerate(lens):           # valid query rows
            r = _rel(got[b, :, :n], want[b, :, :n])
            worst = max(worst, r)
            assert r < REL_L2_MAPS, (i, b, r)
            assert torch.all(got[b, :, :, n:] == 0)
    for i, (s_ref, x_ref) in enumerate(dec_ref):
        blk = dec_w['dec_block_%d' % i]
        s, x = blk['slf_attn_weights'].cpu(), blk['src_attn_weights'].cpu()
        assert s.shape == s_ref.shape and x.shape == x_ref.shape
        rs, rx = _rel(s, s_ref), _rel(x, x_ref)
        worst = max(worst, rs, rx)
        assert rs < REL_L2_MAPS and rx < REL_L2_MAPS, (i, rs, rx)
        assert torch.all(s.triu(1) == 0)
    print(f'{name}: worst map rel_l2 vs the bf16 oracle {worst:.3e}')


@pytest.mark.parametrize('name', CASES)
def test_switch_changes_no_output_and_adds_one_launch_per_site(cases, name):
    c = cases[name]
    model = _model(c)
    _run(model, c, False)          # the first call builds the cached positional tables: keep their launches out of the counts
    y0, enc0, l0, dec0, (e0, d0) = _run(model, c, False)
    y1, enc1, l1, dec1, (e1, d1) = _run(model, c, True)
    nb_enc, nb_dec = len(model.encoder.blocks), len(model.decoder.blocks)
    assert all(v['slf_attn_weights'] is None for v in enc0.values())
    assert all(v['slf_attn_weights'] is None and v['src_attn_weights'] is None for v in dec0.values())
    assert torch.equal(y0, y1) and torch.equal(l0, l1)
    assert e1 - e0 == nb_enc and d1 - d0 == 2 * nb_dec, (e0, e1, d0, d1)
    # inference without a DecoderCache goes through forward; with one it returns None maps
    model.decoder.return_attn_weights = True
    mem, mm = c['mem_ref'].to(DEV), c['mm_ref'].to(DEV)
    with torch.no_grad():
        _, _, attn = model.decoder.inference(c['tgt'][:, :4].to(DEV), mem, mm)
        assert attn['dec_block_0']['src_attn_weights'].shape[-2] == 4
        cache = model.decoder.init_cache(mem, mm, 4)
        _, _, attn = model.decoder.inference(c['tgt'][:, :1].to(DEV), mem, mm, cache)
        assert attn['dec_block_0']['slf_attn_weights'] is None and attn['dec_block_0']['src_attn_weights'] is None


@pytest.mark.parametrize('name', CASES)
def test_recognizer_fills_attn_weights_from_its_encoder_pass(cases, name):
    c = cases[name]
    model = _model(c)
    x, mask = c['x'].to(DEV), c['mask'].to(DEV)
    kw = dict(beam_width=2, nbest=1, max_len=6, penalty=0.6, lamda=5, ngpu=1)
    rec = SpeechToTextRecognizer(model, **kw)
    ids0, sc0, _ = rec.recognize_ids(x, mask)
    assert rec.attn_weights == {} and rec.encode(x, mask)[3] == {}
    model.encoder.return_attn_weights = True
    ids1, sc1, _ = rec.recognize_ids(x, mask)
    assert torch.equal(ids0, ids1) and torch.equal(sc0, sc1)
    got = rec.attn_weights
    assert set(got) == {'encoder', 'decoder'} and got['decoder'] == []
    with torch.no_grad():
        _, _, want = model.encoder(*model.frontend(x, mask))
        sink = []
        model.encode_bf16(x, mask, attn_sink=sink)
    assert list(got['encoder']) == list(want)
    for i, key in enumerate(want):
        g = got['encoder'][key]['slf_attn_weights']
        assert torch.equal(g, sink[i])
        w = want[key]['slf_attn_weights']
        if model.encoder.fuse_abs_posenc():
            # the recognizer's encoder pass fuses x sqrt(d) + PE into the front end's GEMM epilogue, which rounds its input
            # to bf16 once instead of twice: the same maps up to that rounding
            assert _rel(g, w) < 1e-2
        else:
            assert torch.equal(g, w)
    assert rec.encode(x, mask)[3] is rec.attn_weights['encoder']


def test_maps_in_a_cuda_graph_equal_eager(cases):
    c = cases['conformer']
    model = _model(c)
    model.encoder.return_attn_weights = True
    x, mask = c['x'].to(DEV), c['mask'].to(DEV)
    with torch.no_grad():
        fx, fm = model.frontend(x, mask)
        _, _, eager = model.encoder(fx, fm)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            model.encoder(fx, fm)           # warm-up: packs, positional tables, kernel attributes
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            _, _, captured = model.encoder(fx, fm)
        graph.replay()
        torch.cuda.synchronize()
    for key in eager:
        assert torch.equal(captured[key]['slf_attn_weights'], eager[key]['slf_attn_weights']), key


def test_training_produces_no_maps():
    """FusedTrainer's MWER n-best decode runs the recognizer on the model's encoder: with the switch set it still forms no
    maps, and the switch is left as it was."""
    from opentransformer_b200 import train
    from tests.test_gpu_train import _batch, _build, _params
    model, _ = _build(_params(n_enc=1, n_dec=1))
    model.encoder.return_attn_weights = True
    tr = train.FusedTrainer(model.train(), use_graph=False, mwer_nbest=2, mwer_max_len=8)
    x, mask, tgt = _batch(T=200, lens=(200, 180, 191))
    tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV))
    assert tr._recognizer.attn_weights == {}
    assert model.encoder.return_attn_weights is True
