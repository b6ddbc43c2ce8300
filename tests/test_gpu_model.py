"""End-to-end GPU parity of the drop-in modules against the oracle (fp32 reference restatement):
encoder states and decoder logits within the stated tolerance, beam-search integer decisions
bit-exact when driven by the same log-probs, KV-cached decoding == full-prefix recompute."""
import copy
import os

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

# stated tolerances (bf16 operands / activations, fp32 accumulate) -- SURVEY.md 8c
REL_L2_STATES = 2e-2
REL_L2_LOGITS = 2e-2
MAX_ABS_FRAC = 5e-2      # max-abs error <= 5e-2 * ||ref||_inf  (random-init tied embeddings give |logit| ~ 60)


def _params(n_enc=3, n_dec=2, F=80):
    return {'type': 'speech2text', 'frontend_type': 'conv', 'encoder_type': 'transformer',
            'decoder_type': 'transformer',
            'frontend': dict(input_size=F, output_size=256, in_channel=1, mid_channel=64, out_channel=128,
                             kernel_size=[[3, 3], [3, 3]], stride=[2, 2], dropout=0.0, act_func_type='relu',
                             front_end_layer_norm=False),
            'encoder': dict(d_model=256, n_heads=4, d_ff=2048, n_blocks=n_enc, pos_dropout=0.0,
                            slf_attn_dropout=0.0, ffn_dropout=0.0, residual_dropout=0.1, normalize_before=False,
                            concat_after=False, activation='glu', relative_positional=False),
            'decoder': dict(vocab_size=4234, d_model=256, n_heads=4, d_ff=2048, memory_dim=256, n_blocks=n_dec,
                            pos_dropout=0.0, slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0,
                            residual_dropout=0.1, activation='glu', normalize_before=False, concat_after=False,
                            share_embedding=True),
            'ctc_weight': 0.0, 'smoothing': 0.1}


def _build(params, seed=1234):
    torch.manual_seed(seed)
    model = SpeechToText(params).eval()
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if 'norm' in n:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif n.endswith('.bias'):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
        model.decoder.output_layer.bias[1] = -1e4          # SURVEY.md 8(d) config 3: keep all steps alive
    sd = {}
    for part in ('frontend', 'encoder', 'decoder'):
        for k, v in getattr(model, part).state_dict().items():
            sd[f'{part}.{k}'] = v.detach().clone().float()
    return model.to(DEV), sd


def _batch(B, T, F, lens, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, F, generator=g)
    lens = torch.tensor(lens)
    mask = torch.arange(T)[None] < lens[:, None]
    return x * mask.unsqueeze(2), mask


def _rel(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))


def _valid(x, mask):
    return x[mask]


@pytest.mark.parametrize('pre_norm,act', [(False, 'glu'), (True, 'relu')])
def test_frontend_encoder_states_match_oracle(pre_norm, act):
    params = _params()
    params['encoder'].update(normalize_before=pre_norm, activation=act)
    model, sd = _build(params)
    x, mask = _batch(4, 400, 80, [400, 333, 250, 399])
    mem_ref, mmask, fe_ref, layers = om.encode(x, mask, sd, params, return_layers=True)
    with torch.no_grad():
        fe, fmask = model.frontend(x.to(DEV), mask.to(DEV))
        assert torch.equal(fmask.cpu(), mmask)
        r_fe = _rel(fe.cpu(), fe_ref)
        mem, _, attn = model.encoder(fe, fmask)
        mem_fused, lens, B, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
    r_mem = _rel(_valid(mem.cpu(), mmask), _valid(mem_ref, mmask))
    r_fused = _rel(_valid(mem_fused.float().view(B, T2, -1).cpu(), mmask), _valid(mem_ref, mmask))
    print(f'frontend rel_l2={r_fe:.3e}  encoder(module API) rel_l2={r_mem:.3e}  fused rel_l2={r_fused:.3e}')
    assert r_fe < REL_L2_STATES and r_mem < REL_L2_STATES and r_fused < REL_L2_STATES
    assert lens.cpu().tolist() == mmask.sum(1).tolist()
    assert set(attn) == {f'enc_block_{i}' for i in range(3)}


def test_transformer_encoder_relative_positional_matches_oracle():
    """TransformerEncoder(relative_positional=True) (encoder/transformer.py:23-24,46,116-119): Transformer-XL style
    attention without output projection inside the post-norm layer; the oracle path is pinned to the reference by
    tests/golden/small_transformer_relpos.pt."""
    params = _params(n_enc=2, n_dec=1)
    params['encoder'].update(relative_positional=True)
    model, sd = _build(params)
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if n.endswith('posu') or n.endswith('posv'):
                p.copy_(0.3 * torch.randn(p.shape, generator=g))
    sd = {}
    for part in ('frontend', 'encoder', 'decoder'):
        for k, v in getattr(model, part).state_dict().items():
            sd[f'{part}.{k}'] = v.detach().clone().float().cpu()
    x, mask = _batch(3, 400, 80, [400, 300, 255])
    mem_ref, mmask = om.encode(x, mask, sd, params)
    with torch.no_grad():
        fe, fmask = model.frontend(x.to(DEV), mask.to(DEV))
        mem, _, _ = model.encoder(fe, fmask)
        fused, lens, B, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
    r1 = _rel(_valid(mem.cpu(), mmask), _valid(mem_ref, mmask))
    r2 = _rel(_valid(fused.float().view(B, T2, -1).cpu(), mmask), _valid(mem_ref, mmask))
    print(f'rel-pos TransformerEncoder rel_l2 module-API={r1:.3e} fused={r2:.3e}')
    assert r1 < REL_L2_STATES and r2 < REL_L2_STATES


def _conformer_params(n_enc=2, relpos=True):
    p = _params(n_enc=1, n_dec=1)
    p['encoder_type'] = 'conformer'
    p['frontend'].update(mid_channel=64, out_channel=128)
    p['encoder'] = dict(d_model=256, d_ff=768, cov_kernel_size=5, n_heads=4, nblocks=n_enc, pos_dropout=0.0,
                        slf_attn_dropout=0.0, ffn_dropout=0.0, residual_dropout=0.0, conv_dropout=0.0,
                        macaron_style=True, ffn_scale=0.5, conv_bias=True, activation='glu',
                        positional_encoding=True, relative_positional=relpos)
    return p


@pytest.mark.parametrize('relpos', [True, False])
def test_conformer_encoder_states_match_oracle(relpos):
    params = _conformer_params(relpos=relpos)
    model, sd = _build(params)
    g = torch.Generator().manual_seed(11)
    with torch.no_grad():                      # non-trivial BatchNorm running statistics
        for n, b in model.named_buffers():
            if n.endswith('running_mean'):
                b.copy_(0.3 * torch.randn(b.shape, generator=g))
            if n.endswith('running_var'):
                b.copy_(1.0 + 0.5 * torch.rand(b.shape, generator=g))
    sd = {}
    for part in ('frontend', 'encoder', 'decoder'):
        for k, v in getattr(model, part).state_dict().items():
            sd[f'{part}.{k}'] = v.detach().clone().float().cpu() if v.dtype.is_floating_point else v.cpu()
    x, mask = _batch(3, 400, 80, [400, 300, 255])
    mem_ref, mmask, fe_ref, layers = om.encode(x, mask, sd, params, return_layers=True)
    with torch.no_grad():
        fe, fmask = model.frontend(x.to(DEV), mask.to(DEV))
        mem, _, _ = model.encoder(fe, fmask)
        fused, lens, B, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
    r1 = _rel(_valid(mem.cpu(), mmask), _valid(mem_ref, mmask))
    r2 = _rel(_valid(fused.float().view(B, T2, -1).cpu(), mmask), _valid(mem_ref, mmask))
    print(f'conformer(relpos={relpos}) encoder rel_l2 module-API={r1:.3e} fused={r2:.3e}')
    assert r1 < REL_L2_STATES and r2 < REL_L2_STATES


def test_decoder_logits_match_oracle_teacher_forced():
    _decoder_logits_vs_oracle(False, 'glu')


def test_decoder_logits_match_oracle_teacher_forced_prenorm_relu():
    _decoder_logits_vs_oracle(True, 'relu')


def _decoder_logits_vs_oracle(normalize_before, activation):
    params = _params(n_enc=1, n_dec=3)
    params['decoder'].update(normalize_before=normalize_before, activation=activation)
    model, sd = _build(params)
    x, mask = _batch(3, 300, 80, [300, 211, 250])
    mem_ref, mmask = om.encode(x, mask, sd, params)
    g = torch.Generator().manual_seed(5)
    tgt = torch.randint(3, 4234, (3, 31), generator=g)
    tgt[:, 0] = 1
    kw = om.decoder_kwargs(params)
    logits_ref = om.transformer_decoder(tgt[:, :-1], mem_ref, mmask, sd, 'decoder.', **kw)
    with torch.no_grad():
        logits, _ = model.decoder(tgt[:, :-1].to(DEV), mem_ref.to(DEV), mmask.to(DEV))
        lp, _, _ = model.decoder.inference(tgt[:, :7].to(DEV), mem_ref.to(DEV), mmask.to(DEV), None)
        full = model.forward_logits(x.to(DEV), mask.to(DEV), tgt[:, :-1].to(DEV))
    r = _rel(logits.cpu(), logits_ref)
    lp_ref = om.decoder_inference(tgt[:, :7], mem_ref, mmask, sd, 'decoder.', **kw)
    keep = [i for i in range(4234) if i != 1]            # column 1 (EOS) carries the -1e4 bias
    d_lp = float((lp.cpu()[:, keep] - lp_ref[:, keep]).abs().max())
    lim = MAX_ABS_FRAC * float(lp_ref[:, keep].abs().max())
    r_lp = _rel(lp.cpu()[:, keep], lp_ref[:, keep])
    r_full = _rel(full.cpu(), logits_ref)
    print(f'decoder logits rel_l2={r:.3e}  inference log_probs rel_l2={r_lp:.3e} max_abs={d_lp:.3e} (limit {lim:.3e})'
          f'  enc+dec rel_l2={r_full:.3e}')
    assert r < REL_L2_LOGITS and r_full < REL_L2_LOGITS and r_lp < REL_L2_LOGITS and d_lp < lim


def test_model_forward_loss_matches_oracle():
    params = _params(n_enc=1, n_dec=2)
    model, sd = _build(params)
    x, mask = _batch(3, 200, 80, [200, 160, 181])
    g = torch.Generator().manual_seed(9)
    tgt = torch.randint(3, 4234, (3, 12), generator=g)
    tgt[:, 0] = 1
    tgt[0, 9:] = torch.tensor([1, 0, 0])
    tgt[1, 11] = 1
    tgt[2, 6:] = torch.tensor([1, 0, 0, 0, 0, 0])
    loss_ref, _ = om.model_forward_loss(x, mask, tgt, sd, params)
    with torch.no_grad():
        loss, aux = model({'inputs': x.to(DEV), 'mask': mask.to(DEV)}, {'targets': tgt.to(DEV), 'targets_length': None})
    print(f'label-smoothed CE: gpu {float(loss):.5f} oracle {float(loss_ref):.5f}')
    assert aux is None and abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))


def test_beam_search_lockstep_with_oracle():
    _beam_search_lockstep(False, 'glu')


def test_beam_search_lockstep_with_oracle_prenorm_relu():
    _beam_search_lockstep(True, 'relu')


def _beam_search_lockstep(normalize_before, activation):
    """Drive the oracle's beam_step with the CUDA decoder's log-probs: every integer decision of every
    step must be bit-exact, and the KV-cached log-probs must equal the oracle's full-prefix recompute."""
    params = _params(n_enc=1, n_dec=2)
    params['decoder'].update(normalize_before=normalize_before, activation=activation)
    model, sd = _build(params)
    B, beam, max_len = 3, 4, 9
    x, mask = _batch(B, 200, 80, [200, 150, 173])
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
        bd = BeamDecoder(model.decoder, B, beam, T2, max_len, DEV, use_graph=False)
        bd.setup(mem, lens)
        memory = mem.float().view(B, T2, -1).cpu()
        mmask = torch.arange(T2)[None] < lens.cpu()[:, None]
        bm = memory.unsqueeze(1).repeat(1, beam, 1, 1).view(B * beam, T2, -1)
        bmask = mmask.unsqueeze(1).repeat(1, beam, 1).view(B * beam, T2)
        preds = torch.full((B * beam, 1), 1, dtype=torch.long)
        scores = torch.tensor([0.0] + [float('-inf')] * (beam - 1)).repeat(B).unsqueeze(1)
        flag = torch.zeros_like(scores, dtype=torch.bool)
        kw = om.decoder_kwargs(params)
        worst, worst_rel, scale = 0.0, 0.0, 0.0
        for s in range(max_len):
            bd.step()
            lp_gpu = bd.logp.cpu()
            lp_ref = om.decoder_inference(preds, bm, bmask, sd, 'decoder.', **kw)
            alive = ~flag.view(-1)
            worst = max(worst, float((lp_gpu[alive][:, 2:] - lp_ref[alive][:, 2:]).abs().max()))
            worst_rel = max(worst_rel, _rel(lp_gpu[alive][:, 2:], lp_ref[alive][:, 2:]))
            scale = max(scale, float(lp_ref[alive][:, 2:].abs().max()))
            preds, scores, flag = obs.beam_step(lp_gpu, preds, scores, flag, beam)
            assert torch.equal(bd.state.reconstruct(s + 1).cpu(), preds), f'token/parent ids differ at step {s}'
            assert torch.equal(bd.state.scores.cpu(), scores.view(-1)), f'scores differ at step {s}'
        print(f'cached-decoder log-probs vs oracle full recompute: rel_l2<={worst_rel:.3e} max_abs={worst:.3e} '
              f'(|ref|_inf {scale:.3e}) over {max_len} steps')
        assert worst_rel < REL_L2_LOGITS and worst < MAX_ABS_FRAC * scale
        nb, ns = obs.beam_finalize(preds, scores, beam, 2, 0.6, 5)
        gp, gs = bd.state.finalize(0.6, 5, 2)
        assert torch.equal(gp[:, :, :max_len].cpu(), nb)
        torch.testing.assert_close(gs.cpu(), ns, rtol=1e-5, atol=1e-5)


def test_transformer_lm_and_shallow_fusion_lockstep():
    """LM log-probs vs the oracle; beam search with lm_weight: every integer decision bit-exact when the oracle's
    beam_step is fed the CUDA decoder AND CUDA LM log-probs (speech2text.py:102-105)."""
    from opentransformer_b200.lm import TransformerLanguageModel
    lm_params = dict(vocab_size=4234, num_blocks=2, d_model=256, n_heads=4, d_ff=1024, residual_dropout=0.0,
                     smoothing=0.1, share_embedding=True)
    torch.manual_seed(77)
    lm = TransformerLanguageModel(lm_params).eval()
    lm_sd = {'lm.' + k: v.detach().clone().float() for k, v in lm.state_dict().items()}
    lm = lm.to(DEV)
    g = torch.Generator().manual_seed(3)
    toks = torch.randint(2, 4234, (5, 9), generator=g)
    toks[:, 0] = 1
    ref = om.transformer_lm_log_probs(toks, lm_sd, 'lm.', 2, 4, last_frame=False)
    got = lm.predict(toks.to(DEV), last_frame=False).cpu()
    r = _rel(got, ref)
    print(f'transformer LM log-probs rel_l2={r:.3e}')
    assert r < REL_L2_LOGITS
    assert lm.predict(toks.to(DEV), last_frame=True).shape == (5, 1, 4234)

    params = _params(n_enc=1, n_dec=2)
    model, sd = _build(params)
    B, beam, max_len, lmw = 2, 3, 6, 0.3
    x, mask = _batch(B, 160, 80, [160, 131])
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
        bd = BeamDecoder(model.decoder, B, beam, T2, max_len, DEV, use_graph=False)
        bd.setup(mem, lens)
        bd.lm_weight = lmw
        preds = torch.full((B * beam, 1), 1, dtype=torch.long)
        scores = torch.tensor([0.0] + [float('-inf')] * (beam - 1)).repeat(B).unsqueeze(1)
        flag = torch.zeros_like(scores, dtype=torch.bool)
        for s in range(max_len):
            bd.lm_logp = lm.predict(bd.state.reconstruct(s), last_frame=True).squeeze(1).contiguous()
            lm_cpu = bd.lm_logp.cpu()
            bd._step_kernels()
            # bd.logp holds log_softmax(logits) + lmw * lm (the fused kernel materialises it in eager mode)
            dec_lp = bd.logp.cpu() - lmw * lm_cpu
            preds, scores, flag = obs.beam_step(dec_lp, preds, scores, flag, beam, lm_log_probs=lm_cpu, lm_weight=lmw)
            assert torch.equal(bd.state.reconstruct(s + 1).cpu(), preds), f'fusion: ids differ at step {s}'
    rec = SpeechToTextRecognizer(model, lm=lm, lm_weight=lmw, beam_width=beam, nbest=1, max_len=max_len, penalty=0.6,
                                 lamda=5, ngpu=1)
    ids, sc, n = rec.recognize_ids(x.to(DEV), mask.to(DEV))
    assert ids.shape == (B, 1, n)


def test_recognizer_graph_replay_equals_eager_and_decode_step_seam():
    params = _params(n_enc=1, n_dec=2)
    model, sd = _build(params)
    B, beam, max_len = 4, 5, 10
    x, mask = _batch(B, 240, 80, [240, 200, 111, 239])
    xd, md = x.to(DEV), mask.to(DEV)
    rec_g = SpeechToTextRecognizer(model, beam_width=beam, nbest=2, max_len=max_len, penalty=0.6, lamda=5, ngpu=1,
                                   persistent=False)
    rec_e = SpeechToTextRecognizer(model, beam_width=beam, nbest=2, max_len=max_len, penalty=0.6, lamda=5, ngpu=1,
                                   use_graph=False, persistent=False)
    p1, s1, n1 = rec_e.recognize_ids(xd, md)
    p2, s2, n2 = rec_g.recognize_ids(xd, md)
    p3, s3, n3 = rec_g.recognize_ids(xd, md)              # second call re-uses the captured graph
    assert n1 == n2 == n3 == max_len
    assert torch.equal(p1, p2) and torch.equal(p2, p3) and torch.equal(s1, s2) and torch.equal(s2, s3)
    out, scores = rec_g.recognize(xd, md)
    assert torch.equal(out, p2)
    # reference-style seam: decode_step on caller-owned tensors (full-prefix recompute + beam kernel)
    memory, mmask, _, _ = rec_g.encode(xd, md)
    bm = memory.unsqueeze(1).repeat(1, beam, 1, 1).view(B * beam, memory.shape[1], -1)
    bmask = mmask.unsqueeze(1).repeat(1, beam, 1).view(B * beam, -1)
    preds = torch.ones(B * beam, 1, dtype=torch.long, device=DEV)
    scores = torch.tensor([0.0] + [float('-inf')] * (beam - 1), device=DEV).repeat(B).unsqueeze(1)
    flag = torch.zeros_like(scores, dtype=torch.bool)
    with torch.no_grad():
        for _ in range(3):
            preds, _, scores, flag = rec_g.decode_step(preds, bm, bmask, {'decoder': None}, scores, flag)
    assert preds.shape == (B * beam, 4) and scores.shape == (B * beam, 1)
    # 1-best of the seam path (full recompute) and of the cached fast path agree on the first 3 tokens' scores
    print('seam-path scores', scores.view(B, beam)[:, 0].tolist())


def _lockstep_persistent(model, sd, params, x, mask, B, beam, max_len, check_logp=True):
    """Run the persistent cluster kernel for the whole loop with the parity traces on, then drive the oracle's
    beam_step with ITS log-probs step by step: ids / parents / scores must be bit-exact at every step."""
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
        bd = BeamDecoder(model.decoder, B, beam, T2, max_len, DEV, use_graph=False, persistent=True)
        assert bd.persistent, 'persistent decode kernel should support this configuration'
        bd.setup(mem, lens)
        V = model.decoder.vocab_size
        dbg_logp = torch.zeros(max_len, B * beam, V, dtype=torch.float32, device=DEV)
        dbg_scores = torch.zeros(max_len, B * beam, dtype=torch.float32, device=DEV)
        bd.run_persistent(max_len, dbg_logp, dbg_scores)
        torch.cuda.synchronize()
        steps_gpu = int(bd.state.ctrl[0].item())
        memory = mem.float().view(B, T2, -1).cpu()
        mmask = torch.arange(T2)[None] < lens.cpu()[:, None]
        bm = memory.unsqueeze(1).repeat(1, beam, 1, 1).view(B * beam, T2, -1)
        bmask = mmask.unsqueeze(1).repeat(1, beam, 1).view(B * beam, T2)
        preds = torch.full((B * beam, 1), 1, dtype=torch.long)
        scores = torch.tensor([0.0] + [float('-inf')] * (beam - 1)).repeat(B).unsqueeze(1)
        flag = torch.zeros_like(scores, dtype=torch.bool)
        kw = om.decoder_kwargs(params)
        worst, worst_rel, scale, steps_ref = 0.0, 0.0, 1e-9, max_len
        for s in range(max_len):
            lp_gpu = dbg_logp[s].cpu()
            utt_alive = (~flag.view(B, beam)).any(dim=1).repeat_interleave(beam)    # the kernel stops computing ended utterances
            alive = (~flag.view(-1)) & utt_alive
            if check_logp and bool(alive.any()):
                lp_ref = om.decoder_inference(preds, bm, bmask, sd, 'decoder.', **kw)
                worst = max(worst, float((lp_gpu[alive][:, 2:] - lp_ref[alive][:, 2:]).abs().max()))
                worst_rel = max(worst_rel, _rel(lp_gpu[alive][:, 2:], lp_ref[alive][:, 2:]))
                scale = max(scale, float(lp_ref[alive][:, 2:].abs().max()))
            preds, scores, flag = obs.beam_step(lp_gpu, preds, scores, flag, beam)
            assert torch.equal(bd.state.reconstruct(s + 1).cpu(), preds), f'token/parent ids differ at step {s}'
            assert torch.equal(dbg_scores[s].cpu(), scores.view(-1)), f'scores differ at step {s}'
            if bool(flag.all()):
                steps_ref = s + 1
                break
        assert steps_gpu == steps_ref, f'executed step count: kernel {steps_gpu} vs reference loop {steps_ref}'
        assert torch.equal(bd.state.scores.cpu(), scores.view(-1))
        nb, ns = obs.beam_finalize(preds, scores, beam, min(2, beam), 0.6, 5)
        gp, gs = bd.state.finalize(0.6, 5, min(2, beam))
        assert torch.equal(gp[:, :, :steps_ref].cpu(), nb)
        torch.testing.assert_close(gs.cpu(), ns, rtol=1e-6, atol=1e-6)
    return worst, worst_rel, scale, steps_ref


@pytest.mark.parametrize('B,beam,max_len,lens', [(3, 4, 9, [200, 150, 173]), (2, 10, 12, [240, 201]), (5, 1, 6, [160, 160, 120, 99, 140]),
                                                 (1, 16, 5, [170])])
def test_persistent_decode_lockstep_with_oracle(B, beam, max_len, lens):
    params = _params(n_enc=1, n_dec=2)
    model, sd = _build(params)
    x, mask = _batch(B, max(lens), 80, lens)
    worst, worst_rel, scale, steps = _lockstep_persistent(model, sd, params, x, mask, B, beam, max_len)
    print(f'persistent decode (B={B}, beam={beam}): log-probs vs oracle full recompute rel_l2<={worst_rel:.3e} '
          f'max_abs={worst:.3e} (|ref|_inf {scale:.3e}) over {steps} steps; ids / parents / scores bit-exact')
    assert steps == max_len
    assert worst_rel < REL_L2_LOGITS and worst < MAX_ABS_FRAC * scale


def test_persistent_decode_early_end_and_finished_masking():
    """Natural EOS (no -1e4 bias): hypotheses finish at different steps, utterances end at different steps; the kernel's
    history / step count must equal the reference loop's (finished masking, speech2text.py:156-192, early break :66-67).
    (Whether the search ends before max_len depends on the weights: tests/test_gpu_bench_config.py holds the calibrated
    cases that do.)"""
    params = _params(n_enc=1, n_dec=2)
    model, sd = _build(params)
    with torch.no_grad():
        model.decoder.output_layer.bias[1] = 2.0           # EOS likely but not certain
    sd['decoder.output_layer.bias'] = model.decoder.output_layer.bias.detach().float().cpu().clone()
    B, beam, max_len = 6, 4, 14
    lens = [200, 150, 173, 120, 199, 88]
    x, mask = _batch(B, 200, 80, lens)
    worst, worst_rel, scale, steps = _lockstep_persistent(model, sd, params, x, mask, B, beam, max_len, check_logp=False)
    print(f'persistent decode with natural EOS: reference loop executed {steps} of {max_len} steps; history bit-exact')


def test_persistent_equals_per_step_graph_path():
    params = _params(n_enc=1, n_dec=3)
    model, sd = _build(params)
    B, beam, max_len = 4, 5, 10
    x, mask = _batch(B, 240, 80, [240, 200, 111, 239])
    xd, md = x.to(DEV), mask.to(DEV)
    rec_p = SpeechToTextRecognizer(model, beam_width=beam, nbest=2, max_len=max_len, penalty=0.6, lamda=5, ngpu=1,
                                   persistent=True)
    rec_g = SpeechToTextRecognizer(model, beam_width=beam, nbest=2, max_len=max_len, penalty=0.6, lamda=5, ngpu=1,
                                   persistent=False)
    p1, s1, n1 = rec_p.recognize_ids(xd, md)
    p1b, s1b, _ = rec_p.recognize_ids(xd, md)
    p2, s2, n2 = rec_g.recognize_ids(xd, md)
    assert n1 == n2 == max_len
    assert torch.equal(p1, p1b) and torch.equal(s1, s1b), 'persistent kernel must be deterministic'
    same = int((p1 == p2).all(dim=2).sum())
    print(f'persistent vs per-step graph: {same}/{B * 2} n-best sequences identical; scores {s1.view(-1).tolist()} vs {s2.view(-1).tolist()}')
    torch.testing.assert_close(s1, s2, rtol=3e-2, atol=0.3)    # two bf16 pipelines with different rounding points


@pytest.mark.parametrize('B,beam', [(32, 4), (16, 8), (70, 2)])
def test_persistent_full_row_groups_with_even_beam(B, beam):
    """A FULL row group (128 hypotheses) with an even beam: the logits gather of the group's last utterance asks TMA for
    (beam | 1) rows, one past the 128-row tile (out-of-bounds fill), and 70 x 2 spans two groups.  Persistent kernel vs the
    per-step graph path: same hypotheses up to bf16 near-ties, scores within tolerance, deterministic."""
    params = _params(n_enc=1, n_dec=1)
    model, sd = _build(params)
    max_len = 6
    lens = [64 - (i * 7) % 40 for i in range(B)]
    x, mask = _batch(B, 64, 80, lens)
    xd, md = x.to(DEV), mask.to(DEV)
    rec_p = SpeechToTextRecognizer(model, beam_width=beam, nbest=1, max_len=max_len, penalty=0.6, lamda=5, ngpu=1, persistent=True)
    rec_g = SpeechToTextRecognizer(model, beam_width=beam, nbest=1, max_len=max_len, penalty=0.6, lamda=5, ngpu=1, persistent=False)
    p1, s1, n1 = rec_p.recognize_ids(xd, md)
    p1b, s1b, _ = rec_p.recognize_ids(xd, md)
    p2, s2, n2 = rec_g.recognize_ids(xd, md)
    assert next(iter(rec_p._decoders.values())).persistent
    assert n1 == n2 == max_len
    assert torch.equal(p1, p1b) and torch.equal(s1, s1b), 'persistent kernel must be deterministic'
    same = int((p1 == p2).all(dim=2).sum())
    print(f'B={B} beam={beam}: {same}/{B} 1-best identical between the persistent kernel and the graph path')
    assert torch.isfinite(s1).all()
    assert same >= (9 * B) // 10
    torch.testing.assert_close(s1, s2, rtol=3e-2, atol=0.3)


def test_persistent_group_barrier_kinds_give_identical_results():
    """otb_set_decode_barrier: thread-block clusters + barrier.cluster vs plain CTAs + a release/acquire counter in L2.  The
    barrier kind changes scheduling only: hypotheses and scores must be bit-identical."""
    from opentransformer_b200 import ops
    params = _params(n_enc=1, n_dec=2)
    model, sd = _build(params)
    B, beam, max_len = 5, 4, 9
    x, mask = _batch(B, 200, 80, [200, 180, 150, 199, 64])
    xd, md = x.to(DEV), mask.to(DEV)
    rec = SpeechToTextRecognizer(model, beam_width=beam, nbest=2, max_len=max_len, penalty=0.6, lamda=5, ngpu=1, persistent=True)
    out = {}
    try:
        for kind in ('cluster', 'software'):
            ops.set_decode_barrier(kind)
            p_, s_, n_ = rec.recognize_ids(xd, md)
            out[kind] = (p_.clone(), s_.clone(), n_)
    finally:
        ops.set_decode_barrier('default')
    assert next(iter(rec._decoders.values())).persistent
    assert out['cluster'][2] == out['software'][2]
    assert torch.equal(out['cluster'][0], out['software'][0]) and torch.equal(out['cluster'][1], out['software'][1])


def test_end_to_end_best_hypothesis_vs_fp32_oracle():
    """Whole pipeline vs the fp32 oracle: scores of the 1-best within tolerance; report id agreement."""
    params = _params(n_enc=2, n_dec=2)
    model, sd = _build(params)
    B, beam, max_len = 4, 5, 8
    x, mask = _batch(B, 200, 80, [200, 180, 150, 199])
    nb_ref, ns_ref, _, _ = obs.recognize(x, mask, sd, params, beam=beam, nbest=1, max_len=max_len, penalty=0.6, lamda=5)
    rec = SpeechToTextRecognizer(model, beam_width=beam, nbest=1, max_len=max_len, penalty=0.6, lamda=5, ngpu=1)
    p, s, n = rec.recognize_ids(x.to(DEV), mask.to(DEV))
    same = sum(int(torch.equal(p[b, 0].cpu(), nb_ref[b, 0])) for b in range(B))
    print(f'1-best identical to fp32 oracle for {same}/{B} utterances; scores gpu {s.view(-1).tolist()} ref {ns_ref.view(-1).tolist()}')
    torch.testing.assert_close(s.cpu(), ns_ref, rtol=3e-2, atol=0.3)


def test_decoder_kv_cache_through_the_reference_seam():
    _kv_cache_through_the_seam(False, 'glu')


def test_decoder_kv_cache_through_the_reference_seam_prenorm_relu():
    _kv_cache_through_the_seam(True, 'relu')


def _kv_cache_through_the_seam(normalize_before, activation):
    """The cache the reference stubbed out (decoder/transformer.py:92-126,188-203), through its own seam:
    decoder.inference(preds, memory, mask, cache) with cache = decoder.init_cache(...) runs one token per call, and
    SpeechToTextRecognizer.decode_step reorders it by the surviving parents.  Must agree with the full-prefix recompute
    (cache None, the reference's behaviour) and with the oracle in lock-step."""
    params = _params(n_enc=1, n_dec=3)
    params['decoder'].update(normalize_before=normalize_before, activation=activation)
    model, sd = _build(params)
    B, beam, max_len = 3, 4, 8
    x, mask = _batch(B, 200, 80, [200, 150, 173])
    rec = SpeechToTextRecognizer(model, beam_width=beam, nbest=1, max_len=max_len, penalty=0.6, lamda=5, ngpu=1)
    memory, mmask, _, _ = rec.encode(x.to(DEV), mask.to(DEV))
    T2 = memory.shape[1]
    bm = memory.unsqueeze(1).repeat(1, beam, 1, 1).view(B * beam, T2, -1)
    bmask = mmask.unsqueeze(1).repeat(1, beam, 1).view(B * beam, T2)
    kw = om.decoder_kwargs(params)

    def loop(cache):
        preds = torch.ones(B * beam, 1, dtype=torch.long, device=DEV)
        scores = torch.tensor([0.0] + [float('-inf')] * (beam - 1), device=DEV).repeat(B).unsqueeze(1)
        flag = torch.zeros_like(scores, dtype=torch.bool)
        with torch.no_grad():
            for _ in range(max_len):
                preds, cache, scores, flag = rec.decode_step(preds, bm, bmask, cache, scores, flag)
        return preds, scores

    with torch.no_grad():
        dc = model.decoder.init_cache(bm, bmask, max_len, beam=beam)
    p_c, s_c = loop({'decoder': dc})
    p_f, s_f = loop({'decoder': None})
    assert dc.step == max_len
    same = int((p_c == p_f).all(dim=1).sum())
    print(f'KV-cached seam vs full-prefix seam: {same}/{B * beam} hypotheses identical; 1-best scores {s_c.view(B, beam)[:, 0].tolist()} '
          f'vs {s_f.view(B, beam)[:, 0].tolist()}')
    torch.testing.assert_close(s_c, s_f, rtol=3e-2, atol=0.3)
    assert torch.equal(p_c.view(B, beam, -1)[:, 0], p_f.view(B, beam, -1)[:, 0]), '1-best of the cached and the recomputing seam differ'
    # lock-step with the oracle: cached log-probs of the seam drive the oracle's beam_step; ids must be bit-exact
    with torch.no_grad():
        dc = model.decoder.init_cache(bm, bmask, max_len, beam=beam)
        preds = torch.ones(B * beam, 1, dtype=torch.long, device=DEV)
        o_preds = preds.cpu()
        o_scores = torch.tensor([0.0] + [float('-inf')] * (beam - 1)).repeat(B).unsqueeze(1)
        o_flag = torch.zeros_like(o_scores, dtype=torch.bool)
        for s in range(max_len):
            lp, dc, _ = model.decoder.inference(preds, bm, bmask, dc)
            lp_ref = om.decoder_inference(o_preds, bm.cpu(), bmask.cpu(), sd, 'decoder.', **kw)
            alive = ~o_flag.view(-1)
            assert _rel(lp.cpu()[alive][:, 2:], lp_ref[alive][:, 2:]) < REL_L2_LOGITS
            tr = []
            o_preds, o_scores, o_flag = obs.beam_step(lp.cpu(), o_preds, o_scores, o_flag, beam, trace=tr)
            dc.reorder(tr[0]['parent'].to(DEV))        # rows the surviving hypotheses extend (speech2text.py:136)
            preds = o_preds.to(DEV)
