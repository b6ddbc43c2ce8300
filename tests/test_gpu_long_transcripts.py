"""Transcripts past the short-path bounds: the CTC loss up to 1023 labels (64 and fewer take the one-state-per-thread
kernels) and the KV-cached decoder self-attention up to 1023 cached positions (128 and fewer take the one-chunk kernel),
through the ops, the beam search past step 128, the recognizer and joint-CTC / CTCModel training."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops, train
    from opentransformer_b200.recognize import BeamDecoder, SpeechToTextRecognizer
    DEV = torch.device('cuda:0')

from oracle import beam_search as obs
from oracle import train_step as ot

BF = torch.bfloat16


def _rel(a, b):
    return float((a.float().cpu() - b.float().cpu()).norm() / (b.float().cpu().norm() + 1e-20))


# ------------------------------------------------------------------------------------------------ CTC loss
def _long_ctc_batch(L, seed):
    """Five utterances at padded width min(L + 3, 1023): the long target, a short one, long runs of one repeated label,
    one too long for its frames (infeasible) and an empty one."""
    V = 50
    W = min(L + 3, 1023)
    g = torch.Generator().manual_seed(seed)
    T = 2 * L + 40                                  # room for L labels with a blank between every repeated pair
    tgt = torch.randint(1, V, (5, W), generator=g)
    tgt[2, :] = 7
    tgt[2, L // 3:L // 3 + 10] = 8                  # two runs of 7 around a run of 8
    tlen = torch.tensor([L, min(L, 40), L, L, 0], dtype=torch.int32)
    in_len = torch.tensor([T, 100, T, L // 2, T - 5], dtype=torch.int32)
    return V, T, tgt, tlen, in_len


def _torch_ctc(logits, B, T, V, tgt, tlen, in_len):
    x = logits[:, :V].detach().cpu().double().view(B, T, V).requires_grad_(True)
    lp = torch.log_softmax(x, -1).transpose(0, 1)
    ref = F.ctc_loss(lp, tgt, in_len.long(), tlen.long(), blank=0, reduction='mean', zero_infinity=True)
    ref.backward()
    nll = F.ctc_loss(lp.detach(), tgt, in_len.long(), tlen.long(), blank=0, reduction='none', zero_infinity=False)
    return ref, nll, x.grad


@pytest.mark.parametrize('L', [65, 128, 129, 511, 1023])
def test_ctc_loss_long_targets_vs_torch(L):
    V, T, tgt, tlen, in_len = _long_ctc_batch(L, seed=L)
    B = tgt.shape[0]
    g = torch.Generator().manual_seed(3)
    logits = (torch.randn(B * T, 56, generator=g) * 2).to(DEV)
    loss, nll, dl = ops.ctc_loss(logits, B, T, V, in_len.to(DEV), tgt.to(DEV), tlen.to(DEV), 0, want_grad=True)
    ref, ref_nll, ref_grad = _torch_ctc(logits, B, T, V, tgt, tlen, in_len)
    print(f'L {L}: loss gpu {float(loss):.6f} torch {float(ref):.6f}')
    assert abs(float(loss) - float(ref)) < 1e-4 * max(1.0, abs(float(ref)))
    fin = torch.isfinite(ref_nll)
    assert not bool(fin[3]), 'utterance 3 has fewer frames than labels'
    assert torch.equal(torch.isfinite(nll.cpu()), fin)
    torch.testing.assert_close(nll.cpu()[fin].double(), ref_nll[fin], rtol=1e-4, atol=1e-4 * L)
    got = dl.float().cpu().view(B, T, -1)
    assert float(got[:, :, V:].abs().max()) == 0.0
    assert float(got[3].abs().max()) == 0.0, 'infeasible utterance: zero gradient (zero_infinity)'
    for b in range(B):
        assert not bool(got[b, int(in_len[b]):].any()), 'padded frames: zero gradient'
    r = _rel(got[:, :, :V], ref_grad)
    print(f'L {L}: dlogits rel_l2 {r:.3e}')
    assert r < 6e-3


def test_ctc_loss_grad_scale_and_device_scale_at_1023():
    L = 1023
    V, T, tgt, tlen, in_len = _long_ctc_batch(L, seed=5)
    B = tgt.shape[0]
    g = torch.Generator().manual_seed(4)
    logits = (torch.randn(B * T, 56, generator=g) * 2).to(DEV)
    args = (logits, B, T, V, in_len.to(DEV), tgt.to(DEV), tlen.to(DEV), 0)
    _, _, d1 = ops.ctc_loss(*args, want_grad=True)
    _, _, d2 = ops.ctc_loss(*args, want_grad=True, grad_scale=0.25)
    _, _, d3 = ops.ctc_loss(*args, want_grad=True, grad_scale=0.5, scale_dev=torch.tensor([0.5], device=DEV))
    ref = d1.float() * 0.25
    assert _rel(d2, ref) < 8e-3
    assert torch.equal(d2, d3), 'grad_scale 0.5 times a device scale 0.5 is grad_scale 0.25'


# ------------------------------------------------------------------------------------------------ decode self-attention
@pytest.mark.parametrize('dk', [64, 96])
def test_decode_self_attention_long_prefix(dk):
    """The chunked kernel at Lmax 1023 against the fp32 restatement (test_gpu_ops.py's ancestry-cache test), at steps on
    both sides of every 128-key chunk boundary, with a shuffled ancestry table; the newest K/V is appended."""
    N, H, Lmax = 6, 4, 1023
    d = H * dk
    g = torch.Generator().manual_seed(11)
    qkv = torch.randn(N, 3 * d, generator=g).to(BF).to(DEV)
    kc = torch.randn(Lmax, N, d, generator=g).to(BF).to(DEV)
    vc = torch.randn(Lmax, N, d, generator=g).to(BF).to(DEV)
    anc = torch.stack([torch.stack([torch.randperm(N, generator=g) for _ in range(Lmax)], 1) for _ in range(2)])
    anc = anc.to(torch.int32).contiguous().to(DEV)                                      # [2, N, Lmax]
    for step in (0, 127, 128, 129, 255, 256, 700, 1022):
        kcs, vcs = kc.clone(), vc.clone()
        ctrl = torch.tensor([step, 0, 0, 0], dtype=torch.int32, device=DEV)
        out = ops.decode_self_attn(qkv, kcs, vcs, anc, ctrl, N, H, Lmax)
        cur = anc[step & 1].long()
        ks = torch.stack([kc[s, cur[:, s]] for s in range(step)] + [qkv[:, d:2 * d]], 1).float()
        vs = torch.stack([vc[s, cur[:, s]] for s in range(step)] + [qkv[:, 2 * d:]], 1).float()
        q = qkv[:, :d].float().view(N, H, 1, dk)
        sc = (q @ ks.view(N, step + 1, H, dk).transpose(1, 2).transpose(2, 3)) / dk ** 0.5
        ref = (torch.softmax(sc, -1) @ vs.view(N, step + 1, H, dk).transpose(1, 2)).reshape(N, d)
        r = _rel(out, ref)
        print(f'd_k {dk} step {step}: rel_l2 {r:.2e}')
        assert r < 6e-3 and torch.isfinite(out.float()).all()
        assert torch.equal(kcs[step], qkv[:, d:2 * d]) and torch.equal(vcs[step], qkv[:, 2 * d:])
        assert torch.equal(kcs[:step], kc[:step]) and torch.equal(kcs[step + 1:], kc[step + 1:])


# ------------------------------------------------------------------------------------------------ beam search past 128 steps
def _s2t_model(n_enc=1, n_dec=1, ctc_weight=0.0):
    from tests import test_gpu_model as tm
    params = tm._params(n_enc=n_enc, n_dec=n_dec)
    params['ctc_weight'] = ctc_weight
    if ctc_weight:
        params['encoder_output_size'] = 256
    model, sd = tm._build(params)         # EOS logit biased by -1e4: every hypothesis runs to max_len
    return model, tm


@pytest.mark.parametrize('use_graph', [False, True])
def test_beam_search_past_128_steps_lockstep(use_graph):
    """The per-step path (graph and eager) in lockstep with the oracle's beam_step on the GPU's own log-probs for 300
    steps: every token and parent id and every score the same."""
    model, tm = _s2t_model()
    B, beam, max_len = 2, 3, 300
    x, mask = tm._batch(B, 240, 80, [240, 200])
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
        bd = BeamDecoder(model.decoder, B, beam, T2, max_len, DEV, use_graph=use_graph, keep_logp=True)
        assert not bd.persistent
        bd.setup(mem, lens)
        preds = torch.full((B * beam, 1), 1, dtype=torch.long)
        scores = torch.tensor([0.0] + [float('-inf')] * (beam - 1)).repeat(B).unsqueeze(1)
        flag = torch.zeros_like(scores, dtype=torch.bool)
        for s in range(max_len):
            bd.step()
            preds, scores, flag = obs.beam_step(bd.logp.cpu(), preds, scores, flag, beam)
            if s in (127, 128, 129) or s % 50 == 49 or s == max_len - 1:
                assert torch.equal(bd.state.reconstruct(s + 1).cpu(), preds), f'token/parent ids differ at step {s}'
            assert torch.equal(bd.state.scores.cpu(), scores.view(-1)), f'scores differ at step {s}'
        assert not bool(flag.any()), 'every hypothesis must reach step 300'


@pytest.mark.parametrize('ctc_weight', [0.0, 0.3])
def test_recognizer_at_max_len_300(ctc_weight):
    """SpeechToTextRecognizer past the persistent kernel's 128 steps: the search runs all 300 steps, with and without
    the CTC prefix term, and the graph and eager paths give the same n-best.  (With the CTC term, a hypothesis forced
    past its feasible length by the EOS bias may score -inf: only the attention search's scores must be finite.)"""
    model, tm = _s2t_model(ctc_weight=ctc_weight)
    x, mask = tm._batch(2, 1300, 80, [1300, 1250])     # T' > 300: a 300-token hypothesis is feasible for the CTC term
    got = []
    for use_graph in (True, False):
        rec = SpeechToTextRecognizer(model, beam_width=3, nbest=2, max_len=300, ctc_weight=ctc_weight, use_graph=use_graph)
        ids, scores, steps = rec.recognize_ids(x.to(DEV), mask.to(DEV))
        assert int(steps) == 300
        assert ctc_weight > 0 or torch.isfinite(scores).all()
        got.append((ids.cpu(), scores.cpu()))
    assert torch.equal(got[0][0], got[1][0])
    assert torch.equal(got[0][1], got[1][1])


# ------------------------------------------------------------------------------------------------ training
def _speech(T, lens, seed=0):
    g = torch.Generator().manual_seed(seed)
    lens = torch.tensor(lens)
    mask = torch.arange(T)[None] < lens[:, None]
    return torch.randn(len(lens), T, 80, generator=g) * mask.unsqueeze(2), mask


def _long_targets(B, L, V, seed):
    g = torch.Generator().manual_seed(seed)
    tgt = torch.randint(3, V, (B, L + 2), generator=g)
    tgt[:, 0] = 1
    tgt[0, L + 1] = 1                                 # full length: L tokens and the closing <S/E>
    tgt[1, 31:] = torch.tensor([1] + [0] * (L - 30))  # a short transcript beside it
    return tgt


@pytest.mark.parametrize('L', [100, 300])
def test_joint_ctc_long_transcripts_match_oracle(L):
    from tests import test_gpu_train as tt
    params = tt._params(n_enc=1, n_dec=1)
    params['ctc_weight'] = 0.3
    params['encoder_output_size'] = 256
    model, sd = tt._build(params)
    for k, v in model.assistor.state_dict().items():
        sd[f'assistor.{k}'] = v.detach().clone().float().cpu()
    T = 4 * L + 120
    x, mask = _speech(T, (T, T - 100))
    tgt = _long_targets(2, L, 4234, seed=L)
    tlen = torch.tensor([(int((tgt[b, 1:] != 0).sum())) for b in range(2)], dtype=torch.int32)
    assert int(tlen[0]) == L + 1
    loss_ref, g_ref = ot.loss_and_grads(x, mask, tgt, sd, params, truth_length=tlen)
    with torch.no_grad():
        loss, g = train.forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), truth_length=tlen.to(DEV))
    names = [n for n, _ in model.named_parameters()]
    worst = sorted(((_rel(g[n], g_ref[n]), n) for n in names), reverse=True)
    r_all = _rel(torch.cat([g[n].reshape(-1).cpu() for n in names]), torch.cat([g_ref[n].reshape(-1) for n in names]))
    print(f'joint CTC L {L}: loss gpu {float(loss):.5f} oracle {float(loss_ref):.5f}; all grads rel_l2 {r_all:.3e}; '
          'worst ' + ', '.join(f'{n} {r:.2e}' for r, n in worst[:3]))
    assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    # the CTC head and the encoder it feeds at the usual tolerance; the attention decoder's gradients sum bf16 products
    # over L + 1 tokens, so its worst parameter is allowed twice the usual per-parameter error (measured on an H100:
    # decoder.blocks.0.norm3.bias 4.19e-2 at L 100 and 3.27e-2 at L 300, against 4e-2 usually; every other parameter
    # below 3.7e-2)
    worst_ctc = max((_rel(g[n], g_ref[n]), n) for n in names if not n.startswith('decoder.'))
    assert r_all < tt.REL_L2_GRAD_ALL and worst_ctc[0] < tt.REL_L2_GRAD, worst_ctc
    assert worst[0][0] < 2 * tt.REL_L2_GRAD, worst[:3]
    model.eval()
    with torch.no_grad():
        l2, aux = model({'inputs': x.to(DEV), 'mask': mask.to(DEV)}, {'targets': tgt.to(DEV), 'targets_length': tlen})
    assert abs(float(l2) - float(loss_ref)) < 2e-2 * abs(float(loss_ref)) and 'CTCLoss' in aux


def test_ctc_model_training_at_300_tokens():
    from tests import ctc_ref
    from tests import test_gpu_ctc_model as tc
    params = tc._params('transformer')
    model, sd = tc._build(params)
    L, T = 300, 1320
    x, mask = _speech(T, (T, T - 100))
    tgt = _long_targets(2, L, 40, seed=1)
    tlen = (tgt[:, 1:] != 0).sum(1)
    loss_ref, g_ref, _ = ctc_ref.loss_and_grads_train(x, mask, tgt, tlen, sd, params)
    with torch.no_grad():
        loss, g = train.ctc_forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV))
    worst = sorted(((_rel(g[n], g_ref[n]), n) for n in g), reverse=True)
    print(f'CTCModel L {L}: loss gpu {float(loss):.5f} ref {float(loss_ref):.5f}; worst '
          + ', '.join(f'{n} {r:.2e}' for r, n in worst[:3]))
    assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    assert worst[0][0] < tc.REL_L2_GRAD, worst[:3]


def test_ctc_model_fused_trainer_graph_at_300_tokens():
    """FusedTrainer on the CUDA-graph path with 300-token transcripts (the long CTC kernels and their workspace captured in
    the graph): two optimizer steps against the restatement's gradients through the reference's clip + Adam."""
    from tests import ctc_ref
    from tests import test_gpu_ctc_model as tc
    params = tc._params('transformer')
    model, sd = tc._build(params)
    model.train()
    tr = train.FusedTrainer(model, clip_grad=0.05, use_graph=True)
    tr.graph_after = 1
    names = [n for n, _ in tr.params]
    w = {n: sd[n].clone() for n in names}
    m = {n: torch.zeros_like(w[n]) for n in names}
    v = {n: torch.zeros_like(w[n]) for n in names}
    stats = {}
    L, T = 300, 1320
    for opt_step in (1, 2):
        x, mask = _speech(T, (T, T - 100), seed=opt_step)
        tgt = _long_targets(2, L, 40, seed=opt_step)
        tlen = (tgt[:, 1:] != 0).sum(1)
        loss = tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV))
        sd_now = dict(sd)
        sd_now.update({n: w[n] for n in names})
        sd_now.update(stats)
        loss_ref, g_ref, new_stats = ctc_ref.loss_and_grads_train(x, mask, tgt, tlen, sd_now, params)
        stats.update(new_stats)
        assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
        lr = ot.transformer_lr(ot.first_step_index() + opt_step - 1, 256, 12000)
        ot.clip_and_adam(w, {n: g_ref[n] for n in names}, m, v, opt_step, lr, 0.05)
        torch.cuda.synchronize()
        p = dict(model.named_parameters())
        num = sum(float(((p[n].detach().cpu() - w[n]) ** 2).sum()) for n in names)
        den = sum(float(((w[n] - sd[n]) ** 2).sum()) for n in names)
        print(f'CTCModel FusedTrainer graph, L {L}, step {opt_step}: loss {float(loss):.5f} ref {float(loss_ref):.5f}; '
              f'weights rel {(num / den) ** 0.5:.3e}')
        assert (num / den) ** 0.5 < 0.3
    assert len(tr._graphs) >= 1, 'the step must have run as a CUDA graph'


# ------------------------------------------------------------------------------------------------ entry points past step 128
def test_transformer_lm_fusion_lockstep_past_128_steps():
    """Shallow fusion with the Transformer LM re-reading 300-token prefixes: the eager BeamDecoder in lockstep with the
    oracle's beam_step fed the GPU's decoder and LM log-probs, every id and score the same; then
    SpeechToTextRecognizer(lm=...) at max_len 300 returns the oracle's finalised n-best."""
    from opentransformer_b200.lm import TransformerLanguageModel
    from opentransformer_b200.recognize import lm_log_probs
    torch.manual_seed(77)
    lm = TransformerLanguageModel(dict(vocab_size=4234, num_blocks=2, d_model=256, n_heads=4, d_ff=1024, residual_dropout=0.0,
                                       smoothing=0.1, share_embedding=True)).eval().to(DEV)
    model, tm = _s2t_model()
    B, beam, max_len, lmw = 2, 3, 300, 0.3
    x, mask = tm._batch(B, 240, 80, [240, 200])
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
        bd = BeamDecoder(model.decoder, B, beam, T2, max_len, DEV, use_graph=False)
        bd.setup(mem, lens)
        bd.lm_weight = lmw
        preds = torch.full((B * beam, 1), 1, dtype=torch.long)
        scores = torch.tensor([0.0] + [float('-inf')] * (beam - 1)).repeat(B).unsqueeze(1)
        flag = torch.zeros_like(scores, dtype=torch.bool)
        for s in range(max_len):
            bd.lm_logp = lm_log_probs(lm, bd.state.reconstruct(s))
            lm_cpu = bd.lm_logp.cpu()
            bd._step_kernels()
            dec_lp = bd.logp.cpu() - lmw * lm_cpu          # the fused kernel stores decoder + lmw * lm
            preds, scores, flag = obs.beam_step(dec_lp, preds, scores, flag, beam, lm_log_probs=lm_cpu, lm_weight=lmw)
            if s in (127, 128, 129) or s % 50 == 49:
                assert torch.equal(bd.state.reconstruct(s + 1).cpu(), preds), f'fusion: ids differ at step {s}'
        assert torch.equal(bd.state.reconstruct(max_len).cpu(), preds)
        nb, ns = obs.beam_finalize(preds, scores, beam, 2, 0.6, 5)
    rec = SpeechToTextRecognizer(model, lm=lm, lm_weight=lmw, beam_width=beam, nbest=2, max_len=max_len, penalty=0.6,
                                 lamda=5)
    ids, sc, n = rec.recognize_ids(x.to(DEV), mask.to(DEV))
    assert int(n) == max_len
    assert torch.equal(ids[:, :, :max_len].cpu(), nb)
    torch.testing.assert_close(sc.cpu(), ns, rtol=1e-5, atol=1e-5)


def test_joint_ctc_search_lockstep_past_128_steps():
    """ctc_weight 0.3 at max_len 300: the eager BeamDecoder with the CTC term against the float64 restatement
    (tests/ctc_prefix_ref.JointSearch) on the GPU's log-probs: the same live prefixes at every checked step, the same -inf
    pattern, and scores within 1e-3 plus the rounding bound of an fp32 sum over the steps; then SpeechToTextRecognizer returns the same steps on the graph path."""
    from tests import ctc_prefix_ref as cpr
    from tests.test_gpu_ctc_prefix import _joint_model
    model = _joint_model()
    B, beam, P, max_len, w = 2, 3, 6, 300, 0.3
    x, mask = _speech(1300, (1300, 1250))
    x, mask = x.to(DEV), mask.to(DEV)
    V = model.decoder.vocab_size
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x, mask)
        bd = BeamDecoder(model.decoder, B, beam, T2, max_len, DEV, use_graph=False, keep_logp=True, ctc=(model.assistor, w, P))
        bd.setup(mem, lens)
        js = cpr.JointSearch(bd.ctc.lp.view(B, T2, V).cpu(), lens.cpu().tolist(), beam, P, w, 0.0)
        for s in range(max_len):
            bd._step_kernels()
            js.step(bd.logp.cpu().double(), None)
            got, want = bd.state.scores.cpu().double(), js.scores.view(-1)
            assert torch.equal(torch.isfinite(got), torch.isfinite(want)), s
            fin = torch.isfinite(want)
            if bool(fin.any()):
                # fp32 running sums of s + 1 step scores against float64: 1e-3 plus the sum's rounding bound (s + 1) u |score|
                tol = 1e-3 + (s + 1) * 2.0 ** -24 * want[fin].abs()
                assert bool(((got - want)[fin].abs() <= tol).all()), (s, float((got - want)[fin].abs().max()))
            if s in (127, 128, 129) or s % 50 == 49:
                # hypotheses the CTC term rules out (-inf) tie among themselves, and which of the ties fills a slot is not
                # specified: the prefixes of the live ones must agree
                assert s > 129 or bool(fin.any()), f'no live hypothesis at step {s}'
                live = fin.view(-1)
                assert torch.equal(bd.state.reconstruct(s + 1).cpu()[live], js.preds[live]), f'prefixes differ at step {s}'
    rec = SpeechToTextRecognizer(model, ctc_weight=w, ctc_candidates=P, beam_width=beam, nbest=2, max_len=max_len)
    assert int(rec.recognize_ids(x, mask)[2]) == max_len


def test_decoder_cache_seam_past_128_steps():
    """decode_step through DecoderCache for 200 steps: the cached log-probs against the oracle's full-prefix recompute on
    both sides of step 128, the ids in lockstep with the oracle's beam_step, and the recognizer's own decode_step (beam
    kernel + cache reorder) reaching the same prefixes."""
    from oracle import speech_model as om
    from tests import test_gpu_model as tm
    params = tm._params(n_enc=1, n_dec=1)
    model, sd = tm._build(params)
    B, beam, max_len = 2, 3, 200
    x, mask = tm._batch(B, 240, 80, [240, 200])
    rec = SpeechToTextRecognizer(model, beam_width=beam, nbest=1, max_len=max_len, penalty=0.6, lamda=5, ngpu=1)
    memory, mmask, _, _ = rec.encode(x.to(DEV), mask.to(DEV))
    T2 = memory.shape[1]
    bm = memory.unsqueeze(1).repeat(1, beam, 1, 1).view(B * beam, T2, -1)
    bmask = mmask.unsqueeze(1).repeat(1, beam, 1).view(B * beam, T2)
    kw = om.decoder_kwargs(params)
    with torch.no_grad():
        dc = model.decoder.init_cache(bm, bmask, max_len, beam=beam)
        preds = torch.ones(B * beam, 1, dtype=torch.long, device=DEV)
        o_preds = preds.cpu()
        o_scores = torch.tensor([0.0] + [float('-inf')] * (beam - 1)).repeat(B).unsqueeze(1)
        o_flag = torch.zeros_like(o_scores, dtype=torch.bool)
        for s in range(max_len):
            lp, dc, _ = model.decoder.inference(preds, bm, bmask, dc)
            if s in (0, 127, 128, 129, max_len - 1):
                lp_ref = om.decoder_inference(o_preds, bm.cpu(), bmask.cpu(), sd, 'decoder.', **kw)
                r = _rel(lp.cpu()[:, 2:], lp_ref[:, 2:])
                print(f'DecoderCache step {s}: log-probs rel_l2 {r:.3e}')
                assert r < tm.REL_L2_LOGITS
            trace = []
            o_preds, o_scores, o_flag = obs.beam_step(lp.cpu(), o_preds, o_scores, o_flag, beam, trace=trace)
            dc.reorder(trace[0]['parent'].to(DEV))
            preds = o_preds.to(DEV)
        assert dc.step == max_len
        dc2 = model.decoder.init_cache(bm, bmask, max_len, beam=beam)
        p2 = torch.ones(B * beam, 1, dtype=torch.long, device=DEV)
        s2 = torch.tensor([0.0] + [float('-inf')] * (beam - 1), device=DEV).repeat(B).unsqueeze(1)
        f2 = torch.zeros_like(s2, dtype=torch.bool)
        cache = {'decoder': dc2}
        for _ in range(max_len):
            p2, cache, s2, f2 = rec.decode_step(p2, bm, bmask, cache, s2, f2)
    assert torch.equal(p2.cpu(), o_preds)
    assert torch.equal(s2.cpu(), o_scores)


@pytest.mark.parametrize('w', [0.0, 0.3])
def test_recognize_spans_at_max_len_300(w):
    """recognize_spans at max_len 300: the ids, scores and steps of recognize_ids, and the spans of ops.ctc_align called by
    hand on the 1-best plus its closing <S/E>."""
    from tests.test_gpu_ctc_prefix import _joint_model
    model = _joint_model()
    B, max_len = 2, 300
    x, mask = _speech(1300, (1300, 1250))
    x, mask = x.to(DEV), mask.to(DEV)
    rec = SpeechToTextRecognizer(model, ctc_weight=w, beam_width=3, nbest=2, max_len=max_len, penalty=0.6, lamda=5)
    ids, sc, n = rec.recognize_ids(x, mask)
    ids2, sc2, n2, spans = rec.recognize_spans(x, mask)
    assert int(n) == max_len
    assert n == n2 and torch.equal(ids, ids2) and torch.equal(sc, sc2)
    assert spans.shape == (B, n + 1, 2) and spans.dtype == torch.int32
    V = model.decoder.vocab_size
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x, mask)
        lp = ops.log_softmax(model.assistor.logits_bf16(mem), V).view(B, T2, V)
    tgt = torch.cat((ids[:, 0], torch.full((B, 1), 1, dtype=torch.int64, device=DEV)), 1)
    n_tok = [row.index(1) + 1 for row in tgt.cpu().tolist()]
    _, _, want, _ = ops.ctc_align(lp, lens, tgt, torch.tensor(n_tok, dtype=torch.int32, device=DEV))
    assert torch.equal(spans, want)


def test_attention_rescoring_at_max_len_300():
    """apply_rescoring with max_len 300 on 1300-frame utterances (the CTC n-best runs past 128 tokens): the rescored
    n-best against the restatement (tests/rescore_ref.py) on the same first-pass hypotheses."""
    from opentransformer_b200.recognize import ctc_decode
    from tests import rescore_ref as rr
    from tests import test_gpu_rescore as trs
    model, sd, params = trs._speech_model(ctc_weight=0.3, eos_bias=0.0)
    B, beam, nbest, w = 2, 4, 2, 0.7
    V = model.decoder.vocab_size
    x, mask = _speech(1300, (1300, 1250), seed=2)
    x, mask = x.to(DEV), mask.to(DEV)
    rec = SpeechToTextRecognizer(model, beam_width=beam, nbest=nbest, max_len=300, apply_rescoring=True, rescore_weight=w)
    ids, scores, steps = rec.recognize_ids(x, mask)
    with torch.no_grad():
        mem, mem_len, _, T2 = model.encode_bf16(x, mask)
        cids, cn, csc = ctc_decode(model.assistor.logits_bf16(mem), mem_len, B, T2, V, 0, 'beam', beam)
    hyps = [[rr.cut(cids[b, k].tolist(), int(cn[b, k])) for k in range(beam)] for b in range(B)]
    longest = max(len(y) for row in hyps for y in row)
    print(f'apply_rescoring: longest first-pass hypothesis {longest} tokens, steps {steps}')
    assert ids.shape == (B, nbest, steps) and steps == longest + 1
    lens = (ids == 1).int().argmax(dim=2)
    dec = trs._decoder_second(model, sd, params, mem, mem_len, T2)
    trs._check_against_restatement(ids.cpu(), lens.cpu(), scores.cpu(), hyps, csc.cpu().tolist(), lambda b, y: [dec(b, y)],
                                   w, nbest)


def test_fused_trainer_mwer_nbest_past_128_steps():
    """FusedTrainer(mwer_nbest=2, mwer_max_len=200) with the EOS logit biased down, so the n-best decode runs all 200
    steps: the graph and eager paths decode the same n-best (identical losses) and the weights agree as in
    test_gpu_mwer.py's graph-against-eager test."""
    from tests.test_gpu_train import _batch, _build, _params
    params = _params(n_enc=1, n_dec=1)
    x, mask, tgt = (t.to(DEV) for t in _batch())
    runs = []
    for use_graph in (False, True):
        model, _ = _build(params)
        with torch.no_grad():
            model.decoder.output_layer.bias[1] = -30.0
        tr = train.FusedTrainer(model.train(), clip_grad=0.05, use_graph=use_graph, mwer_nbest=2, mwer_max_len=200)
        tr.graph_after = 1
        losses = [float(tr.step(x, mask, tgt)) for _ in range(2)]
        runs.append((losses, tr.flat_p.clone(), len(tr._graphs)))
    print('MWER past 128 steps: losses eager', runs[0][0], 'graph', runs[1][0])
    assert all(torch.isfinite(torch.tensor(r[0])).all() for r in runs)
    assert runs[1][2] >= 1
    assert runs[0][0] == runs[1][0]
    differ = int((runs[0][1] != runs[1][1]).sum())
    assert differ <= 1e-3 * runs[0][1].numel()
    assert float((runs[0][1] - runs[1][1]).abs().max()) <= 5e-8
