"""GPU checks of the low-frame-rate front ends (`concat`, `concat-with-linear`): otb_frame_stack bit for bit against
nn.Unfold + a bf16 cast, the front ends and whole encoders against the bf16-policy oracle, the recognizers in lock-step with
the oracle's beam step on the persistent and the per-step graph paths, the CTC recognizer and its spans, and training
(loss and every gradient, FusedTrainer with and without the graph, MixSpeech) against the fp32 restatement."""
import pytest
import torch
import torch.nn.functional as F

from tests import concat_frontend_ref as cref
from tests import ctc_ref
from tests import train_options_ref as tor

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops, train
    from opentransformer_b200.model import encoder_frames_to_input
    from opentransformer_b200.recognize import BeamDecoder, CTCRecognizer, SpeechToTextRecognizer
    from tests import test_gpu_model as tgm
    from tests import test_gpu_ctc_model as tgc
    DEV = torch.device('cuda:0')

from oracle import beam_search as obs
from oracle import speech_model as om
from oracle import train_step as ot

REL_L2_STATES = 2e-2
REL_L2_GRAD = 4e-2


def _rel(a, b):
    return float((a.float().cpu() - b.float().cpu()).norm() / (b.float().cpu().norm() + 1e-20))


# ------------------------------------------------------------------------------------------------ otb_frame_stack
def _unfold_ref(x, n, s, T2):
    """nn.Unfold over the zero-padded [T, F] plane, T2 rows (past T_p as well) -> f32 [B*T2, n F]."""
    B, T, Fd = x.shape
    need = (T2 - 1) * s + n
    xp = F.pad(x, (0, 0, 0, max(0, need - T)))
    y = torch.nn.Unfold(kernel_size=(n, Fd), stride=s)(xp.unsqueeze(1)).transpose(1, 2)[:, :T2]
    return y.reshape(B * T2, n * Fd)


@pytest.mark.parametrize('B,T,Fd,n,s,extra', [
    (3, 1000, 80, 4, 4, 0), (2, 37, 80, 3, 3, 0), (2, 2, 5, 6, 6, 0), (3, 23, 5, 7, 3, 2), (1, 9, 13, 4, 2, 3),
    (2, 50, 3, 1, 1, 0), (4, 101, 40, 5, 2, 1)])
def test_frame_stack_is_bit_exact(B, T, Fd, n, s, extra):
    """Ragged T, T < n, n F not a multiple of 8 (padding columns zero), rows past T_p (extra) and F % 4 != 0 (scalar
    loads); canary columns past the written width stay as they were."""
    g = torch.Generator().manual_seed(T * 7 + n)
    x = torch.randn(B, T, Fd, generator=g)
    Tp = T + (s - (T - n) % s) % s
    T2 = (Tp - n) // s + 1 + extra
    W = (n * Fd + 7) // 8 * 8
    out = torch.full((B * T2, W + 16), 7.0, dtype=torch.bfloat16, device=DEV)
    ops.frame_stack(x.to(DEV), n, s, T2, out=out)
    got = out.cpu()
    want = _unfold_ref(x, n, s, T2).to(torch.bfloat16)
    assert torch.equal(got[:, :n * Fd], want)
    assert bool((got[:, n * Fd:W] == 0).all()) and bool((got[:, W:] == 7.0).all())
    # the epilogue y * alpha + table[i], within bf16 rounding of the fp32 expression
    table = torch.randn(T2, n * Fd, generator=g)
    y = ops.frame_stack(x.to(DEV), n, s, T2, alpha=16.0, table=table.to(DEV)).cpu()
    ref = (_unfold_ref(x, n, s, T2) * 16.0 + table.repeat(B, 1))
    torch.testing.assert_close(y[:, :n * Fd].float(), ref, rtol=2 ** -8, atol=1e-6)
    assert bool((y[:, n * Fd:] == 0).all())


def test_frame_stack_refuses_bad_arguments():
    x = torch.zeros(1, 8, 5, device=DEV)
    with pytest.raises(ValueError, match='table'):
        ops.frame_stack(x, 2, 2, 4, table=torch.zeros(4, 9, device=DEV))
    with pytest.raises(ValueError, match='out'):
        ops.frame_stack(x, 2, 2, 4, out=torch.zeros(4, 8, dtype=torch.bfloat16, device=DEV))
    with pytest.raises(RuntimeError, match='>= 1'):
        ops.frame_stack(x, 2, 0, 4)


# ------------------------------------------------------------------------------------------------ models
def _s2t_params(left=3, right=0, rate=40, F_in=80, ctc=0.0):
    p = tgm._params(n_enc=2, n_dec=2, F=F_in)
    p['frontend_type'] = 'concat-with-linear'
    p['frontend'] = dict(input_size=F_in, output_size=256, left_frames=left, right_frames=right, frame_rate=rate, dropout=0.0)
    p['ctc_weight'] = ctc
    p['encoder_output_size'] = 256
    p['decoder']['share_embedding'] = False
    return p


def _s2t_build(params, training=False):
    """tests/test_gpu_model._build, with every key of the model (the joint-CTC head's as well) in the oracle's dict.  For
    training, the decoder embedding is scaled by 0.12 as tests/test_gpu_train._build does: it keeps the logits O(1)."""
    model, _ = tgm._build(params)
    if training:
        with torch.no_grad():
            model.decoder.embedding.weight.mul_(0.12)
    return model, {k: v.detach().cpu().float() for k, v in model.state_dict().items()}


def _ctc_params(encoder_type, frontend_type='concat'):
    p = tgc._params(encoder_type)
    p['frontend_type'] = frontend_type
    if frontend_type == 'concat':
        p['frontend'] = dict(input_size=64, left_frames=2, right_frames=1, frame_rate=20)           # n 4, s 2: 256 wide
    else:
        p['frontend'] = dict(input_size=80, output_size=256, left_frames=3, right_frames=0, frame_rate=40, dropout=0.0)
    return p


# Training inputs have std 0.1.  Under an abs-pos encoder the stacked features reach the first block multiplied by
# sqrt(d) = 16; unit-variance features then saturate its softmax, and the fp32 gradients of its projections hinge on the
# bf16 rounding of the forward, so the comparison with the fp32 restatement would measure that, not the implementation.
X_SCALE = 0.1


def _ctc_batch(Fd, B=3, T=200, L=10, lens=(200, 160, 181), V=40, seed=0, scale=X_SCALE):
    x, mask, tgt, tlen = tgc._batch(B, T, L, lens, V, seed)
    g = torch.Generator().manual_seed(seed + 100)
    x = scale * torch.randn(B, T, Fd, generator=g) * mask.unsqueeze(2)
    return x, mask, tgt, tlen


def _s2t_batch(seed=0):
    x, mask = tgm._batch(3, 200, 20, [200, 160, 181], seed=seed)
    _, _, tgt, tlen = tgc._batch(V=4234, seed=seed)
    return X_SCALE * x, mask, tgt, tlen


@pytest.mark.parametrize('kind', ['concat-with-linear', 'concat'])
def test_front_end_and_encoder_match_the_bf16_oracle(kind):
    if kind == 'concat-with-linear':
        params = _s2t_params(left=2, right=1, rate=30)          # n 4, s 3: n F 320
        model, sd = _s2t_build(params)
        Fd = 80
    else:
        params = _ctc_params('transformer')
        model, sd = tgc._build(params)
        Fd = 64
    x, mask = tgm._batch(4, 400, Fd, [400, 333, 250, 399])
    with cref.frontend_of(params):
        mem_ref, mmask, fe_ref, _ = om.encode(x, mask, sd, params, policy='bf16', return_layers=True)
    with torch.no_grad():
        fe, fmask = model.frontend(x.to(DEV), mask.to(DEV))
        mem, lens, B, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
    assert torch.equal(fmask.cpu(), mmask) and lens.cpu().tolist() == mmask.sum(1).tolist()
    assert T2 == model.frontend.output_length(400) == mmask.shape[1]
    r_fe, r_mem = _rel(fe.cpu(), fe_ref), _rel(mem.float().view(B, T2, -1).cpu()[mmask], mem_ref[mmask])
    print(f'{kind}: front end rel_l2 {r_fe:.3e}, encoder rel_l2 {r_mem:.3e}')
    if kind == 'concat':           # the stacked features, rounded once to bf16
        assert torch.equal(fe.cpu(), fe_ref.to(torch.bfloat16).float())
    assert r_fe < 1e-2 and r_mem < REL_L2_STATES


def _graph_lockstep(model, sd, params, x, mask, beam, max_len):
    """The per-step graph path of BeamDecoder driven against the oracle's beam_step: ids, parents and scores bit-exact."""
    B = x.shape[0]
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
        bd = BeamDecoder(model.decoder, B, beam, T2, max_len, DEV, use_graph=True, keep_logp=True)
        assert not bd.persistent
        bd.setup(mem, lens)
        preds = torch.full((B * beam, 1), 1, dtype=torch.long)
        scores = torch.tensor([0.0] + [float('-inf')] * (beam - 1)).repeat(B).unsqueeze(1)
        flag = torch.zeros_like(scores, dtype=torch.bool)
        for s in range(max_len):
            bd.step()
            preds, scores, flag = obs.beam_step(bd.logp.cpu(), preds, scores, flag, beam)
            assert torch.equal(bd.state.reconstruct(s + 1).cpu(), preds), f'token/parent ids differ at step {s}'
            assert torch.equal(bd.state.scores.cpu(), scores.view(-1)), f'scores differ at step {s}'
    return T2


def test_recognizer_lockstep_persistent_and_graph_paths():
    """T' <= 256 (n 4, s 4 on 1000 frames: 250) takes the persistent kernel; s 3 gives T' 333 > 256, which takes the
    per-step graph path, as the conv front end's long batches do."""
    params = _s2t_params()
    model, sd = _s2t_build(params)
    x, mask = tgm._batch(3, 1000, 80, [1000, 801, 977])
    tgm._lockstep_persistent(model, sd, params, x, mask, 3, 4, 8)
    rec = SpeechToTextRecognizer(model, beam_width=4, nbest=1, max_len=8, penalty=0.6, lamda=5, ngpu=1)
    rec.recognize_ids(x.to(DEV), mask.to(DEV))
    assert next(iter(rec._decoders.values())).persistent
    params3 = _s2t_params(left=3, right=0, rate=30)
    model3, sd3 = _s2t_build(params3)
    assert _graph_lockstep(model3, sd3, params3, x, mask, 4, 8) == 333
    rec3 = SpeechToTextRecognizer(model3, beam_width=4, nbest=1, max_len=8, penalty=0.6, lamda=5, ngpu=1)
    rec3.recognize_ids(x.to(DEV), mask.to(DEV))
    assert not next(iter(rec3._decoders.values())).persistent


@pytest.mark.parametrize('mode,beam', [('greedy', 1), ('beam', 10)])
def test_ctc_recognizer_and_spans(mode, beam):
    """CTCRecognizer over a concat front end: its ids are exactly the restatement's decode of the model's own log-probs,
    which follow the bf16-policy oracle; recognize_spans' windows, through encoder_frames_to_input, hold the stacked
    frames of each token."""
    params = _ctc_params('transformer')
    model, sd = tgc._build(params)
    x, mask, _, _ = _ctc_batch(64, scale=1.0)
    rec = CTCRecognizer(model, beam_width=beam, mode=mode, idx2unit={i: f'u{i}' for i in range(40)})
    ids, nout, _ = rec.recognize_ids(x.to(DEV), mask.to(DEV))
    with torch.no_grad():
        lp, n = model.inference(x.to(DEV), mask.to(DEV))
        logits, _, B, T2 = model.logits_bf16(x.to(DEV), mask.to(DEV))
    with cref.frontend_of(params):
        lp_ref, n_ref = ctc_ref.log_probs(x, mask, sd, params, policy='bf16')
    assert torch.equal(n.cpu().long(), n_ref.long())
    valid = torch.arange(T2)[None] < n_ref[:, None]
    assert _rel(lp.cpu()[valid], lp_ref[valid]) < 2e-2
    lp_c = lp.cpu()
    if mode == 'beam':
        lp_k, tok_k = ops.ctc_frame_topk(logits, B, T2, 40, n, 40)
        lp_k, tok_k = lp_k.view(B, T2, -1).cpu(), tok_k.view(B, T2, -1).cpu()
    for b in range(B):
        L = int(n[b])
        if mode == 'greedy':
            own = ctc_ref.greedy_collapse(lp_c[b].argmax(-1), L)
        else:
            fr = [list(zip(tok_k[b, t].tolist(), lp_k[b, t].tolist())) for t in range(L)]
            own = list(ctc_ref.prefix_beam_search(fr, beam, fp32=True)[0][0])
        assert ids[b, 0, :int(nout[b, 0])].tolist() == own, b
    _, _, _, spans = rec.recognize_spans(x.to(DEV), mask.to(DEV))
    fe = model.frontend
    win = encoder_frames_to_input(spans.cpu(), frontend=fe)
    s, nfr = fe.stride, fe.nframes
    for b in range(B):
        for k in range(int(nout[b, 0])):
            t0, t1 = spans[b, k].tolist()
            if t0 < 0:
                continue
            assert win[b, k].tolist() == [s * t0, s * (t1 - 1) + nfr]
            for t in range(t0, t1):                # every stacked frame of the token's encoder frames lies in the window
                assert win[b, k, 0] <= s * t and s * t + nfr <= win[b, k, 1]


# ------------------------------------------------------------------------------------------------ training
def _compare_grads(g, g_ref, names, label):
    zero = [n for n in names if n.endswith('depthwise_conv.bias')]
    worst = sorted(((_rel(g[n], g_ref[n]), n) for n in names if n not in zero), reverse=True)
    print(f'{label}: worst ' + ', '.join(f'{n} {r:.2e}' for r, n in worst[:4]))
    assert worst[0][0] < REL_L2_GRAD, worst[:3]


def test_speech2text_training_matches_restatement():
    """concat-with-linear (n 3, s 3: n F 60, K padded to 64) + Transformer encoder + joint CTC: the loss and every
    gradient, frontend.linear.* included, through forward_backward and through the loss.backward() seam."""
    params = _s2t_params(left=1, right=1, rate=30, F_in=20, ctc=0.3)
    params['encoder']['residual_dropout'] = params['decoder']['residual_dropout'] = 0.0
    model, sd = _s2t_build(params, training=True)
    x, mask, tgt, tlen = _s2t_batch()
    loss_ref, g_ref = cref.speech2text_loss_and_grads(x, mask, tgt, tlen, sd, params)
    model.train()
    with torch.no_grad():
        loss, g = train.forward_backward(model, x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV))
    names = [n for n, _ in model.named_parameters()]
    assert set(g) == set(names) and 'frontend.linear.weight' in g
    assert tuple(g['frontend.linear.weight'].shape) == (256, 60)
    assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    _compare_grads(g, g_ref, names, 'speech2text concat-with-linear')
    for p in model.parameters():
        p.grad = None
    lo, _ = model({'inputs': x.to(DEV), 'mask': mask.to(DEV)}, {'targets': tgt.to(DEV), 'targets_length': tlen.to(DEV)})
    lo.backward()
    assert _rel(model.frontend.linear.weight.grad, g_ref['frontend.linear.weight']) < REL_L2_GRAD


@pytest.mark.parametrize('encoder_type,frontend_type', [('conformer', 'concat'), ('transformer', 'concat'),
                                                        ('conformer', 'concat-with-linear')])
def test_ctc_model_training_matches_restatement(encoder_type, frontend_type):
    params = _ctc_params(encoder_type, frontend_type)
    model, sd = tgc._build(params)
    Fd = params['frontend']['input_size']
    x, mask, tgt, tlen = _ctc_batch(Fd)
    with cref.frontend_of(params):
        loss_ref, g_ref, stats_ref = ctc_ref.loss_and_grads_train(x, mask, tgt, tlen, sd, params)
    with torch.no_grad():
        loss, g = train.ctc_forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV))
    want = {n for n, v in g_ref.items() if v is not None}
    assert set(g) == want
    assert any(n.startswith('frontend.') for n in g) == (frontend_type == 'concat-with-linear')
    assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    _compare_grads(g, g_ref, sorted(g), f'ctc {encoder_type} {frontend_type}')
    bufs = dict(model.named_buffers())
    for n, v in stats_ref.items():
        assert _rel(bufs[n], v) < 1e-3, n


def test_fused_trainer_graph_equals_eager():
    """A few FusedTrainer steps give the same weights with the CUDA graph on and off."""
    params = _s2t_params(left=1, right=1, rate=30, F_in=20, ctc=0.3)
    weights = []
    for use_graph in (False, True):
        model, _ = _s2t_build(params, training=True)
        tr = train.FusedTrainer(model.train(), clip_grad=5.0, accum_steps=1, use_graph=use_graph)
        for step in range(3):
            x, mask, tgt, tlen = _s2t_batch(seed=step)
            tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV), truth_length=tlen.to(DEV))
        torch.cuda.synchronize()
        weights.append({n: p.detach().cpu().clone() for n, p in model.named_parameters()})
    worst = max(float((weights[0][n] - weights[1][n]).abs().max()) for n in weights[0])
    print(f'graph vs eager after 3 steps: max |dw| {worst:.2e}')
    assert worst < 1e-6


def test_fused_trainer_follows_the_oracle_step():
    """Two optimizer steps (2 accumulated micro-batches each) of a concat CTCModel: clip + Adam as the reference trainer."""
    params = _ctc_params('transformer', 'concat-with-linear')
    model, sd = tgc._build(params)
    tr = train.FusedTrainer(model.train(), clip_grad=0.05, accum_steps=2, use_graph=True)
    names = [n for n, _ in tr.params]
    w = {n: sd[n].clone() for n in names}
    m = {n: torch.zeros_like(w[n]) for n in names}
    v = {n: torch.zeros_like(w[n]) for n in names}
    for opt_step in (1, 2):
        acc = None
        for micro in range(2):
            x, mask, tgt, tlen = _ctc_batch(80, seed=10 * opt_step + micro)
            tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV))
            sd_now = dict(sd)
            sd_now.update(w)
            with cref.frontend_of(params):
                _, g_ref, _ = ctc_ref.loss_and_grads_train(x, mask, tgt, tlen, sd_now, params)
            acc = {n: g_ref[n] / 2 for n in names} if acc is None else {n: acc[n] + g_ref[n] / 2 for n in names}
        ot.clip_and_adam(w, acc, m, v, opt_step, ot.transformer_lr(ot.first_step_index() + opt_step - 1, 256, 12000), 0.05)
        torch.cuda.synchronize()
        p = dict(model.named_parameters())
        num = sum(float(((p[n].detach().cpu() - w[n]) ** 2).sum()) for n in names)
        den = sum(float(((w[n] - sd[n]) ** 2).sum()) for n in names)
        print(f'step {opt_step}: rel {(num / den) ** 0.5:.3e}')
        assert (num / den) ** 0.5 < 0.3


def test_mixspeech_step_matches_oracle():
    """One MixSpeech micro-step (features mixed before the front end) against the oracle at the same lambda."""
    params = _ctc_params('transformer', 'concat-with-linear')
    model, sd = tgc._build(params)
    x, mask, tgt, tlen = _ctc_batch(80, B=4, lens=(200, 160, 181, 120))
    tr = train.FusedTrainer(model.train(), accum_steps=2, use_graph=False, mixspeech=True)
    loss = tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV), truth_length=tlen.to(DEV))
    lam = float(tr.last_lambda)
    xm, mm = tor.mix(x, mask, lam)
    xm, mm = torch.from_numpy(xm), torch.from_numpy(mm)
    losses, grads = [], []
    for k in range(2):
        with cref.frontend_of(params):
            l_k, g_k, _ = ctc_ref.loss_and_grads_train(xm, mm, tgt[k::2], tlen[k::2], sd, params)
        losses.append(float(l_k))
        grads.append(g_k)
    loss_ref = lam * losses[0] + (1 - lam) * losses[1]
    names = [n for n, _ in tr.params]
    g = {n: 2.0 * tr.sink[n] for n in names}
    g_ref = {n: lam * grads[0][n] + (1 - lam) * grads[1][n] for n in names}
    assert abs(float(loss) - loss_ref) < 2e-2 * abs(loss_ref)
    _compare_grads(g, g_ref, names, f'mixspeech lambda {lam:.3f}')
