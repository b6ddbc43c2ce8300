"""GPU checks of the conv front end at kernel sizes and strides other than the shipped 3x3 / stride 2: conv1 and the conv2
implicit GEMM against F.conv2d on the same bf16 operands, the backward chain (im2col, col2im + ReLU', conv1's weight
gradient) against autograd, the recognizers and recognize_spans against the bf16-policy oracle, and training
(forward_backward, ctc_forward_backward, FusedTrainer with and without the graph) against the fp32 restatement and the
reference's own gradients (tests/golden/live_ref_conv_frontend.pt)."""
import copy
import os

import pytest
import torch
import torch.nn.functional as F

from tests import concat_frontend_ref as cref
from tests import conv_frontend_ref as vref
from tests import ctc_ref
from tests.test_head_dim_96 import synth_state_dict
from tests.test_transformer_lm_ref import sample

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops, train
    from opentransformer_b200.model import CTCModel, SpeechToText, encoder_frames_to_input
    from opentransformer_b200.recognize import CTCRecognizer, SpeechToTextRecognizer
    from tests import test_gpu_ctc_model as tgc
    from tests import test_gpu_model as tgm
    from tests import test_gpu_train as ttr
    DEV = torch.device('cuda:0')

from oracle import speech_model as om

BF = torch.bfloat16
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'live_ref_conv_frontend.pt')
# (kernel_size, stride) as a YAML writes them: shipped, 6x, [[5,5],[3,3]] at [3,2], [1,2], asymmetric pairs
GEOMETRIES = [([[3, 3], [3, 3]], [2, 2]), ([[3, 3], [3, 3]], [2, 3]), ([[5, 5], [3, 3]], [3, 2]), ([[3, 3], [3, 3]], [1, 2]),
              ([[3, 5], [5, 3]], [[2, 1], [2, 2]]), ([[7, 7], [2, 4]], [[1, 4], [4, 1]])]
IDS = ['shipped', '6x', 'k5k3-s3s2', 's1s2', 'asym', 'k7k2-wide']
REL_L2_STATES = 2e-2
REL_L2_GRAD = 4e-2


def _rel(a, b):
    return float((a.float().cpu() - b.float().cpu()).norm() / (b.float().cpu().norm() + 1e-20))


def _geom(ks, st):
    (k1, s1), (k2, s2) = vref.layers({'kernel_size': ks, 'stride': st})
    return (*k1, *s1, *k2, *s2)


def _rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize('ks,st', GEOMETRIES, ids=IDS)
@pytest.mark.parametrize('C1', [64, 96, 256])
def test_conv1_and_conv2_match_conv2d(ks, st, C1):
    """Ragged batch; conv1 on fp32 inputs (bf16 output), conv2 on the same bf16 operands as F.conv2d; the right frequency
    padding conv2 reads is zero.  C1 96 runs conv2 on its 128-channel zero-padded buffer, as the module does."""
    geom = _geom(ks, st)
    kt1, kf1, st1, sf1, kt2, kf2, st2, sf2 = geom
    B, T, Fd, C2 = 3, 157, 80, 64
    x = _rnd(B, T, Fd, seed=1)
    x[1, 120:] = 0
    T1, F1, T2, F2, T1p, F1p = ops.conv_sizes(T, Fd, geom)
    C1p = (C1 + 63) // 64 * 64
    w1 = torch.zeros(C1p, 1, kt1, kf1, device=DEV)
    w1[:C1] = _rnd(C1, 1, kt1, kf1, scale=0.3, seed=2)
    b1 = torch.zeros(C1p, device=DEV)
    b1[:C1] = _rnd(C1, scale=0.1, seed=3)
    h1 = ops.conv1_relu(x, w1, b1, geom=geom)
    assert tuple(h1.shape) == (B, T1p, F1p, C1p)
    r1 = torch.relu(F.conv2d(x.unsqueeze(1), w1, b1, stride=(st1, sf1), padding=(0, kf1 // 2)))
    assert r1.shape[2:] == (T1, F1)
    got1 = h1[:, :T1, :F1].permute(0, 3, 1, 2).float()
    assert _rel(got1, r1) < 4e-3
    assert float(h1[:, :T1, F1:].float().abs().sum()) == 0.0
    w2 = _rnd(C2, C1p, kt2, kf2, scale=(kt2 * kf2 * C1) ** -0.5, seed=4)
    w2[:, C1:] = 0
    b2 = _rnd(C2, scale=0.1, seed=5)
    w2p = w2.permute(0, 2, 3, 1).reshape(C2, kt2 * kf2 * C1p).to(BF).contiguous()
    h2 = ops.conv2_relu(h1, w2p, b2, B, T, Fd, geom=geom)
    r2 = torch.relu(F.conv2d(got1, w2.to(BF).float(), b2, stride=(st2, sf2), padding=(0, kf2 // 2)))   # [B,C2,T2,F2]
    want = r2.permute(0, 2, 3, 1).reshape(B * T2, F2 * C2)
    assert _rel(h2, want) < 4e-3, _rel(h2, want)


@pytest.mark.parametrize('ks,st', [([[3, 3], [3, 3]], [1, 2]), ([[1, 3], [3, 3]], [[1, 1], [1, 2]])], ids=['s1s2', 'f128'])
def test_conv2_with_f2_near_128(ks, st):
    """F2 127 and 128: one output row per M tile, the widest TMA box conv2 takes; F2 129 is refused."""
    geom = _geom(ks, st)
    for Fd, ok in ((253, True), (255, True), (257, False)):
        T1, F1, T2, F2, _, _ = ops.conv_sizes(60, Fd, geom)
        x = _rnd(2, 60, Fd, seed=Fd)
        w1, b1 = _rnd(64, 1, geom[0], geom[1], scale=0.3, seed=6), _rnd(64, scale=0.1, seed=7)
        h1 = ops.conv1_relu(x, w1, b1, geom=geom)
        w2 = _rnd(16, 64, 3, 3, scale=(9 * 64) ** -0.5, seed=8)
        w2p = w2.permute(0, 2, 3, 1).reshape(16, 9 * 64).to(BF).contiguous()
        if not ok:
            with pytest.raises(RuntimeError, match='F2 > 128'):
                ops.conv2_relu(h1, w2p, b1[:16].contiguous(), 2, 60, Fd, geom=geom)
            continue
        h2 = ops.conv2_relu(h1, w2p, b1[:16].contiguous(), 2, 60, Fd, geom=geom)
        r1 = h1[:, :T1, :F1].permute(0, 3, 1, 2).float()
        r2 = torch.relu(F.conv2d(r1, w2.to(BF).float(), b1[:16], stride=(geom[6], geom[7]), padding=(0, 1)))
        assert F2 in (127, 128) and _rel(h2, r2.permute(0, 2, 3, 1).reshape(2 * T2, F2 * 16)) < 4e-3


@pytest.mark.parametrize('ks,st', GEOMETRIES, ids=IDS)
def test_backward_chain_matches_autograd(ks, st):
    """dW2 (= dpre2^T im2col), dcol -> col2im + ReLU' -> dpre1, conv1's tap and bias gradients, against autograd of the
    fp32 convolutions on the kernels' own bf16 activations."""
    geom = _geom(ks, st)
    kt1, kf1, st1, sf1, kt2, kf2, st2, sf2 = geom
    B, T, Fd, C1, C2 = 2, 131, 40, 64, 32
    x = _rnd(B, T, Fd, seed=11)
    T1, F1, T2, F2, _, _ = ops.conv_sizes(T, Fd, geom)
    w1, b1 = _rnd(C1, 1, kt1, kf1, scale=0.3, seed=12), _rnd(C1, scale=0.1, seed=13)
    w2 = _rnd(C2, C1, kt2, kf2, scale=(kt2 * kf2 * C1) ** -0.5, seed=14)
    h1 = ops.conv1_relu(x, w1, b1, geom=geom)
    dpre2 = _rnd(B * T2 * F2, C2, scale=0.1, seed=15).to(BF)
    col = ops.conv_im2col(h1, B, T, Fd, C1, geom=geom)
    dw2 = ops.linear_wgrad(dpre2, col).view(C2, kt2, kf2, C1).permute(0, 3, 1, 2)
    w2p = w2.permute(0, 2, 3, 1).reshape(C2, kt2 * kf2 * C1).to(BF)
    dcol = ops.linear(dpre2, w2p.t().contiguous())
    dpre1 = ops.conv_col2im_relu(dcol, h1, B, T, Fd, C1, geom=geom)
    g1 = ops.conv1_wgrad(dpre1, x, B, T, Fd, C1, geom=geom)
    # autograd on the same operands
    a1 = h1[:, :T1, :F1].permute(0, 3, 1, 2).float().requires_grad_(True)
    w2r = w2.to(BF).float().requires_grad_(True)
    y2 = F.conv2d(a1, w2r, None, stride=(st2, sf2), padding=(0, kf2 // 2))
    y2.backward(dpre2.float().view(B, T2, F2, C2).permute(0, 3, 1, 2))
    assert _rel(dw2, w2r.grad) < 1e-2
    da1 = a1.grad * (a1.detach() > 0)
    got = dpre1[:, :T1, :F1].permute(0, 3, 1, 2)
    assert _rel(got, da1) < 1e-2
    assert float(dpre1[:, T1:].float().abs().sum()) == 0.0 and float(dpre1[:, :, F1:].float().abs().sum()) == 0.0
    w1r, b1r = w1.clone().requires_grad_(True), b1.clone().requires_grad_(True)
    y1 = F.conv2d(x.unsqueeze(1), w1r, b1r, stride=(st1, sf1), padding=(0, kf1 // 2))
    y1.backward(got.float())
    assert tuple(g1.shape) == (C1, kt1 * kf1 + 1)
    assert _rel(g1[:, :kt1 * kf1].reshape(C1, 1, kt1, kf1), w1r.grad) < 1e-3 and _rel(g1[:, -1], b1r.grad) < 1e-3


# ------------------------------------------------------------------------------------------------ models
def _s2t(ks, st, mid=64, ln=False):
    p = tgm._params(n_enc=2, n_dec=2)
    p['frontend'].update(kernel_size=ks, stride=st, mid_channel=mid, front_end_layer_norm=ln)
    return p


@pytest.mark.parametrize('ks,st', GEOMETRIES, ids=IDS)
def test_front_end_and_encoder_match_the_bf16_oracle(ks, st):
    params = _s2t(ks, st, mid=96, ln=ks[0] == [5, 5])
    model, sd = tgm._build(params)
    x, mask = tgm._batch(4, 400, 80, [400, 333, 250, 399])
    with vref.conv_frontend_of(params):
        mem_ref, mmask, fe_ref, _ = om.encode(x, mask, sd, params, policy='bf16', return_layers=True)
    with torch.no_grad():
        fe, fmask = model.frontend(x.to(DEV), mask.to(DEV))
        mem, lens, B, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
    assert torch.equal(fmask.cpu(), mmask) and lens.cpu().tolist() == mmask.sum(1).tolist()
    assert T2 == model.frontend.output_length(400) == mmask.shape[1]
    r_fe, r_mem = _rel(fe, fe_ref), _rel(mem.float().view(B, T2, -1).cpu()[mmask], mem_ref[mmask])
    print(f'{ks} {st}: T2 {T2}, front end rel_l2 {r_fe:.3e}, encoder rel_l2 {r_mem:.3e}')
    assert r_fe < 1e-2 and r_mem < REL_L2_STATES


@pytest.mark.parametrize('ks,st', GEOMETRIES[1:3], ids=IDS[1:3])
def test_recognizer_lockstep(ks, st):
    """The persistent decode kernel in lock-step with the oracle's beam step over a 6x front end, and the public call."""
    params = _s2t(ks, st)
    model, sd = tgm._build(params)
    x, mask = tgm._batch(3, 600, 80, [600, 451, 577])
    with vref.conv_frontend_of(params):
        tgm._lockstep_persistent(model, sd, params, x, mask, 3, 4, 8)
    rec = SpeechToTextRecognizer(model, beam_width=4, nbest=1, max_len=8, penalty=0.6, lamda=5, ngpu=1)
    ids, _, n = rec.recognize_ids(x.to(DEV), mask.to(DEV))
    assert n == 8 and ids.shape == (3, 1, 8)


@pytest.mark.parametrize('ks,st', [GEOMETRIES[1], GEOMETRIES[4]], ids=['6x', 'asym'])
def test_ctc_recognizer_and_spans(ks, st):
    params = tgc._params('transformer')
    params['frontend'].update(kernel_size=ks, stride=st)
    model, sd = tgc._build(params)
    x, mask, _, _ = tgc._batch()
    rec = CTCRecognizer(model, beam_width=1, mode='greedy', idx2unit={i: f'u{i}' for i in range(40)})
    ids, nout, _ = rec.recognize_ids(x.to(DEV), mask.to(DEV))
    with torch.no_grad():
        lp, n = model.inference(x.to(DEV), mask.to(DEV))
    with vref.conv_frontend_of(params):
        lp_ref, n_ref = ctc_ref.log_probs(x, mask, sd, params, policy='bf16')
    assert torch.equal(n.cpu().long(), n_ref.long())
    valid = torch.arange(lp.shape[1])[None] < n_ref[:, None]
    assert _rel(lp.cpu()[valid], lp_ref[valid]) < 2e-2
    for b in range(x.shape[0]):
        assert ids[b, 0, :int(nout[b, 0])].tolist() == ctc_ref.greedy_collapse(lp.cpu()[b].argmax(-1), int(n[b]))
    _, _, _, spans = rec.recognize_spans(x.to(DEV), mask.to(DEV))
    s, w = model.frontend.input_window()
    win = encoder_frames_to_input(spans.cpu(), frontend=model.frontend)
    for b in range(x.shape[0]):
        for k in range(int(nout[b, 0])):
            t0, t1 = spans[b, k].tolist()
            if t0 >= 0:
                assert win[b, k].tolist() == [s * t0, s * (t1 - 1) + w]


# ------------------------------------------------------------------------------------------------ training
def _compare_grads(g, g_ref, names, label):
    worst = sorted(((_rel(g[n], g_ref[n]), n) for n in names), reverse=True)
    print(f'{label}: worst ' + ', '.join(f'{n} {r:.2e}' for r, n in worst[:4]))
    assert worst[0][0] < REL_L2_GRAD, worst[:3]


def _s2t_train_batch(seed=0):
    x, mask, tgt = ttr._batch(T=300, lens=(300, 260, 281), seed=seed)
    return x, mask, tgt, (tgt[:, 1:] != 0).sum(1)


def _s2t_train(ks, st, ln):
    """tests/test_gpu_train's model (dropout 0, embedding scaled so that the logits stay O(1)) with joint CTC 0.3."""
    params = ttr._params()
    params['frontend'].update(kernel_size=ks, stride=st, front_end_layer_norm=ln)
    params.update(ctc_weight=0.3, encoder_output_size=256)
    params['decoder']['share_embedding'] = False
    model, _ = ttr._build(params)
    if ln:      # unit-variance features times sqrt(d) saturate the first block's softmax, as unscaled inputs would
        with torch.no_grad():
            model.frontend.layer_norm.weight.mul_(0.1)
    return params, model, {k: v.detach().cpu().float() for k, v in model.state_dict().items()}


@pytest.mark.parametrize('ks,st,ln', [(*GEOMETRIES[1], True), (*GEOMETRIES[4], False)], ids=['6x-ln', 'asym'])
def test_speech2text_training_matches_restatement(ks, st, ln):
    """forward_backward and the loss.backward() seam: loss and every gradient, frontend.* included."""
    params, model, sd = _s2t_train(ks, st, ln)
    x, mask, tgt, tlen = _s2t_train_batch()
    with vref.conv_frontend_of(params):
        loss_ref, g_ref = cref.speech2text_loss_and_grads(x, mask, tgt, tlen, sd, params)
    model.train()
    with torch.no_grad():
        loss, g = train.forward_backward(model, x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV))
    names = [n for n, _ in model.named_parameters()]
    assert set(g) == set(names) and ('frontend.layer_norm.weight' in g) == ln
    assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    # the front end and the encoder at the per-parameter bound; the decoder's cross-attention query projections, whose
    # small gradients hinge on the bf16 rounding of the memory, within 1e-1; all gradients together within 2e-2
    _compare_grads(g, g_ref, [n for n in names if not n.startswith('decoder.')], f'speech2text {ks} {st}')
    assert max(_rel(g[n], g_ref[n]) for n in names if n.startswith('decoder.')) < 1e-1
    r_all = _rel(torch.cat([g[n].reshape(-1).cpu() for n in names]), torch.cat([g_ref[n].reshape(-1) for n in names]))
    assert r_all < 2e-2, r_all
    for p in model.parameters():
        p.grad = None
    lo, _ = model({'inputs': x.to(DEV), 'mask': mask.to(DEV)}, {'targets': tgt.to(DEV), 'targets_length': tlen.to(DEV)})
    lo.backward()
    assert _rel(model.frontend.conv1.conv_layer.weight.grad, g_ref['frontend.conv1.conv_layer.weight']) < REL_L2_GRAD


@pytest.mark.parametrize('ks,st', GEOMETRIES[1:], ids=IDS[1:])
def test_ctc_model_training_matches_restatement(ks, st):
    params = tgc._params('transformer')
    params['frontend'].update(kernel_size=ks, stride=st)
    model, sd = tgc._build(params)
    x, mask, tgt, tlen = tgc._batch()
    x = 0.1 * x
    with vref.conv_frontend_of(params):
        loss_ref, g_ref, _ = ctc_ref.loss_and_grads_train(x, mask, tgt, tlen, sd, params)
    with torch.no_grad():
        loss, g = train.ctc_forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV))
    assert set(g) == {n for n, v in g_ref.items() if v is not None}
    assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    _compare_grads(g, g_ref, sorted(g), f'ctc {ks} {st}')


@pytest.mark.parametrize('kind', ['speech2text', 'ctc'])
def test_training_matches_the_live_reference(kind):
    """The reference's own loss and gradients (6x geometries, front_end_layer_norm in speech2text) against the port's
    forward_backward / ctc_forward_backward."""
    c = torch.load(GOLDEN, weights_only=False)[kind]
    sd = synth_state_dict(c['sd_shapes'], c['sd_seed'])
    model = (SpeechToText if kind == 'speech2text' else CTCModel)(c['params'])
    model.load_state_dict(sd, strict=True)
    model.to(DEV).train()
    args = (c['x'].to(DEV), c['mask'].to(DEV), c['tgt'].to(DEV), c['tlen'].to(DEV))
    with torch.no_grad():
        loss, g = (train.forward_backward if kind == 'speech2text' else train.ctc_forward_backward)(model, *args)
    assert abs(float(loss) - float(c['loss_ref'])) < 2e-2 * abs(float(c['loss_ref']))
    want = {n: v for n, v in c['g_ref'].items() if v is not None}
    assert set(g) == set(want)
    worst = sorted(((_rel(sample(g[n].float().cpu()), v), n) for n, v in want.items()), reverse=True)
    print(f'{kind} vs the live reference: worst ' + ', '.join(f'{n} {r:.2e}' for r, n in worst[:4]))
    assert worst[0][0] < REL_L2_GRAD, worst[:3]


def test_fused_trainer_graph_equals_eager_and_mixspeech_runs():
    """A few FusedTrainer steps at the asymmetric geometry with front_end_layer_norm give the same weights with the CUDA
    graph on and off; a MixSpeech step at the 6x geometry runs and moves the weights."""
    weights = []
    for use_graph in (False, True):
        _, model, _ = _s2t_train(*GEOMETRIES[4], True)
        tr = train.FusedTrainer(model.train(), clip_grad=5.0, accum_steps=1, use_graph=use_graph)
        for step in range(3):
            x, mask, tgt, tlen = _s2t_train_batch(seed=step)
            tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV), truth_length=tlen.to(DEV))
        torch.cuda.synchronize()
        weights.append({n: p.detach().cpu().clone() for n, p in model.named_parameters()})
    worst = max(float((weights[0][n] - weights[1][n]).abs().max()) for n in weights[0])
    print(f'graph vs eager after 3 steps: max |dw| {worst:.2e}')
    assert worst < 1e-6
    params = tgc._params('transformer')
    params['frontend'].update(kernel_size=GEOMETRIES[1][0], stride=GEOMETRIES[1][1])
    model, sd = tgc._build(params)
    x, mask, tgt, tlen = tgc._batch(B=4, lens=(200, 160, 181, 120))
    tr = train.FusedTrainer(model.train(), accum_steps=2, use_graph=False, mixspeech=True)
    loss = tr.step(0.1 * x.to(DEV), mask.to(DEV), tgt.to(DEV), truth_length=tlen.to(DEV))
    assert torch.isfinite(torch.as_tensor(float(loss)))
    assert all(torch.isfinite(tr.sink[n]).all() for n, _ in tr.params)
    assert float(tr.sink['frontend.conv1.conv_layer.weight'].abs().sum()) > 0


def test_dropout_front_end_recognizes_like_dropout_zero():
    params = _s2t(*GEOMETRIES[2])
    model, _ = tgm._build(params)
    p2 = copy.deepcopy(params)
    p2['frontend']['dropout'] = 0.1
    m2 = SpeechToText(p2).eval()
    m2.load_state_dict(model.state_dict())
    m2.to(DEV)
    x, mask = tgm._batch(2, 300, 80, [300, 211])
    with torch.no_grad():
        a = model.encode_bf16(x.to(DEV), mask.to(DEV))[0]
        b = m2.encode_bf16(x.to(DEV), mask.to(DEV))[0]
    assert torch.equal(a, b)
