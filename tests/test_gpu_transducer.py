"""The transducer on the GPU: each kernel of csrc/rnnt.cu on its own operands against float64, the chunked output layer,
the whole training pass against the bf16-policy restatement (tests/rnnt_ref.py), the training entry points, and greedy
search in lockstep with a restatement driven by the GPU's own joint log-probs."""
import pytest
import torch

from opentransformer_b200 import ops, train
from opentransformer_b200.model import TransducerModel
from opentransformer_b200.recognize import TransducerRecognizer
from oracle import train_step as ot
from tests import rnnt_ref
from tests.test_rnnt_ref import params

pytestmark = pytest.mark.gpu
DEV = 'cuda'
REL_L2_GRAD = 4e-2


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _ulp_bf16(x):
    """One bf16 ulp at |x| (float64)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def _bf(x):
    return x.to(ops.BF16).double()


def _lens(t, u):
    return torch.tensor(t, dtype=torch.int32, device=DEV), torch.tensor(u, dtype=torch.int32, device=DEV)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize('B,T,U1,D,t_len,u_len', [(3, 5, 4, 64, [5, 1, 3], [3, 0, 2]), (2, 7, 9, 520, [7, 6], [8, 1])])
def test_joint_matches_float64(B, T, U1, D, t_len, u_len):
    g = torch.Generator().manual_seed(D)
    ep = torch.randn(B * T, D, generator=g).to(ops.BF16).to(DEV)
    pp = torch.randn(B * U1, D, generator=g).to(ops.BF16).to(DEV)
    tl, ul = _lens(t_len, u_len)
    out = ops.rnnt_joint(ep, pp, B, T, U1, tl, ul).double().cpu().view(B, T, U1, D)
    want = torch.tanh(ep.double().cpu().view(B, T, 1, D) + pp.double().cpu().view(B, 1, U1, D))
    for b in range(B):
        want[b, t_len[b]:] = 0
        want[b, :, u_len[b] + 1:] = 0
    assert bool(((out - want).abs() <= _ulp_bf16(want)).all())
    full = ops.rnnt_joint(ep, pp, B, T, U1).double().cpu().view(B, T, U1, D)      # no lengths: every node
    assert bool(((full - torch.tanh(ep.double().cpu().view(B, T, 1, D) + pp.double().cpu().view(B, 1, U1, D))).abs()
                 <= _ulp_bf16(full)).all())


@pytest.mark.parametrize('B,T,U1,D,t_len,u_len', [(3, 5, 4, 64, [5, 1, 3], [3, 0, 2]), (2, 9, 6, 320, [9, 2], [5, 5])])
def test_joint_bwd_matches_float64(B, T, U1, D, t_len, u_len):
    g = torch.Generator().manual_seed(D + 1)
    h = torch.tanh(torch.randn(B * T * U1, D, generator=g)).to(ops.BF16)
    dh = torch.randn(B * T * U1, D, generator=g).to(ops.BF16)
    tl, ul = _lens(t_len, u_len)
    dep, dpp = ops.rnnt_joint_bwd(dh.to(DEV), h.to(DEV), B, T, U1, tl, ul)
    dz = (dh.double() * (1 - h.double() ** 2)).view(B, T, U1, D)
    for b in range(B):
        dz[b, t_len[b]:] = 0
        dz[b, :, u_len[b] + 1:] = 0
    # the bf16 outputs against the float64 sums rounded to bf16 (the rounding alone is a rel-L2 of about 1.5e-3)
    assert _rel(dep, _bf(dz.sum(2).reshape(B * T, D))) < 1e-3
    assert _rel(dpp, _bf(dz.sum(1).reshape(B * U1, D))) < 1e-3
    again = ops.rnnt_joint_bwd(dh.to(DEV), h.to(DEV), B, T, U1, tl, ul)
    assert torch.equal(again[0], dep) and torch.equal(again[1], dpp)


def _lattice(B, T, U1, V, t_len, u_len, seed, scale=2.0):
    g = torch.Generator().manual_seed(seed)
    ld = (V + 7) // 8 * 8
    logits = torch.full((B * T * U1, ld), float('nan'))
    logits[:, :V] = scale * torch.randn(B * T * U1, V, generator=g)
    labels = torch.randint(1, V, (B, max(U1 - 1, 1)), generator=g, dtype=torch.int32)
    return logits, labels, _lens(t_len, u_len)


def _ref_logprob(logits, labels, B, T, U1, V, t_len, u_len):
    x = logits[:, :V].double().view(B, T, U1, V)
    lse = torch.logsumexp(x, -1)
    lpb = x[..., 0] - lse
    lpy = torch.full((B, T, U1), float('-inf'), dtype=torch.float64)
    for b in range(B):
        for u in range(u_len[b]):
            lpy[b, :, u] = x[b, :, u, int(labels[b, u])] - lse[b, :, u]
    return lse, lpb, lpy


@pytest.mark.parametrize('chunk', [7, 13, 1000])
def test_logprob_matches_float64(chunk):
    B, T, U1, V = 3, 6, 5, 37
    t_len, u_len = [6, 1, 4], [4, 0, 2]
    logits, labels, (tl, ul) = _lattice(B, T, U1, V, t_len, u_len, seed=chunk)
    rows = B * T * U1
    lp = torch.full((rows, 3), float('nan'), device=DEV)
    for r0 in range(0, rows, chunk):            # chunk boundaries that cut utterances and frames
        ops.rnnt_logprob(logits[r0:r0 + chunk].to(DEV), r0, V, B, T, U1, tl, ul, labels.to(DEV), lp)
    lp = lp.cpu().double().view(B, T, U1, 3)
    lse, lpb, lpy = _ref_logprob(logits, labels, B, T, U1, V, t_len, u_len)
    for b in range(B):
        n = (slice(0, t_len[b]), slice(0, u_len[b] + 1))
        for k, want in ((0, lse), (1, lpb), (2, lpy)):
            got, w = lp[b][n][..., k], want[b][n]
            fin = torch.isfinite(w)
            assert torch.equal(torch.isfinite(got), fin)
            if bool(fin.any()):
                assert float(((got - w).abs()[fin] / w.abs()[fin].clamp_min(1.0)).max()) < 1e-6
        assert float(lp[b, t_len[b]:].abs().sum()) == 0 and float(lp[b, :, u_len[b] + 1:].abs().sum()) == 0


def _ref_node_grads(lpb, lpy, B, T, U1, t_len, u_len):
    """float64 autograd of the batch-mean loss with respect to every node's two log-probs."""
    gb, gy = torch.zeros(B, T, U1, dtype=torch.float64), torch.zeros(B, T, U1, dtype=torch.float64)
    nll = []
    for b in range(B):
        Tb, Ub = t_len[b], u_len[b]
        a = lpb[b, :Tb, :Ub + 1].clone().requires_grad_(True)
        c = lpy[b, :Tb, :Ub].clone().requires_grad_(True)
        loss = rnnt_ref.lattice_nll(a, c)
        (loss / B).backward()
        nll.append(float(loss))
        gb[b, :Tb, :Ub + 1] = a.grad
        gy[b, :Tb, :Ub] = c.grad
    return torch.tensor(nll, dtype=torch.float64), gb, gy


@pytest.mark.parametrize('case', ['ragged', 'long', 'short'])
def test_loss_and_node_grads_match_float64(case):
    if case == 'ragged':
        B, T, U1, t_len, u_len = 4, 9, 6, [9, 1, 5, 7], [5, 0, 3, 5]
    elif case == 'long':                    # U_b = 1023 labels
        B, T, U1, t_len, u_len = 2, 12, 1024, [12, 5], [1023, 40]
    else:                                   # T_b = 1 with labels, U_b = 0 with frames
        B, T, U1, t_len, u_len = 3, 4, 3, [1, 4, 1], [2, 0, 0]
    V = 11
    logits, labels, (tl, ul) = _lattice(B, T, U1, V, t_len, u_len, seed=U1)
    lp = torch.empty(B * T * U1, 3, device=DEV)
    ops.rnnt_logprob(logits.to(DEV), 0, V, B, T, U1, tl, ul, labels.to(DEV), lp)
    loss, nll, grad = ops.rnnt_loss(lp, B, T, U1, tl, ul, grad_scale=0.5)
    lp64 = lp.cpu().double().view(B, T, U1, 3)
    want_nll, gb, gy = _ref_node_grads(lp64[..., 1], lp64[..., 2], B, T, U1, t_len, u_len)
    assert float(((nll.cpu().double() - want_nll).abs() / want_nll.abs()).max()) < 1e-5
    assert abs(float(loss) - float(want_nll.mean())) < 1e-5 * float(want_nll.mean())
    grad = grad.cpu().double().view(B, T, U1, 2) / 0.5
    for got, want in ((grad[..., 0], gb), (grad[..., 1], gy)):
        err = (got - want).abs() / want.abs().max()
        assert float(err.max()) < 1e-5, float(err.max())
    # a device scale multiplies the host one
    _, _, g2 = ops.rnnt_loss(lp, B, T, U1, tl, ul, grad_scale=0.5, scale_dev=torch.tensor([2.0], device=DEV))
    _, _, g1 = ops.rnnt_loss(lp, B, T, U1, tl, ul, grad_scale=1.0)
    assert torch.equal(g2, g1)


def test_dlogits_matches_float64():
    B, T, U1, V = 2, 5, 4, 29
    t_len, u_len = [5, 3], [3, 1]
    logits, labels, (tl, ul) = _lattice(B, T, U1, V, t_len, u_len, seed=9)
    logits[:, V:] = 0.0
    rows = B * T * U1
    lp = torch.empty(rows, 3, device=DEV)
    ops.rnnt_logprob(logits.to(DEV), 0, V, B, T, U1, tl, ul, labels.to(DEV), lp)
    _, _, grad = ops.rnnt_loss(lp, B, T, U1, tl, ul)
    dz = torch.cat([ops.rnnt_dlogits(logits[r0:r0 + 11].to(DEV), r0, V, B, T, U1, tl, ul, labels.to(DEV), lp, grad)
                    for r0 in range(0, rows, 11)])
    x = logits[:, :V].double().view(B, T, U1, V).requires_grad_(True)
    loss = rnnt_ref.batch_loss(x, labels, torch.tensor(t_len), torch.tensor(u_len))
    loss.backward()
    want = torch.zeros(rows, dz.shape[1], dtype=torch.float64)
    want[:, :V] = x.grad.reshape(rows, V)
    assert _rel(dz, _bf(want)) < 1e-3
    assert float(dz[:, V:].float().abs().sum()) == 0


# ------------------------------------------------------------------------------------------------ the model
def _build(p, seed=1234):
    torch.manual_seed(seed)
    model = TransducerModel(p)
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for n, t in model.named_parameters():
            if 'norm' in n:
                t.add_(0.1 * torch.randn(t.shape, generator=g))
            elif n.endswith('.bias'):
                t.add_(0.05 * torch.randn(t.shape, generator=g))
        for n, b in model.named_buffers():
            if n.endswith('running_mean'):
                b.normal_(0.0, 0.1, generator=g)
            elif n.endswith('running_var'):
                b.uniform_(0.8, 1.2, generator=g)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    return model.to(DEV), sd


def _batch(B=3, T=120, L=9, lens=(120, 96, 109), V=40, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, 80, generator=g)
    lens = torch.tensor(lens)
    mask = torch.arange(T)[None] < lens[:, None]
    x = x * mask.unsqueeze(2)
    tgt = torch.randint(2, V, (B, L), generator=g)
    tgt[:, 0] = 1
    tgt[0, L - 3:] = torch.tensor([1, 0, 0])
    tgt[1, L - 1] = 1
    tgt[2, 2:] = torch.tensor([1] + [0] * (L - 3))          # one label
    return x, mask, tgt, (tgt[:, 1:] != 0).sum(1)


def _replay(model, B, T2, U1, p_enc, p_dec, seed):
    """The product's dropout masks, as the restatement's drop((prefix, k), tensor)."""
    masks = {}
    per = train._enc_sites(model.encoder)
    d = model.encoder.d_model
    if p_enc > 0:
        for i in range(len(model.encoder.blocks)):
            for k in range(per):
                m = ops.dropout_mask(B * T2, d, p_enc, seed, train.ENC_SITE + per * i + k).cpu().view(B, -1, d).float()
                masks[(f'encoder.blocks.{i}', k)] = m / (1.0 - p_enc)
    H = model.decoder.hidden_size
    for k in range(model.decoder.num_layers - 1):
        m = ops.dropout_mask(U1 * B, H, p_dec, seed, train.RNNT_SITE + k).cpu().view(U1, B, H).transpose(0, 1).float()
        masks[('decoder.rnn', k)] = m / (1.0 - p_dec)
    return lambda s, t: t * masks[s]


@pytest.mark.parametrize('encoder_type,layers,rate', [('transformer', 1, 0.0), ('transformer', 2, 0.1), ('conformer', 1, 0.0),
                                                      ('conformer', 2, 0.1)])
def test_training_matches_restatement(encoder_type, layers, rate):
    p = params(encoder_type, layers=layers, dropout=rate, rate=rate)
    model, sd = _build(p)
    x, mask, tgt, tlen = _batch()
    seed = torch.tensor([777], dtype=torch.int32, device=DEV)
    T2 = ops.conv_geometry(x.shape[1], 80)[2]
    drop = _replay(model, x.shape[0], T2, tgt.shape[1] - 1, rate, rate, seed) if rate > 0 else None
    loss_ref, g_ref, _ = rnnt_ref.loss_and_grads(x, mask, tgt, tlen, sd, p, drop=drop)
    with torch.no_grad():
        loss, g = train.transducer_forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV),
                                                    drop_seed=seed)
    assert set(g) == {n for n, _ in model.named_parameters() if g_ref[n] is not None}
    zero = [n for n in g if n.endswith('depthwise_conv.bias')]
    worst = sorted(((_rel(g[n], g_ref[n]), n) for n in g if n not in zero), reverse=True)
    print(f'{encoder_type} layers {layers} rate {rate}: loss gpu {float(loss):.5f} ref {float(loss_ref):.5f}; worst '
          + ', '.join(f'{n} {r:.2e}' for r, n in worst[:4]))
    assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    assert worst[0][0] < REL_L2_GRAD, worst[:3]


def test_chunked_output_layer_is_budget_independent():
    p = params()
    model, _ = _build(p)
    x, mask, tgt, tlen = _batch()
    pk = train.EncoderPack(model, with_decoder=False)
    op = train.transducer_operands(model, pk)
    out = []
    for budget in (None, 4 * 48 * 13):          # the default, and 13 rows per chunk (chunks cut frames and utterances)
        with torch.no_grad():
            mem, tr = train._encoder_fwd(model.train(), pk, x.to(DEV), mask.to(DEV), None)
            g = train.Grads()
            loss, dmem = train.transducer_head(model, op, mem, tr.B, tr.T2, tr.lengths, tgt.to(DEV), tlen.to(DEV), g=g,
                                               workspace_bytes=budget)
        out.append((loss, dmem, g))
    assert torch.equal(out[0][0], out[1][0])
    for n in out[0][2]:
        assert _rel(out[1][2][n], out[0][2][n]) < 1e-6, n
    assert _rel(out[1][1], out[0][1]) < 1e-2


def test_autograd_seam_and_modes():
    p = params()
    model, sd = _build(p)
    x, mask, tgt, tlen = _batch()
    inputs, targets = {'inputs': x.to(DEV), 'mask': mask.to(DEV)}, {'targets': tgt.to(DEV), 'targets_length': tlen.to(DEV)}
    model.train()
    loss, aux = model(inputs, targets)
    assert aux is None and loss.requires_grad
    (loss * 0.5).backward()
    loss_ref, g_ref, _ = rnnt_ref.loss_and_grads(x, mask, tgt, tlen, sd, p)
    used = [(n, t) for n, t in model.named_parameters()]
    assert all(t.grad is not None for _, t in used)
    r = _rel(torch.cat([t.grad.reshape(-1) for _, t in used]), 0.5 * torch.cat([g_ref[n].reshape(-1) for n, _ in used]))
    assert r < 2e-2, r
    with torch.no_grad():
        l_nograd, _ = model(inputs, targets)
        model.eval()
        l_eval, _ = model(inputs, targets)
    assert abs(float(l_nograd) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    assert abs(float(l_eval) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))


def _trainer_run(use_graph, steps=2):
    p = params()
    model, sd = _build(p)
    model.train()
    tr = train.FusedTrainer(model, clip_grad=0.05, accum_steps=2, use_graph=use_graph)
    losses = []
    for opt_step in range(1, steps + 1):
        for micro in range(2):
            x, mask, tgt, tlen = _batch(seed=0)        # one geometry, so the graph path captures and replays
            # read now: on the graph path the loss is the graph's output buffer, which the next replay overwrites
            losses.append(float(tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV))))
    torch.cuda.synchronize()
    return model, sd, tr, losses


def test_fused_trainer_follows_the_oracle_step_graph_and_eager():
    """Two optimizer steps over 2 accumulated micro-batches: clip + Adam as the reference trainer, with and without the
    graph.  Every micro-step's loss is the same bits with and without the graph; the weights agree to the order of the fp32
    atomics in the backward's column sums and embedding gradient (shared with every model's backward)."""
    runs = {}
    for use_graph in (False, True):
        model, sd, tr, losses = _trainer_run(use_graph)
        assert tr._graphs if use_graph else not tr._graphs
        runs[use_graph] = ({n: t.detach().clone() for n, t in model.named_parameters()}, losses)
    print('losses eager', runs[False][1], 'graph', runs[True][1])
    assert runs[False][1] == runs[True][1]
    p = params()
    _, sd = _build(p)
    names = [n for n, _ in tr.params]
    w = {n: sd[n].clone() for n in names}
    m = {n: torch.zeros_like(w[n]) for n in names}
    v = {n: torch.zeros_like(w[n]) for n in names}
    for opt_step in (1, 2):
        acc = None
        for micro in range(2):
            x, mask, tgt, tlen = _batch(seed=0)
            sd_now = dict(sd)
            sd_now.update({n: w[n] for n in names})
            _, g_ref, _ = rnnt_ref.loss_and_grads(x, mask, tgt, tlen, sd_now, p)
            acc = {n: g_ref[n] / 2 for n in names} if acc is None else {n: acc[n] + g_ref[n] / 2 for n in names}
        lr = ot.transformer_lr(ot.first_step_index() + opt_step - 1, 256, 12000)
        ot.clip_and_adam(w, acc, m, v, opt_step, lr, 0.05)
    for use_graph in (False, True):
        got = runs[use_graph][0]
        num = sum(float(((got[n].cpu() - w[n]) ** 2).sum()) for n in names)
        den = sum(float(((w[n] - sd[n]) ** 2).sum()) for n in names)
        print(f'graph={use_graph}: rel {(num / den) ** 0.5:.3e}')
        assert (num / den) ** 0.5 < 0.3
    num = sum(float(((runs[True][0][n] - runs[False][0][n]) ** 2).sum()) for n in names)
    den = sum(float(((runs[False][0][n].cpu() - sd[n]) ** 2).sum()) for n in names)
    assert (num / den) ** 0.5 < 1e-4


def test_mixspeech_micro_step_matches_oracle():
    """One MixSpeech micro-step: lambda L(mix, y_even) + (1 - lambda) L(mix, y_odd), gradients alike."""
    p = params()
    model, sd = _build(p)
    model.train()
    tr = train.FusedTrainer(model, accum_steps=1, use_graph=False, mixspeech=True)
    x, mask, tgt, tlen = _batch(B=4, lens=(120, 96, 109, 100), seed=3)
    batch = model.train_batch(x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV))
    tr.flat_bf16.copy_(tr.flat_p)
    loss = tr._micro_mix(batch)
    lam = float(tr.last_lambda)
    xm = lam * x[0::2] + (1 - lam) * x[1::2]
    mm = mask[0::2] | mask[1::2]
    l1, g1, _ = rnnt_ref.loss_and_grads(xm, mm, tgt[0::2], tlen[0::2], sd, p)
    l2, g2, _ = rnnt_ref.loss_and_grads(xm, mm, tgt[1::2], tlen[1::2], sd, p)
    want = lam * l1 + (1 - lam) * l2
    assert abs(float(loss) - float(want)) < 2e-2 * abs(float(want))
    names = [n for n, _ in tr.params]
    got = torch.cat([tr.sink[n].reshape(-1).cpu() for n in names])
    ref = torch.cat([(lam * g1[n] + (1 - lam) * g2[n]).reshape(-1) for n in names])
    assert _rel(got, ref) < REL_L2_GRAD


# ------------------------------------------------------------------------------------------------ greedy search
def test_greedy_step_kernel_matches_float64():
    B, T, D, H, L, V, max_len = 4, 3, 16, 8, 2, 9, 3
    g = torch.Generator().manual_seed(3)
    logits = torch.randn(B, V, generator=g)
    lp = torch.log_softmax(logits.double(), -1)
    val, idx = torch.empty(B, 1, device=DEV), torch.empty(B, 1, dtype=torch.int32, device=DEV)
    logp = torch.empty(B, 16, device=DEV)
    logits[1] = -logits[1].abs()
    logits[1, 0] = 5.0                                      # row 1 takes blank
    lp = torch.log_softmax(logits.double(), -1)
    ops.logsoftmax_topk(logits.to(DEV), V, 1, out_val=val, out_idx=idx, out_logp=logp)
    i32 = dict(dtype=torch.int32, device=DEV)
    t_len = torch.tensor([3, 2, 0, 3], **i32)
    frame = torch.tensor([0, 1, 0, 2], **i32)
    n_sym = torch.tensor([0, 0, 0, 2], **i32)              # row 3 is at the per-frame cap
    n_out = torch.tensor([max_len - 1, 0, 0, 0], **i32)
    ids = torch.zeros(B, max_len, **i32)
    score = torch.tensor([0.5, 0.0, 0.0, -1.0], device=DEV)
    active = torch.tensor([3], **i32)
    h, c = torch.zeros(L, B, H, device=DEV), torch.zeros(L, B, H, device=DEV)
    pp = torch.zeros(B, D, dtype=ops.BF16, device=DEV)
    hn, cn = torch.randn(L, B, H, device=DEV), torch.randn(L, B, H, device=DEV)
    ppn = torch.randn(B, D, device=DEV).to(ops.BF16)
    ep = torch.randn(B * T, D, device=DEV).to(ops.BF16)
    ep_cur = torch.zeros(B, D, dtype=ops.BF16, device=DEV)
    ops.rnnt_greedy_step(idx.view(-1), logp, hn, cn, ppn, h, c, pp, ep, T, ep_cur, t_len, frame, n_sym, n_out, ids, 2, score,
                         active)
    best = logits.argmax(-1)
    assert int(best[0]) != 0 and int(best[3]) != 0
    # row 0 emits its arg-max as its last token
    assert ids[0].tolist() == [0, 0, int(best[0])] and int(n_out[0]) == max_len and torch.equal(h[:, 0], hn[:, 0])
    assert torch.equal(pp[0], ppn[0]) and int(frame[0]) == 0
    assert abs(float(score[0]) - (0.5 + float(lp[0, best[0]]))) < 1e-6
    # row 1 takes blank on its last frame and ends (and so does row 3 below)
    assert int(frame[1]) == 2 and int(active) == 1 and abs(float(score[1]) - float(lp[1, 0])) < 1e-6
    assert float(h[:, 1].abs().sum()) == 0
    # row 2 has no frame: untouched; row 3 is capped: blank, next frame... past its last frame (3): ends
    assert float(score[2]) == 0.0 and int(frame[2]) == 0
    assert int(frame[3]) == 3 and int(n_sym[3]) == 0 and abs(float(score[3]) - (-1.0 + float(lp[3, 0]))) < 1e-6
    # a row that moves to a frame it still has copies that frame's encoder projection
    frame2 = torch.tensor([0, 0, 0, 0], **i32)
    ops.rnnt_greedy_step(idx.view(-1), logp, hn, cn, ppn, h, c, pp, ep, T, ep_cur, torch.tensor([3, 3, 3, 3], **i32), frame2,
                         torch.zeros(B, **i32), torch.zeros(B, **i32), ids, 2, score, active)
    assert torch.equal(ep_cur[1], ep[1 * T + 1])


def _tie_free_model(seed, x, mask):
    """A random model whose greedy search emits on some frames and not others: the output layer scaled up (tie-free
    arg-maxes) and the blank bias set to the median margin of the best label over blank at the first predictor state."""
    p = params(layers=2, V=24)
    model, _ = _build(p, seed)
    model.eval()
    with torch.no_grad():
        model.joint.output_layer.weight.mul_(4.0)
        mem, lengths, B, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
        op = model._pack.get()
        ep = ops.linear(mem, op['enc'].w, op['enc'].b, ops.EPI_BIAS)
        y, _, _, _ = train.lstm_stack_fwd(ops.embedding(torch.zeros(B, dtype=torch.long, device=DEV), op['emb']), op['layers'],
                                          1, B)
        pp = ops.linear(y, op['dec_w'])
        logits = ops.linear(ops.rnnt_joint(ep, pp, B, T2, 1), op['out_w'], op['out_b'], ops.EPI_BIAS, out_f32=True)
        margin = logits[:, 1:24].max(-1).values - logits[:, 0]
        model.joint.output_layer.bias[0] += float(margin.median())
    return model


def _greedy_restatement(model, mem, lengths, max_sym, max_len):
    """The greedy search in fp64 host code over the GPU's own joint log-probs: every step asks the GPU for the joint's
    log-probs at the state the restatement holds, and makes the decision itself."""
    op = model._pack.get()
    B = len(lengths)
    T2 = mem.shape[0] // B
    ep = ops.linear(mem, op['enc'].w, op['enc'].b, ops.EPI_BIAS).view(B, T2, -1)
    out = []
    for b in range(B):
        tok = torch.zeros(1, dtype=torch.long, device=DEV)
        x = ops.embedding(tok, op['emb'])
        y, h, c, _ = train.lstm_stack_fwd(x, op['layers'], 1, 1)
        pp = ops.linear(y, op['dec_w'])
        t, n_sym, ids, score = 0, 0, [], 0.0
        while t < int(lengths[b]):
            hj = ops.rnnt_joint(ep[b, t:t + 1].contiguous(), pp, 1, 1, 1)
            logits = ops.linear(hj, op['out_w'], op['out_b'], ops.EPI_BIAS, out_f32=True, n_out=model.joint.ld_logits)
            lp = torch.log_softmax(logits[0, :model.vocab_size].double().cpu(), -1)
            k = int(lp.argmax()) if (n_sym < max_sym and len(ids) < max_len) else 0
            score += float(lp[k])
            if k:
                ids.append(k)
                n_sym += 1
                x = ops.embedding(torch.tensor([k], device=DEV), op['emb'])
                y, h, c, _ = train.lstm_stack_fwd(x, op['layers'], 1, 1, hidden=(h, c))
                pp = ops.linear(y, op['dec_w'])
            else:
                t, n_sym = t + 1, 0
        out.append((ids, score))
    return out


@pytest.mark.parametrize('max_sym,max_len', [(5, 1023), (1, 1023), (3, 4)])
def test_greedy_search_in_lockstep_with_restatement(max_sym, max_len):
    x, mask, _, _ = _batch(lens=(120, 60, 97), seed=5)
    model = _tie_free_model(11, x, mask)
    res = {}
    for use_graph in (False, True):
        rec = TransducerRecognizer(model, max_symbols_per_frame=max_sym, max_len=max_len, use_graph=use_graph)
        res[use_graph] = [t.clone() for t in rec.recognize_ids(x.to(DEV), mask.to(DEV))]
    for a, b in zip(res[False], res[True]):
        assert torch.equal(a, b)
    ids, n, sc = res[True]
    with torch.no_grad():
        mem, lengths, B, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
        want = _greedy_restatement(model, mem, lengths.cpu(), max_sym, max_len)
    print(max_sym, max_len, [(len(w), s) for w, s in want], n.tolist())
    for b, (w_ids, w_score) in enumerate(want):
        assert ids[b, :int(n[b])].tolist() == w_ids
        assert float(ids[b, int(n[b]):].abs().sum()) == 0
        assert abs(float(sc[b]) - w_score) <= 1e-5 * abs(w_score)
    assert all(0 < len(w) for w, _ in want)
    if max_len == 4:
        assert max(len(w) for w, _ in want) == 4
    else:
        assert all(len(w) < 5 * int(t) for (w, _), t in zip(want, lengths.cpu()))      # blank is taken on some frames
    text = TransducerRecognizer(model, max_symbols_per_frame=max_sym, max_len=max_len).recognize(x.to(DEV), mask.to(DEV))
    assert text == [w for w, _ in want]
