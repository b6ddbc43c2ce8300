"""GPU tests of Conformer training (d_model 256, 64-wide heads): the new kernels against torch autograd in fp64 / fp32, and
the whole training step against the fp32 training-mode restatement (tests/conformer_train_ref.py) -- loss, every gradient,
the BatchNorm running statistics, residual dropout with replayed masks, joint CTC, the fused optimizer step and the public
`loss.backward()` seam."""
import copy

import pytest
import torch

import bench
from tests import conformer_train_ref as ref

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops, train
    from opentransformer_b200.model import SpeechToText
    DEV = torch.device('cuda:0')

from oracle import speech_model as om
from oracle import train_step as ot

REL_L2_GRAD = 4e-2        # per-parameter gradient, bf16 activations / gradients vs the fp32 restatement (as the Transformer)
REL_L2_GRAD_ALL = 2e-2    # all gradients concatenated
BF16 = torch.bfloat16


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize('d,k', [(256, 5), (384, 5), (256, 15)])
def test_conv_module_training_kernels_match_autograd(d, k):
    """otb_conformer_conv_train / _bwd: depthwise conv of the masked GLU output + BatchNorm with batch statistics + swish,
    the running-statistics update, and every gradient, against fp64 autograd."""
    g = torch.Generator().manual_seed(d + k)
    B, T = 3, 61
    lens = torch.tensor([61, 40, 17], dtype=torch.int32)
    mask = torch.arange(T)[None] < lens[:, None].long()
    x = torch.randn(B * T, d, generator=g).to(BF16)
    w = 0.3 * torch.randn(d, k, generator=g)
    wb = 0.2 * torch.randn(d, generator=g)
    gamma, beta = 1 + 0.2 * torch.randn(d, generator=g), 0.2 * torch.randn(d, generator=g)
    rm, rv = 0.1 * torch.randn(d, generator=g), 1 + 0.1 * torch.rand(d, generator=g)
    nbt = torch.tensor(7, dtype=torch.int64)
    dy = torch.randn(B * T, d, generator=g).to(BF16)
    rm_d, rv_d, nbt_d = rm.to(DEV), rv.to(DEV), nbt.to(DEV)
    out, c, stats = ops.conformer_conv_train(x.to(DEV), lens.to(DEV), w.to(DEV), wb.to(DEV), gamma.to(DEV), beta.to(DEV), rm_d, rv_d,
                                             nbt_d, B, T)
    dx, dw, dwb, dg, db = ops.conformer_conv_bwd(dy.to(DEV), x.to(DEV), lens.to(DEV), w.to(DEV), gamma.to(DEV), beta.to(DEV), c, stats,
                                                 B, T)
    torch.cuda.synchronize()
    X = x.double().view(B, T, d).masked_fill(~mask.unsqueeze(2), 0.0).requires_grad_()
    W, WB, G, Bt = (t.double().clone().requires_grad_() for t in (w, wb, gamma, beta))
    rm64, rv64 = rm.double().clone(), rv.double().clone()
    C = torch.nn.functional.conv1d(X.transpose(1, 2), W.unsqueeze(1), WB, padding=(k - 1) // 2, groups=d)
    A = torch.nn.functional.batch_norm(C, rm64, rv64, G, Bt, True, 0.1, 1e-5)
    S = (A * torch.sigmoid(A)).transpose(1, 2).masked_fill(~mask.unsqueeze(2), 0.0)
    (S * dy.double().view(B, T, d)).sum().backward()
    assert _rel(c.cpu(), C.detach().transpose(1, 2).reshape(B * T, d)) < 1e-5
    assert _rel(out.cpu(), S.detach().reshape(B * T, d)) < 1e-2
    assert _rel(rm_d.cpu(), rm64) < 1e-5 and _rel(rv_d.cpu(), rv64) < 1e-5
    assert int(nbt_d) == 8
    want_dx = X.grad.masked_fill(~mask.unsqueeze(2), 0.0).reshape(B * T, d)
    assert float(dx.cpu().view(B, T, d)[~mask].abs().max()) == 0.0
    for name, a, b_ in (('dx', dx, want_dx), ('dw', dw, W.grad), ('dgamma', dg, G.grad), ('dbeta', db, Bt.grad)):
        assert _rel(a, b_) < 1e-2, (name, _rel(a, b_))
    # the conv bias feeds BatchNorm, whose batch mean removes any per-channel constant: its exact gradient is zero, and the
    # kernel's fp32 sum over the rows of dc leaves only rounding noise
    assert float(WB.grad.norm()) < 1e-9 * float(W.grad.norm())
    assert float(dwb.norm()) < 1e-4 * float(W.grad.norm()), float(dwb.norm()) / float(W.grad.norm())
    # accumulate: a second backward adds the same gradients on top
    ops.conformer_conv_bwd(dy.to(DEV), x.to(DEV), lens.to(DEV), w.to(DEV), gamma.to(DEV), beta.to(DEV), c, stats, B, T, dw=dw, dwb=dwb,
                           dgamma=dg, dbeta=db, accumulate=True)
    assert _rel(dg.cpu(), 2 * G.grad) < 1e-2 and _rel(dw.cpu(), 2 * W.grad) < 1e-2


def test_dropout_add_uses_the_dropout_mask_of_its_site():
    g = torch.Generator().manual_seed(3)
    M, N, p, site, T = 300, 256, 0.1, 17, 100
    x = torch.randn(M, N, generator=g).to(BF16).to(DEV)
    r = torch.randn(M, N, generator=g).to(BF16).to(DEV)
    seed = torch.tensor([4321], dtype=torch.int32, device=DEV)
    keep = ops.dropout_mask(M, N, p, seed, site).float()
    out = ops.dropout_add(x, r, p, seed, site, alpha=0.5)
    assert _rel(out, r.double() + 0.5 * x.double() * keep / (1 - p)) < 5e-3
    assert float((keep.mean() - (1 - p)).abs()) < 0.01
    # resid None + row mask: the backward of a masked, dropped site
    lens = torch.tensor([100, 40, 0], dtype=torch.int32, device=DEV)
    rows = (torch.arange(M, device=DEV) % T < lens.long().repeat_interleave(T)).float()[:, None]
    out = ops.dropout_add(x, None, p, seed, site, row_len=lens, row_period=T)
    assert _rel(out, x.double() * keep * rows / (1 - p)) < 5e-3
    assert torch.equal(ops.dropout_add(x, r), (x.float() + r.float()).to(BF16))


# ------------------------------------------------------------------------------------------------ whole model
def _params(rate=0.0, ctc=0.0):
    p = copy.deepcopy(bench.conformer_params())
    p['frontend'].update(mid_channel=64, out_channel=128)
    p['encoder'].update(nblocks=2, residual_dropout=rate)
    p['decoder'].update(n_blocks=2, residual_dropout=rate)
    p['ctc_weight'] = ctc
    if ctc:
        p['encoder_output_size'] = 256
    return p


def _build(params, seed=1234):
    torch.manual_seed(seed)
    model = SpeechToText(params)
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if 'norm' in n:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif n.endswith('.bias'):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
        model.decoder.embedding.weight.mul_(0.12)
        for n, b in model.named_buffers():
            if n.endswith('running_mean'):
                b.normal_(0.0, 0.1, generator=g)
            elif n.endswith('running_var'):
                b.uniform_(0.8, 1.2, generator=g)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    return model.to(DEV), sd


def _batch(B=3, T=200, L=12, lens=(200, 160, 181), seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, 80, generator=g)
    lens = torch.tensor(lens)
    mask = torch.arange(T)[None] < lens[:, None]
    x = x * mask.unsqueeze(2)
    tgt = torch.randint(3, 4234, (B, L), generator=g)
    tgt[:, 0] = 1
    tgt[0, L - 3:] = torch.tensor([1, 0, 0])
    tgt[1, L - 1] = 1
    tgt[2, L // 2:] = torch.tensor([1] + [0] * (L - L // 2 - 1))
    tlen = (tgt[:, 1:] != 0).sum(1)
    return x, mask, tgt, tlen


def _replay(model, B, T2, L, p, seed):
    """The product's mask of every dropout site, as the restatement's drop((prefix, k), tensor)."""
    masks = {}
    for site, part, _ in train.dropout_sites(model):
        i, k = divmod(site - (train.ENC_SITE if part == 'encoder' else train.DEC_SITE), 3)
        rows = B * T2 if part == 'encoder' else B * L
        masks[(f'{part}.blocks.{i}', k)] = ops.dropout_mask(rows, 256, p, seed, site).cpu().view(B, -1, 256).float()
    return lambda s, t: t * masks[s] / (1.0 - p)


def _compare(model, sd, params, x, mask, tgt, tlen, seed=None, drop=None, label=''):
    use_tlen = tlen if params['ctc_weight'] > 0 else None
    loss_ref, g_ref, stats_ref = ref.loss_and_grads_train(x, mask, tgt, sd, params, truth_length=use_tlen, drop=drop)
    with torch.no_grad():
        loss, g = train.forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), drop_seed=seed,
                                         truth_length=use_tlen.to(DEV) if use_tlen is not None else None)
    names = [n for n, _ in model.named_parameters()]
    assert set(g) == {n for n in names if g_ref[n] is not None}
    assert all(g_ref[n] is None for n in names if '.post_ffn.' in n)
    # depthwise_conv.bias feeds BatchNorm with batch statistics, which removes any per-channel constant: its exact gradient
    # is zero and both sides hold rounding noise only, so it is held to an absolute bound against the conv weight gradient
    # instead of a relative one
    zero = [n for n in g if n.endswith('depthwise_conv.bias')]
    for n in zero:
        wn = n[:-len('bias')] + 'weight'
        ratio = float(g[n].norm()) / float(g_ref[wn].norm())
        print(f'{n}: |grad| / |weight grad| = {ratio:.2e} (reference {float(g_ref[n].norm()) / float(g_ref[wn].norm()):.2e})')
        assert ratio < 1e-3
    worst = sorted(((_rel(g[n], g_ref[n]), n) for n in g if n not in zero), reverse=True)
    r_all = _rel(torch.cat([g[n].reshape(-1).cpu() for n in g]), torch.cat([g_ref[n].reshape(-1) for n in g]))
    print(f'{label}: loss gpu {float(loss):.5f} ref {float(loss_ref):.5f}; all grads rel_l2 {r_all:.3e}; worst '
          + ', '.join(f'{n} {r:.2e}' for r, n in worst[:5]))
    assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    assert r_all < REL_L2_GRAD_ALL
    assert worst[0][0] < REL_L2_GRAD, worst[:3]
    bufs = dict(model.named_buffers())
    for n, want in stats_ref.items():
        assert _rel(bufs[n], want) < 1e-3, (n, _rel(bufs[n], want))
    return loss_ref


def test_whole_model_gradients_match_training_restatement():
    params = _params()
    model, sd = _build(params)
    x, mask, tgt, tlen = _batch()
    _compare(model, sd, params, x, mask, tgt, tlen, label='conformer')
    assert int(dict(model.named_buffers())['encoder.blocks.0.conv.batch_norm.num_batches_tracked']) == 1


def test_whole_model_with_residual_dropout_and_replayed_masks():
    params = _params(rate=0.1)
    model, sd = _build(params)
    x, mask, tgt, tlen = _batch()
    B, T2, L = x.shape[0], ops.conv_geometry(x.shape[1], 80)[2], tgt.shape[1] - 1
    seed = torch.tensor([12345], dtype=torch.int32, device=DEV)
    drop = _replay(model, B, T2, L, 0.1, seed)
    loss_ref = _compare(model, sd, params, x, mask, tgt, tlen, seed=seed, drop=drop, label='conformer, dropout 0.1')
    loss_nodrop, _ = ref.loss_train(x, mask, tgt, sd, params)
    assert abs(float(loss_ref) - float(loss_nodrop)) > 1e-4, 'the replayed masks must change the network'


def test_whole_model_with_joint_ctc():
    params = _params(ctc=0.3)
    model, sd = _build(params)
    x, mask, tgt, tlen = _batch()
    _compare(model, sd, params, x, mask, tgt, tlen, label='conformer, joint CTC 0.3')


@pytest.mark.parametrize('use_graph', [False, True])
def test_fused_trainer_steps_follow_the_reference_update(use_graph):
    """Two optimizer steps with accumulation 2: clip + lr(3), lr(4) + Adam over every parameter except post_ffn.*, which
    stays bit-identical; the running statistics follow the restatement's."""
    params = _params()
    model, sd = _build(params)
    model.train()
    post = {n: p.detach().clone() for n, p in model.named_parameters() if '.post_ffn.' in n}
    tr = train.FusedTrainer(model, lr=1e-3, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6, clip_grad=0.05, model_size=256,
                            warmup_steps=12000, accum_steps=2, use_graph=use_graph)
    names = [n for n, _ in model.named_parameters() if n not in post]
    w = {n: sd[n].clone() for n in names}
    m = {n: torch.zeros_like(w[n]) for n in names}
    v = {n: torch.zeros_like(w[n]) for n in names}
    stats = {n: sd[n].clone() for n in sd if 'running_' in n}
    for opt_step in (1, 2):
        acc = None
        for micro in range(2):
            x, mask, tgt, _ = _batch(seed=10 * opt_step + micro)
            loss = tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV))
            sd_now = dict(sd)
            sd_now.update(w)
            sd_now.update(stats)
            if params['decoder'].get('share_embedding', False):
                sd_now['decoder.output_layer.weight'] = w['decoder.embedding.weight']
            loss_ref, g_ref, stats = ref.loss_and_grads_train(x, mask, tgt, sd_now, params)
            assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
            acc = {n: g_ref[n] / 2 for n in names} if acc is None else {n: acc[n] + g_ref[n] / 2 for n in names}
        lr = ot.transformer_lr(ot.first_step_index() + opt_step - 1, 256, 12000)
        ot.clip_and_adam(w, acc, m, v, opt_step, lr, 0.05)
        torch.cuda.synchronize()
        cur = dict(model.named_parameters())
        num = sum(float(((cur[n].detach().cpu() - w[n]) ** 2).sum()) for n in names)
        den = sum(float(((w[n] - sd[n]) ** 2).sum()) for n in names)
        print(f'optimizer step {opt_step} (graph {use_graph}): ||w_gpu - w_ref|| / ||w_ref - w_init|| = {(num / den) ** 0.5:.3e}')
        assert (num / den) ** 0.5 < 0.3
        bufs = dict(model.named_buffers())
        for n, want in stats.items():
            assert _rel(bufs[n], want) < 2e-3, (n, _rel(bufs[n], want))
    for n, p in model.named_parameters():
        if n in post:
            assert torch.equal(p.detach(), post[n]), n
    assert int(dict(model.named_buffers())['encoder.blocks.1.conv.batch_norm.num_batches_tracked']) == 4


def test_public_seam_and_eval_after_training():
    """model.train(); loss.backward() fills .grad of every parameter but post_ffn.*; the next eval-mode encoder forward
    uses the updated running statistics."""
    params = _params()
    model, sd = _build(params)
    x, mask, tgt, _ = _batch()
    model.train()
    loss, _ = model({'inputs': x.to(DEV), 'mask': mask.to(DEV)}, {'targets': tgt.to(DEV), 'targets_length': None})
    loss.backward()
    for n, p in model.named_parameters():
        if '.post_ffn.' in n:
            assert p.grad is None, n
        else:
            assert p.grad is not None and p.grad.shape == p.shape, n
    _, _, stats = ref.loss_and_grads_train(x, mask, tgt, sd, params)
    sd_eval = dict(sd)
    sd_eval.update(stats)
    mem_ref, mmask = om.encode(x, mask, sd_eval, params)
    model.eval()
    with torch.no_grad():
        mem, _, _, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
    got = mem.float().view(x.shape[0], T2, -1).cpu()
    r = _rel(got[mmask], mem_ref[mmask])
    stale, _ = om.encode(x, mask, sd, params)
    print(f'eval after training: rel_l2 {r:.3e} (against the stale statistics {_rel(got[mmask], stale[mmask]):.3e})')
    assert r < 2e-2


def test_train_mode_without_gradients_uses_batch_statistics():
    """model.train() under torch.no_grad() (a validation loop that does not call eval()): the loss is the training-mode
    forward's (BatchNorm with batch statistics), and the running statistics move, as in the reference."""
    params = _params()
    model, sd = _build(params)
    x, mask, tgt, _ = _batch()
    model.train()
    with torch.no_grad():
        loss, _ = model({'inputs': x.to(DEV), 'mask': mask.to(DEV)}, {'targets': tgt.to(DEV), 'targets_length': None})
    loss_ref, stats = ref.loss_train(x, mask, tgt, sd, params)
    loss_eval, _ = om.model_forward_loss(x, mask, tgt, sd, params)
    print(f'train mode, no grad: loss gpu {float(loss):.5f} ref {float(loss_ref):.5f} (eval-mode loss {float(loss_eval):.5f})')
    assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    bufs = dict(model.named_buffers())
    for n, want in stats.items():
        assert _rel(bufs[n], want) < 1e-3, n
