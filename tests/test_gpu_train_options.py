"""GPU tests of FusedTrainer's training options: otb_mixspeech against tests/train_options_ref.py and torch's fp32
expression, one MixSpeech micro-step against the oracles with each pass's dropout masks replayed, the autograd seam under
the reference's own MixSpeech loop, MixSpeech optimizer steps (graph and eager), the gradient noise of the fused Adam
launch against the restatement, and resuming from state_dict / a reference-style checkpoint."""
import copy

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops, train
    from opentransformer_b200.model import CTCModel, SpeechToText
    DEV = torch.device('cuda:0')

from oracle import speech_model as om
from oracle import train_step as ot
from tests import conformer_train_ref as conf_ref
from tests import ctc_ref
from tests import train_options_ref as ref
from tests.test_gpu_train import REL_L2_GRAD, REL_L2_GRAD_ALL, _params as speech_params, _build as speech_build

P_DROP = 0.1


def _rel(a, b):
    return float((a.float().cpu() - b.float().cpu()).norm() / (b.float().cpu().norm() + 1e-20))


def _ulps(a, b):
    return np.abs(a.astype(np.float64) - b) / np.spacing(np.abs(b).astype(np.float32)).astype(np.float64)


# ------------------------------------------------------------------------------------------------ otb_mixspeech
@pytest.mark.parametrize('B,T,F', [(4, 50, 80), (5, 37, 3), (2, 1, 1), (9, 201, 80)])
def test_mixspeech_kernel_matches_restatement_and_torch(B, T, F):
    g = torch.Generator().manual_seed(B * 1000 + T)
    x = (torch.randn(B, T, F, generator=g) + 0.25).to(DEV)          # padded frames hold non-zero values too
    mask = (torch.rand(B, T, generator=g) > 0.4).to(DEV)
    lam = torch.empty(3, dtype=torch.float32, device=DEV)
    for seed, step in ((12345, 1), (7, 2 ** 31 - 1), (2 ** 31 - 2, 77)):
        s = torch.tensor([seed], dtype=torch.int32, device=DEV)
        t = torch.tensor([step], dtype=torch.int32, device=DEV)
        xm, mm = ops.mixspeech(x, mask, s, t, 0.5, lam)
        want = ref.mix_lambda(seed, step)
        got = lam.cpu().numpy()
        assert _ulps(got[:1], np.array([want]))[0] <= 1.0, (got[0], want)
        lt = lam[0]
        n = B // 2 * 2
        assert torch.equal(xm, x[0:n:2] * lt + x[1:n:2] * (1 - lt))              # trainer.py:172-173, fp32
        assert torch.equal(mm, torch.max(mask[0:n:2], mask[1:n:2]))
        assert float(lam[1]) == np.float32(got[0] * np.float32(0.5)) and float(lam[2]) == np.float32((np.float32(1) - got[0]) * np.float32(0.5))
        xr, mr = ref.mix(x.cpu(), mask.cpu(), got[0])
        assert np.array_equal(xm.cpu().numpy(), xr) and np.array_equal(mm.cpu().numpy(), mr)


# ------------------------------------------------------------------------------------------------ MixSpeech micro-step
def _batch(B=5, T=200, L=12, V=4234, lens=(200, 160, 181, 120, 199, 150, 170), seed=0, low=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, 80, generator=g)
    lens = torch.tensor(lens[:B])
    mask = torch.arange(T)[None] < lens[:, None]
    x = x * mask.unsqueeze(2)
    tgt = torch.randint(low, V, (B, L), generator=g)
    tgt[:, 0] = 1
    for b in range(B):
        n = L - 1 - (3 * b) % 5
        tgt[b, n] = 1
        tgt[b, n + 1:] = 0
    return x, mask, tgt, (tgt[:, 1:] != 0).sum(1).to(torch.int32)


def _speech_masks(model, P, T2, L, seed):
    masks = {}
    for site, part, rate in train.dropout_sites(model):
        rows = P * T2 if part == 'encoder' else P * L
        i, k = divmod(site - (train.ENC_SITE if part == 'encoder' else train.DEC_SITE), 2 if part == 'encoder' else 3)
        masks[(f'{part}.blocks.{i}', k)] = ops.dropout_mask(rows, 256, rate, seed, site).cpu().view(P, -1, 256).float()
    return lambda s, t: t * masks[s] / (1.0 - P_DROP)


def _case(kind):
    """(model, sd, params, oracle(x, mask, tgt, tlen, sd, drop) -> (loss, grads, stats), batch, uses truth_length)"""
    if kind == 'speech':
        params = speech_params(n_enc=2, n_dec=1)
        params['ctc_weight'] = 0.3
        params['encoder_output_size'] = 256
        for part in ('encoder', 'decoder'):
            params[part]['residual_dropout'] = P_DROP
        model, sd = speech_build(params)
        for k, v in model.assistor.state_dict().items():
            sd[f'assistor.{k}'] = v.detach().clone().float().cpu()

        def oracle(x, mask, tgt, tlen, sd, drop):
            om.set_dropout(drop)
            try:
                loss, g = ot.loss_and_grads(x, mask, tgt, sd, params, truth_length=tlen)
            finally:
                om.set_dropout(None)
            return loss, g, {}
        return model, sd, params, oracle, _batch(), True
    if kind == 'ctc':
        from tests.test_gpu_ctc_model import _params as ctc_params, _build as ctc_build
        params = ctc_params('transformer')
        model, sd = ctc_build(params)

        def oracle(x, mask, tgt, tlen, sd, drop):
            return ctc_ref.loss_and_grads_train(x, mask, tgt, tlen, sd, params, drop=drop)
        return model, sd, params, oracle, _batch(L=10, V=40, low=2), True
    from tests.test_gpu_conformer_train import _params as conf_params, _build as conf_build
    params = conf_params()
    model, sd = conf_build(params)

    def oracle(x, mask, tgt, tlen, sd, drop):
        return conf_ref.loss_and_grads_train(x, mask, tgt, sd, params, drop=drop)
    # 3 utterances per pass, the batch the Conformer's tolerances were set on (test_gpu_conformer_train.py): with 2, the
    # rel-pos band's gradients (pos_proj, posv) come out at 4.5e-2 of the fp32 restatement
    return model, sd, params, oracle, _batch(B=7), False


@pytest.mark.parametrize('kind', ['speech', 'ctc', 'conformer'])
def test_mixspeech_micro_step_matches_oracle(kind):
    """One micro-step (accumulation 2, so the flat buffer holds the scaled gradient before any update): the two passes
    against the oracle run with the same lambda and each pass's masks; lambda L1 + (1 - lambda) L2 and the weighted sum of
    the gradients; a Conformer's running statistics move twice."""
    model, sd, params, oracle, (x, mask, tgt, tlen), with_len = _case(kind)
    model.train()
    tr = train.FusedTrainer(model, accum_steps=2, use_graph=False, mixspeech=True)
    s0 = int(tr.drop_seed)
    nbt = {n: int(b) for n, b in model.named_buffers() if n.endswith('num_batches_tracked')}
    loss = tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV), truth_length=tlen.to(DEV) if with_len else None)
    lam = float(tr.last_lambda)
    assert 0.0 < lam < 1.0
    xm, mm = ref.mix(x, mask, lam)
    xm, mm = torch.from_numpy(xm), torch.from_numpy(mm)
    n = x.shape[0] // 2 * 2
    P, T2, L = n // 2, ops.conv_geometry(x.shape[1], 80)[2], tgt.shape[1] - 1
    sd_now, losses, grads = dict(sd), [], []
    for k in range(2):
        drop = None
        if kind == 'speech':
            drop = _speech_masks(model, P, T2, L, torch.tensor([s0 + 1 + k], dtype=torch.int32, device=DEV))
        l_k, g_k, stats = oracle(xm, mm, tgt[k:n:2], tlen[k:n:2], sd_now, drop)
        sd_now.update(stats)
        losses.append(float(l_k))
        grads.append(g_k)
    loss_ref = lam * losses[0] + (1 - lam) * losses[1]
    names = [n_ for n_, _ in tr.params]
    g = {n_: 2.0 * tr.sink[n_] for n_ in names}
    g_ref = {n_: lam * grads[0][n_] + (1 - lam) * grads[1][n_] for n_ in names}
    zero = [n_ for n_ in names if n_.endswith('depthwise_conv.bias')]
    for n_ in zero:
        assert float(g[n_].norm()) < 1e-3 * float(g_ref[n_[:-len('bias')] + 'weight'].norm())
    worst = sorted(((_rel(g[n_], g_ref[n_]), n_) for n_ in names if n_ not in zero), reverse=True)
    r_all = _rel(torch.cat([g[n_].reshape(-1).cpu() for n_ in names if n_ not in zero]),
                 torch.cat([g_ref[n_].reshape(-1) for n_ in names if n_ not in zero]))
    print(f'{kind}: lambda {lam:.4f}; loss gpu {float(loss):.5f} oracle {loss_ref:.5f}; all grads rel_l2 {r_all:.3e}; worst '
          + ', '.join(f'{n_} {r:.2e}' for r, n_ in worst[:3]))
    assert abs(float(loss) - loss_ref) < 2e-2 * abs(loss_ref)
    assert r_all < REL_L2_GRAD_ALL and worst[0][0] < REL_L2_GRAD, worst[:3]
    bufs = dict(model.named_buffers())
    for n_, want in sd_now.items():      # two updates: the bound of the Conformer's multi-step test (2e-3), not one update's
        if 'running_' in n_:
            assert _rel(bufs[n_], want) < 2e-3, (n_, _rel(bufs[n_], want))
    for n_, c in nbt.items():
        assert int(bufs[n_]) == c + 2, n_
    if kind == 'conformer':
        assert nbt


def test_autograd_seam_runs_the_reference_mixspeech_loop():
    """trainer.py:155-201 written out over this project's model through the autograd seam (two model() calls, one
    backward), with the trainer's lambda, against the FusedTrainer micro-step.  The trainer scales the loss gradient by
    lambda / accum_steps before its bf16 rounding, the seam scales the finished gradients: the two agree to the bf16
    rounding of the scaled loss gradient, not to fp32 rounding (measured: 1.6e-3 over all gradients, 3.0e-2 on the worst
    parameter)."""
    params = speech_params(n_enc=1, n_dec=1)
    params['ctc_weight'] = 0.3
    params['encoder_output_size'] = 256
    model, _ = speech_build(params)
    seam = copy.deepcopy(model).train()
    model.train()
    x, mask, tgt, tlen = _batch()
    x, mask, tgt, tlen = x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV)
    tr = train.FusedTrainer(model, accum_steps=2, use_graph=False, mixspeech=True)
    tr.step(x, mask, tgt, truth_length=tlen)
    lambda_ = tr.last_lambda.reshape(1).clone()
    # the reference's lines, as written (batch_size even, mix_coeffs repeated over [P, T, C])
    batch_size, t_, c_ = x.shape
    num_coeffs = batch_size // 2
    batch_size = num_coeffs * 2
    mix_coeffs = lambda_.unsqueeze(1).unsqueeze(1).repeat(num_coeffs, t_, c_)
    new_inputs = {'inputs': x[0:batch_size:2] * mix_coeffs + x[1:batch_size:2] * (1 - mix_coeffs),
                  'mask': torch.max(mask[0:batch_size:2], mask[1:batch_size:2])}
    target_1 = {'targets_length': tlen[0:batch_size:2], 'targets': tgt[0:batch_size:2]}
    target_2 = {'targets_length': tlen[1:batch_size:2], 'targets': tgt[1:batch_size:2]}
    loss_1, _ = seam(new_inputs, target_1)
    loss_2, _ = seam(new_inputs, target_2)
    loss = lambda_ * loss_1 + (1 - lambda_) * loss_2
    loss = torch.mean(loss) / 2
    loss.backward()
    names = [n for n, _ in tr.params]
    sp = dict(seam.named_parameters())
    r = _rel(torch.cat([sp[n].grad.reshape(-1) for n in names]), torch.cat([tr.sink[n].reshape(-1) for n in names]))
    worst = max(_rel(sp[n].grad, tr.sink[n]) for n in names)
    print(f'seam vs FusedTrainer micro-step: all grads rel_l2 {r:.3e}, worst parameter {worst:.3e}')
    assert r < 4e-3 and worst < REL_L2_GRAD


@pytest.mark.parametrize('use_graph', [False, True])
def test_mixspeech_optimizer_steps_follow_the_oracle(use_graph):
    """Two MixSpeech optimizer steps with accumulation 2 (lambda drawn per micro-step): clip + lr(3), lr(4) + Adam as the
    oracle's clip_and_adam on the oracle's MixSpeech gradients.  The graph path draws the same lambdas as the eager one."""
    params = speech_params(n_enc=1, n_dec=1)
    model, sd = speech_build(params)
    model.train()
    torch.manual_seed(99)
    tr = train.FusedTrainer(model, clip_grad=0.05, accum_steps=2, use_graph=use_graph, mixspeech=True)
    names = [n for n, _ in model.named_parameters()]
    w = {n: sd[n].clone() for n in names}
    m = {n: torch.zeros_like(w[n]) for n in names}
    v = {n: torch.zeros_like(w[n]) for n in names}
    lams = []
    for opt_step in (1, 2):
        acc = {n: torch.zeros_like(w[n]) for n in names}
        for micro in range(2):
            x, mask, tgt, _ = _batch(B=4, seed=10 * opt_step + micro)
            loss = tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV))
            lam = float(tr.last_lambda)
            lams.append(lam)
            xm, mm = (torch.from_numpy(a) for a in ref.mix(x, mask, lam))
            sd_now = dict(sd)
            sd_now.update(w)
            sd_now['decoder.output_layer.weight'] = w['decoder.embedding.weight']
            l1, g1 = ot.loss_and_grads(xm, mm, tgt[0::2], sd_now, params)
            l2, g2 = ot.loss_and_grads(xm, mm, tgt[1::2], sd_now, params)
            loss_ref = lam * float(l1) + (1 - lam) * float(l2)
            assert abs(float(loss) - loss_ref) < 2e-2 * abs(loss_ref)
            for n in names:
                acc[n] += (lam * g1[n] + (1 - lam) * g2[n]) / 2
        lr = ot.transformer_lr(ot.first_step_index() + opt_step - 1, 256, 12000)
        ot.clip_and_adam(w, acc, m, v, opt_step, lr, 0.05)
        torch.cuda.synchronize()
        num = sum(float(((p.detach().cpu() - w[n]) ** 2).sum()) for n, p in model.named_parameters())
        den = sum(float(((w[n] - sd[n]) ** 2).sum()) for n in names)
        print(f'MixSpeech graph={use_graph} step {opt_step}: rel {(num / den) ** 0.5:.3e}; lambdas {lams}')
        assert (num / den) ** 0.5 < 0.3
    want = ref.mix_lambda(int(tr.mix_seed), np.arange(1, 5))
    assert (_ulps(np.array(lams, dtype=np.float32), want) <= 1.0).all(), (lams, want)


# ------------------------------------------------------------------------------------------------ gradient noise
def _flat(spans, n, seed):
    g = torch.Generator().manual_seed(seed)
    live = torch.zeros(n, dtype=torch.bool)
    for o, k in spans:
        live[o:o + k] = True
    return live, g


def _adam_ref(p, g, m, v, live, sigma, key, coef, lr, t, b1, b2, eps, wd):
    """float64 restatement of one clip + noise + Adam step on the live elements."""
    z = np.zeros(p.shape[0])
    idx = np.nonzero(live)[0]
    z[idx] = ref.normal(key, idx)
    gi = g * coef + sigma * z * live + wd * p
    m2 = b1 * m + (1 - b1) * gi
    v2 = b2 * v + (1 - b2) * gi * gi
    p2 = p - lr / (1 - b1 ** t) * m2 / (np.sqrt(v2) / np.sqrt(1 - b2 ** t) + eps)
    return p2, m2, v2, z


def test_adam_noise_matches_restatement():
    spans = [(0, 1000), (1000, 3), (1008, 4099), (5112, 7)]
    n = 5120
    live, gen = _flat(spans, n, 0)
    mask = ops.noise_bitmask(n, spans).to(DEV)
    seed = torch.tensor([424242], dtype=torch.int32, device=DEV)
    # sigma = 1, zero gradient, beta1 = 0, wd = 0: m holds the drawn noise itself
    p = torch.zeros(n, device=DEV)
    g = torch.zeros(n, device=DEV)
    m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    sumsq = torch.zeros(1, device=DEV)
    counters = torch.tensor([0, 2, 0], dtype=torch.int32, device=DEV)
    hyper = torch.zeros(4, device=DEV)
    ops.sumsq(g, sumsq)
    ops.adam_step_sched(p, g, m, v, sumsq, 5.0, 1e-3, 256, 0, 1.0, (0.0, 0.98), 1e-9, 0.0, counters, hyper,
                        noise_std=1.0, noise_seed=seed, noise_mask=mask)
    zg = m.cpu().numpy()
    idx = np.nonzero(live.numpy())[0]
    z = ref.normal(ref.noise_key(424242, 1), idx)
    tol = 4 * np.spacing(np.maximum(np.abs(z), 1.0).astype(np.float32)).astype(np.float64)
    err = np.abs(zg[idx] - z)
    print(f'noise: max error {err.max():.3e}, {float((err / tol).max()):.2f} of the 4-ulp bound')
    assert (err <= tol).all()
    assert not m.cpu()[~live].any() and not p.cpu()[~live].any() and not v.cpu()[~live].any()
    assert counters.tolist() == [1, 3, 0]
    # sigma = 0.01 on a real-looking state: p, m, v within 1e-6 relative of the float64 restatement
    p0 = torch.randn(n, generator=gen) * live
    g0 = torch.randn(n, generator=gen) * 0.1 * live
    m0 = torch.randn(n, generator=gen) * 0.01 * live
    v0 = torch.rand(n, generator=gen) * 1e-3 * live
    outs = []
    for _ in range(2):                              # the same seed twice: bit-identical
        p, g, m, v = (t.clone().to(DEV) for t in (p0, g0, m0, v0))
        counters = torch.tensor([4, 6, 0], dtype=torch.int32, device=DEV)
        ops.sumsq(g, sumsq)
        ops.adam_step_sched(p, g, m, v, sumsq, 5.0, 1e-3, 256, 12000, 1.0, (0.9, 0.98), 1e-9, 1e-6, counters, hyper,
                            noise_std=0.01, noise_seed=seed, noise_mask=mask)
        outs.append((p.cpu(), m.cpu(), v.cpu()))
    assert all(torch.equal(a, b) for a, b in zip(*outs))
    total = float(torch.sqrt((g0.double() ** 2).sum()))
    coef = min(1.0, 5.0 / (total + 1e-6))
    lr = ot.transformer_lr(7, 256, 12000)
    p2, m2, v2, _ = _adam_ref(p0.double().numpy(), g0.double().numpy(), m0.double().numpy(), v0.double().numpy(),
                              live.numpy(), 0.01, ref.noise_key(424242, 5), coef, lr, 5, 0.9, 0.98, 1e-9, 1e-6)
    for got, want, name in zip(outs[0], (p2, m2, v2), 'pmv'):
        r = float(np.abs(got.double().numpy() - want).max() / np.abs(want).max())
        print(f'{name}: max relative error {r:.2e}')
        assert r < 1e-6, name
        assert not got[~live].any(), name
    # a different step draws different noise: the noise differs from the sigma = 0 update
    p, g, m, v = (t.clone().to(DEV) for t in (p0, g0, m0, v0))
    counters = torch.tensor([4, 6, 0], dtype=torch.int32, device=DEV)
    ops.sumsq(g, sumsq)
    ops.adam_step_sched(p, g, m, v, sumsq, 5.0, 1e-3, 256, 12000, 1.0, (0.9, 0.98), 1e-9, 1e-6, counters, hyper)
    assert not torch.equal(m.cpu(), outs[0][1])


def test_nan_step_with_noise_changes_nothing():
    n = 64
    spans = [(0, 60)]
    mask = ops.noise_bitmask(n, spans).to(DEV)
    seed = torch.tensor([5], dtype=torch.int32, device=DEV)
    p, m, v = torch.randn(n, device=DEV), torch.rand(n, device=DEV), torch.rand(n, device=DEV)
    g = torch.randn(n, device=DEV)
    g[3] = float('nan')
    before = [t.clone() for t in (p, m, v)]
    sumsq = torch.zeros(1, device=DEV)
    counters = torch.tensor([3, 5, 0], dtype=torch.int32, device=DEV)
    hyper = torch.zeros(4, device=DEV)
    ops.sumsq(g, sumsq)
    ops.adam_step_sched(p, g, m, v, sumsq, 5.0, 1e-3, 256, 12000, 1.0, (0.9, 0.98), 1e-9, 1e-6, counters, hyper,
                        noise_std=0.01, noise_seed=seed, noise_mask=mask)
    assert all(torch.equal(a, b) for a, b in zip((p, m, v), before))
    assert counters.tolist() == [3, 5, 1]


def test_trainers_with_noise_keep_gaps_zero_and_differ_from_noise_free():
    params = speech_params(n_enc=1, n_dec=1)
    model, _ = speech_build(params)
    model.train()
    tr = train.FusedTrainer(model, grad_noise=0.01, use_graph=False)
    x, mask, tgt, _ = _batch(B=3)
    for _ in range(2):
        tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV))
    live = torch.zeros(tr.flat_p.numel(), dtype=torch.bool)
    for o, k in tr.offsets.values():
        live[o:o + k] = True
    for buf in (tr.flat_p, tr.m, tr.v):
        assert not buf.cpu()[~live].any()
    assert tr.counters.tolist() == [2, 4, 0]


# ------------------------------------------------------------------------------------------------ resume
def _resume_setup():
    params = speech_params(n_enc=1, n_dec=1)
    params['ctc_weight'] = 0.3
    params['encoder_output_size'] = 256
    for part in ('encoder', 'decoder'):
        params[part]['residual_dropout'] = P_DROP
    return params


def _resume_trainer(params, seed=5):
    model, _ = speech_build(params)
    model.train()
    torch.manual_seed(seed)
    return model, train.FusedTrainer(model, clip_grad=5.0, accum_steps=1, use_graph=True, mixspeech=True, grad_noise=0.01)


def test_resume_continues_the_same_run(tmp_path):
    """4 steps straight against 2 steps, torch.save, a fresh model and trainer, load, 2 more steps (dropout, MixSpeech,
    gradient noise and the CUDA graph all on).  The counters, seeds and lambdas are equal; the weights and moments agree to
    the order of the kernels' fp32 atomics (the gradient norm and the embedding gradient accumulate with atomics)."""
    params = _resume_setup()
    batches = [_batch(B=4, seed=50 + i) for i in range(4)]

    def run(tr, idx):
        lams = []
        for i in idx:
            x, mask, tgt, tlen = batches[i]
            tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV), truth_length=tlen.to(DEV))
            lams.append(float(tr.last_lambda))
        return lams

    model_a, tr_a = _resume_trainer(params)
    p_init = tr_a.flat_p.clone()
    lams_a = run(tr_a, range(4))
    model_b, tr_b = _resume_trainer(params)
    lams_b = run(tr_b, range(2))
    path = tmp_path / 'latest_optimizer.pt'
    torch.save({'model': model_b.state_dict(), 'optim': tr_b.state_dict()}, path)
    del model_b, tr_b
    ck = torch.load(path, weights_only=False)
    model_c, tr_c = _resume_trainer(params, seed=777)          # other seeds until the checkpoint is loaded
    model_c.load_state_dict(ck['model'])
    tr_c.load_state_dict(ck['optim'])
    lams_b += run(tr_c, range(2, 4))
    assert lams_a == lams_b, (lams_a, lams_b)
    assert tr_a.counters.tolist() == tr_c.counters.tolist() == [4, 6, 0]
    for name in ('drop_seed', 'mix_seed', 'mix_step', 'noise_seed'):
        assert torch.equal(getattr(tr_a, name), getattr(tr_c, name)), name
    exact = all(torch.equal(getattr(tr_a, b), getattr(tr_c, b)) for b in ('flat_p', 'm', 'v'))
    dp = float((tr_c.flat_p - tr_a.flat_p).norm() / (tr_a.flat_p - p_init).norm())
    rm, rv = _rel(tr_c.m, tr_a.m), _rel(tr_c.v, tr_a.v)
    print(f'resume: bit-identical {exact}; p {dp:.2e} of the update, m {rm:.2e}, v {rv:.2e}')
    assert dp < 1e-3 and rm < 1e-3 and rv < 1e-3


def test_resume_from_a_reference_style_checkpoint():
    """The oracle's loop (clip_and_adam with transformer_lr) for 2 steps, saved as trainer.py:280-288 does through
    torch.optim.Adam; FusedTrainer loads it and its next step follows the oracle's third step (lr(5), Adam step 3)."""
    params = speech_params(n_enc=1, n_dec=1)
    model, sd = speech_build(params)
    names = [n for n, _ in model.named_parameters()]
    w = {n: sd[n].clone() for n in names}
    m = {n: torch.zeros_like(w[n]) for n in names}
    v = {n: torch.zeros_like(w[n]) for n in names}

    def oracle_step(t, seed):
        x, mask, tgt, _ = _batch(B=3, seed=seed)
        sd_now = dict(sd)
        sd_now.update(w)
        sd_now['decoder.output_layer.weight'] = w['decoder.embedding.weight']
        _, g = ot.loss_and_grads(x, mask, tgt, sd_now, params)
        ot.clip_and_adam(w, g, m, v, t, ot.transformer_lr(ot.first_step_index() + t - 1, 256, 12000), 0.05)
        return x, mask, tgt

    for t in (1, 2):
        oracle_step(t, 30 + t)
    cpu_params = {n: torch.nn.Parameter(w[n].clone()) for n in names}
    adam = torch.optim.Adam(list(cpu_params.values()), lr=1e-3, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6)
    for n, p_ in cpu_params.items():
        adam.state[p_] = {'step': torch.tensor(2.0), 'exp_avg': m[n].clone(), 'exp_avg_sq': v[n].clone()}
    ckpt = {'global_step': 2 + 2, 'optim': adam.state_dict()}
    with torch.no_grad():
        for n, p_ in model.named_parameters():
            p_.copy_(w[n].to(DEV))
    w_prev = {n: w[n].clone() for n in names}
    model.train()
    tr = train.FusedTrainer(model, clip_grad=0.05, accum_steps=1, use_graph=False)
    tr.load_state_dict(ckpt)
    assert tr.counters.tolist() == [2, 4, 0]
    x, mask, tgt = oracle_step(3, 33)
    tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV))
    assert tr.counters.tolist() == [3, 5, 0]
    assert abs(tr.lr() - ot.transformer_lr(5, 256, 12000)) < 1e-12
    torch.cuda.synchronize()
    num = sum(float(((p_.detach().cpu() - w[n]) ** 2).sum()) for n, p_ in model.named_parameters())
    den = sum(float(((w[n] - w_prev[n]) ** 2).sum()) for n in names)
    print(f'step after a reference-style checkpoint: ||w_gpu - w_oracle|| / ||w_oracle step|| = {(num / den) ** 0.5:.3e}')
    assert (num / den) ** 0.5 < 0.3
