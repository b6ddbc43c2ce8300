"""Training the Transformer language model on the GPU (lm.transformer_forward_backward, the autograd seam of
TransformerLanguageModel.forward and train.FusedTrainer) against the bf16-policy oracle of tests/transformer_lm_ref.py, which
tests/test_transformer_lm_ref.py pins to the reference's own module.  Tolerances are those of tests/test_gpu_train.py: loss
within 2e-2 relative, every gradient within 4e-2 relative L2, all gradients concatenated within 2e-2."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops, train
    from opentransformer_b200.lm import TLM_SITE, TransformerLanguageModel, transformer_forward_backward
    from opentransformer_b200.recognize import lm_log_probs
    DEV = torch.device('cuda:0')

from oracle import speech_model as om
from oracle import train_step as ot
from tests import transformer_lm_ref as tr
from tests.test_transformer_lm_ref import TLM_YAML

REL_LOSS = 2e-2
REL_L2_GRAD = 4e-2
REL_L2_GRAD_ALL = 2e-2
V = 300


def _params(tied=True, dropout=0.0, blocks=2):
    return dict(type='transformer_lm', vocab_size=V, num_blocks=blocks, d_model=256, n_heads=4, d_ff=1024,
                residual_dropout=dropout, smoothing=0.1, share_embedding=tied)


def _lm(params, seed=1234):
    torch.manual_seed(seed)
    lm = TransformerLanguageModel(params)
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for n, p in lm.named_parameters():
            if 'norm' in n:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif n.endswith('.bias'):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
        # keeps the logits O(1), so the loss is sensitive to every layer: at N(0, 1) the tied LM starts out predicting its
        # input token with logits ~ sqrt(d) * |E|, a saturated softmax whose bias gradients are differences of near-equal sums
        lm.embedding.weight.mul_(0.02)
    sd = {k: v.detach().clone().float() for k, v in lm.state_dict().items()}
    return lm.to(DEV), sd


def _batch(N, L, seed=3):
    """inputs / targets i64 [N, L]: BOS + tokens and tokens + EOS, PAD after each row's length; row 0 is full, the other
    rows are shorter by different amounts (at L = 1 every row is full)."""
    g = torch.Generator().manual_seed(seed)
    toks = torch.randint(2, V, (N, L), generator=g)
    inputs = torch.cat([torch.ones(N, 1, dtype=torch.long), toks[:, :-1]], 1)
    targets = toks.clone()
    for b in range(N):
        n = max(1, L - (L * b) // N - b)
        targets[b, n - 1] = 1
        targets[b, n:] = 0
        inputs[b, n:] = 0
    return inputs, targets


def _rel(a, b):
    return float((a.float().cpu() - b.float().cpu()).norm() / (b.float().cpu().norm() + 1e-20))


def _check(what, loss, g, loss_ref, g_ref, names, scale=1.0):
    assert set(names) == set(g_ref) == set(g), (set(names) ^ set(g_ref), set(names) ^ set(g))
    for n in names:
        assert g[n].shape == g_ref[n].shape and torch.isfinite(g[n]).all(), n
    worst = sorted(((_rel(g[n], scale * g_ref[n]), n) for n in names), reverse=True)
    r_all = _rel(torch.cat([g[n].reshape(-1).cpu() for n in names]), scale * torch.cat([g_ref[n].reshape(-1) for n in names]))
    print(f'{what}: loss gpu {float(loss):.5f} oracle {float(loss_ref):.5f}; all grads rel_l2 {r_all:.3e}; worst '
          + ', '.join(f'{n} {r:.2e}' for r, n in worst[:3]))
    assert abs(float(loss) - float(loss_ref)) < REL_LOSS * abs(float(loss_ref))
    assert r_all < REL_L2_GRAD_ALL
    assert worst[0][0] < REL_L2_GRAD, worst[:3]


def _masks(seed, N, L, blocks, p):
    """The product's keep masks of every residual-dropout site, keyed like the oracle's replay hook."""
    return {(f'blocks.{i}', k): ops.dropout_mask(N * L, 256, p, seed, TLM_SITE + 2 * i + k).cpu().float().view(N, L, 256)
            for i in range(blocks) for k in range(2)}


def _oracle(inputs, targets, sd, params, masks=None):
    p = params['residual_dropout']
    if masks is not None:
        om.set_dropout(lambda site, t: t * masks[site] / (1.0 - p))
    try:
        return tr.transformer_lm_loss_and_grads(inputs, targets, sd, params, policy='bf16')
    finally:
        om.set_dropout(None)


@pytest.mark.parametrize('L', [1, 47, 130])
@pytest.mark.parametrize('tied', [True, False])
def test_gradients_match_oracle(tied, L):
    """Loss and every parameter gradient; L = 130 crosses the attention kernels' 128-row tile."""
    params = _params(tied=tied)
    lm, sd = _lm(params)
    inputs, targets = _batch(4, L)
    loss_ref, g_ref = _oracle(inputs, targets, sd, params)
    with torch.no_grad():
        loss, g = transformer_forward_backward(lm.train(), inputs.to(DEV), targets.to(DEV))
    _check(f'tied={tied} L={L}', loss, g, loss_ref, g_ref, [n for n, _ in lm.named_parameters()])


def test_residual_dropout_with_replayed_masks():
    """residual_dropout 0.1: the oracle applies the product's masks, which have the right rate, differ between sites and
    change the loss."""
    params = _params(tied=True, dropout=0.1)
    lm, sd = _lm(params)
    inputs, targets = _batch(4, 47)
    N, L = inputs.shape
    seed = torch.tensor([777], dtype=torch.int32, device=DEV)
    masks = _masks(seed, N, L, 2, 0.1)
    keep = torch.stack([m.mean() for m in masks.values()])
    assert float((keep - 0.9).abs().max()) < 0.01, keep.tolist()
    ms = list(masks.values())
    assert all(not torch.equal(ms[i], ms[j]) for i in range(len(ms)) for j in range(i)), 'sites must draw different masks'
    loss_ref, g_ref = _oracle(inputs, targets, sd, params, masks)
    loss_nodrop, _ = _oracle(inputs, targets, sd, params)
    assert abs(float(loss_ref) - float(loss_nodrop)) > 1e-4, 'the replayed masks must change the network'
    with torch.no_grad():
        loss, g = transformer_forward_backward(lm.train(), inputs.to(DEV), targets.to(DEV), drop_seed=seed)
    _check('residual dropout 0.1', loss, g, loss_ref, g_ref, [n for n, _ in lm.named_parameters()])


def test_autograd_seam_and_predict_after_an_optimizer_step():
    """lm.train(); loss, _ = lm(inputs, targets); loss.backward() fills every .grad, scaled by the upstream gradient; two
    calls draw different masks; after an optimizer step predict() and the shallow-fusion term use the new weights."""
    params = _params(tied=True, dropout=0.1)
    lm, sd = _lm(params)
    inputs, targets = _batch(4, 20)
    x, y = inputs.to(DEV), targets.to(DEV)
    lm.eval()
    before = lm.predict(x, last_frame=False)
    fusion_before = lm_log_probs(lm, x)
    lm.train()
    loss, aux = lm({'inputs': x}, {'targets': y})
    seed = lm._drop_seed.clone()
    assert aux is None and loss.requires_grad
    (loss * 0.5).backward()
    names = [n for n, _ in lm.named_parameters()]
    loss_ref, g_ref = _oracle(inputs, targets, sd, params, _masks(seed, *inputs.shape, 2, 0.1))
    _check('autograd seam x 0.5', loss.detach(), {n: p.grad for n, p in lm.named_parameters()}, loss_ref, g_ref, names, scale=0.5)
    loss2, _ = lm({'inputs': x}, {'targets': y})
    assert not torch.equal(lm._drop_seed, seed) and float(loss2) != float(loss)
    with torch.no_grad():
        loss3, _ = lm({'inputs': x}, {'targets': y})         # train() without gradients: the training forward, dropout on
    assert float(loss3) not in (float(loss), float(loss2))
    opt = torch.optim.Adam(lm.parameters(), lr=1e-3, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6)
    torch.nn.utils.clip_grad_norm_(lm.parameters(), 5.0)
    opt.step()
    lm.eval()
    after = lm.predict(x, last_frame=False)
    sd_new = {k: v.detach().cpu().float() for k, v in lm.state_dict().items()}
    ref = om.transformer_lm_log_probs(inputs, sd_new, '', 2, 4, last_frame=False, policy='bf16')
    r = _rel(after, ref)
    print(f'predict after the optimizer step: rel_l2 {r:.3e} vs the oracle on the updated state dict')
    assert r < REL_LOSS and not torch.equal(after, before)
    fusion = lm_log_probs(lm, x)
    assert torch.allclose(fusion, after[:, -1], rtol=0, atol=1e-5) and not torch.equal(fusion, fusion_before)
    with torch.no_grad():
        l_eval, _ = lm({'inputs': x}, {'targets': y})
    assert abs(float(l_eval) - float(tr.transformer_lm_loss(inputs, targets, sd_new, '', params, 'bf16'))) < REL_LOSS * float(l_eval)


@pytest.mark.parametrize('use_graph', [False, True])
def test_fused_trainer_steps_match_oracle(use_graph):
    """Two optimizer steps of 2 accumulated micro-batches: the weights follow the oracle's clip + lr(3), lr(4) + Adam."""
    params = _params(tied=True)
    lm, sd = _lm(params)
    lm.train()
    tr_ = train.FusedTrainer(lm, lr=1e-3, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6, clip_grad=0.05, model_size=256,
                             warmup_steps=12000, accum_steps=2, use_graph=use_graph)
    names = [n for n, _ in lm.named_parameters()]
    w = {n: sd[n].clone() for n in names}
    m = {n: torch.zeros_like(w[n]) for n in names}
    v = {n: torch.zeros_like(w[n]) for n in names}
    for opt_step in (1, 2):
        acc = None
        for micro in range(2):
            inputs, targets = _batch(4, 30, seed=10 * opt_step + micro)
            loss = tr_.step(inputs.to(DEV), targets.to(DEV))
            sd_now = dict(sd)
            sd_now.update(w)
            sd_now['output_project.weight'] = w['embedding.weight']
            loss_ref, g_ref = _oracle(inputs, targets, sd_now, params)
            assert abs(float(loss) - float(loss_ref)) < REL_LOSS * abs(float(loss_ref))
            acc = {n: g_ref[n] / 2 for n in names} if acc is None else {n: acc[n] + g_ref[n] / 2 for n in names}
        lr = ot.transformer_lr(ot.first_step_index() + opt_step - 1, 256, 12000)
        assert abs(lr - tr_.lr()) < 1e-12
        ot.clip_and_adam(w, acc, m, v, opt_step, lr, 0.05)
        torch.cuda.synchronize()
        num = sum(float(((p.detach().cpu() - w[n]) ** 2).sum()) for n, p in lm.named_parameters())
        den = sum(float(((w[n] - sd[n]) ** 2).sum()) for n in names)
        print(f'optimizer step {opt_step}: ||w_gpu - w_oracle|| / ||w_oracle - w_init|| = {(num / den) ** 0.5:.3e}')
        assert (num / den) ** 0.5 < 0.3
    assert bool(tr_._graphs) == use_graph
    assert set(lm.state_dict()) >= set(names)


def test_fused_trainer_graph_replays():
    """Without dropout the graph's micro-steps compute the eager ones bit for bit; with dropout every replay draws fresh
    masks (4 micro-steps of one optimizer step: the weights do not move in between)."""
    batches = [_batch(4, 30, seed=s) for s in range(4)]
    losses = {}
    for use_graph in (False, True):
        lm, _ = _lm(_params(tied=False))
        tr_ = train.FusedTrainer(lm.train(), accum_steps=4, use_graph=use_graph)
        losses[use_graph] = [float(tr_.step(x.to(DEV), y.to(DEV))) for x, y in batches]
    assert losses[False] == losses[True], losses
    lm, _ = _lm(_params(tied=True, dropout=0.1))
    tr_ = train.FusedTrainer(lm.train(), accum_steps=4, use_graph=True)
    x, y = batches[0][0].to(DEV), batches[0][1].to(DEV)
    dropped = [float(tr_.step(x, y)) for _ in range(4)]
    print('FusedTrainer losses with dropout, one batch (captured at the 2nd step, replayed from the 3rd):', dropped)
    assert len(tr_._graphs) == 1 and len(set(dropped)) == 4


def test_shipped_transformer_lm_yaml_trains_with_the_graph():
    """transformer_lm.yaml (vocab 4233, 6 blocks, residual_dropout 0.1, tied) through FusedTrainer with the CUDA graph on one
    fixed 16 x 48 batch: the loss is finite and falls over 30 optimizer steps.  The warm-up is shortened to 100 steps so that
    30 steps move the weights (at the shipped 12000 the learning rate stays below 2e-6)."""
    torch.manual_seed(0)
    lm = TransformerLanguageModel(TLM_YAML).to(DEV).train()
    tr_ = train.FusedTrainer(lm, lr=1e-3, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6, clip_grad=5.0, model_size=256,
                             warmup_steps=100, accum_steps=1, use_graph=True)
    g = torch.Generator().manual_seed(5)
    toks = torch.randint(2, 4233, (16, 49), generator=g)
    x, y = toks[:, :-1].contiguous().to(DEV), toks[:, 1:].contiguous().to(DEV)
    losses = [float(tr_.step(x, y)) for _ in range(30)]
    print('transformer_lm.yaml, 30 FusedTrainer steps:', [round(v, 3) for v in losses])
    assert all(torch.isfinite(torch.tensor(losses)))
    assert len(tr_._graphs) == 1 and tr_.skipped_steps == 0
    assert sum(losses[-5:]) / 5 < sum(losses[:5]) / 5 - 0.5


# kernel launches of one speech FusedTrainer micro-step (tests/test_gpu_train.py's 1 + 1 block model, its _batch()),
# counted on the commit before the language model could train: without and with residual_dropout 0.1
SPEECH_MICRO_LAUNCHES = {0.0: 105, 0.1: 110}
ADAM_LAUNCHES = 3       # otb_sumsq + otb_adam_step_sched


@pytest.mark.parametrize('rate', [0.0, 0.1])
def test_speech_micro_step_launches_eager_and_replayed(rate):
    """A speech micro-step launches its recorded kernels eagerly, its captured graph holds them, and a replay counts
    them."""
    from tests.test_gpu_train import _batch as speech_batch, _build, _params as speech_params
    params = speech_params(n_enc=1, n_dec=1)
    params['encoder']['residual_dropout'] = rate
    params['decoder']['residual_dropout'] = rate
    x, mask, tgt = (t.to(DEV) for t in speech_batch())
    model, _ = _build(params)
    tr_ = train.FusedTrainer(model.train(), accum_steps=2, use_graph=False)
    counts = []
    for _ in range(3):                          # micro-step, micro-step + optimizer step, micro-step
        n0 = ops.COUNTERS['launches']
        tr_.step(x, mask, tgt)
        counts.append(ops.COUNTERS['launches'] - n0)
    assert counts[1:] == [SPEECH_MICRO_LAUNCHES[rate] + ADAM_LAUNCHES, SPEECH_MICRO_LAUNCHES[rate]], counts
    model, _ = _build(params)
    tr_ = train.FusedTrainer(model.train(), accum_steps=2, use_graph=True)
    tr_.step(x, mask, tgt)
    tr_.step(x, mask, tgt)                      # the second sighting captures the graph
    (ent,) = tr_._graphs.values()
    assert ent[0].launches == SPEECH_MICRO_LAUNCHES[rate], ent[0].launches
    n0 = ops.COUNTERS['launches']
    tr_.step(x, mask, tgt)                      # a replay, no optimizer step
    assert ops.COUNTERS['launches'] - n0 == SPEECH_MICRO_LAUNCHES[rate]
