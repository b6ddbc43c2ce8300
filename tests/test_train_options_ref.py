"""CPU tests of FusedTrainer's training options: the distributions of MixSpeech's lambda and of the gradient noise
(tests/train_options_ref.py restates csrc/counter_rng.cuh), the optimizer checkpoint format against torch.optim.Adam, the
refusals (all before any device work: FusedTrainer constructs on CPU tensors without a kernel) and the noise seed across
two gloo ranks."""
import copy
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from scipy import stats

import bench
from opentransformer_b200.lm import TransformerLanguageModel
from opentransformer_b200.model import CTCModel, SpeechToText
from opentransformer_b200.train import FusedTrainer, unused_parameters
from tests import train_options_ref as ref
from tests.test_dp_gloo import _free_port
from tests.test_transformer_lm_ref import _cuda_calls_fail, small_params


def test_lambda_follows_beta_half_half():
    seeds = np.arange(100_000, dtype=np.uint64) * np.uint64(2654435761) + np.uint64(17)
    lam = ref.mix_lambda(seeds, 1)
    p = stats.kstest(lam, stats.beta(0.5, 0.5).cdf).pvalue
    assert p > 1e-3, p
    assert lam.min() > 0.0 and lam.max() < 1.0
    # successive micro-steps of one trainer, too
    p2 = stats.kstest(ref.mix_lambda(12345, np.arange(100_000)), stats.beta(0.5, 0.5).cdf).pvalue
    assert p2 > 1e-3, p2


def test_noise_is_standard_normal():
    z = ref.normal(ref.noise_key(987654321, 1), np.arange(1_000_000))
    p = stats.kstest(z[:100_000], stats.norm.cdf).pvalue
    assert p > 1e-3, p
    assert abs(z.mean()) < 0.01 and abs(z.std() - 1.0) < 0.01, (z.mean(), z.std())
    assert np.isfinite(z).all()
    # another step draws other numbers
    z2 = ref.normal(ref.noise_key(987654321, 2), np.arange(1000))
    assert abs(np.corrcoef(z[:1000], z2)[0, 1]) < 0.1


def test_mix_restatement_is_the_reference_expression():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(5, 7, 3, generator=g)
    mask = torch.rand(5, 7, generator=g) > 0.5
    lam = torch.tensor([0.3141], dtype=torch.float32)
    xm, mm = ref.mix(x, mask, float(lam))
    want = x[0:4:2] * lam + x[1:4:2] * (1 - lam)            # trainer.py:172-173, odd last utterance dropped
    assert np.array_equal(xm, want.numpy())
    assert np.array_equal(mm, torch.max(mask[0:4:2], mask[1:4:2]).numpy())


def _speech_params(vocab=50, encoder='transformer'):
    p = {'type': 'speech2text', 'frontend_type': 'conv', 'encoder_type': 'transformer', 'decoder_type': 'transformer',
         'frontend': dict(input_size=80, output_size=128, in_channel=1, mid_channel=16, out_channel=16,
                          kernel_size=[[3, 3], [3, 3]], stride=[2, 2], dropout=0.0, act_func_type='relu',
                          front_end_layer_norm=False),
         'encoder': dict(d_model=128, n_heads=2, d_ff=256, n_blocks=1, pos_dropout=0.0, slf_attn_dropout=0.0,
                         ffn_dropout=0.0, residual_dropout=0.0, normalize_before=False, concat_after=False,
                         activation='glu', relative_positional=False),
         'decoder': dict(vocab_size=vocab, d_model=128, n_heads=2, d_ff=256, memory_dim=128, n_blocks=1,
                         pos_dropout=0.0, slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0,
                         residual_dropout=0.0, activation='glu', normalize_before=False, concat_after=False,
                         share_embedding=True),
         'ctc_weight': 0.0, 'smoothing': 0.1}
    if encoder == 'conformer':
        p = copy.deepcopy(bench.conformer_params())
        p['frontend'].update(mid_channel=16, out_channel=16)
        p['encoder'].update(nblocks=2)
        p['decoder'].update(n_blocks=1)
    return p


def _reference_adam_file(model, k=3, seed=0, lr=1e-4):
    """k torch.optim.Adam steps with synthetic gradients on the reference's parameter list, saved as trainer.py:280-288
    does (a Conformer's post_ffn gets no gradient, as in the reference's loop)."""
    skip = unused_parameters(model)
    named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
    opt = torch.optim.Adam([p for _, p in named], lr=lr, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6)
    g = torch.Generator().manual_seed(seed)
    for _ in range(k):
        for n, p in named:
            p.grad = None if n in skip else torch.randn(p.shape, generator=g)
        opt.step()
    return {'global_step': 2 + k, 'optim': copy.deepcopy(opt.state_dict())}, opt


def test_load_reproduces_a_reference_file_and_state_dict_goes_back_into_torch():
    torch.manual_seed(0)
    model = SpeechToText(_speech_params())
    ckpt, opt = _reference_adam_file(copy.deepcopy(model))
    tr = FusedTrainer(model, warmup_steps=12000)
    tr.load_state_dict(ckpt)
    assert tr.counters.tolist() == [3, 5, 0]
    named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
    state = ckpt['optim']['state']
    for i, (n, p) in enumerate(named):
        o, k = tr.offsets[n]
        assert torch.equal(tr.m[o:o + k].view(p.shape), state[i]['exp_avg']), n
        assert torch.equal(tr.v[o:o + k].view(p.shape), state[i]['exp_avg_sq']), n
    # the alignment gaps stay zero
    live = torch.zeros(tr.m.numel(), dtype=torch.bool)
    for o, k in tr.offsets.values():
        live[o:o + k] = True
    assert not tr.m[~live].any() and not tr.v[~live].any()
    # and back: what state_dict writes, torch's Adam loads, with equal tensors
    out = tr.state_dict()
    assert out['global_step'] == 5 and out['fused_trainer']['skipped_steps'] == 0
    fresh = torch.optim.Adam([p for _, p in named], lr=1.0, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6)
    fresh.load_state_dict(out['optim'])
    for i, (n, p) in enumerate(named):
        st = fresh.state[p]
        assert float(st['step']) == 3.0
        assert torch.equal(st['exp_avg'], state[i]['exp_avg']) and torch.equal(st['exp_avg_sq'], state[i]['exp_avg_sq']), n
    g = out['optim']['param_groups'][0]
    assert g['betas'] == (0.9, 0.98) and g['eps'] == 1e-9 and g['weight_decay'] == 1e-6 and not g['amsgrad']


def test_the_file_replaces_betas_eps_and_weight_decay():
    torch.manual_seed(0)
    model = SpeechToText(_speech_params())
    ckpt, _ = _reference_adam_file(copy.deepcopy(model), k=1)
    ckpt['optim']['param_groups'][0].update(betas=(0.8, 0.9), eps=1e-8, weight_decay=0.0)
    tr = FusedTrainer(model)
    tr.load_state_dict(ckpt)
    assert tr.betas == (0.8, 0.9) and tr.eps == 1e-8 and tr.wd == 0.0


def test_a_fresh_trainer_saves_no_state():
    torch.manual_seed(0)
    tr = FusedTrainer(SpeechToText(_speech_params()), mixspeech=True, grad_noise=0.01)
    out = tr.state_dict()
    assert out['global_step'] == 2 and out['optim']['state'] == {}
    own = out['fused_trainer']
    assert own['mix_step'] == 0 and own['noise_seed'] is not None and own['drop_seed'] is not None
    tr2 = FusedTrainer(SpeechToText(_speech_params()), mixspeech=True, grad_noise=0.01)
    tr2.load_state_dict(out)
    assert tr2.counters.tolist() == [0, 2, 0] and int(tr2.noise_seed) == own['noise_seed']
    assert int(tr2.mix_seed) == own['mix_seed'] and int(tr2.drop_seed) == own['drop_seed']


def test_conformer_post_ffn_has_no_state():
    torch.manual_seed(0)
    model = SpeechToText(_speech_params(encoder='conformer'))
    skip = unused_parameters(model)
    assert skip
    ckpt, _ = _reference_adam_file(copy.deepcopy(model), k=2)
    tr = FusedTrainer(model)
    tr.load_state_dict(ckpt)
    out = tr.state_dict()
    names = [n for n, p in model.named_parameters() if p.requires_grad]
    assert out['optim']['param_groups'][0]['params'] == list(range(len(names)))
    assert {names[i] for i in range(len(names)) if i not in out['optim']['state']} == skip
    for i in out['optim']['state']:
        assert torch.equal(out['optim']['state'][i]['exp_avg'], ckpt['optim']['state'][i]['exp_avg'])


def _trainer(monkeypatch=None):
    torch.manual_seed(0)
    model = SpeechToText(_speech_params())
    ckpt, _ = _reference_adam_file(copy.deepcopy(model), k=2)
    return model, FusedTrainer(model), ckpt


def test_refusals_come_before_device_work(monkeypatch):
    model, tr, ckpt = _trainer()
    _cuda_calls_fail(monkeypatch)
    bad = dict(ckpt)
    del bad['global_step']
    with pytest.raises(ValueError, match='global_step'):
        tr.load_state_dict(bad)
    bad = copy.deepcopy(ckpt)
    bad['optim']['param_groups'][0]['params'] = bad['optim']['param_groups'][0]['params'][:-1]
    with pytest.raises(ValueError, match='parameters'):
        tr.load_state_dict(bad)
    bad = copy.deepcopy(ckpt)
    bad['optim']['state'][0]['exp_avg'] = bad['optim']['state'][0]['exp_avg'][..., :1]
    with pytest.raises(ValueError, match='shape'):
        tr.load_state_dict(bad)
    bad = copy.deepcopy(ckpt)
    bad['optim']['param_groups'][0]['amsgrad'] = True
    with pytest.raises(ValueError, match='amsgrad'):
        tr.load_state_dict(bad)
    bad = copy.deepcopy(ckpt)
    bad['optim']['state'][1]['step'] = torch.tensor(7.0)
    with pytest.raises(ValueError, match='unequal'):
        tr.load_state_dict(bad)
    with pytest.raises(ValueError, match='grad_noise'):
        FusedTrainer(SpeechToText(_speech_params()), grad_noise=-0.1)
    lm = TransformerLanguageModel(small_params(True))
    with pytest.raises(NotImplementedError, match='MixSpeech'):
        FusedTrainer(lm, mixspeech=True)
    mtr = FusedTrainer(SpeechToText(_speech_params()), mixspeech=True)
    x, mask, truth = torch.zeros(1, 40, 80), torch.ones(1, 40, dtype=torch.bool), torch.ones(1, 5, dtype=torch.long)
    with pytest.raises(ValueError, match='at least 2'):
        mtr.step(x, mask, truth)


def test_default_trainer_draws_no_new_seeds():
    """With every new argument at its default the constructor consumes torch's RNG as before and allocates nothing new."""
    torch.manual_seed(0)
    model = SpeechToText(_speech_params())
    torch.manual_seed(5)
    tr = FusedTrainer(model)
    after = torch.rand(1)
    torch.manual_seed(5)
    torch.randint(0, 2 ** 31 - 1, (1,), dtype=torch.int32)          # the dropout seed, the one draw of the parent
    assert torch.equal(after, torch.rand(1))
    assert tr.mix_seed is None and tr.noise_seed is None and tr.noise_mask is None and tr.last_lambda is None


def test_ctc_model_has_the_mix_contract():
    assert CTCModel.mix_batch is SpeechToText.mix_batch
    assert not hasattr(TransformerLanguageModel, 'mix_batch')


def _noise_worker(rank, world, port, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    torch.manual_seed(0)
    model = SpeechToText(_speech_params())
    torch.manual_seed(100 + rank)                # ranks built with different torch seeds
    tr = FusedTrainer(model, grad_noise=0.01, mixspeech=True)
    q.put((rank, int(tr.noise_seed), int(tr.mix_seed)))
    dist.destroy_process_group()


def test_noise_seed_is_the_first_ranks():
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_noise_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = sorted(q.get(timeout=180) for _ in range(2))
    for p in ps:
        p.join(timeout=60)
    torch.manual_seed(100)
    torch.randint(0, 2 ** 31 - 1, (1,), dtype=torch.int32)           # dropout seed
    mix0 = int(torch.randint(0, 2 ** 31 - 1, (1,), dtype=torch.int32))
    noise0 = int(torch.randint(0, 2 ** 31 - 1, (1,), dtype=torch.int32))
    assert res == [(0, noise0, mix0), (1, noise0, mix0)]
