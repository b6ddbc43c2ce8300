"""Training the Transformer language model (model/lm.py:94-141, transformer_lm.yaml) without a GPU: its fp32 restatement
(tests/transformer_lm_ref.py) against the reference's own TransformerLanguageModel in train() (tests/golden/
live_ref_transformer_lm.pt, made by tests/golden/make_live_ref_transformer_lm.py), the port's state_dict against the
reference's for transformer_lm.yaml, and the configurations the training path refuses before any device work."""
import os

import pytest
import torch

from tests import transformer_lm_ref as tr

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, 'golden', 'live_ref_transformer_lm.pt')

# egs/aishell/conf/transformer_lm.yaml, model section
TLM_YAML = dict(type='transformer_lm', vocab_size=4233, num_blocks=6, d_model=256, n_heads=4, d_ff=1024, residual_dropout=0.1,
                smoothing=0.1, share_embedding=True)


def small_params(tied):
    return dict(type='transformer_lm', vocab_size=40, num_blocks=2, d_model=128, n_heads=2, d_ff=256, residual_dropout=0.0,
                smoothing=0.1, share_embedding=tied)


def small_batch():
    """inputs [3, 11] (BOS + tokens, PAD after each length), targets [3, 11] (tokens + EOS, PAD-padded); row 0 is full."""
    g = torch.Generator().manual_seed(6)
    toks = torch.randint(2, 40, (3, 11), generator=g)
    lens = torch.tensor([11, 7, 2])
    inputs = torch.cat([torch.ones(3, 1, dtype=torch.long), toks[:, :-1]], 1)
    targets = toks.clone()
    for b, n in enumerate(lens.tolist()):
        targets[b, n - 1] = 1
        targets[b, n:] = 0
        inputs[b, n:] = 0
    return inputs, targets


def synth_state_dict(shapes, seed, tied):
    """Deterministic weights for the given {key: shape}: uniform(-0.3, 0.3) in key order, LayerNorm weights 1 + that; a tied
    output_project.weight is the embedding."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shape in shapes.items():
        sd[k] = torch.rand(shape, generator=g) * 0.6 - 0.3
        if '.norm' in k and k.endswith('.weight'):
            sd[k] += 1.0
    if tied:
        sd['output_project.weight'] = sd['embedding.weight']
    return sd


def sample(grad):
    """The elements of a gradient the fixture stores: all of a tensor of up to 4096 elements, else a fixed random quarter
    of them (seeded by the size), which keeps the fixture under 1 MB."""
    flat = grad.reshape(-1)
    if flat.numel() <= 4096:
        return flat.clone()
    idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(flat.numel()))[:flat.numel() // 4]
    return flat[idx].clone()


@pytest.fixture(scope='module')
def fixture():
    return torch.load(FIXTURE)


def _rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize('which', ['tied', 'untied'])
def test_oracle_matches_reference(fixture, which):
    """fp32 oracle vs the reference's forward in train() and loss.backward() on the same weights: only summation order
    differs, so 1e-5 relative on the loss and 1e-4 relative L2 on every gradient (on its stored elements)."""
    c = fixture[which]
    sd = synth_state_dict(c['sd_shapes'], c['sd_seed'], which == 'tied')
    loss, grads = tr.transformer_lm_loss_and_grads(c['inputs'], c['targets'], sd, c['params'])
    assert abs(float(loss) - float(c['loss'])) < 1e-5 * abs(float(c['loss']))
    assert set(grads) == set(c['grads'])
    for k, ref in c['grads'].items():
        assert _rel(sample(grads[k]), ref) < 1e-4, k


def test_fixture_batch_is_ragged_with_a_full_row(fixture):
    inputs, targets = fixture['tied']['inputs'], fixture['tied']['targets']
    counts = (targets != 0).sum(1)
    assert int(counts.max()) == targets.shape[1] and len(set(counts.tolist())) == targets.shape[0]
    assert torch.equal(inputs, small_batch()[0]) and torch.equal(targets, small_batch()[1])


def test_state_dict_matches_reference_transformer_lm_yaml(fixture):
    from opentransformer_b200.lm import LanguageModel
    lm = LanguageModel['transformer_lm'](TLM_YAML)
    assert lm.model_type == 'transformer_lm'
    assert {k: tuple(v.shape) for k, v in lm.state_dict().items()} == fixture['transformer_lm_yaml_keys']
    assert lm.output_project.weight is lm.embedding.weight


def _cuda_calls_fail(monkeypatch):
    """Any CUDA work from here on fails the test: the refusals must come first."""
    from opentransformer_b200 import _lib

    def no_device(*a, **k):
        raise AssertionError('device work before the refusal')
    monkeypatch.setattr(_lib, 'lib', no_device)
    monkeypatch.setattr(torch.cuda, 'current_stream', no_device)


def test_training_refuses_heads_that_are_not_64_wide(monkeypatch):
    """d_model 192 with 2 heads (96 wide) loads and predicts, but its training path raises before any device work: the
    public seam with and without gradients, the forward / backward function and FusedTrainer."""
    from opentransformer_b200 import lm as lm_mod
    from opentransformer_b200.train import FusedTrainer
    lm = lm_mod.TransformerLanguageModel(dict(small_params(True), d_model=192, n_heads=2))
    inputs, targets = small_batch()
    _cuda_calls_fail(monkeypatch)
    lm.train()
    for call in (lambda: lm({'inputs': inputs}, {'targets': targets}),
                 lambda: lm_mod.transformer_forward_backward(lm, inputs, targets),
                 lambda: FusedTrainer(lm)):
        with pytest.raises(NotImplementedError, match='64-wide attention heads only'):
            call()
    with torch.no_grad(), pytest.raises(NotImplementedError, match='64-wide attention heads only'):
        lm({'inputs': inputs}, {'targets': targets})


def test_fused_trainer_refuses_the_recurrent_lm(monkeypatch):
    from opentransformer_b200.lm import RecurrentLanguageModel
    from opentransformer_b200.train import FusedTrainer
    from tests.test_rnnlm_ref import small_params as rnn_params
    _cuda_calls_fail(monkeypatch)
    with pytest.raises(NotImplementedError, match='step-linear'):
        FusedTrainer(RecurrentLanguageModel(rnn_params(True)))


def test_unused_parameters_of_a_language_model():
    from opentransformer_b200.lm import TransformerLanguageModel
    from opentransformer_b200.train import unused_parameters
    assert unused_parameters(TransformerLanguageModel(small_params(False))) == set()


def test_dropout_sites_are_distinct():
    from opentransformer_b200 import lm, train
    tlm = {lm.TLM_SITE + 2 * i + k for i in range(64) for k in range(2)}
    rnn = {lm.RNNLM_SITE + k for k in range(64)}
    speech = {train.ENC_SITE + 3 * i + k for i in range(64) for k in range(3)} | {train.DEC_SITE + 3 * i + k for i in range(64)
                                                                                for k in range(3)}
    assert not (tlm & rnn) and not (tlm & speech)
