"""The recurrent language model (model/lm.py:31-90, rnnlm.yaml) without a GPU: its fp32 restatement (tests/rnnlm_ref.py) against the reference's own
RecurrentLanguageModel (tests/golden/live_ref_rnnlm.pt, made by tests/golden/make_live_ref_rnnlm.py), the port's state_dict
against the reference's for rnnlm.yaml, the registry, and the configurations the CUDA path refuses."""
import os

import pytest
import torch

from tests import rnnlm_ref as rr

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, 'golden', 'live_ref_rnnlm.pt')

# egs/aishell/conf/rnnlm.yaml, model section
RNNLM_YAML = dict(type='rnn_lm', vocab_size=4233, num_layers=2, hidden_size=1024, residual_dropout=0.1, smoothing=0.1, dropout=0.1,
                  share_embedding=True)
H100_SMS, H100_SMEM_OPTIN = 132, 232448


def small_params(tied):
    return dict(type='rnn_lm', vocab_size=40, num_layers=2, hidden_size=64, residual_dropout=0.1, smoothing=0.1, dropout=0.0,
                share_embedding=tied)


def small_batch():
    """inputs [3, 9] (BOS + tokens, PAD after each length), targets [3, 9] (tokens + EOS, PAD-padded)."""
    g = torch.Generator().manual_seed(5)
    toks = torch.randint(2, 40, (3, 9), generator=g)
    lens = torch.tensor([9, 6, 3])
    inputs = torch.cat([torch.ones(3, 1, dtype=torch.long), toks[:, :-1]], 1)
    targets = toks.clone()
    for b, n in enumerate(lens.tolist()):
        targets[b, n - 1] = 1
        targets[b, n:] = 0
        inputs[b, n:] = 0
    return inputs, targets


def synth_state_dict(shapes, seed, tied):
    """Deterministic weights for the given {key: shape}: uniform(-0.3, 0.3) in key order; a tied output_project.weight is the
    embedding."""
    g = torch.Generator().manual_seed(seed)
    sd = {k: torch.rand(shape, generator=g) * 0.6 - 0.3 for k, shape in shapes.items()}
    if tied:
        sd['output_project.weight'] = sd['embedding.weight']
    return sd


@pytest.fixture(scope='module')
def fixture():
    return torch.load(FIXTURE)


def _rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize('which', ['tied', 'untied'])
def test_oracle_matches_reference(fixture, which):
    """fp32 oracle vs the reference run on the same weights: only summation order differs, so 1e-5 relative."""
    c = fixture[which]
    tied = which == 'tied'
    sd = synth_state_dict(c['sd_shapes'], c['sd_seed'], tied)
    lp, (h, cc) = rr.rnn_lm_predict(c['inputs'], sd, '', 2)
    assert _rel(lp, c['log_probs']) < 1e-5 and _rel(h, c['h_n']) < 1e-5 and _rel(cc, c['c_n']) < 1e-5
    lp1, hid = rr.rnn_lm_predict(c['inputs'][:, :4], sd, '', 2)
    lp2, (h2, c2) = rr.rnn_lm_predict(c['inputs'][:, 4:], sd, '', 2, hidden=hid)
    assert _rel(torch.cat([lp1, lp2], 1), c['carried_log_probs']) < 1e-5
    assert _rel(h2, c['carried_h_n']) < 1e-5 and _rel(c2, c['carried_c_n']) < 1e-5
    loss, grads = rr.rnn_lm_loss_and_grads(c['inputs'], c['targets'], sd, c['params'])
    assert abs(float(loss) - float(c['loss'])) < 1e-5 * abs(float(c['loss']))
    assert set(grads) == set(c['grads'])
    for k, ref in c['grads'].items():
        assert _rel(grads[k], ref) < 1e-4, k


def test_state_dict_matches_reference_rnnlm_yaml(fixture):
    from opentransformer_b200.lm import LanguageModel
    lm = LanguageModel['rnn_lm'](RNNLM_YAML)
    assert lm.model_type == 'recurrent_lm'
    assert {k: tuple(v.shape) for k, v in lm.state_dict().items()} == fixture['rnnlm_yaml_keys']
    assert lm.output_project.weight is lm.embedding.weight
    assert lm.init_hidden_states(3, 'cpu').shape == (2, 3, 1024)


def test_registry():
    from opentransformer_b200.lm import LanguageModel, RecurrentLanguageModel, TransformerLanguageModel
    assert LanguageModel['rnn_lm'] is RecurrentLanguageModel and LanguageModel['transformer_lm'] is TransformerLanguageModel


def test_limits_raise():
    from opentransformer_b200 import build, ops
    from opentransformer_b200.lm import RecurrentLanguageModel
    with pytest.raises(NotImplementedError, match='multiple of 8'):
        RecurrentLanguageModel(dict(RNNLM_YAML, hidden_size=1020))
    build.build()
    assert ops.lstm_config(1024, H100_SMS, H100_SMEM_OPTIN)[0] == 8          # 128 CTAs of 8 units
    assert ops.lstm_config(64, H100_SMS, H100_SMEM_OPTIN)[0] == 8
    with pytest.raises(NotImplementedError, match='multiple of 8'):
        ops.lstm_config(1020, H100_SMS, H100_SMEM_OPTIN)
    with pytest.raises(NotImplementedError, match='does not fit'):
        ops.lstm_config(2048, H100_SMS, H100_SMEM_OPTIN)                  # 16 units x 4 gates x 2048 x bf16 = 256 KB
