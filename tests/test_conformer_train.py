"""CPU checks of Conformer training: which configurations the training path accepts and refuses (before any device work),
its dropout sites and unused parameters, and the fp32 training-mode restatement the GPU tests compare against, pinned
to the reference's own modules in train()."""
import copy
import os

import pytest
import torch

import bench
from tests import conformer_train_ref as ref
from tests.test_head_dim_96 import CONFORMER_BASELINE, synth_state_dict


def _params(**enc):
    p = copy.deepcopy(bench.conformer_params())       # BASELINE config 4: d_model 256, 4 heads, d_ff 768 GLU, k 5
    p['encoder'].update(nblocks=2, residual_dropout=0.1)
    p['encoder'].update(enc)
    p['decoder'].update(n_blocks=1)
    return p


def _model(params):
    from opentransformer_b200.model import SpeechToText
    return SpeechToText(params)


def test_config4_conformer_is_accepted():
    from opentransformer_b200.train import TrainPack
    pk = TrainPack(_model(_params()))
    assert pk.conformer and len(pk.enc) == 2
    p = pk.enc[0]
    assert p['wext'].shape == (4 * 256, 256) and p['bext'].shape == (4 * 256,)
    assert p['dw'].shape == (256, 5)


def test_conv_dropout_is_accepted_and_ignored():
    """The reference builds ConformerConvolutionModule.dropout and never applies it (module/conformer.py:34,36-57)."""
    from opentransformer_b200.train import TrainPack
    TrainPack(_model(_params(conv_dropout=0.3)))


def test_d_model_384_conformer_is_refused_for_its_96_wide_heads():
    from opentransformer_b200.train import TrainPack
    with pytest.raises(NotImplementedError, match='64-wide attention heads'):
        TrainPack(_model(copy.deepcopy(CONFORMER_BASELINE)))


@pytest.mark.parametrize('flag,match', [
    (dict(macaron_style=False), 'macaron_style'),
    (dict(conv_first=True), 'conv_first'),
    (dict(relative_positional=False), 'relative positional'),
    (dict(ffn_dropout=0.1), 'only residual_dropout'),
    (dict(pos_dropout=0.1), 'pos_dropout'),
])
def test_out_of_scope_conformer_flags_are_refused(flag, match):
    from opentransformer_b200.train import TrainPack
    with pytest.raises(NotImplementedError, match=match):
        TrainPack(_model(_params(**flag)))


def test_relpos_transformer_encoder_is_refused():
    from opentransformer_b200.train import TrainPack
    p = bench.model_params()
    p['encoder'].update(n_blocks=1, relative_positional=True)
    p['decoder'].update(n_blocks=1)
    with pytest.raises(NotImplementedError, match='absolute positions'):
        TrainPack(_model(p))


def test_three_dropout_sites_per_conformer_block_clear_of_the_decoder():
    from opentransformer_b200.train import DEC_SITE, dropout_sites
    sites = dropout_sites(_model(_params()))
    enc = [s for s, part, _ in sites if part == 'encoder']
    assert enc == list(range(6))
    assert all(s >= DEC_SITE for s, part, _ in sites if part == 'decoder')
    assert all(r == 0.1 for _, _, r in sites)


def test_post_ffn_is_the_only_unused_parameter_group():
    from opentransformer_b200.train import unused_parameters
    m = _model(_params())
    unused = unused_parameters(m)
    assert unused and all('.post_ffn.' in n for n in unused)
    assert len(unused) == 2 * 4          # w_1 / w_2 weight and bias, two blocks


def test_training_restatement_equals_live_reference_in_train_mode():
    """The oracle's Conformer block in train() (tests/conformer_train_ref.py) against the REFERENCE's own SpeechToText in
    train() (tests/golden/live_ref_conformer_train.pt, from make_live_ref_conformer_train.py): loss, every parameter
    gradient (post_ffn.* gets none), and the BatchNorm running statistics after the forward -- batch statistics over the
    padded frames too, unbiased running_var."""
    c = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'live_ref_conformer_train.pt'),
                   weights_only=False)
    sd = synth_state_dict(c['sd_shapes'], c['sd_seed'])
    loss, grads, stats = ref.loss_and_grads_train(c['x'], c['mask'], c['tgt'], sd, c['params'], truth_length=c['tlen'])
    torch.testing.assert_close(loss, c['loss_ref'], rtol=1e-5, atol=1e-5)
    g_ref = c['g_ref']
    assert set(grads) == set(g_ref), set(grads) ^ set(g_ref)
    none = sorted(n for n, g in g_ref.items() if g is None)
    assert none and all('.post_ffn.' in n for n in none)
    for n in grads:
        if g_ref[n] is None:
            assert grads[n] is None, n
        else:
            torch.testing.assert_close(grads[n], g_ref[n], rtol=2e-4, atol=2e-6, msg=lambda m, n=n: f'{n}: {m}')
    for n, want in c['stats_ref'].items():
        if 'num_batches' in n:
            assert int(want) == 1
            continue
        torch.testing.assert_close(stats[n], want, rtol=1e-5, atol=1e-6, msg=lambda m, n=n: f'{n}: {m}')
