"""CPU checks of the layer options training takes beside GLU / ReLU and residual_dropout: the gelu, tanh and swish
feed-forwards and the attention's output dropout (slf_attn_dropout, src_attn_dropout).

The fp32 restatement the GPU tests compare against (oracle/speech_model.py, tests/conformer_train_ref.py) is pinned here to
the reference's own modules in train() (tests/golden/live_ref_layer_options.pt, from make_live_ref_layer_options.py),
including the placement of the attention dropout, with the masks torch drew replayed.  Then what TrainPack accepts and
refuses, and the dropout site ids, all before any device work."""
import os

import pytest
import torch

from oracle import speech_model as om
from oracle import train_step as ot
from tests import conformer_train_ref as conf_ref
from tests.test_head_dim_96 import synth_state_dict
from tests.test_gpu_train import _params as speech_params

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'live_ref_layer_options.pt')


def _fixture():
    return torch.load(FIXTURE, weights_only=False)


def _grads(c):
    """The reference's gradients of a case: name -> tensor (the fixture keeps them as one flat fp32 tensor)."""
    out, o = {}, 0
    for n, shape in zip(c['g_names'], c['g_shapes']):
        k = int(torch.Size(shape).numel())
        out[n] = c['g_flat'][o:o + k].view(shape)
        o += k
    assert o == c['g_flat'].numel()
    return out


def _replay(c):
    """oracle.set_dropout's fn for the masks the reference drew: every mask recorded on (block, sub-layer), scaled."""
    p = c['params']
    rate = {'res': p['encoder']['residual_dropout'], 'attn': p['encoder']['slf_attn_dropout']}
    assert p['decoder']['residual_dropout'] == rate['res'] and p['decoder']['slf_attn_dropout'] == rate['attn']
    assert p['decoder']['src_attn_dropout'] == rate['attn']

    def drop(site, t):
        for kind in ('attn', 'res'):
            m = c['masks'].get(site + (kind,))
            if m is not None:
                t = t * m.float() / (1.0 - rate[kind])
        return t
    return drop


@pytest.mark.parametrize('name', ['postnorm-gelu', 'postnorm-tanh', 'postnorm-swish', 'prenorm-gelu', 'prenorm-tanh',
                                  'prenorm-swish', 'conformer-swish', 'attn-dropout'])
def test_restatement_equals_live_reference(name):
    f = _fixture()
    b, c = f['batch'], f['cases'][name]
    sd = synth_state_dict(c['sd_shapes'], c['sd_seed'])
    sd = {k: v for k, v in sd.items() if k.split('.')[0] in ('frontend', 'encoder', 'decoder', 'assistor')}
    if name.startswith('conformer'):
        loss, grads, _ = conf_ref.loss_and_grads_train(b['x'], b['mask'], b['tgt'], sd, c['params'], truth_length=b['tlen'])
    elif name == 'attn-dropout':
        om.set_dropout(_replay(c))
        try:
            loss, grads = ot.loss_and_grads(b['x'], b['mask'], b['tgt'], sd, c['params'])
        finally:
            om.set_dropout(None)
    else:
        loss, grads = ot.loss_and_grads(b['x'], b['mask'], b['tgt'], sd, c['params'])
    torch.testing.assert_close(loss, c['loss_ref'], rtol=1e-5, atol=1e-5)
    g_ref = _grads(c)
    assert set(n for n, g in grads.items() if g is not None) == set(g_ref)
    assert all('.post_ffn.' in n for n in c['g_none']), c['g_none']      # a Conformer's post_ffn: read by no forward
    for n, want in g_ref.items():
        torch.testing.assert_close(grads[n], want, rtol=2e-4, atol=2e-6, msg=lambda m, n=n: f'{n}: {m}')


def test_attention_dropout_changes_the_reference_loss():
    """The recorded masks matter: without them the restatement gives another loss."""
    f = _fixture()
    b, c = f['batch'], f['cases']['attn-dropout']
    sd = synth_state_dict(c['sd_shapes'], c['sd_seed'])
    sd = {k: v for k, v in sd.items() if k.split('.')[0] in ('frontend', 'encoder', 'decoder')}
    loss, _ = ot.loss_and_grads(b['x'], b['mask'], b['tgt'], sd, c['params'])
    assert abs(float(loss) - float(c['loss_ref'])) > 1e-3
    assert {k[2] for k in c['masks']} == {'attn', 'res'}


def _model(params):
    from opentransformer_b200.model import SpeechToText
    torch.manual_seed(0)
    return SpeechToText(params)


@pytest.mark.parametrize('act', ['gelu', 'tanh', 'swish'])
@pytest.mark.parametrize('pre', [False, True])
def test_trainpack_accepts_the_activations(act, pre):
    from opentransformer_b200.train import TrainPack
    p = speech_params(n_enc=1, n_dec=1)
    for part in ('encoder', 'decoder'):
        p[part]['activation'] = act
        p[part]['normalize_before'] = pre
    pk = TrainPack(_model(p))
    assert pk.enc[0]['act'] == act and pk.dec[0]['act'] == act


def test_trainpack_accepts_the_attention_dropout():
    from opentransformer_b200 import train
    p = speech_params(n_enc=2, n_dec=1)
    p['encoder']['slf_attn_dropout'] = 0.1
    p['decoder']['slf_attn_dropout'] = 0.2
    p['decoder']['src_attn_dropout'] = 0.3
    model = _model(p)
    pk = train.TrainPack(model)
    assert pk.rates == {'encoder': [0.0, 0.0], 'decoder': [0.0]}           # residual_dropout 0: the attention's masks alone
    assert pk.attn_rates == {'encoder': [(0.1, 0.0)] * 2, 'decoder': [(0.2, 0.3, 0.0)]}
    with pytest.raises(ValueError, match='drop_seed'):                   # refused before any device work
        train.forward_backward(model, torch.zeros(1, 40, 80), torch.ones(1, 40, dtype=torch.bool), torch.ones(1, 3, dtype=torch.long))


@pytest.mark.parametrize('key,part', [('ffn_dropout', 'encoder'), ('ffn_dropout', 'decoder')])
def test_ffn_dropout_is_still_refused(key, part):
    from opentransformer_b200.train import TrainPack
    p = speech_params(n_enc=1, n_dec=1)
    p[part]['slf_attn_dropout'] = 0.1
    p[part][key] = 0.1
    with pytest.raises(NotImplementedError, match='only residual_dropout'):
        TrainPack(_model(p))


def test_pos_dropout_is_still_refused():
    from opentransformer_b200.train import TrainPack
    p = speech_params(n_enc=1, n_dec=1)
    p['encoder']['pos_dropout'] = 0.1
    with pytest.raises(NotImplementedError, match='pos_dropout'):
        TrainPack(_model(p))


def test_attention_rate_out_of_range_is_refused():
    from opentransformer_b200.train import TrainPack
    p = speech_params(n_enc=1, n_dec=1)
    p['decoder']['src_attn_dropout'] = 1.0
    with pytest.raises(ValueError, match='src_attn_dropout'):
        TrainPack(_model(p))


def test_attention_sites_are_a_range_of_their_own():
    """ATTN_SITE + the residual site: clear of every residual range (encoder, decoder, MWER, the language models'), and
    turning the attention dropout on leaves the residual sites as they were."""
    from opentransformer_b200 import lm, train
    p = speech_params(n_enc=12, n_dec=6)
    for part in ('encoder', 'decoder'):
        p[part]['residual_dropout'] = 0.1
    before = train.dropout_sites(_model(p))
    p['encoder']['slf_attn_dropout'] = 0.1
    p['decoder']['slf_attn_dropout'] = 0.1
    p['decoder']['src_attn_dropout'] = 0.1
    model = _model(p)
    assert train.dropout_sites(model) == before
    attn = train.attn_dropout_sites(model)
    assert len(attn) == 12 + 2 * 6
    ids = [s for s, _, _ in attn]
    assert len(set(ids)) == len(ids) and min(ids) >= train.ATTN_SITE
    residual = {s for s, _, _ in before}
    mwer = {train.MWER_SITE + 3 * i + k for i in range(6) for k in range(3)}
    lms = {lm.TLM_SITE + k for k in range(2 * 12)} | {lm.RNNLM_SITE + k for k in range(8)}
    assert not set(ids) & (residual | mwer | lms)
    assert ids[:2] == [train.ATTN_SITE + 0, train.ATTN_SITE + 2]                          # encoder layer i: 2 i + 0
    assert (train.ATTN_SITE + train.DEC_SITE, 'decoder', 0.1) in attn and (train.ATTN_SITE + train.DEC_SITE + 1, 'decoder', 0.1) in attn
