"""CPU checks of the low-frame-rate front ends (`concat`, `concat-with-linear`): the restatement (tests/concat_frontend_ref.py)
against the reference's own modules (tests/golden/live_ref_concat_frontend.pt), the port's geometry against the reference
module's for every small configuration, the registry, kwargs and state_dict keys, and the refusals, which come before any
device work."""
import copy
import os

import pytest
import torch

from tests import concat_frontend_ref as cref
from tests import ctc_ref
from tests.test_head_dim_96 import synth_state_dict
from tests.test_transformer_lm_ref import _cuda_calls_fail, sample

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'live_ref_concat_frontend.pt')


@pytest.fixture(scope='module')
def fixture():
    return torch.load(GOLDEN, weights_only=False)


def _fe(c):
    return {'left_frames': c['left'], 'right_frames': c['right'], 'frame_rate': c['frame_rate']}


def test_restated_front_ends_equal_the_reference(fixture):
    """Outputs and masks exactly, for T - n a multiple of the stride and not, T < n, n = 1 and ragged masks."""
    for c in fixture['frontend']:
        y, m = cref.concat_frontend(c['x'], c['mask'], {}, '', _fe(c), False)
        assert torch.equal(y, c['y']) and torch.equal(m, c['mask_out']), (c['left'], c['right'], c['frame_rate'])
        sd = synth_state_dict(c['sd_shapes'], c['sd_seed'])              # keys linear.weight / linear.bias
        yl, ml = cref.concat_frontend(c['x'], c['mask'], sd, '', _fe(c), True)
        torch.testing.assert_close(yl, c['y_linear'], rtol=1e-6, atol=1e-6)
        assert torch.equal(ml, c['mask_out'])


def test_port_geometry_equals_the_reference_module(fixture):
    """T' and the output mask's length of the port's module, for T 1..64 and every (n, s) with right < s <= 4; where the
    reference's nn.Unfold fails the port raises ValueError."""
    from opentransformer_b200.modules import ConcatFeatureFrontEnd
    fes = {}
    for left, right, rate, T, T2, n_valid in fixture['geometry'].tolist():
        fe = fes.setdefault((left, right, rate), ConcatFeatureFrontEnd(1, left, right, rate))
        mask = torch.arange(T)[None] < T - T // 3
        if T2 < 0:
            with pytest.raises(ValueError, match='fewer than'):
                fe.output_length(T)
            with pytest.raises(ValueError, match='fewer than'):
                fe.output_mask(mask)
            continue
        m = fe.output_mask(mask)
        assert (fe.output_length(T), int(m.sum())) == (T2, n_valid) and m.shape[1] == T2, (left, right, rate, T)
        assert cref.geometry(T, left, right, rate)[4] == T2


def test_speech2text_restatement_equals_live_reference(fixture):
    """SpeechToText (concat-with-linear, Transformer encoder, joint CTC) in train(): loss and every gradient."""
    c = fixture['speech2text']
    sd = synth_state_dict(c['sd_shapes'], c['sd_seed'])
    loss, grads = cref.speech2text_loss_and_grads(c['x'], c['mask'], c['tgt'], c['tlen'], sd, c['params'])
    torch.testing.assert_close(loss, c['loss_ref'], rtol=1e-5, atol=1e-5)
    assert set(grads) == set(c['g_ref'])
    assert 'frontend.linear.weight' in grads
    for n, want in c['g_ref'].items():
        torch.testing.assert_close(sample(grads[n]), want, rtol=2e-4, atol=2e-6, msg=lambda m, n=n: f'{n}: {m}')


def test_ctc_model_restatement_equals_live_reference(fixture):
    """CTCModel (concat, rel-pos Conformer) in train(): loss, every gradient (post_ffn.* none) and BatchNorm statistics."""
    c = fixture['ctc']
    sd = synth_state_dict(c['sd_shapes'], c['sd_seed'])
    with cref.frontend_of(c['params']):
        loss, grads, stats = ctc_ref.loss_and_grads_train(c['x'], c['mask'], c['tgt'], c['tlen'], sd, c['params'])
    torch.testing.assert_close(loss, c['loss_ref'], rtol=1e-5, atol=1e-5)
    assert set(grads) == set(c['g_ref']) and not any(n.startswith('frontend.') for n in grads)
    for n, want in c['g_ref'].items():
        if want is None:
            assert grads[n] is None and '.post_ffn.' in n, n
            continue
        torch.testing.assert_close(sample(grads[n]), want, rtol=2e-4, atol=2e-6, msg=lambda m, n=n: f'{n}: {m}')
    for n, want in c['stats_ref'].items():
        if 'num_batches' not in n:
            torch.testing.assert_close(stats[n], want, rtol=1e-5, atol=1e-6, msg=lambda m, n=n: f'{n}: {m}')


def test_registry_kwargs_and_state_dict_keys_match_the_reference(fixture):
    from opentransformer_b200.model import BuildFrontEnd, CTCModel, SpeechToText
    from opentransformer_b200.modules import ConcatFeatureFrontEnd, ConcatWithLinearFrontEnd, ConvFrontEnd
    assert BuildFrontEnd == {'concat': ConcatFeatureFrontEnd, 'concat-with-linear': ConcatWithLinearFrontEnd,
                             'conv': ConvFrontEnd}
    fe = ConcatWithLinearFrontEnd(input_size=80, output_size=256, left_frames=3, right_frames=0, frame_rate=40, dropout=0.0)
    assert (fe.nframes, fe.stride, fe.output_size, fe.linear.in_features, fe.linear.out_features) == (4, 4, 320, 320, 256)
    assert set(fe.state_dict()) == {'linear.weight', 'linear.bias'}
    assert ConcatFeatureFrontEnd(80, 2, 0).state_dict() == {} and ConcatFeatureFrontEnd(80, 2, 0).stride == 3
    for kind, cls in (('speech2text', SpeechToText), ('ctc', CTCModel)):
        c = fixture[kind]
        ref_sd = synth_state_dict(c['sd_shapes'], c['sd_seed'])
        m = cls(c['params'])
        assert {k: (tuple(v.shape), str(v.dtype).replace('torch.', '')) for k, v in m.state_dict().items()} == c['sd_shapes']
        m.load_state_dict(ref_sd, strict=True)                  # a reference state_dict loads key for key
        assert all(torch.equal(m.state_dict()[k], v) for k, v in ref_sd.items())


def test_encoder_frames_to_input_takes_the_front_ends_window():
    from opentransformer_b200.model import encoder_frames_to_input
    from opentransformer_b200.modules import ConcatFeatureFrontEnd
    spans = torch.tensor([[[0, 1], [2, 5], [-1, -1]]])
    assert encoder_frames_to_input(spans).tolist() == [[[0, 7], [8, 23], [-1, -1]]]
    fe = ConcatFeatureFrontEnd(80, 2, 1, 30)                # n 4, s 3: frame t stacks [3t, 3t + 4)
    assert encoder_frames_to_input(spans, frontend=fe).tolist() == [[[0, 4], [6, 16], [-1, -1]]]
    sec = encoder_frames_to_input(spans, 0.01, frontend=fe)
    assert sec.dtype == torch.float64 and sec[0, 1].tolist() == pytest.approx([0.06, 0.16]) and sec[0, 2].tolist() == [-1, -1]


@pytest.mark.parametrize('kwargs,exc,match', [
    (dict(left_frames=3, right_frames=4, frame_rate=40), ValueError, 'less than the stride'),
    (dict(left_frames=0, right_frames=1, frame_rate=10), ValueError, 'less than the stride'),
    (dict(left_frames=3, right_frames=0, frame_rate=9), ValueError, 'frame_rate'),
])
def test_constructor_refusals(kwargs, exc, match):
    from opentransformer_b200.modules import ConcatFeatureFrontEnd, ConcatWithLinearFrontEnd
    with pytest.raises(exc, match=match):
        ConcatFeatureFrontEnd(80, **kwargs)
    with pytest.raises(exc, match=match):
        ConcatWithLinearFrontEnd(80, 256, **kwargs)


def test_dropout_is_refused():
    from opentransformer_b200.modules import ConcatWithLinearFrontEnd
    with pytest.raises(NotImplementedError, match='dropout'):
        ConcatWithLinearFrontEnd(80, 256, 3, 0, 40, dropout=0.1)


def test_too_short_input_is_refused_before_any_device_work(monkeypatch, fixture):
    """T_p < n: the front end, the recognizer's encode and the training pass raise ValueError before any CUDA call."""
    from opentransformer_b200.model import CTCModel, SpeechToText
    from opentransformer_b200.modules import ConcatWithLinearFrontEnd
    _cuda_calls_fail(monkeypatch)
    fe = ConcatWithLinearFrontEnd(5, 16, 5, 1, 20).eval()   # n 7, s 2: T 4 pads to 4
    x, mask = torch.zeros(1, 4, 5), torch.ones(1, 4, dtype=torch.bool)
    for call in (lambda: fe.forward_bf16(x), lambda: fe(x, mask), lambda: fe.inference(x, mask, None)):
        with pytest.raises(ValueError, match='fewer than'):
            call()
    params = copy.deepcopy(fixture['speech2text']['params'])
    params['frontend'].update(left_frames=5, right_frames=1, frame_rate=20)                 # n 7, s 2: T 4 pads to 5
    m = SpeechToText(params)
    x1, mask1 = torch.zeros(2, 4, 20), torch.ones(2, 4, dtype=torch.bool)
    tgt, tlen = torch.tensor([[1, 5, 1], [1, 6, 1]]), torch.tensor([2, 2])
    with pytest.raises(ValueError, match='fewer than'):
        m.eval().encode_bf16(x1, mask1)
    with pytest.raises(ValueError, match='fewer than'):
        m.train()({'inputs': x1, 'mask': mask1}, {'targets': tgt, 'targets_length': tlen})
    cm = CTCModel(fixture['ctc']['params']).train()                          # n 4, s 2: T 2 pads to 2
    with pytest.raises(ValueError, match='fewer than'):
        cm({'inputs': torch.zeros(1, 2, 32), 'mask': torch.ones(1, 2, dtype=torch.bool)},
           {'targets': tgt[:1], 'targets_length': tlen[:1]})
