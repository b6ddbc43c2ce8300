"""CPU checks of the conv front end at any kernel size and stride: the restatement (tests/conv_frontend_ref.py) against the
reference's own modules (tests/golden/live_ref_conv_frontend.pt), the port's geometry, masks and input window against the
reference module's for every supported (k, s), the C geometry against the Python one, state_dict keys and shapes, and the
refusals, which come before any device work."""
import copy
import ctypes
import os

import pytest
import torch

from tests import concat_frontend_ref as cref
from tests import conv_frontend_ref as vref
from tests import ctc_ref
from tests.test_head_dim_96 import synth_state_dict
from tests.test_transformer_lm_ref import _cuda_calls_fail, sample

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'live_ref_conv_frontend.pt')


@pytest.fixture(scope='module')
def fixture():
    return torch.load(GOLDEN, weights_only=False)


def test_restated_front_end_equals_the_reference(fixture):
    """Outputs and masks of every stored geometry, with and without front_end_layer_norm, on a ragged batch."""
    for c in fixture['frontend']:
        kw = c['kwargs']
        sd = synth_state_dict(c['sd_shapes'], c['sd_seed'])
        y, m = vref.conv_frontend(c['x'], c['mask'], sd, '', kw, layer_norm_out=kw['front_end_layer_norm'])
        torch.testing.assert_close(y, c['y'], rtol=1e-5, atol=1e-5)
        assert torch.equal(m, c['mask_out']), (kw['kernel_size'], kw['stride'])


def test_port_and_c_geometry_equal_the_reference_module(fixture):
    """T', the output mask and input_window of the port's module for T 1..64 and every (k, s) in 1..7 x 1..4; where the
    reference's conv2d raises the port raises ValueError.  The C entry point (otb_conv_geometry) agrees."""
    from opentransformer_b200 import _lib
    from opentransformer_b200.modules import ConvFrontEnd
    fes = {}
    lib = _lib.lib()
    out = (ctypes.c_int * 6)()
    for k, s, T, T2, n_mask in fixture['geometry'].tolist():
        fe = fes.setdefault((k, s), ConvFrontEnd(9, 32, mid_channel=8, out_channel=16, kernel_size=[k, k], stride=[s, s]))
        mask = torch.arange(T)[None] < T - T // 3
        if T2 < 0:
            with pytest.raises(ValueError, match='too short'):
                fe.output_length(T)
            with pytest.raises(ValueError, match='too short'):
                fe.output_mask(mask)
            assert lib.otb_conv_geometry(T, 9, k, k, s, s, k, k, s, s, out) != 0
            continue
        m = fe.output_mask(mask)
        assert (fe.output_length(T), m.shape[1]) == (T2, n_mask), (k, s, T)
        assert lib.otb_conv_geometry(T, 9, k, k, s, s, k, k, s, s, out) == 0
        assert list(out)[:4] == [v for hw in fe.sizes(T) for v in hw]
        assert fe.input_window() == (s * s, k + (k - 1) * s)


def test_module_masks_and_sizes_on_the_stored_geometries(fixture):
    """The port's output_mask and conv output sizes on the stored asymmetric geometries (int and pair kwargs mixed)."""
    from opentransformer_b200.modules import ConvFrontEnd
    for c in fixture['frontend']:
        fe = ConvFrontEnd(**c['kwargs'])
        T = c['x'].shape[1]
        assert torch.equal(fe.output_mask(c['mask']), c['mask_out'])
        assert fe.output_length(T) == c['y'].shape[1]
        assert (fe.conv1.output_size, fe.conv2.output_size) == c['output_size']
        assert fe.sizes(T)[1][1] == c['output_size'][1]


def test_speech2text_restatement_equals_live_reference(fixture):
    """SpeechToText (conv front end at stride [2, 3] with front_end_layer_norm, joint CTC) in train(): every gradient."""
    c = fixture['speech2text']
    sd = synth_state_dict(c['sd_shapes'], c['sd_seed'])
    with vref.conv_frontend_of(c['params']):
        loss, grads = cref.speech2text_loss_and_grads(c['x'], c['mask'], c['tgt'], c['tlen'], sd, c['params'])
    torch.testing.assert_close(loss, c['loss_ref'], rtol=1e-5, atol=1e-5)
    assert set(grads) == set(c['g_ref']) and 'frontend.layer_norm.weight' in grads
    for n, want in c['g_ref'].items():
        torch.testing.assert_close(sample(grads[n]), want, rtol=2e-4, atol=2e-6, msg=lambda m, n=n: f'{n}: {m}')


def test_ctc_model_restatement_equals_live_reference(fixture):
    """CTCModel (conv front end, kernels [[5, 5], [3, 3]] at stride [3, 2]) in train(): loss and every gradient."""
    c = fixture['ctc']
    sd = synth_state_dict(c['sd_shapes'], c['sd_seed'])
    with vref.conv_frontend_of(c['params']):
        loss, grads, _ = ctc_ref.loss_and_grads_train(c['x'], c['mask'], c['tgt'], c['tlen'], sd, c['params'])
    torch.testing.assert_close(loss, c['loss_ref'], rtol=1e-5, atol=1e-5)
    assert set(grads) == {n for n, v in c['g_ref'].items() if v is not None}
    for n, want in c['g_ref'].items():
        torch.testing.assert_close(sample(grads[n]), want, rtol=2e-4, atol=2e-6, msg=lambda m, n=n: f'{n}: {m}')


def test_state_dict_keys_and_shapes_match_the_reference(fixture):
    from opentransformer_b200.model import CTCModel, SpeechToText
    from opentransformer_b200.modules import ConvFrontEnd
    for c in fixture['frontend']:
        fe = ConvFrontEnd(**c['kwargs'])
        assert {k: (tuple(v.shape), str(v.dtype).replace('torch.', '')) for k, v in fe.state_dict().items()} == c['sd_shapes']
    for kind, cls in (('speech2text', SpeechToText), ('ctc', CTCModel)):
        c = fixture[kind]
        ref_sd = synth_state_dict(c['sd_shapes'], c['sd_seed'])
        m = cls(c['params'])
        assert {k: (tuple(v.shape), str(v.dtype).replace('torch.', '')) for k, v in m.state_dict().items()} == c['sd_shapes']
        m.load_state_dict(ref_sd, strict=True)


def test_reference_kwargs_are_accepted():
    """act_func_type is ignored (the reference always applies relu); dropout is accepted for recognition."""
    from opentransformer_b200.modules import ConvFrontEnd
    fe = ConvFrontEnd(80, 256, mid_channel=64, out_channel=64, kernel_size=[3, [5, 3]], stride=[[2, 3], 2], dropout=0.1,
                      act_func_type='swish', front_end_layer_norm=True)
    assert fe.geom == (3, 3, 2, 3, 5, 3, 2, 2) and fe.input_window() == (4, 3 + 4 * 2)
    assert fe.sizes(100) == [(49, 27), (23, 14)]


@pytest.mark.parametrize('kernel_size,stride', [([[8, 3], [3, 3]], [2, 2]), ([[3, 3], [3, 0]], [2, 2]),
                                                ([[3, 3], [3, 3]], [5, 2]), ([[3, 3], [3, 3]], [[2, 2], [1, 5]]),
                                                ([0, 3], [2, 2])])
def test_out_of_range_geometry_is_refused_at_construction(kernel_size, stride):
    from opentransformer_b200.modules import ConvFrontEnd
    with pytest.raises(NotImplementedError, match='kernel sizes 1..7 and strides 1..4'):
        ConvFrontEnd(80, 256, kernel_size=kernel_size, stride=stride)


def _s2t_params(fixture, **frontend):
    params = copy.deepcopy(fixture['speech2text']['params'])
    params['frontend'].update(frontend)
    return params


def test_too_short_input_is_refused_before_any_device_work(monkeypatch, fixture):
    """T shorter than one output frame: the front end, the recognizer's encode and the training pass raise ValueError
    before any CUDA call."""
    from opentransformer_b200.model import CTCModel, SpeechToText
    from opentransformer_b200.modules import ConvFrontEnd
    _cuda_calls_fail(monkeypatch)
    fe = ConvFrontEnd(20, 64, mid_channel=8, out_channel=16, kernel_size=[[5, 5], [3, 3]], stride=[3, 2]).eval()
    x, mask = torch.zeros(1, 10, 20), torch.ones(1, 10, dtype=torch.bool)    # T1 = 2 < 3
    for call in (lambda: fe.forward_bf16(x), lambda: fe(x, mask), lambda: fe.inference(x, mask, None)):
        with pytest.raises(ValueError, match='too short'):
            call()
    m = SpeechToText(_s2t_params(fixture))                                       # stride [2, 3]: T 6 gives T1 2 < 3
    x1, mask1 = torch.zeros(2, 6, 20), torch.ones(2, 6, dtype=torch.bool)
    tgt, tlen = torch.tensor([[1, 5, 1], [1, 6, 1]]), torch.tensor([2, 2])
    with pytest.raises(ValueError, match='too short'):
        m.eval().encode_bf16(x1, mask1)
    with pytest.raises(ValueError, match='too short'):
        m.train()({'inputs': x1, 'mask': mask1}, {'targets': tgt, 'targets_length': tlen})
    cm = CTCModel(fixture['ctc']['params']).train()
    with pytest.raises(ValueError, match='too short'):
        cm({'inputs': torch.zeros(1, 4, 16), 'mask': torch.ones(1, 4, dtype=torch.bool)},
           {'targets': tgt[:1], 'targets_length': tlen[:1]})


def test_training_refuses_front_end_dropout_and_a_wide_front_layer_norm(monkeypatch, fixture):
    from opentransformer_b200.model import SpeechToText
    from opentransformer_b200.train import TrainPack
    _cuda_calls_fail(monkeypatch)
    with pytest.raises(NotImplementedError, match='front-end dropout 0.1'):
        TrainPack(SpeechToText(_s2t_params(fixture, dropout=0.1)))
    params = _s2t_params(fixture, output_size=320)
    for part in ('encoder', 'decoder'):
        params[part].update(d_model=320, n_heads=5)
    params['decoder']['memory_dim'] = params['encoder_output_size'] = 320
    with pytest.raises(NotImplementedError, match='front_end_layer_norm over output_size 320'):
        TrainPack(SpeechToText(params))
    SpeechToText(_s2t_params(fixture, dropout=0.1)).eval()          # recognition takes it: dropout is the identity there
