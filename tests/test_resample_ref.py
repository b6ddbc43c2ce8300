"""The float64 resampling restatement (tests/resample_ref.py) against torchaudio.functional.resample, and the host-side
refusals of ops.resample and FbankExtractor's rate / speed arguments, before any device work."""
import math

import numpy as np
import pytest
import torch

from tests import resample_ref as rr

ta = pytest.importorskip('torchaudio')

PAIRS = ((16000, 14400), (16000, 17600), (8000, 16000), (44100, 16000), (22050, 16000), (16000, 8000), (32000, 16000),
         (48000, 16000))


def _signal(L, seed):
    g = np.random.default_rng(seed)
    t = np.arange(L)
    return 0.5 * np.sin(2 * np.pi * 0.013 * t) + 0.3 * np.sin(2 * np.pi * 0.41 * t + 1.0) + 0.2 * g.standard_normal(L)


@pytest.mark.parametrize('orig,new', PAIRS)
def test_restatement_equals_torchaudio_in_float64(orig, new):
    o, _ = rr.reduced(orig, new)
    for L in sorted({1, 2, 23, 24, 25, o, 16007, 3 * orig}):
        x = _signal(L, L)
        ref = ta.functional.resample(torch.from_numpy(x), orig, new).numpy()
        got = rr.resample(x, orig, new)
        assert got.shape == ref.shape == (rr.out_length(L, orig, new),)
        assert got.shape[0] == math.ceil(new * L / orig)
        err = float(np.abs(got - ref).max()) if L else 0.0
        assert err < 1e-12, (orig, new, L, err)


def test_table_sizes_match_the_formula():
    # the phase tables the kernel's shared memory has to hold, from the formula
    for (orig, new), (o, n, w) in {(16000, 14400): (10, 9, 7), (16000, 17600): (10, 11, 7), (8000, 16000): (1, 2, 7),
                                   (44100, 16000): (441, 160, 17), (22050, 16000): (441, 320, 9)}.items():
        h, width = rr.phase_table(orig, new)
        assert rr.reduced(orig, new) == (o, n) and width == w and h.shape == (n, 2 * w + o)


def test_equal_rates_pass_through():
    x = _signal(101, 3)
    assert np.array_equal(rr.resample(x, 16000, 16000), x)


@pytest.fixture
def no_device(monkeypatch):
    """Arm it after building what the test needs: from then on every way to reach the GPU fails loudly."""
    from opentransformer_b200 import _lib

    def refuse(*a, **k):
        raise AssertionError('reached the device')

    def arm():
        for name in ('current_device', 'current_stream', 'init', 'synchronize', 'set_device'):
            monkeypatch.setattr(torch.cuda, name, refuse)
        monkeypatch.setattr(_lib, 'lib', refuse)
        monkeypatch.setattr(torch.Tensor, 'cuda', refuse)
        monkeypatch.setattr(torch.Tensor, 'to', refuse)
        monkeypatch.setattr(torch, 'randint', refuse)
    return arm


def test_op_refusals_come_before_any_device_work(no_device):
    from opentransformer_b200 import ops
    x, lens = torch.zeros(2, 100), torch.full((2,), 100, dtype=torch.int32)
    no_device()
    for orig, new in ((0, 16000), (16000, -1), (16000.5, 16000), (16000, '8000'), ([16000], 8000), ([16000, 8000, 8000], 8000),
                      (torch.tensor([16000.0, 8000.0]), 8000), (True, 8000), (2 ** 31, 8000)):
        with pytest.raises(ValueError):
            ops.resample(x, lens, orig, new)
    with pytest.raises(ValueError, match='int32'):
        ops.resample(torch.zeros(1, 2 ** 20), lens[:1], 1, 4096)
    with pytest.raises(ValueError, match='shorter'):
        ops.resample(x, lens, 8000, 16000, width=150)
    with pytest.raises(AssertionError, match='reached the device'):   # the fixture does refuse device work
        torch.cuda.current_stream()


def test_extractor_refusals_come_before_any_device_work(no_device):
    from opentransformer_b200.features import FbankExtractor
    fe = FbankExtractor(device='cpu', speed_perturb=True)
    one_hz = FbankExtractor(sample_rate=1, frame_length_ms=2000.0, frame_shift_ms=1000.0, device='cpu', speed_perturb=True)
    w, lens = torch.zeros(3, 400), torch.full((3,), 400, dtype=torch.int32)
    no_device()
    bad = [dict(sample_rate=0), dict(sample_rate=[16000, 8000]), dict(sample_rate=[16000, 8000, 22050.5]),
           dict(sample_rate=-8000), dict(speeds=[1.0, 0.9]), dict(speeds=[1.0, 0.0, 1.1]), dict(speeds=[1.0, -0.9, 1.1]),
           dict(speeds=[1.0, float('nan'), 1.1]), dict(speeds=[1.0, 1e-5, 1.1]), dict(sample_rate=1, speeds=[1.0, 1.0, 2 ** 20]),
           dict(sample_rate=2 ** 31 - 1, speeds=[1.0, 1.0, 2 ** 18]), dict(speeds=[1.0, 'fast', 1.1])]
    for kw in bad:
        with pytest.raises(ValueError):
            fe(w, lens, **kw)
    with pytest.raises(ValueError, match='target rates'):      # int(1 * 0.9) = 0
        one_hz(w, lens)
    with pytest.raises(ValueError, match='int32'):
        fe(torch.zeros(1, 2 ** 20), lens[:1], sample_rate=1)
    with pytest.raises(AssertionError, match='reached the device'):
        fe(w, lens)


def test_from_config_leaves_speed_perturb_off():
    from opentransformer_b200.features import FbankExtractor
    data = {'num_mel_bins': 80, 'normalization': True, 'speed_perturb': True}
    for is_eval in (False, True):
        fe = FbankExtractor.from_config(data, sample_rate=16000, is_eval=is_eval, device='cpu')
        assert not fe.speed_perturb
    assert FbankExtractor(device='cpu').speed_rates == [14400, 16000, 17600]
    assert FbankExtractor(sample_rate=22050, device='cpu').speed_rates == [19845, 22050, 24255]
