"""The audio front end at any sample rate, without a GPU: the mel filterbank and frame geometry against
torchaudio.compliance.kaldi (the reference's fbank, data/audio.py:117-120) at the FFT sizes other than 512, the YAML
`data:` section read the way AudioDataset.__init__ reads it (audio.py:31-73), and the refusals that must come before any
device work."""
import numpy as np
import pytest
import torch

ta = pytest.importorskip('torchaudio')
kaldi = ta.compliance.kaldi

RATES = (8000, 11025, 22050, 44100, 48000)


@pytest.mark.parametrize('n_fft,sr', [(256, 8000), (1024, 22050), (2048, 44100), (2048, 48000)])
def test_mel_banks_equal_kaldi_at_other_fft_sizes(n_fft, sr):
    from opentransformer_b200.features import mel_banks
    for nb in (40, 80):
        ref, _ = kaldi.get_mel_banks(nb, n_fft, float(sr), 20.0, 0.0, 100.0, -500.0, 1.0)
        bank, rng = mel_banks(nb, n_fft, sr)
        assert bank.shape == (nb, n_fft // 2)
        torch.testing.assert_close(bank, ref, rtol=1e-3, atol=1e-5)
        for f in range(nb):
            lo, hi = int(rng[f, 0]), int(rng[f, 1])
            assert hi > lo and float(bank[f, :lo].abs().sum()) == 0.0 and float(bank[f, hi:].abs().sum()) == 0.0


@pytest.mark.parametrize('sr', RATES)
def test_frame_geometry_matches_kaldi(sr):
    from opentransformer_b200.features import FbankExtractor
    fe = FbankExtractor(num_mel_bins=80, sample_rate=sr, device='cpu')
    _, shift, size, padded = kaldi._get_waveform_and_window_properties(torch.zeros(1, sr), -1, float(sr), 10.0, 25.0, True, 0.97)
    assert (fe.frame_len, fe.frame_shift) == (size, shift)
    assert fe.bank.shape == (80, padded // 2) and fe.window.shape == (size,)
    g = torch.Generator().manual_seed(sr)
    for n in (size, size + 1, size + shift - 1, size + shift, sr + 7):
        w = torch.randn(1, n, generator=g)
        assert fe.n_frames(n) == kaldi.fbank(w, num_mel_bins=80, sample_frequency=float(sr), dither=0.0).shape[0]
    assert fe.n_frames(size - 1) == 0


def _data_section(**kw):
    # the data section of egs/aishell/conf/conformer_baseline.yaml with its augmentations switched by kw
    d = {'name': 'aishell', 'vocab': 'egs/aishell/data/vocab', 'batch_size': 16, 'dataset_type': 'online',
         'feature_extractor': 'torchaudio', 'num_mel_bins': 80, 'normalization': True, 'spec_augment': True,
         'speed_perturb': False, 'volume_perturb': False, 'gaussian_noise': 0.0,
         'spec_augment_config': {'freq_mask_num': 2, 'time_mask_num': 2, 'freq_mask_rate': 0.3, 'time_mask_rate': 0.05}}
    d.update(kw)
    return d


def test_from_config_turns_on_what_audio_dataset_would():
    from opentransformer_b200.features import FbankExtractor
    p = _data_section(volume_perturb=True, gaussian_noise=0.1, speed_perturb=True)
    fe = FbankExtractor.from_config(p, sample_rate=8000, device='cpu')
    assert (fe.F, fe.sr, fe.normalization) == (80, 8000, True)
    assert fe.volume_perturb and fe.gaussian_noise == 0.1 and fe.spec_augment
    assert fe.spec_augment_config == p['spec_augment_config']
    assert fe.gmean is None and fe.gstd is None
    ev = FbankExtractor.from_config(p, sample_rate=8000, is_eval=True, device='cpu')
    assert not ev.volume_perturb and ev.gaussian_noise == 0.0 and not ev.spec_augment and ev.normalization
    off = FbankExtractor.from_config(_data_section(spec_augment=False, normalization=False), device='cpu')
    assert not off.volume_perturb and off.gaussian_noise == 0.0 and not off.spec_augment and not off.normalization
    bare = {'num_mel_bins': 40, 'normalization': False}          # optional keys absent: everything off, as in AudioDataset
    fe = FbankExtractor.from_config(bare, device='cpu')
    assert fe.F == 40 and not (fe.volume_perturb or fe.gaussian_noise or fe.spec_augment or fe.normalization)


def test_from_config_loads_global_cmvn(tmp_path):
    from opentransformer_b200.features import FbankExtractor
    mean, std = np.linspace(-2.0, 3.0, 80), np.linspace(0.5, 1.5, 80)
    prefix = str(tmp_path / 'global_cmvn')
    np.save(prefix + '.mean.npy', mean)
    np.save(prefix + '.std.npy', std)
    fe = FbankExtractor.from_config(_data_section(global_cmvn=prefix), device='cpu')
    assert fe.gmean.dtype == torch.float32 and fe.gstd.dtype == torch.float32
    torch.testing.assert_close(fe.gmean, torch.from_numpy(mean).float())
    torch.testing.assert_close(fe.gstd, torch.from_numpy(std).float())
    # AudioDataset reads global_cmvn only when normalization is on
    assert FbankExtractor.from_config(_data_section(global_cmvn=prefix, normalization=False), device='cpu').gmean is None


@pytest.fixture
def no_device(monkeypatch):
    """Every way the extractor reaches the GPU fails loudly."""
    from opentransformer_b200 import _lib

    def refuse(*a, **k):
        raise AssertionError('reached the device')
    for name in ('current_device', 'current_stream', 'init', 'synchronize', 'set_device'):
        monkeypatch.setattr(torch.cuda, name, refuse)
    monkeypatch.setattr(_lib, 'lib', refuse)
    monkeypatch.setattr(torch.Tensor, 'cuda', refuse)


def test_refusals_come_before_any_device_work(no_device):
    from opentransformer_b200.features import FbankExtractor
    with pytest.raises(NotImplementedError, match='2048'):
        FbankExtractor(sample_rate=48000, frame_length_ms=100.0)             # 4800-sample frames
    with pytest.raises(NotImplementedError, match='2048'):
        FbankExtractor.from_config(_data_section(), sample_rate=96000)      # 25 ms at 96 kHz = 2400 samples
    for kind in ('psf', 'python_speech_feature'):
        with pytest.raises(NotImplementedError, match='psf'):
            FbankExtractor.from_config(_data_section(feature_extractor=kind))
    with pytest.raises(ValueError):
        FbankExtractor.from_config(_data_section(feature_extractor='librosa'))
    with pytest.raises(AssertionError, match='reached the device'):          # the fixture does refuse device work
        FbankExtractor(sample_rate=48000)
