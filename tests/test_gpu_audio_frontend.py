"""The device audio front end at any sample rate and with the reference's training augmentations, against
torchaudio.compliance.kaldi.fbank (data/audio.py:117-120) and the reference's volume_perturb / normalization /
gaussian_noise / spec_augment order (audio.py:112-136)."""
import math
import random

import numpy as np
import pytest
import torch

ta = pytest.importorskip('torchaudio')
kaldi = ta.compliance.kaldi

pytestmark = pytest.mark.gpu

RATES = (8000, 16000, 22050, 32000, 44100, 48000)


def _waves(sr, seed=5):
    """Ragged tones + noise + DC at rate sr; the third is one sample shorter than a 25 ms frame."""
    g = torch.Generator().manual_seed(seed)
    frame = int(sr * 25.0 * 0.001)
    out = []
    for n, f0 in ((sr, 220.0), (int(1.47 * sr), 997.0), (frame - 1, 50.0), (int(0.51 * sr) + 3, 0.21 * sr)):
        t = torch.arange(n) / float(sr)
        w = (0.3 * torch.sin(2 * math.pi * f0 * t) + 0.1 * torch.sin(2 * math.pi * 1.7 * f0 * t + 1.0)
             + 0.02 * torch.randn(n, generator=g) + 0.05)
        out.append(w)
    return out


def _check_padding(feats, lens, mask):
    for b in range(feats.shape[0]):
        n = int(lens[b])
        assert int(mask[b].sum()) == n and bool(mask[b, :n].all())
        if n < feats.shape[1]:
            assert float(feats[b, n:].abs().max()) == 0.0


@pytest.mark.parametrize('sr', RATES)
def test_fbank_matches_kaldi_at_every_rate(sr):
    from opentransformer_b200.features import FbankExtractor
    waves = _waves(sr)
    fe = FbankExtractor(num_mel_bins=80, sample_rate=sr, normalization=False)
    feats, lens, mask = fe(waves)
    _check_padding(feats, lens, mask)
    assert int(lens[2]) == 0
    for b, w in enumerate(waves):
        n = int(lens[b])
        if n == 0:
            continue
        ref = kaldi.fbank(w.unsqueeze(0), num_mel_bins=80, sample_frequency=float(sr), dither=0.0)
        assert ref.shape == (n, 80)
        got = feats[b, :n].cpu()
        print(f'{sr} Hz utt {b}: {n} frames, max |diff| {float((got - ref).abs().max()):.2e}')
        torch.testing.assert_close(got, ref, rtol=1e-3, atol=2e-3)


@pytest.mark.parametrize('sr', (8000, 16000, 48000))
def test_explicit_gains_scale_the_waveform_before_fbank(sr):
    from opentransformer_b200.features import FbankExtractor
    waves = _waves(sr)
    waves[1][sr // 4: sr // 4 + sr // 5] = 0.0          # a run of exact zeros: whole frames at the eps floor
    gains = [0.83, 1.2, 1.0, 10 ** (-1.6 / 20)]
    feats, lens, mask = FbankExtractor(num_mel_bins=80, sample_rate=sr, normalization=False)(waves, gains=gains)
    _check_padding(feats, lens, mask)
    for b, w in enumerate(waves):
        n = int(lens[b])
        if n == 0:
            continue
        ref = kaldi.fbank((w * gains[b]).unsqueeze(0), num_mel_bins=80, sample_frequency=float(sr), dither=0.0)
        torch.testing.assert_close(feats[b, :n].cpu(), ref, rtol=1e-3, atol=2e-3)
    f = feats[1, :int(lens[1])]
    top, bottom = f.max(dim=1).values, f.min(dim=1).values
    silent = (top == bottom) & (top < -15.0)            # log(eps) in every bin: the frames of exact zeros sit on the floor
    assert int(silent.sum()) >= 10


@pytest.mark.parametrize('normalization', [True, False])
def test_explicit_noise_is_added_after_cmvn(normalization):
    from opentransformer_b200.features import FbankExtractor
    waves = _waves(16000)
    fe = FbankExtractor(num_mel_bins=80, normalization=normalization)
    x, lens, mask = fe(waves)
    noise = torch.randn(len(waves), 80, generator=torch.Generator().manual_seed(3))
    y, lens2, mask2 = fe(waves, noise=noise)
    assert torch.equal(lens, lens2) and torch.equal(mask, mask2)
    _check_padding(y, lens, mask)
    exp = (x + noise.to(x.device)[:, None, :]) * mask[:, :, None]
    torch.testing.assert_close(y, exp, rtol=0, atol=0)
    gm, gs = torch.linspace(-1, 1, 80), torch.linspace(0.5, 2.0, 80)
    if normalization:                                   # global CMVN takes the noise in the same store
        fg = FbankExtractor(num_mel_bins=80, global_mean=gm, global_std=gs)
        xg, _, _ = fg(waves)
        yg, _, _ = fg(waves, noise=noise)
        torch.testing.assert_close(yg, (xg + noise.to(x.device)[:, None, :]) * mask[:, :, None], rtol=0, atol=0)


def test_drawn_gains_are_the_reference_distribution():
    from opentransformer_b200.features import FbankExtractor
    B, sr = 4096, 16000
    g = torch.Generator().manual_seed(11)
    w = 0.3 * torch.sin(2 * math.pi * 440.0 * torch.arange(800) / sr) + 0.05 * torch.randn(B, 800, generator=g)
    lens = torch.full((B,), 800, dtype=torch.int32)
    plain = FbankExtractor(normalization=False)
    base, n, _ = plain(w, lens)
    fe = FbankExtractor(normalization=False, volume_perturb=True, generator=torch.Generator('cuda').manual_seed(1))
    pert, _, _ = fe(w, lens)
    # power scales by g^2, so every log-mel energy of an utterance moves by the same 2 ln g, except where the max(e, eps)
    # floor holds one of the two (after pre-emphasis a low mel bin of a noise frame falls there now and then) or fp32
    # rounding of the spectrum is large against a tiny energy
    T = int(n[0])
    base, pert = base[:, :T].flatten(1), pert[:, :T].flatten(1)
    d = pert - base
    ok = (base > -10.0) & (pert > -10.0)
    assert float(ok.float().mean()) > 0.99
    two_ln_g = d.masked_fill(~ok, float('nan')).nanmedian(dim=1).values
    assert float(((d - two_ln_g[:, None]).abs() * ok).max()) < 1e-3
    gains = torch.exp(two_ln_g / 2).cpu()
    lo, hi = 10 ** -0.08, 10 ** 0.08
    assert float(gains.min()) >= lo - 1e-4 and float(gains.max()) <= hi + 1e-4
    db = 20 * torch.log10(gains)
    assert float(db.min()) < -1.5 and float(db.max()) > 1.5 and abs(float(db.mean())) < 0.1   # U(-1.6, 1.6) dB


def test_drawn_noise_is_one_vector_per_utterance_of_std_sigma():
    from opentransformer_b200.features import FbankExtractor
    B, sr, sigma = 4096, 16000, 0.25
    g = torch.Generator().manual_seed(12)
    w = 0.2 * torch.randn(B, 1200, generator=g)
    lens = torch.full((B,), 1200, dtype=torch.int32)
    ev, n, mask = FbankExtractor()(w, lens)
    fe = FbankExtractor(gaussian_noise=sigma, generator=torch.Generator('cuda').manual_seed(2))
    tr, _, _ = fe(w, lens)
    T = int(n[0])
    assert T >= 5
    d = tr - ev
    vec = d[:, 0, :]
    assert float((d[:, :T] - vec[:, None, :]).abs().max()) < 1e-5      # the same F-vector on every valid frame
    std = float(vec.std())
    print(f'noise std over {B} utterances: {std:.4f} (sigma {sigma})')
    assert abs(std - sigma) < 0.05 * sigma and abs(float(vec.mean())) < 0.05 * sigma


def test_seeded_generator_repeats_and_draws_advance():
    from opentransformer_b200.features import FbankExtractor
    waves = _waves(22050)

    def run(seed):
        fe = FbankExtractor(sample_rate=22050, volume_perturb=True, gaussian_noise=0.1,
                            generator=torch.Generator('cuda').manual_seed(seed))
        return fe(waves)[0], fe(waves)[0]
    a1, a2 = run(4)
    b1, b2 = run(4)
    assert torch.equal(a1, b1) and torch.equal(a2, b2)
    assert not torch.equal(a1, a2)


def test_spec_augment_runs_last_with_the_host_rng():
    from opentransformer_b200 import augment
    from opentransformer_b200.features import FbankExtractor
    waves = _waves(16000)
    cfg = {'freq_mask_num': 2, 'time_mask_num': 2, 'freq_mask_rate': 0.3, 'time_mask_rate': 0.05}
    noise = torch.randn(len(waves), 80, generator=torch.Generator().manual_seed(9))
    x, lens, mask = FbankExtractor()(waves, noise=noise)
    np.random.seed(21)
    random.seed(21)
    y, _, _ = FbankExtractor(spec_augment=True, spec_augment_config=cfg)(waves, noise=noise)
    np.random.seed(21)
    random.seed(21)
    exp = x.clone()
    for b in range(len(waves)):
        bands = augment.draw_bands(int(lens[b]), 80, **cfg)
        for j in range(2):
            exp[b, :, bands[2 * j]:bands[2 * j] + bands[2 * j + 1]] = 0.0
            exp[b, bands[4 + 2 * j]:bands[4 + 2 * j] + bands[5 + 2 * j], :] = 0.0
    assert torch.equal(y, exp) and not torch.equal(y, x)


def test_from_config_in_eval_equals_a_plain_extractor():
    from opentransformer_b200.features import FbankExtractor
    data = {'num_mel_bins': 80, 'normalization': True, 'spec_augment': True, 'volume_perturb': True, 'gaussian_noise': 0.1,
            'speed_perturb': True, 'spec_augment_config': {'freq_mask_num': 2, 'time_mask_num': 2}}
    for sr in (8000, 44100):
        waves = _waves(sr)
        got = FbankExtractor.from_config(data, sample_rate=sr, is_eval=True)(waves)
        ref = FbankExtractor(num_mel_bins=80, sample_rate=sr)(waves)
        for a, b in zip(got, ref):
            assert torch.equal(a, b)
