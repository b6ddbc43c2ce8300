"""The device resampler (ops.resample, csrc/resample.cu) against the float64 restatement of torchaudio's resample, and
FbankExtractor's speed perturbation and mixed input rates against torchaudio's resample followed by kaldi.fbank
(otrans/data/audio.py:63-67,106-110: resample_waveform(w, sr, int(sr * ratio)), then fbank at sr)."""
import math
import random

import numpy as np
import pytest
import torch

from tests import resample_ref as rr

ta = pytest.importorskip('torchaudio')
kaldi = ta.compliance.kaldi
F = ta.functional

pytestmark = pytest.mark.gpu

RATES = (8000, 16000, 22050, 32000, 44100, 48000)


def _tone(n, sr, seed):
    """Audio of peak about 1: two tones, noise and a DC offset."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n, dtype=torch.float64) / sr
    f0 = 97.0 + 31.0 * seed
    w = 0.5 * torch.sin(2 * math.pi * f0 * t) + 0.3 * torch.sin(2 * math.pi * 0.37 * sr * t + 1.0)
    return (w + 0.1 * torch.randn(n, generator=g, dtype=torch.float64) + 0.05).float()


def _run(rows):
    """rows: (length, orig, new), resampled in one launch from a NaN-padded batch; checks every row -> the largest error."""
    from opentransformer_b200 import ops
    B, N = len(rows), max(r[0] for r in rows) + 37
    x = torch.full((B, N), float('nan'))
    waves = []
    for b, (L, o, n) in enumerate(rows):
        waves.append(_tone(L, o, b))
        x[b, :L] = waves[-1]
    lens = torch.tensor([r[0] for r in rows], dtype=torch.int32)
    out, out_len = ops.resample(x.cuda(), lens.cuda(), [r[1] for r in rows], [r[2] for r in rows])
    out, out_len = out.cpu(), out_len.cpu()
    assert out.shape == (B, ops.resample_width(N, [r[1] for r in rows], [r[2] for r in rows]))
    worst = 0.0
    for b, (L, o, n) in enumerate(rows):
        m = int(out_len[b])
        assert m == rr.out_length(L, o, n) == math.ceil(n * L / o)
        assert float(out[b, m:].abs().max()) == 0.0 if m < out.shape[1] else True      # the tail is zero, never NaN
        if o == n:
            assert torch.equal(out[b, :m], waves[b])                                    # bit for bit
            continue
        if m == 0:
            continue
        ref = rr.resample(waves[b].double().numpy(), o, n)
        err = float(np.abs(out[b, :m].double().numpy() - ref).max())
        print(f'{o} -> {n}, {L} samples: max |err| {err:.2e}')
        assert err < 2e-5, (o, n, L, err)
        worst = max(worst, err)
    return worst


def test_ragged_mixed_pairs_in_one_launch():
    rows = [(16000 * 3 + 7, 16000, 14400), (16000 * 2, 16000, 17600), (8000 + 3, 8000, 16000), (44100 * 2 - 5, 44100, 16000),
            (22050 + 11, 22050, 16000), (1, 16000, 17600), (2, 44100, 16000), (25, 16000, 8000), (441, 44100, 16000),
            (32000 + 1, 32000, 16000), (48000, 48000, 16000), (16000 + 5, 16000, 16000), (0, 16000, 17600),
            (12345, 11025, 16000), (5000, 16000, 44100), (20000, 44100, 16001)]
    _run(rows)


def test_long_rows_keep_the_phase():
    # 60 s rows: i / o near 10^6, where a float32 i / o - j / n would lose the phase
    _run([(48000 * 60, 48000, 16000), (16000 * 60, 16000, 17600), (16000 * 60 - 3, 16000, 14400)])


def test_output_width_and_tails():
    from opentransformer_b200 import ops
    x = torch.randn(3, 1000, device='cuda')
    lens = torch.tensor([1000, 10, 500], dtype=torch.int32, device='cuda')
    out, out_len = ops.resample(x, lens, [16000, 16000, 8000], [17600, 17600, 16000])
    assert out.shape == (3, 2000)                       # ceil(2 * 1000): the 8 -> 16 kHz row bounds the width
    assert out_len.cpu().tolist() == [1100, 11, 1000]
    for b, m in enumerate(out_len.cpu().tolist()):
        assert float(out[b, m:].abs().max()) == 0.0
    wide, wl = ops.resample(x, lens, [16000, 16000, 8000], [17600, 17600, 16000], width=2100)
    assert torch.equal(wide[:, :2000], out) and float(wide[:, 2000:].abs().max()) == 0.0 and torch.equal(wl, out_len)


def _fbank_ref(w, sr_in, sr, speed=1.0):
    y = F.resample(w.unsqueeze(0), sr_in, int(sr * speed))
    return kaldi.fbank(y, num_mel_bins=80, sample_frequency=float(sr), dither=0.0)


def _waves(sr):
    return [_tone(int(1.3 * sr), sr, 1), _tone(int(0.7 * sr) + 13, sr, 2), _tone(int(2.1 * sr) - 1, sr, 3)]


@pytest.mark.parametrize('sr', RATES)
def test_explicit_speeds_match_torchaudio_then_kaldi(sr):
    from opentransformer_b200.features import FbankExtractor
    waves = _waves(sr)
    speeds = [0.9, 1.0, 1.1]
    feats, lens, mask = FbankExtractor(num_mel_bins=80, sample_rate=sr, normalization=False)(waves, speeds=speeds)
    for b, w in enumerate(waves):
        ref = _fbank_ref(w, sr, sr, speeds[b])
        n = int(lens[b])
        assert n == ref.shape[0] and int(mask[b].sum()) == n
        got = feats[b, :n].cpu()
        print(f'{sr} Hz speed {speeds[b]}: {n} frames, max |diff| {float((got - ref).abs().max()):.2e}')
        torch.testing.assert_close(got, ref, rtol=1e-3, atol=2e-3)
        assert float(feats[b, n:].abs().max()) == 0.0 if n < feats.shape[1] else True


def test_speeds_of_one_change_nothing():
    from opentransformer_b200.features import FbankExtractor
    for sr in (16000, 44100):
        waves = _waves(sr)
        fe = FbankExtractor(sample_rate=sr)
        for a, b in zip(fe(waves), fe(waves, speeds=[1.0] * len(waves), sample_rate=sr)):
            assert torch.equal(a, b)


def test_mixed_input_rates_into_one_extractor():
    from opentransformer_b200.features import FbankExtractor
    rates = [8000, 22050, 44100, 48000, 16000]
    waves = [_tone(int(s * (0.8 + 0.3 * i)), s, i) for i, s in enumerate(rates)]
    for speeds in (None, [1.1, 0.9, 1.0, 1.1, 0.9]):
        feats, lens, _ = FbankExtractor(num_mel_bins=80, normalization=False)(waves, sample_rate=rates, speeds=speeds)
        for b, w in enumerate(waves):
            ref = _fbank_ref(w, rates[b], 16000, 1.0 if speeds is None else speeds[b])
            n = int(lens[b])
            assert n == ref.shape[0]
            torch.testing.assert_close(feats[b, :n].cpu(), ref, rtol=1e-3, atol=2e-3)


def test_drawn_speeds_are_the_documented_draw():
    from opentransformer_b200.features import SPEEDS, FbankExtractor
    waves = _waves(16000) * 3
    B = len(waves)
    fe = FbankExtractor(speed_perturb=True, generator=torch.Generator('cuda').manual_seed(7))
    got = fe(waves)
    pick = torch.randint(3, (B,), generator=torch.Generator('cuda').manual_seed(7), device='cuda').tolist()
    assert len(set(pick)) > 1
    ref = FbankExtractor()(waves, speeds=[SPEEDS[k] for k in pick])
    for a, b in zip(got, ref):
        assert torch.equal(a, b)
    again = fe(waves)                                    # the generator advances
    assert not all(torch.equal(a, b) for a, b in zip(got, again))


def test_drawn_speeds_spread_over_the_three_ratios():
    from opentransformer_b200.features import FbankExtractor
    B, n = 3000, 2000
    w = torch.randn(B, n, generator=torch.Generator().manual_seed(1)) * 0.1
    lens = torch.full((B,), n, dtype=torch.int32)
    fe = FbankExtractor(speed_perturb=True, generator=torch.Generator('cuda').manual_seed(3))
    _, frames, _ = fe(w, lens)
    # 2000 samples become 1800 / 2000 / 2200: 9 / 11 / 12 frames of 400 with shift 160
    share = [float((frames == t).float().mean()) for t in (9, 11, 12)]
    print('speed shares 0.9 / 1.0 / 1.1:', share)
    assert abs(sum(share) - 1.0) < 1e-6 and all(0.25 <= s <= 0.42 for s in share)


def test_every_augmentation_equals_the_explicit_path():
    from opentransformer_b200.features import SPEEDS, FbankExtractor
    cfg = {'freq_mask_num': 2, 'time_mask_num': 2, 'freq_mask_rate': 0.3, 'time_mask_rate': 0.05}
    waves = _waves(22050)
    B = len(waves)
    fe = FbankExtractor(sample_rate=22050, speed_perturb=True, volume_perturb=True, gaussian_noise=0.1, spec_augment=True,
                        spec_augment_config=cfg, generator=torch.Generator('cuda').manual_seed(5))
    np.random.seed(8)
    random.seed(8)
    got = fe(waves)
    g = torch.Generator('cuda').manual_seed(5)
    pick = torch.randint(3, (B,), generator=g, device='cuda').tolist()
    db = torch.empty(B, dtype=torch.float32, device='cuda').uniform_(-1.6, 1.6, generator=g)
    noise = torch.empty(B, 80, dtype=torch.float32, device='cuda').normal_(0.0, 0.1, generator=g)
    np.random.seed(8)
    random.seed(8)
    ref = FbankExtractor(sample_rate=22050, spec_augment=True, spec_augment_config=cfg)(
        waves, speeds=[SPEEDS[k] for k in pick], gains=torch.pow(10.0, db / 20.0), noise=noise)
    for a, b in zip(got, ref):
        assert torch.equal(a, b)
