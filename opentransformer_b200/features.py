"""Log-mel filterbank features + CMVN on the GPU (SURVEY.md 8f row 3): the step immediately before the hot path.

Mirror of what otrans/data/audio.py:112-136 does on DataLoader worker CPUs per utterance,

    wavform *= 10 ** (random.uniform(-1.6, 1.6) / 20)                      # volume_perturb (training only)
    feature = ta.compliance.kaldi.fbank(wavform, num_mel_bins=..., sample_frequency=..., dither=0.0)
    feature = normalization(feature)            # (x - mean) / std over the whole utterance, or global CMVN
    feature += torch.normal(torch.zeros(F), std=gaussian_noise)           # one vector per utterance (training only)
    feature = spec_augment(feature)             # opentransformer_b200/augment.py (training only)

batched on the device (csrc/fbank.cu): at thousands of utterances per second per GPU the CPU front end is the next wall.
The mel filterbank follows Kaldi's definition as published by torchaudio.compliance.kaldi.get_mel_banks (mel(f) = 1127
ln(1 + f / 700), num_bins + 2 equally spaced mel points between low_freq and Nyquist, triangles over the first N/2 FFT bins).
The FFT has round_to_power_of_two(frame_len) points, at most 2048 (25 ms frames at sample rates up to 81.9 kHz).  The
features are at the extractor's sample rate; input at other rates, given per row, is resampled to it on the device
(csrc/resample.cu) in the same pass as speed perturbation.
"""
import math

import numpy as np
import torch

from . import _lib, augment, ops
from ._lib import check

MAX_FFT = 2048          # csrc/fbank.cu: shared-memory buffers of one frame
SPEEDS = (0.9, 1.0, 1.1)  # speed perturbation ratios, otrans/data/audio.py:106 random.choice([0.9, 1.0, 1.1])


def _mel(f):
    return 1127.0 * math.log(1.0 + f / 700.0)


def mel_banks(num_bins, n_fft, sample_rate, low_freq=20.0, high_freq=0.0):
    """-> (bank f32 [num_bins, n_fft/2], range i32 [num_bins, 2]) triangular weights and their non-zero [lo, hi) bin ranges."""
    nyq = 0.5 * sample_rate
    if high_freq <= 0.0:
        high_freq += nyq
    nb = n_fft // 2
    width = sample_rate / n_fft
    lo, hi = _mel(low_freq), _mel(high_freq)
    delta = (hi - lo) / (num_bins + 1)
    mel = torch.tensor([_mel(width * i) for i in range(nb)], dtype=torch.float32).unsqueeze(0)
    b = torch.arange(num_bins, dtype=torch.float32).unsqueeze(1)
    left, center, right = lo + b * delta, lo + (b + 1.0) * delta, lo + (b + 2.0) * delta
    bank = torch.clamp(torch.minimum((mel - left) / (center - left), (right - mel) / (right - center)), min=0.0)
    rng = torch.zeros(num_bins, 2, dtype=torch.int32)
    for f in range(num_bins):
        nz = torch.nonzero(bank[f] > 0).view(-1)
        if len(nz):
            rng[f, 0], rng[f, 1] = int(nz[0]), int(nz[-1]) + 1
    return bank.contiguous(), rng


def povey_window(n):
    return torch.hann_window(n, periodic=False, dtype=torch.float32).pow(0.85)


class FbankExtractor:
    """Batched fbank (+ CMVN, + the reference's training augmentations) on the device.  ``__call__(waves)`` takes a list of
    1-D float waveforms (as ta.load returns them, any length) or a padded f32 [B, N] tensor with ``lengths`` and returns
    what collate_fn_with_eos_bos builds (data/loader.py:66-108): features f32 [B, Tmax, F] zero padded, feature lengths,
    bool mask [B, Tmax].

    ``speed_perturb`` resamples each waveform from sample_rate to int(sample_rate * ratio), ratio drawn from SPEEDS
    (0.9, 1.0, 1.1), and computes the fbank at sample_rate, as the reference's commented-out speed perturbation does
    (otrans/data/audio.py:63-67,106-110); ``volume_perturb`` scales each waveform by 10 ** (U(-1.6, 1.6) / 20) before the
    fbank, ``gaussian_noise`` = sigma adds one N(0, sigma) vector of F values per utterance to its valid frames after CMVN,
    and ``spec_augment`` masks bands last with ``augment.spec_augment_`` (``spec_augment_config`` are its keyword
    arguments).  The speeds, the gains and the noise are drawn on the device from ``generator`` (a CUDA torch.Generator;
    torch's default one if None), in that order; SpecAugment draws its bands on the host with the reference's RNG calls.
    All four are off by default."""

    def __init__(self, num_mel_bins=80, sample_rate=16000, frame_length_ms=25.0, frame_shift_ms=10.0, preemphasis=0.97,
                 normalization=True, global_mean=None, global_std=None, device=None, volume_perturb=False, gaussian_noise=0.0,
                 spec_augment=False, spec_augment_config=None, generator=None, speed_perturb=False):
        self.F, self.sr = num_mel_bins, sample_rate
        self.frame_len = int(sample_rate * frame_length_ms * 0.001)
        self.frame_shift = int(sample_rate * frame_shift_ms * 0.001)
        if not 2 <= self.frame_len <= MAX_FFT:
            raise NotImplementedError(f'fbank kernel takes frames of 2 .. {MAX_FFT} samples (a FFT of at most {MAX_FFT} points); '
                                      f'{frame_length_ms} ms at {sample_rate} Hz is {self.frame_len}')
        n_fft = 1 << (self.frame_len - 1).bit_length()               # round_to_power_of_two
        self.device = torch.device(device if device is not None else torch.cuda.current_device())
        bank, rng = mel_banks(num_mel_bins, n_fft, sample_rate)
        self.bank, self.range = bank.to(self.device), rng.to(self.device)
        self.window = povey_window(self.frame_len).to(self.device)
        self.preemph = preemphasis
        self.normalization = normalization
        self.gmean = global_mean.float().to(self.device).contiguous() if global_mean is not None else None
        self.gstd = global_std.float().to(self.device).contiguous() if global_std is not None else None
        # with normalization off the CMVN pass only adds the noise: global statistics 0 / 1 store x itself
        self.unit_stats = None if normalization else (torch.zeros(num_mel_bins, device=self.device),
                                                      torch.ones(num_mel_bins, device=self.device))
        self.volume_perturb = bool(volume_perturb)
        self.gaussian_noise = float(gaussian_noise)
        self.spec_augment = bool(spec_augment)
        self.spec_augment_config = dict(spec_augment_config or {})
        self.generator = generator
        self.speed_perturb = bool(speed_perturb)
        # target rates of the three speeds, from float64 on the host as the reference computes them
        self.speed_rates = [int(sample_rate * s) for s in SPEEDS]
        self._speed_rates_d = None

    @classmethod
    def from_config(cls, data_params, sample_rate=16000, is_eval=False, device=None):
        """The extractor AudioDataset(data_params, ..., is_eval) stands for (otrans/data/audio.py:31-73): num_mel_bins,
        normalization with the optional global_cmvn prefix (<prefix>.mean.npy / .std.npy), and in training spec_augment
        (+ spec_augment_config), volume_perturb and gaussian_noise.  speed_perturb is accepted and ignored, as the reference
        has it commented out; to speed-perturb, pass ``speed_perturb=True`` to the constructor.  The reference calls
        spec_augment(feature) with its defaults; the shipped configs set the same values, and here spec_augment_config is
        passed on."""
        p = data_params
        kind = p.get('feature_extractor', 'torchaudio')
        if kind in ('psf', 'python_speech_feature'):
            raise NotImplementedError('feature_extractor psf (python_speech_features.logfbank) is not built; use torchaudio')
        if kind not in ('torchaudio', 'ta'):
            raise ValueError(f'unknown feature_extractor {kind!r}')
        gmean = gstd = None
        if p['normalization'] and 'global_cmvn' in p:
            gmean = torch.from_numpy(np.load(p['global_cmvn'] + '.mean.npy'))
            gstd = torch.from_numpy(np.load(p['global_cmvn'] + '.std.npy'))
        train = not is_eval
        return cls(num_mel_bins=p['num_mel_bins'], sample_rate=sample_rate, normalization=p['normalization'], global_mean=gmean,
                   global_std=gstd, device=device, volume_perturb=train and bool(p.get('volume_perturb', False)),
                   gaussian_noise=float(p.get('gaussian_noise', 0.0)) if train else 0.0,
                   spec_augment=train and bool(p.get('spec_augment', False)),
                   spec_augment_config=p.get('spec_augment_config') if train else None)

    def n_frames(self, n_samples):
        return 0 if n_samples < self.frame_len else 1 + (n_samples - self.frame_len) // self.frame_shift

    def _resample_plan(self, B, N, sample_rate, speeds):
        """Host half of the rate / speed step -> None when no row changes rate, else (input rates [B], target rates [B] or
        None when the speeds are drawn on the device, output width).  Raises ValueError on a bad argument."""
        src = ops.resample_rates(self.sr if sample_rate is None else sample_rate, B, 'sample_rate')
        if speeds is None:
            if not self.speed_perturb:
                if src == [self.sr] * B:
                    return None
                dst = [self.sr] * B
                return self._checked(src, dst, ops.resample_width(N, src, dst))
            if min(self.speed_rates) < 1:
                raise ValueError(f'speed perturbation at {self.sr} Hz gives target rates {self.speed_rates}')
            return self._checked(src, None, ops.resample_width(N, src, [max(self.speed_rates)] * B))
        if isinstance(speeds, torch.Tensor):
            speeds = speeds.tolist()
        speeds = list(speeds)
        if len(speeds) != B:
            raise ValueError(f'speeds must be one ratio per utterance, {B}, got {len(speeds)}')
        dst = []
        for s in speeds:
            try:
                s = float(s)
            except (TypeError, ValueError):
                raise ValueError(f'speed ratios must be numbers, got {s!r}') from None
            if not (s > 0.0 and math.isfinite(s)) or not 1 <= int(self.sr * s) <= ops.INT32_MAX:
                raise ValueError(f'speed ratio {s} at {self.sr} Hz gives no positive int32 target rate')
            dst.append(int(self.sr * s))
        if dst == src:
            return None
        return self._checked(src, dst, ops.resample_width(N, src, dst))

    @staticmethod
    def _checked(src, dst, width):
        if width > ops.INT32_MAX:
            raise ValueError(f'resampling gives {width} samples per utterance, past int32')
        return src, dst, width

    def __call__(self, waves, lengths=None, gains=None, noise=None, sample_rate=None, speeds=None):
        """``gains`` f32 [B] (linear factors) and ``noise`` f32 [B, F] replace what volume_perturb / gaussian_noise would
        draw, for checking exact values; either applies whether or not its option is on.  ``speeds`` (one ratio per
        utterance) likewise replaces the speed_perturb draw.

        ``sample_rate`` is the rate of the input, one int or one per utterance (default: the extractor's).  A row at another
        rate is resampled to the extractor's, or, when it is also speed-perturbed, straight to int(sr * ratio) in the same
        pass.  Order, as the reference's: resample -> volume gain (applied where the fbank loads the samples) -> fbank ->
        CMVN + noise -> SpecAugment."""
        if isinstance(waves, (list, tuple)):
            lens = [int(w.numel()) for w in waves]
            N = max(lens)
            buf = torch.zeros(len(waves), N, dtype=torch.float32)
            for i, w in enumerate(waves):
                buf[i, :lens[i]] = w.reshape(-1).float()
            waves, lengths = buf, torch.tensor(lens, dtype=torch.int32)
        plan = self._resample_plan(waves.shape[0], waves.shape[1], sample_rate, speeds)
        waves = waves.to(self.device, torch.float32).contiguous()
        lengths = lengths.to(self.device, torch.int32).contiguous()
        B, N = waves.shape
        if plan is not None:
            src, dst, width = plan
            if dst is None:                     # drawn on the device, before the gains and the noise
                if self._speed_rates_d is None:
                    self._speed_rates_d = torch.tensor(self.speed_rates, dtype=torch.int32, device=self.device)
                pick = torch.randint(len(SPEEDS), (B,), generator=self.generator, device=self.device)
                dst = self._speed_rates_d[pick]
                src = torch.tensor(src, dtype=torch.int32).to(self.device)
            waves, lengths = ops.resample(waves, lengths, src, dst, width=width)
            B, N = waves.shape
        if gains is None and self.volume_perturb:
            db = torch.empty(B, dtype=torch.float32, device=self.device).uniform_(-1.6, 1.6, generator=self.generator)
            gains = torch.pow(10.0, db / 20.0)
        if noise is None and self.gaussian_noise > 0.0:
            noise = torch.empty(B, self.F, dtype=torch.float32, device=self.device).normal_(0.0, self.gaussian_noise,
                                                                                             generator=self.generator)
        if gains is not None:
            gains = torch.as_tensor(gains, dtype=torch.float32).to(self.device).contiguous()
            if gains.shape != (B,):
                raise ValueError(f'gains must be [B] = [{B}], got {tuple(gains.shape)}')
        if noise is not None:
            noise = torch.as_tensor(noise, dtype=torch.float32).to(self.device).contiguous()
            if noise.shape != (B, self.F):
                raise ValueError(f'noise must be [B, F] = [{B}, {self.F}], got {tuple(noise.shape)}')
        frames = torch.tensor([self.n_frames(int(n)) for n in lengths.cpu().tolist()], dtype=torch.int32)
        Tmax = max(1, int(frames.max()))
        out = torch.empty(B, Tmax, self.F, dtype=torch.float32, device=self.device)
        st = ops._stream()
        check(_lib.lib().otb_fbank(ops._p(waves), N, ops._p(lengths), ops._p(gains), B, ops._p(self.window), ops._p(self.bank),
                                   ops._p(self.range), ops._p(out), Tmax, self.F, self.frame_len, self.frame_shift, self.preemph, st),
              'otb_fbank')
        ops._count()
        frames_d = frames.to(self.device)
        if self.normalization or noise is not None:
            gmean, gstd = (self.gmean, self.gstd) if self.normalization else self.unit_stats
            check(_lib.lib().otb_utt_cmvn(ops._p(out), B, Tmax, self.F, ops._p(frames_d), ops._p(gmean), ops._p(gstd),
                                          ops._p(noise), st), 'otb_utt_cmvn')
            ops._count()
        if self.spec_augment:
            augment.spec_augment_(out, frames.tolist(), **self.spec_augment_config)
        mask = torch.arange(Tmax, device=self.device)[None] < frames_d[:, None]
        return out, frames_d, mask
