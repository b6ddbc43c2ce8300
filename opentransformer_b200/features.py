"""Log-mel filterbank features + CMVN on the GPU (SURVEY.md 8f row 3): the step immediately before the hot path.

Mirror of what otrans/data/audio.py:117-133 does on DataLoader worker CPUs per utterance,

    feature = ta.compliance.kaldi.fbank(wavform, num_mel_bins=..., sample_frequency=..., dither=0.0)
    feature = normalization(feature)            # (x - mean) / std over the whole utterance, or global CMVN
    feature = spec_augment(feature)             # opentransformer_b200/augment.py

batched on the device (csrc/fbank.cu): at thousands of utterances per second per GPU the CPU front end is the next wall.
The mel filterbank follows Kaldi's definition as published by torchaudio.compliance.kaldi.get_mel_banks (mel(f) = 1127
ln(1 + f / 700), num_bins + 2 equally spaced mel points between low_freq and Nyquist, triangles over the first N/2 FFT bins).
"""
import math

import torch

from . import _lib, ops
from ._lib import check


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
    """Batched fbank (+ CMVN) on the device.  ``__call__(waves)`` takes a list of 1-D float waveforms (as ta.load returns
    them, any length) or a padded f32 [B, N] tensor with ``lengths`` and returns what collate_fn_with_eos_bos builds
    (data/loader.py:66-108): features f32 [B, Tmax, F] zero padded, feature lengths, bool mask [B, Tmax]."""

    def __init__(self, num_mel_bins=80, sample_rate=16000, frame_length_ms=25.0, frame_shift_ms=10.0, preemphasis=0.97,
                 normalization=True, global_mean=None, global_std=None, device=None):
        self.F, self.sr = num_mel_bins, sample_rate
        self.frame_len = int(sample_rate * frame_length_ms * 0.001)
        self.frame_shift = int(sample_rate * frame_shift_ms * 0.001)
        n_fft = 1 << (self.frame_len - 1).bit_length()               # round_to_power_of_two
        if n_fft != 512:
            raise NotImplementedError('fbank kernel is built for a 512-point FFT (25 ms frames at 16 kHz)')
        self.device = torch.device(device if device is not None else torch.cuda.current_device())
        bank, rng = mel_banks(num_mel_bins, n_fft, sample_rate)
        self.bank, self.range = bank.to(self.device), rng.to(self.device)
        self.window = povey_window(self.frame_len).to(self.device)
        self.preemph = preemphasis
        self.normalization = normalization
        self.gmean = global_mean.float().to(self.device).contiguous() if global_mean is not None else None
        self.gstd = global_std.float().to(self.device).contiguous() if global_std is not None else None

    def n_frames(self, n_samples):
        return 0 if n_samples < self.frame_len else 1 + (n_samples - self.frame_len) // self.frame_shift

    def __call__(self, waves, lengths=None):
        if isinstance(waves, (list, tuple)):
            lens = [int(w.numel()) for w in waves]
            N = max(lens)
            buf = torch.zeros(len(waves), N, dtype=torch.float32)
            for i, w in enumerate(waves):
                buf[i, :lens[i]] = w.reshape(-1).float()
            waves, lengths = buf, torch.tensor(lens, dtype=torch.int32)
        waves = waves.to(self.device, torch.float32).contiguous()
        lengths = lengths.to(self.device, torch.int32).contiguous()
        B, N = waves.shape
        frames = torch.tensor([self.n_frames(int(n)) for n in lengths.cpu().tolist()], dtype=torch.int32)
        Tmax = max(1, int(frames.max()))
        out = torch.empty(B, Tmax, self.F, dtype=torch.float32, device=self.device)
        st = ops._stream()
        check(_lib.lib().otb_fbank(ops._p(waves), N, ops._p(lengths), B, ops._p(self.window), ops._p(self.bank), ops._p(self.range),
                                   ops._p(out), Tmax, self.F, self.frame_len, self.frame_shift, self.preemph, st), 'otb_fbank')
        ops._count()
        frames_d = frames.to(self.device)
        if self.normalization:
            check(_lib.lib().otb_utt_cmvn(ops._p(out), B, Tmax, self.F, ops._p(frames_d), ops._p(self.gmean), ops._p(self.gstd), st),
                  'otb_utt_cmvn')
            ops._count()
        mask = torch.arange(Tmax, device=self.device)[None] < frames_d[:, None]
        return out, frames_d, mask
