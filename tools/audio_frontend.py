"""The device audio front end (features.FbankExtractor) at 32 utterances x 10 s, at 8, 16, 22.05, 44.1 and 48 kHz:

  - the extractor end to end on device-resident padded waveforms (fbank + utterance CMVN), without and with the training
    augmentations (volume_perturb, gaussian_noise 0.1, SpecAugment with the shipped config);
  - otb_fbank alone, with the bytes it must move (the waveforms read once, the features written once) over its time
    against the H100 SXM data sheet's 3.35 TB/s;
  - torchaudio.compliance.kaldi.fbank on the host's cores for the same batch, one utterance after another as the
    reference's AudioDataset does, with torch's intra-op threads.

CUDA events after warm-up; each figure is the median of --reps repetitions of the mean over --iters calls.  The card, its
power limit and its maximum SM clock are read in the same run.

    python tools/audio_frontend.py [--iters 20] [--reps 5] [--host-reps 1]
    python tools/audio_frontend.py --dump DIR

--dump writes the 16 kHz features (raw log-mel and utterance-normalised) of a fixed-seed batch to DIR/fbank_16k.bin and
prints its SHA-1; it uses only FbankExtractor(num_mel_bins, sample_rate, normalization), so two builds of the project can
be compared byte for byte.
"""
import argparse
import hashlib
import math
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from opentransformer_b200 import _lib, ops  # noqa: E402
from opentransformer_b200.features import FbankExtractor  # noqa: E402

B, SECONDS, F = 32, 10.0, 80
RATES = (8000, 16000, 22050, 44100, 48000)
HBM_BYTES_PER_S = 3.35e12
SPEC_AUGMENT = {'freq_mask_num': 2, 'time_mask_num': 2, 'freq_mask_rate': 0.3, 'time_mask_rate': 0.05}


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else 'unknown'


def batch(sr, seed=0, seconds=SECONDS, n=B):
    """n utterances of tones + noise at rate sr, from 0.55 to 1.0 times `seconds` long -> (padded f32 [n, N], lengths)."""
    g = torch.Generator().manual_seed(seed)
    N = int(seconds * sr)
    lens = [N - (N * 9 * i) // (20 * n) for i in range(n)]
    t = torch.arange(N) / float(sr)
    f0 = 100.0 + 900.0 * torch.rand(n, 1, generator=g)
    w = 0.3 * torch.sin(2 * math.pi * f0 * t) + 0.05 * torch.randn(n, N, generator=g)
    for i, m in enumerate(lens):
        w[i, m:] = 0.0
    return w, torch.tensor(lens, dtype=torch.int32)


def timed(fn, iters, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(reps):
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / iters)
    return statistics.median(out), min(out), max(out)


def dump(directory):
    os.makedirs(directory, exist_ok=True)
    w, lens = batch(16000, seed=1234, seconds=4.0, n=8)
    waves = [w[i, :int(lens[i])] for i in range(len(lens))]
    parts = []
    for norm in (False, True):
        feats, flen, _ = FbankExtractor(num_mel_bins=F, sample_rate=16000, normalization=norm)(waves)
        torch.cuda.synchronize()
        parts += [feats.cpu().contiguous().numpy().tobytes(), flen.cpu().to(torch.int32).numpy().tobytes()]
    blob = b''.join(parts)
    path = os.path.join(directory, 'fbank_16k.bin')
    with open(path, 'wb') as f:
        f.write(blob)
    print(f'{path}: {len(blob)} bytes, sha1 {hashlib.sha1(blob).hexdigest()}')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--host-reps', type=int, default=1)
    ap.add_argument('--dump', metavar='DIR')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/audio_frontend.py measures on the GPU; none is visible')
    if a.dump:
        dump(a.dump)
        return
    import torchaudio
    dev = torch.device('cuda:0')
    print(f'card: {card()}; host: {os.cpu_count()} cores, torch intra-op threads {torch.get_num_threads()}')
    print(f'{B} utterances x {SECONDS:.0f} s (lengths 0.55 .. 1.0 x), {F} mel bins; ms per batch, median [min, max] of {a.reps}')
    print('| rate | frame / FFT | frames | extractor | + augmentation | otb_fbank alone | bytes | HBM share | kaldi.fbank on the host | speed-up |')
    print('|---|---|---|---|---|---|---|---|---|---|')
    for sr in RATES:
        w, lens = batch(sr)
        wd, ld = w.to(dev), lens.to(dev)
        plain = FbankExtractor(num_mel_bins=F, sample_rate=sr, device=dev)
        aug = FbankExtractor(num_mel_bins=F, sample_rate=sr, device=dev, volume_perturb=True, gaussian_noise=0.1,
                             spec_augment=True, spec_augment_config=SPEC_AUGMENT,
                             generator=torch.Generator('cuda').manual_seed(0))
        t_plain = timed(lambda: plain(wd, ld), a.iters, a.reps)
        t_aug = timed(lambda: aug(wd, ld), a.iters, a.reps)
        feats, flen, _ = plain(wd, ld)
        Tmax = feats.shape[1]
        out = torch.empty_like(feats)
        st = ops._stream()

        def kernel():
            _lib.check(_lib.lib().otb_fbank(ops._p(wd), wd.shape[1], ops._p(ld), None, B, ops._p(plain.window),
                                            ops._p(plain.bank), ops._p(plain.range), ops._p(out), Tmax, F, plain.frame_len,
                                            plain.frame_shift, plain.preemph, st), 'otb_fbank')
        t_kernel = timed(kernel, a.iters, a.reps)
        nbytes = 4 * int(lens.sum()) + 4 * B * Tmax * F
        share = nbytes / (t_kernel[0] * 1e-3) / HBM_BYTES_PER_S
        host = []
        for _ in range(a.host_reps):
            t0 = time.perf_counter()
            for i in range(B):
                torchaudio.compliance.kaldi.fbank(w[i:i + 1, :int(lens[i])], num_mel_bins=F, sample_frequency=float(sr),
                                                  dither=0.0)
            host.append((time.perf_counter() - t0) * 1e3)
        t_host = statistics.median(host)
        n_fft = plain.bank.shape[1] * 2
        fmt = lambda t: f'{t[0]:.3f} [{t[1]:.3f}, {t[2]:.3f}]'
        print(f'| {sr / 1000:g} kHz | {plain.frame_len} / {n_fft} | {int(flen.sum())} | {fmt(t_plain)} | {fmt(t_aug)} | '
              f'{fmt(t_kernel)} | {nbytes / 1e6:.1f} MB | {100 * share:.1f} % | {t_host:.1f} | {t_host / t_plain[0]:.0f}x |')


if __name__ == '__main__':
    main()
