"""Resampling on the device (ops.resample, csrc/resample.cu) and speed perturbation in the audio front end, at 32
utterances x 10 s (lengths 0.55 .. 1.0 x):

  - otb_resample alone at 16 -> 17.6 kHz, 16 -> 14.4 kHz and 44.1 -> 16 kHz, with the bytes it must move (the input rows
    read once, the output written once, from the shapes) over its time against the H100 SXM data sheet's 3.35 TB/s;
  - the 16 kHz extractor end to end on device-resident waveforms, without and with speed_perturb;
  - torchaudio.functional.resample on the host's cores for the same batch, one utterance after another as the
    reference's AudioDataset would, with torch's intra-op threads.

CUDA events after warm-up; each figure is the median of --reps repetitions of the mean over --iters calls.  The card, its
power limit and its maximum SM clock are read in the same run.

    python tools/speed_perturb.py [--iters 20] [--reps 5] [--host-reps 1]
"""
import argparse
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from opentransformer_b200 import _lib, ops  # noqa: E402
from opentransformer_b200.features import FbankExtractor  # noqa: E402
from tools.audio_frontend import B, F, HBM_BYTES_PER_S, batch, card, timed  # noqa: E402

PAIRS = ((16000, 17600), (16000, 14400), (44100, 16000))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--host-reps', type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/speed_perturb.py measures on the GPU; none is visible')
    import torchaudio
    dev = torch.device('cuda:0')
    fmt = lambda t: f'{t[0]:.3f} [{t[1]:.3f}, {t[2]:.3f}]'
    print(f'card: {card()}; host: {os.cpu_count()} cores, torch intra-op threads {torch.get_num_threads()}')
    print(f'{B} utterances x 10 s (lengths 0.55 .. 1.0 x); ms per batch, median [min, max] of {a.reps}')
    print('| rate pair | output samples | otb_resample alone | bytes | HBM share | torchaudio resample on the host | speed-up |')
    print('|---|---|---|---|---|---|---|')
    for orig, new in PAIRS:
        w, lens = batch(orig)
        wd, ld = w.to(dev), lens.to(dev)
        out, out_len = ops.resample(wd, ld, orig, new)
        rates = torch.tensor([[orig] * B, [new] * B], dtype=torch.int32, device=dev)
        width = out.shape[1]
        st = ops._stream()

        def kernel():
            _lib.check(_lib.lib().otb_resample(ops._p(wd), wd.shape[1], ops._p(ld), ops._p(rates[0]), ops._p(rates[1]),
                                               ops._p(out), width, ops._p(out_len), B, width, st), 'otb_resample')
        t_kernel = timed(kernel, a.iters, a.reps)
        n_out = int(out_len.sum())
        nbytes = 4 * int(lens.sum()) + 4 * B * width
        share = nbytes / (t_kernel[0] * 1e-3) / HBM_BYTES_PER_S
        host = []
        for _ in range(a.host_reps):
            t0 = time.perf_counter()
            for i in range(B):
                torchaudio.functional.resample(w[i:i + 1, :int(lens[i])], orig, new)
            host.append((time.perf_counter() - t0) * 1e3)
        t_host = statistics.median(host)
        print(f'| {orig / 1000:g} -> {new / 1000:g} kHz | {n_out} | {fmt(t_kernel)} | {nbytes / 1e6:.1f} MB | {100 * share:.1f} % | '
              f'{t_host:.1f} | {t_host / t_kernel[0]:.0f}x |')

    w, lens = batch(16000)
    wd, ld = w.to(dev), lens.to(dev)
    plain = FbankExtractor(num_mel_bins=F, device=dev)
    speed = FbankExtractor(num_mel_bins=F, device=dev, speed_perturb=True, generator=torch.Generator('cuda').manual_seed(0))
    t_plain = timed(lambda: plain(wd, ld), a.iters, a.reps)
    t_speed = timed(lambda: speed(wd, ld), a.iters, a.reps)
    print()
    print('| 16 kHz extractor (fbank + utterance CMVN) | ms per batch |')
    print('|---|---|')
    print(f'| plain | {fmt(t_plain)} |')
    print(f'| speed_perturb | {fmt(t_speed)} |')


if __name__ == '__main__':
    main()
