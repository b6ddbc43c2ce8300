"""Float64 restatement of band-limited resampling (torchaudio.functional.resample at its defaults: sinc_interp_hann,
lowpass_filter_width 6, rolloff 0.99), written from the formula csrc/resample.cu implements:

    g = gcd(orig, new), o = orig / g, n = new / g, base = 0.99 min(o, n), w = ceil(6 o / base)
    y[j] = sum_{i in [q o - w, q o + w + o)} x[i] h(t),   j = q n + p,   t = base (i n - j o) / (o n) clamped to [-6, 6]
    h(t) = cos^2(pi t / 12) sinc(pi t) base / o

with x[i] = 0 outside [0, L) and ceil(n L / o) outputs.  t is formed from the integer numerator i n - j o."""
import math

import numpy as np

WIDTH, ROLLOFF = 6, 0.99


def reduced(orig, new):
    g = math.gcd(orig, new)
    return orig // g, new // g


def out_length(L, orig, new):
    o, n = reduced(orig, new)
    return -(-n * L // o)


def phase_table(orig, new):
    """-> (h float64 [n, 2w + o], w): h[p, k] weights x[q o - w + k] in output q n + p."""
    o, n = reduced(orig, new)
    base = ROLLOFF * min(o, n)
    w = math.ceil(WIDTH * o / base)
    i_rel = np.arange(-w, w + o, dtype=np.int64)[None, :]
    p = np.arange(n, dtype=np.int64)[:, None]
    num = i_rel * n - p * o                        # i n - j o with i = q o + i_rel, j = q n + p
    t = np.clip(base * num.astype(np.float64) / (o * n), -WIDTH, WIDTH)
    h = np.cos(np.pi * t / (2 * WIDTH)) ** 2 * np.sinc(t) * (base / o)
    return h, w


def resample(x, orig, new):
    """x: 1-D float array -> float64 array of ceil(n L / o) samples."""
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    if orig == new:
        return x.copy()
    o, n = reduced(orig, new)
    h, w = phase_table(orig, new)
    L = x.shape[0]
    frames = L // o + 1
    pad = np.zeros(frames * o + 2 * w + o, dtype=np.float64)
    pad[w:w + L] = x
    cols = np.lib.stride_tricks.as_strided(pad, shape=(frames, 2 * w + o), strides=(o * pad.strides[0], pad.strides[0]))
    y = (cols @ h.T).reshape(-1)                   # [frames, n] -> j = q n + p
    return y[:out_length(L, orig, new)]
