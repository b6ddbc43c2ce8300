"""float64 / numpy restatement of the random numbers of FusedTrainer's training options (csrc/counter_rng.cuh) and of the
MixSpeech mix (csrc/mixspeech.cu), vectorised over seeds, steps and element indices."""
import numpy as np

M32 = np.uint64(0xFFFFFFFF)


def mix32(x):
    """lowbias32 on uint32 values (computed in uint64, masked to 32 bits)."""
    x = np.asarray(x, dtype=np.uint64) & M32
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x7FEB352D)) & M32
    x ^= x >> np.uint64(15)
    x = (x * np.uint64(0x846CA68B)) & M32
    x ^= x >> np.uint64(16)
    return x


def rng_key(seed, counter):
    return mix32(mix32(np.asarray(seed, dtype=np.uint64) & M32) ^ (np.asarray(counter, dtype=np.uint64) & M32))


def u01(h):
    """The top 23 bits as (k + 0.5) / 2^23 (exact in fp32 and in float64)."""
    return ((np.asarray(h, dtype=np.uint64) >> np.uint64(9)).astype(np.float64) + 0.5) * 2.0 ** -23


def mix_lambda(seed, step):
    """MixSpeech's lambda = sin^2(pi u / 2) ~ Beta(1/2, 1/2), float64 (the kernel rounds it once to fp32)."""
    return np.sin(0.5 * np.pi * u01(rng_key(seed, step))) ** 2


def normal(key, idx):
    """The standard normal of element idx under key (Box-Muller on the counters 2 idx and 2 idx + 1), float64."""
    c = 2 * np.asarray(idx, dtype=np.uint64)
    k = mix32(np.uint64(key) ^ (c >> np.uint64(32)))
    u1 = u01(mix32(k ^ (c & M32)))
    u2 = u01(mix32(k ^ ((c + np.uint64(1)) & M32)))
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


def noise_key(seed, t):
    """The key of Adam step t's noise under the noise seed."""
    return int(rng_key(seed, t))


def mix(x, mask, lam):
    """MixSpeech of numpy / torch arrays x [B, T, F] and mask [B, T] for an fp32 lambda: the reference's fp32 expression
    x0 * lam + x1 * (1 - lam), each product rounded, then the sum -> (x_mix, mask_mix) as fp32 / bool numpy arrays."""
    x = np.asarray(x, dtype=np.float32)
    n = x.shape[0] // 2 * 2
    lam = np.float32(lam)
    om = np.float32(np.float32(1.0) - lam)
    x_mix = (x[0:n:2] * lam).astype(np.float32) + (x[1:n:2] * om).astype(np.float32)
    mask = np.asarray(mask, dtype=bool)
    return x_mix.astype(np.float32), mask[0:n:2] | mask[1:n:2]
