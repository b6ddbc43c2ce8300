// Counter-based random numbers of the training options (MixSpeech's mixing weight, gradient noise): pure functions of a
// seed and counters read from device memory, so that a captured CUDA graph draws fresh values on every replay, nothing is
// stored, and a run resumed from a checkpoint continues the same sequence.  tests/train_options_ref.py restates them.
#pragma once
#include <stdint.h>

namespace otb {

// lowbias32: a bijective 32-bit integer mixer (xor-shift / multiply rounds)
__host__ __device__ __forceinline__ uint32_t mix32(uint32_t x) {
    x ^= x >> 16;
    x *= 0x7FEB352Du;
    x ^= x >> 15;
    x *= 0x846CA68Bu;
    x ^= x >> 16;
    return x;
}

// the key of one draw: (seed, counter) -> 32 bits
__host__ __device__ __forceinline__ uint32_t rng_key(uint32_t seed, uint32_t counter) { return mix32(mix32(seed) ^ counter); }

// the top 23 bits of h as a uniform in (0, 1): (k + 0.5) / 2^23, never 0 or 1.  23 bits, not 24: k + 0.5 must fit the
// 24-bit fp32 significand for the value to be exact
__host__ __device__ __forceinline__ float rng_u01(uint32_t h) { return ((float)(h >> 9) + 0.5f) * 1.1920928955078125e-7f; }

// MixSpeech's lambda ~ Beta(1/2, 1/2) (the arcsine law): lambda = sin^2(pi u / 2) with u uniform, evaluated in fp64 and
// rounded once
__device__ __forceinline__ float mix_lambda(uint32_t seed, uint32_t step) {
    const double s = sinpi(0.5 * (double)rng_u01(rng_key(seed, step)));
    return (float)(s * s);
}

// a standard normal for element i under `key` (Box-Muller on the uniforms of the counters 2i and 2i + 1), fp32 with the
// accurate logf / cospif
__device__ __forceinline__ float normal_at(uint32_t key, size_t i) {
    const uint64_t c = 2ull * (uint64_t)i;
    const uint32_t k = mix32(key ^ (uint32_t)(c >> 32));
    const float u1 = rng_u01(mix32(k ^ (uint32_t)c)), u2 = rng_u01(mix32(k ^ (uint32_t)(c + 1)));
    return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}

}  // namespace otb
