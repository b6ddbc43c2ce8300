// Counter-based dropout mask shared by the forward GEMM epilogue, the backward replay and the test export.
// The reference draws nn.Dropout masks from torch's Philox stream (encoder/transformer.py:32-33,54,61;
// decoder/transformer.py:36-38), which no other implementation can reproduce; what has to match is the distribution
// (Bernoulli(1-p), scaled by 1/(1-p)) and that forward and backward of one step see the SAME mask.  keep(seed, site, row,
// col) is a pure function -- a 32-bit mix of the per-step seed (read from device memory, so that a captured CUDA graph
// draws a fresh mask on every replay), the dropout site (layer / sub-layer) and the element index -- so nothing is stored.
#pragma once
#include <stdint.h>

namespace otb {

__host__ __device__ __forceinline__ uint32_t drop_hash(uint32_t seed, uint32_t site, uint32_t row, uint32_t col) {
    uint32_t h = seed * 0x9E3779B1u + site * 0x85EBCA77u + 0x27D4EB2Fu;
    h ^= row * 0xC2B2AE3Du;
    h = (h ^ (h >> 16)) * 0x7FEB352Du;
    h ^= col * 0x165667B1u;
    h = (h ^ (h >> 15)) * 0x846CA68Bu;
    return h ^ (h >> 16);
}
__host__ __device__ __forceinline__ bool drop_keep(uint32_t seed, uint32_t site, uint32_t row, uint32_t col, uint32_t thresh) {
    return drop_hash(seed, site, row, col) >= thresh;      // P(keep) = 1 - thresh / 2^32
}
inline uint32_t drop_threshold(float p) {
    if (p <= 0.f) return 0u;
    const double t = (double)p * 4294967296.0;
    return t >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)t;
}
// the scale of two independent masks on one tensor (attention-output dropout under the residual dropout), rounded once
inline float drop_scale2(float p, float p2) {
    return (float)(1.0 / ((1.0 - (double)p) * (1.0 - (double)p2)));
}

}  // namespace otb
