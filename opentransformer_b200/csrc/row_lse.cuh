// The log-sum-exp of one fp32 logits row, read once by one warp: otb_token_logprob's row reduction, shared with the
// transducer's lattice log-probs (rnnt.cu).  Each lane folds the float4s lane, lane + 32, ... in that order with an online
// max / sum-exp, and the lanes combine by a fixed xor tree, so the result does not depend on scheduling: two calls are
// bit-identical.  x must be 16-byte aligned.
#pragma once
#include <math.h>

namespace otb {

static constexpr int ROW_LSE_UNROLL = 4;      // float4 loads in flight per lane

// (m, s) <- the online log-sum-exp state after the values whose maximum is mg >= m (-inf-safe)
__device__ __forceinline__ float rescale(float s, float m, float mg) { return m == mg ? s : s * expf(m - mg); }

// -> (m, s) in every lane: m = max_k x[k], s = sum_k exp(x[k] - m) over k < V; logsumexp = m + logf(s)
__device__ __forceinline__ void warp_row_lse(const float* __restrict__ x, int V, int lane, float& m_out, float& s_out) {
    const float4* x4 = reinterpret_cast<const float4*>(x);
    const int nv = V >> 2;
    float m = -INFINITY, s = 0.f;
    for (int i0 = lane; i0 < nv; i0 += 32 * ROW_LSE_UNROLL) {
        float4 v[ROW_LSE_UNROLL];
#pragma unroll
        for (int j = 0; j < ROW_LSE_UNROLL; ++j) {
            const int i = i0 + 32 * j;
            v[j] = i < nv ? __ldcs(x4 + i) : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
        }
        float mg = m;
#pragma unroll
        for (int j = 0; j < ROW_LSE_UNROLL; ++j) mg = fmaxf(mg, fmaxf(fmaxf(v[j].x, v[j].y), fmaxf(v[j].z, v[j].w)));
        if (mg == -INFINITY) continue;
        float acc = rescale(s, m, mg);
#pragma unroll
        for (int j = 0; j < ROW_LSE_UNROLL; ++j)
            acc += expf(v[j].x - mg) + expf(v[j].y - mg) + expf(v[j].z - mg) + expf(v[j].w - mg);
        s = acc;
        m = mg;
    }
    for (int i = 4 * nv + lane; i < V; i += 32) {     // the last V % 4 columns
        const float xv = x[i];
        const float mg = fmaxf(m, xv);
        if (mg == -INFINITY) continue;
        s = rescale(s, m, mg) + expf(xv - mg);
        m = mg;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, m, o);
        const float os = __shfl_xor_sync(0xffffffffu, s, o);
        const float mg = fmaxf(m, om);
        if (mg != -INFINITY) s = rescale(s, m, mg) + rescale(os, om, mg);
        m = mg;
    }
    m_out = m;
    s_out = s;
}

}  // namespace otb
