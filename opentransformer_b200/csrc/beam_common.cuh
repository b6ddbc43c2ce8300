// Device helpers shared by the beam-search kernels (beam.cu) and the persistent decode kernel
// (decode_group.cu): comparison rule (ties -> LOWER index, torch.topk's tie order is implementation-defined),
// the warp arg-max step built on it, per-lane sorted candidate lists and a warp-wide top-k.  Both decode paths
// select through `better` / `warp_best`, which is what keeps their ids bit-exact with each other.
#pragma once
#include <math.h>

#include "ptx.cuh"

namespace otb {

static constexpr int KMAX = 16;
static constexpr long long EOS_ID = 1;  // otrans/data/__init__.py:9-10 (BOS == EOS == 1)

__device__ __forceinline__ bool better(float va, int ia, float vb, int ib) {
    return (va > vb) || (va == vb && ia < ib);
}

// Warp-wide arg-max of (bv, bi) under `better`: every lane ends with the winner.
__device__ __forceinline__ void warp_best(float& bv, int& bi) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
}

// Per-lane sorted (descending) list of the K best (value, index) pairs, statically indexed.
struct TopList {
    float v[KMAX];
    int i[KMAX];
    __device__ __forceinline__ void init() {
#pragma unroll
        for (int j = 0; j < KMAX; ++j) { v[j] = -INFINITY; i[j] = 0x7fffffff; }
    }
    __device__ __forceinline__ void push(float val, int idx) {
        if (!better(val, idx, v[KMAX - 1], i[KMAX - 1])) return;
        v[KMAX - 1] = val;
        i[KMAX - 1] = idx;
#pragma unroll
        for (int j = KMAX - 1; j > 0; --j) {
            if (better(v[j], i[j], v[j - 1], i[j - 1])) {
                const float tv = v[j]; v[j] = v[j - 1]; v[j - 1] = tv;
                const int ti = i[j]; i[j] = i[j - 1]; i[j - 1] = ti;
            }
        }
    }
    __device__ __forceinline__ void pop() {
#pragma unroll
        for (int j = 0; j < KMAX - 1; ++j) { v[j] = v[j + 1]; i[j] = i[j + 1]; }
        v[KMAX - 1] = -INFINITY;
        i[KMAX - 1] = 0x7fffffff;
    }
};

// Warp-wide top-k over `n` values produced by `get(idx)`; results (sorted, descending, ties -> lower
// index) written by lane 0 to out_v/out_i[0..k).
template <typename F>
__device__ __forceinline__ void warp_topk(F get, int n, int k, float* out_v, int* out_i) {
    const int lane = threadIdx.x & 31;
    TopList tl;
    tl.init();
    for (int idx = lane; idx < n; idx += 128) {   // 4 independent loads in flight, then the branchy insertions
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = (idx + 32 * j < n) ? get(idx + 32 * j) : -INFINITY;
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (idx + 32 * j < n) tl.push(v[j], idx + 32 * j);
    }
    for (int r = 0; r < k; ++r) {
        float bv = tl.v[0];
        int bi = tl.i[0];
        warp_best(bv, bi);
        if (tl.i[0] == bi && tl.v[0] == bv) tl.pop();  // indices are unique -> exactly one lane pops
        if (lane == 0) { out_v[r] = bv; out_i[r] = bi; }
    }
}

}  // namespace otb
