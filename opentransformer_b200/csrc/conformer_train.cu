// Conformer convolution module in training mode (module/conformer.py:36-57 under autograd):
//
//   c   = depthwise_conv(mask(g)) + conv bias          g = GLU output [B*T, d], padded frames read as zero (conformer.py:46)
//   a   = (c - mean) * invstd * gamma + beta           nn.BatchNorm1d in train(): batch statistics over ALL B*T positions,
//                                                      padded frames included; biased variance for the normalisation
//   out = mask(a * sigmoid(a))                         swish; padded frames written as zero (the reference zeroes them after
//                                                      pointwise_conv2, a row-wise Linear, so the two are the same network)
//
// and the running-statistics update of BatchNorm (momentum 0.1, unbiased variance for running_var, num_batches_tracked + 1),
// done on the device so that a captured CUDA graph performs it on every replay.  The backward recomputes a from c and
// the saved (mean, invstd).  Everything is HBM-bound fp32 SIMT: c and dc are kept in fp32, the statistics and every reduction
// are fp32 (per-CTA partial sums in shared memory, one atomic per channel and CTA).
//
// The depthwise weight is nn.Conv1d's own layout, w [d, k] (d, 1, k squeezed); k is odd, padding (k - 1) / 2.
#include <math.h>

#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

namespace {

// Reduction layout: CTA = 32 groups of 8 channels (256 channels) x 8 row lanes; the CTAs along y stride over the rows.
constexpr int RL = 8;

__device__ __forceinline__ void load8(const bf16* p, float (&v)[8]) {
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    const float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y), c = unpack_bf16(u.z), d = unpack_bf16(u.w);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
__device__ __forceinline__ void load8(const float* p, float (&v)[8]) {
    const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void store8(float* p, const float (&v)[8]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void store8(bf16* p, const float (&v)[8]) {
    uint4 u;
    u.x = pack_bf16(v[0], v[1]); u.y = pack_bf16(v[2], v[3]); u.z = pack_bf16(v[4], v[5]); u.w = pack_bf16(v[6], v[7]);
    *reinterpret_cast<uint4*>(p) = u;
}
// Valid frames of an utterance: t < min(len, T).  A length above T means every frame is valid; the conv taps are bounded by
// the clamped length too, so they never read the next utterance's rows (or past the buffer, for the last one).
__device__ __forceinline__ int valid_len(const int* len, int row, int T) { return min(len[row / T], T); }
__device__ __forceinline__ bool row_valid(const int* len, int row, int T) { return row % T < valid_len(len, row, T); }

// Sum the 8 row lanes' partials of this CTA and add them to out[col .. col + 8) (one atomic per channel and CTA).
__device__ __forceinline__ void reduce_add(float (&red)[RL][256], const float (&acc)[8], float* out, int d) {
    const int cg = threadIdx.x & 31, rl = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < 8; ++j) red[rl][cg * 8 + j] = acc[j];
    __syncthreads();
    const int c = blockIdx.x * 256 + threadIdx.x;
    if (c < d) {
        float s = 0.f;
#pragma unroll
        for (int r = 0; r < RL; ++r) s += red[r][threadIdx.x];
        atomicAdd(out + c, s);
    }
}

// ---- forward
// c = depthwise conv of the masked input + bias (fp32), and the per-channel sum of c into stats[0, :]
__global__ void __launch_bounds__(256) dwconv_sum_kernel(const bf16* __restrict__ x, const int* __restrict__ len,
                                                         const float* __restrict__ w, const float* __restrict__ wb,
                                                         float* __restrict__ c, float* __restrict__ stats, int M, int T, int d,
                                                         int k) {
    __shared__ float red[RL][256];
    const int col = blockIdx.x * 256 + (threadIdx.x & 31) * 8, rl = threadIdx.x >> 5, pad = (k - 1) / 2;
    float sum[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (col < d) {
        for (int row = blockIdx.y * RL + rl; row < M; row += gridDim.y * RL) {
            const int t = row % T, n = valid_len(len, row, T);
            float acc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = wb ? wb[col + j] : 0.f;
            for (int tap = 0; tap < k; ++tap) {
                const int tt = t + tap - pad;
                if (tt < 0 || tt >= n) continue;       // zero padding of the conv, and the masked (padded) frames
                float xv[8];
                load8(x + (size_t)(row + tap - pad) * d + col, xv);
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] = fmaf(xv[j], w[(col + j) * k + tap], acc[j]);
            }
            store8(c + (size_t)row * d + col, acc);
#pragma unroll
            for (int j = 0; j < 8; ++j) sum[j] += acc[j];
        }
    }
    reduce_add(red, sum, stats, d);
}

// sum of (c - mean)^2 into stats[1, :] (two passes: no cancellation between E[c^2] and mean^2)
__global__ void __launch_bounds__(256) bn_var_kernel(const float* __restrict__ c, float* __restrict__ stats, int M, int d) {
    __shared__ float red[RL][256];
    const int col = blockIdx.x * 256 + (threadIdx.x & 31) * 8, rl = threadIdx.x >> 5;
    float q[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (col < d) {
        float mean[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) mean[j] = stats[col + j] / (float)M;
        for (int row = blockIdx.y * RL + rl; row < M; row += gridDim.y * RL) {
            float v[8];
            load8(c + (size_t)row * d + col, v);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float e = v[j] - mean[j];
                q[j] = fmaf(e, e, q[j]);
            }
        }
    }
    reduce_add(red, q, stats + d, d);
}

// stats [2, d]: (sum, centred sum of squares) -> (mean, invstd); running_* = (1 - momentum) running_* + momentum * batch
// (running_var with the unbiased variance, nn.BatchNorm1d); num_batches_tracked += 1
__global__ void __launch_bounds__(256) bn_finalize_kernel(float* __restrict__ stats, float* __restrict__ run_mean,
                                                          float* __restrict__ run_var, long long* __restrict__ n_batches, int M,
                                                          int d, float momentum, float eps) {
    for (int ch = threadIdx.x; ch < d; ch += blockDim.x) {
        const float mean = stats[ch] / (float)M, var = stats[d + ch] / (float)M;
        stats[ch] = mean;
        stats[d + ch] = rsqrtf(var + eps);
        if (run_mean) run_mean[ch] = (1.f - momentum) * run_mean[ch] + momentum * mean;
        if (run_var) run_var[ch] = (1.f - momentum) * run_var[ch] + momentum * (M > 1 ? var * (float)M / (float)(M - 1) : var);
    }
    if (threadIdx.x == 0 && n_batches) *n_batches += 1;
}

__device__ __forceinline__ void bn_affine(const float* c, const float* stats, const float* gamma, const float* beta, int col, int d,
                                          float (&a)[8], float (&xh)[8]) {
    load8(c, a);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        xh[j] = (a[j] - stats[col + j]) * stats[d + col + j];
        a[j] = fmaf(xh[j], gamma[col + j], beta[col + j]);
    }
}

// out = mask(swish(BN(c))) -> bf16; thread = (row, 8 channels)
__global__ void __launch_bounds__(256) bn_swish_kernel(const float* __restrict__ c, const float* __restrict__ stats,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       const int* __restrict__ len, bf16* __restrict__ out, int M, int T, int d) {
    const int cg = d / 8;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)M * cg) return;
    const int row = (int)(i / cg), col = (int)(i % cg) * 8;
    float a[8], xh[8];
    bn_affine(c + (size_t)row * d + col, stats, gamma, beta, col, d, a, xh);
    const bool ok = row_valid(len, row, T);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = ok ? a[j] * __fdividef(1.0f, 1.0f + __expf(-a[j])) : 0.f;
    store8(out + (size_t)row * d + col, a);
}

// ---- backward
// da = mask * dy * swish'(a), swish'(a) = s (1 + a (1 - s)), s = sigmoid(a)
__device__ __forceinline__ void swish_bwd(const bf16* dy, bool ok, float (&a)[8], float (&da)[8]) {
    float g[8];
    load8(dy, g);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float s = __fdividef(1.0f, 1.0f + __expf(-a[j]));
        da[j] = ok ? g[j] * s * (1.0f + a[j] * (1.0f - s)) : 0.f;
    }
}

// red [2, d] (zeroed by the launcher) += (sum da, sum da * xhat): dbeta and dgamma of this pass
__global__ void __launch_bounds__(256) bn_bwd_reduce_kernel(const bf16* __restrict__ dy, const float* __restrict__ c,
                                                            const float* __restrict__ stats, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, const int* __restrict__ len,
                                                            float* __restrict__ red_out, int M, int T, int d) {
    __shared__ float red[RL][256];
    const int col = blockIdx.x * 256 + (threadIdx.x & 31) * 8, rl = threadIdx.x >> 5;
    float s1[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, s2[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (col < d) {
        for (int row = blockIdx.y * RL + rl; row < M; row += gridDim.y * RL) {
            float a[8], xh[8], da[8];
            bn_affine(c + (size_t)row * d + col, stats, gamma, beta, col, d, a, xh);
            swish_bwd(dy + (size_t)row * d + col, row_valid(len, row, T), a, da);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                s1[j] += da[j];
                s2[j] = fmaf(da[j], xh[j], s2[j]);
            }
        }
    }
    reduce_add(red, s1, red_out, d);
    __syncthreads();
    reduce_add(red, s2, red_out + d, d);
}

// dc = gamma * invstd * (da - mean(da) - xhat * mean(da * xhat))  (fp32); block 0 also hands dbeta / dgamma to the caller
__global__ void __launch_bounds__(256) bn_bwd_dx_kernel(const bf16* __restrict__ dy, const float* __restrict__ c,
                                                        const float* __restrict__ stats, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, const int* __restrict__ len,
                                                        const float* __restrict__ red, float* __restrict__ dc,
                                                        float* __restrict__ dgamma, float* __restrict__ dbeta, int accumulate,
                                                        int M, int T, int d) {
    if (blockIdx.x == 0) {
        for (int ch = threadIdx.x; ch < d; ch += blockDim.x) {
            dbeta[ch] = (accumulate ? dbeta[ch] : 0.f) + red[ch];
            dgamma[ch] = (accumulate ? dgamma[ch] : 0.f) + red[d + ch];
        }
    }
    const int cg = d / 8;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)M * cg) return;
    const int row = (int)(i / cg), col = (int)(i % cg) * 8;
    float a[8], xh[8], da[8];
    bn_affine(c + (size_t)row * d + col, stats, gamma, beta, col, d, a, xh);
    swish_bwd(dy + (size_t)row * d + col, row_valid(len, row, T), a, da);
    const float inv_m = 1.0f / (float)M;
#pragma unroll
    for (int j = 0; j < 8; ++j)
        da[j] = gamma[col + j] * stats[d + col + j] * (da[j] - red[col + j] * inv_m - xh[j] * red[d + col + j] * inv_m);
    store8(dc + (size_t)row * d + col, da);
}

// dx[t] = mask * sum_tap w[tap] dc[t - tap + pad]: the transposed depthwise conv, over the conv's output rows [0, T)
__global__ void __launch_bounds__(256) dwconv_bwd_dx_kernel(const float* __restrict__ dc, const int* __restrict__ len,
                                                            const float* __restrict__ w, bf16* __restrict__ dx, int M, int T,
                                                            int d, int k) {
    const int cg = d / 8;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)M * cg) return;
    const int row = (int)(i / cg), col = (int)(i % cg) * 8, t = row % T, pad = (k - 1) / 2;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (row_valid(len, row, T)) {
        for (int tap = 0; tap < k; ++tap) {
            const int tt = t - tap + pad;
            if (tt < 0 || tt >= T) continue;
            float v[8];
            load8(dc + (size_t)(row - tap + pad) * d + col, v);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = fmaf(v[j], w[(col + j) * k + tap], acc[j]);
        }
    }
    store8(dx + (size_t)row * d + col, acc);
}

// dw[ch, tap] += sum_rows dc[row] * mask(x)[row + tap - pad] (blockIdx.z = tap), and the conv bias gradient at z = k
__global__ void __launch_bounds__(256) dwconv_wgrad_kernel(const float* __restrict__ dc, const bf16* __restrict__ x,
                                                           const int* __restrict__ len, float* __restrict__ dw,
                                                           float* __restrict__ dwb, int M, int T, int d, int k) {
    __shared__ float red[RL][256];
    const int col = blockIdx.x * 256 + (threadIdx.x & 31) * 8, rl = threadIdx.x >> 5, pad = (k - 1) / 2, tap = blockIdx.z;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (col < d) {
        for (int row = blockIdx.y * RL + rl; row < M; row += gridDim.y * RL) {
            float g[8];
            load8(dc + (size_t)row * d + col, g);
            if (tap == k) {
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] += g[j];
                continue;
            }
            const int tt = row % T + tap - pad;
            if (tt < 0 || tt >= valid_len(len, row, T)) continue;
            float v[8];
            load8(x + (size_t)(row + tap - pad) * d + col, v);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = fmaf(g[j], v[j], acc[j]);
        }
    }
    const int cgi = threadIdx.x & 31;
#pragma unroll
    for (int j = 0; j < 8; ++j) red[rl][cgi * 8 + j] = acc[j];
    __syncthreads();
    const int ch = blockIdx.x * 256 + threadIdx.x;
    if (ch < d) {
        float s = 0.f;
#pragma unroll
        for (int r = 0; r < RL; ++r) s += red[r][threadIdx.x];
        if (tap == k)
            atomicAdd(dwb + ch, s);
        else
            atomicAdd(dw + (size_t)ch * k + tap, s);
    }
}

dim3 reduce_grid(int M, int d, int z = 1) {
    int gy = (M + 4 * RL - 1) / (4 * RL);      // at least 4 rows per thread
    if (gy > 128) gy = 128;
    return dim3((d + 255) / 256, gy, z);
}

const char* check_shape(int B, int T, int d, int k) {
    if (B < 1 || T < 1) return "conformer conv: empty batch";
    if (d % 8) return "conformer conv: d must be a multiple of 8";
    if (k < 1 || !(k & 1)) return "conformer conv: the kernel size must be odd";
    return nullptr;
}

}  // namespace

const char* conv_bn_train_launch(cudaStream_t st, const bf16* x, const int* len, const float* w, const float* wb, const float* gamma,
                                 const float* beta, float* run_mean, float* run_var, long long* n_batches, float momentum, float eps,
                                 float* c, float* stats, bf16* out, int B, int T, int d, int k) {
    if (const char* e = check_shape(B, T, d, k)) return e;
    const int M = B * T;
    cudaError_t e = cudaMemsetAsync(stats, 0, (size_t)2 * d * sizeof(float), st);
    if (e != cudaSuccess) return cudaGetErrorString(e);
    const char* err;
    if ((err = launch<dwconv_sum_kernel>(reduce_grid(M, d), 256, 0, st, x, len, w, wb, c, stats, M, T, d, k))) return err;
    if ((err = launch<bn_var_kernel>(reduce_grid(M, d), 256, 0, st, c, stats, M, d))) return err;
    if ((err = launch<bn_finalize_kernel>(1, 256, 0, st, stats, run_mean, run_var, n_batches, M, d, momentum, eps))) return err;
    const size_t n = (size_t)M * (d / 8);
    return launch<bn_swish_kernel>((unsigned)((n + 255) / 256), 256, 0, st, c, stats, gamma, beta, len, out, M, T, d);
}

const char* conv_bn_bwd_launch(cudaStream_t st, const bf16* dy, const bf16* x, const int* len, const float* w, const float* gamma,
                               const float* beta, const float* c, const float* stats, float* red, float* dc, bf16* dx, float* dw,
                               float* dwb, float* dgamma, float* dbeta, int accumulate, int B, int T, int d, int k) {
    if (const char* e = check_shape(B, T, d, k)) return e;
    const int M = B * T;
    cudaError_t e = cudaMemsetAsync(red, 0, (size_t)2 * d * sizeof(float), st);
    if (e == cudaSuccess && !accumulate) e = cudaMemsetAsync(dw, 0, (size_t)d * k * sizeof(float), st);
    if (e == cudaSuccess && !accumulate && dwb) e = cudaMemsetAsync(dwb, 0, (size_t)d * sizeof(float), st);
    if (e != cudaSuccess) return cudaGetErrorString(e);
    const char* err;
    if ((err = launch<bn_bwd_reduce_kernel>(reduce_grid(M, d), 256, 0, st, dy, c, stats, gamma, beta, len, red, M, T, d))) return err;
    const size_t n = (size_t)M * (d / 8);
    const unsigned grid = (unsigned)((n + 255) / 256);
    if ((err = launch<bn_bwd_dx_kernel>(grid, 256, 0, st, dy, c, stats, gamma, beta, len, red, dc, dgamma, dbeta, accumulate, M, T, d)))
        return err;
    if ((err = launch<dwconv_bwd_dx_kernel>(grid, 256, 0, st, dc, len, w, dx, M, T, d, k))) return err;
    return launch<dwconv_wgrad_kernel>(reduce_grid(M, d, dwb ? k + 1 : k), 256, 0, st, dc, x, len, dw, dwb, M, T, d, k);
}

}  // namespace otb
