// HBM-bound kernels of the training step (backward of the row-wise ops, reductions, optimizer).
// Each kernel cites the reference forward it differentiates; the reference itself relies on torch autograd
// (otrans/train/trainer.py:206-234: loss.backward(), clip_grad_norm_, optimizer.step()).
#include <math.h>

#include "counter_rng.cuh"
#include "dropout.cuh"
#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

__device__ __forceinline__ void unpack8(const uint4& u, float (&v)[8]) {
    const float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y), c = unpack_bf16(u.z), d = unpack_bf16(u.w);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
__device__ __forceinline__ uint4 pack8(const float (&v)[8]) {
    uint4 u;
    u.x = pack_bf16(v[0], v[1]); u.y = pack_bf16(v[2], v[3]); u.z = pack_bf16(v[4], v[5]); u.w = pack_bf16(v[6], v[7]);
    return u;
}
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }

// ------------------------------------------------------------------------------------------------
// Bias gradient: out[n] = sum_m x[m, n]   (d/d bias of nn.Linear, attention.py:68 / ffn.py:39-41 ...)
// x bf16 [M, N] (ldx); out f32 [N], zeroed by the launcher.  CTA = 64 columns x a row slice; thread = 8 columns.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) colsum_kernel(const bf16* __restrict__ x, int ldx, float* __restrict__ out, int M, int N) {
    __shared__ float red[32][65];
    const int cg = threadIdx.x & 7, rl = threadIdx.x >> 3;          // 8 column groups x 32 row lanes
    const int col = blockIdx.x * 64 + cg * 8;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (col < N) {
        for (int m = blockIdx.y * 32 + rl; m < M; m += gridDim.y * 32) {
            float v[8];
            unpack8(*reinterpret_cast<const uint4*>(x + (size_t)m * ldx + col), v);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] += v[j];
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) red[rl][cg * 8 + j] = acc[j];
    __syncthreads();
    if (threadIdx.x < 64) {
        float s = 0.f;
#pragma unroll 8
        for (int r = 0; r < 32; ++r) s += red[r][threadIdx.x];
        const int c = blockIdx.x * 64 + threadIdx.x;
        if (c < N) atomicAdd(out + c, s);
    }
}

const char* colsum_launch(cudaStream_t st, const bf16* x, int ldx, float* out, int M, int N, int accumulate) {
    if (N % 8 || ldx % 8) return "colsum: N and ldx must be multiples of 8";
    cudaError_t e = accumulate ? cudaSuccess : cudaMemsetAsync(out, 0, (size_t)N * 4, st);
    if (e != cudaSuccess) return cudaGetErrorString(e);
    int gy = (M + 255) / 256;
    if (gy > 64) gy = 64;
    if (gy < 1) gy = 1;
    return launch<colsum_kernel>(dim3((N + 63) / 64, gy), 256, 0, st, x, ldx, out, M, N);
}

// ------------------------------------------------------------------------------------------------
// LayerNorm backward (nn.LayerNorm, eps 1e-5; encoder/transformer.py:54-56,61-63, decoder/transformer.py:60-88).
//   y = (z - mean) * rstd * gamma + beta ;  dz = rstd * (g - mean(g) - xhat * mean(g * xhat)),  g = dy * gamma
//   dgamma += dy * xhat ; dbeta += dy     (fp32, atomics; zeroed by the launcher)
// z, dy, dz bf16 [M, N], N <= 256 (one 16-byte chunk per lane); statistics are recomputed from z.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(const bf16* __restrict__ dy, int lddy, const bf16* __restrict__ z,
                                                            int ldz, const float* __restrict__ gamma, bf16* __restrict__ dz,
                                                            int lddz, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                            float eps, int M, int N) {
    __shared__ float sg[8][256], sb[8][256];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int col = lane * 8;
    const bool live = col < N;
    float gam[8], ag[8], ab[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { gam[j] = live ? gamma[col + j] : 0.f; ag[j] = 0.f; ab[j] = 0.f; }
    const float inv_n = 1.0f / (float)N;
    for (int row = blockIdx.x * 8 + warp; row < M; row += gridDim.x * 8) {
        float zv[8], dv[8];
        if (live) {
            unpack8(*reinterpret_cast<const uint4*>(z + (size_t)row * ldz + col), zv);
            unpack8(*reinterpret_cast<const uint4*>(dy + (size_t)row * lddy + col), dv);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) { zv[j] = 0.f; dv[j] = 0.f; }
        }
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) s += zv[j];
        const float mean = warp_sum(s) * inv_n;
        float q = 0.f;
        if (live) {
#pragma unroll
            for (int j = 0; j < 8; ++j) { const float d = zv[j] - mean; q += d * d; }
        }
        const float rstd = rsqrtf(warp_sum(q) * inv_n + eps);
        float s1 = 0.f, s2 = 0.f, xh[8], g[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            xh[j] = live ? (zv[j] - mean) * rstd : 0.f;
            g[j] = dv[j] * gam[j];
            s1 += g[j];
            s2 += g[j] * xh[j];
            ag[j] += dv[j] * xh[j];
            ab[j] += dv[j];
        }
        s1 = warp_sum(s1) * inv_n;
        s2 = warp_sum(s2) * inv_n;
        if (live) {
            float o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = rstd * (g[j] - s1 - xh[j] * s2);
            *reinterpret_cast<uint4*>(dz + (size_t)row * lddz + col) = pack8(o);
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) { sg[warp][col + j] = ag[j]; sb[warp][col + j] = ab[j]; }
    __syncthreads();
    if ((int)threadIdx.x < N) {
        float a = 0.f, b = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) { a += sg[w][threadIdx.x]; b += sb[w][threadIdx.x]; }
        atomicAdd(dgamma + threadIdx.x, a);
        atomicAdd(dbeta + threadIdx.x, b);
    }
}

const char* layernorm_bwd_launch(cudaStream_t st, const bf16* dy, int lddy, const bf16* z, int ldz, const float* gamma,
                                 bf16* dz, int lddz, float* dgamma, float* dbeta, float eps, int M, int N, int accumulate) {
    if (N % 8 || N > 256 || lddy % 8 || ldz % 8 || lddz % 8) return "layernorm_bwd: N must be a multiple of 8, <= 256";
    cudaError_t e = accumulate ? cudaSuccess : cudaMemsetAsync(dgamma, 0, (size_t)N * 4, st);
    if (e == cudaSuccess && !accumulate) e = cudaMemsetAsync(dbeta, 0, (size_t)N * 4, st);
    if (e != cudaSuccess) return cudaGetErrorString(e);
    int grid = (M + 7) / 8;
    if (grid > 4 * num_sms()) grid = 4 * num_sms();
    return launch<layernorm_bwd_kernel>(grid, 256, 0, st, dy, lddy, z, ldz, gamma, dz, lddz, dgamma, dbeta, eps, M, N);
}

// ------------------------------------------------------------------------------------------------
// GLU (ffn.py:18,34 F.glu): u = [a | g] bf16 [M, 2F] -> h = a * sigmoid(g) bf16 [M, F], and its backward
//   da = dh * sigmoid(g) ; dg = dh * a * sigmoid(g) * (1 - sigmoid(g))
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) glu_fwd_kernel(const bf16* __restrict__ u, bf16* __restrict__ h, int M, int F) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int cpr = F / 8;
    if (i >= (size_t)M * cpr) return;
    const int row = (int)(i / cpr), c = (int)(i % cpr) * 8;
    float a[8], g[8], o[8];
    unpack8(*reinterpret_cast<const uint4*>(u + (size_t)row * 2 * F + c), a);
    unpack8(*reinterpret_cast<const uint4*>(u + (size_t)row * 2 * F + F + c), g);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = a[j] * sigmoidf_(g[j]);
    *reinterpret_cast<uint4*>(h + (size_t)row * F + c) = pack8(o);
}
__global__ void __launch_bounds__(256) glu_bwd_kernel(const bf16* __restrict__ dh, const bf16* __restrict__ u,
                                                      bf16* __restrict__ du, int M, int F) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int cpr = F / 8;
    if (i >= (size_t)M * cpr) return;
    const int row = (int)(i / cpr), c = (int)(i % cpr) * 8;
    float a[8], g[8], d[8], da[8], dg[8];
    unpack8(*reinterpret_cast<const uint4*>(u + (size_t)row * 2 * F + c), a);
    unpack8(*reinterpret_cast<const uint4*>(u + (size_t)row * 2 * F + F + c), g);
    unpack8(*reinterpret_cast<const uint4*>(dh + (size_t)row * F + c), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float s = sigmoidf_(g[j]);
        da[j] = d[j] * s;
        dg[j] = d[j] * a[j] * s * (1.0f - s);
    }
    *reinterpret_cast<uint4*>(du + (size_t)row * 2 * F + c) = pack8(da);
    *reinterpret_cast<uint4*>(du + (size_t)row * 2 * F + F + c) = pack8(dg);
}
const char* glu_launch(cudaStream_t st, const bf16* u, const bf16* dh, bf16* out, int M, int F) {
    if (F % 8) return "glu: F must be a multiple of 8";
    const size_t n = (size_t)M * (F / 8);
    const unsigned grid = (unsigned)((n + 255) / 256);
    return dh ? launch<glu_bwd_kernel>(grid, 256, 0, st, dh, u, out, M, F) : launch<glu_fwd_kernel>(grid, 256, 0, st, u, out, M, F);
}

// ------------------------------------------------------------------------------------------------
// The other feed-forward activations (ffn.py:15-41: w_2(dropout(act(w_1 x)))) for training, un-fused from the w_1 GEMM so
// that the backward reads the bf16 pre-activation u:  h = act(u);  du = dh * act'(u).  ACT is the epilogue id of the same
// activation (the recognition path fuses it into the GEMM epilogue):
//   EPI_GELU   F.gelu, erf form          act'(u) = Phi(u) + u phi(u)
//   EPI_TANH   torch.tanh                act'(u) = 1 - tanh(u)^2
//   EPI_SWISH  u * sigmoid(u)            act'(u) = s (1 + u (1 - s)),  s = sigmoid(u)
// bf16 [n] contiguous, fp32 math; thread = 8 elements (one 16-byte load per operand), the last thread takes n % 8 singly.
// ------------------------------------------------------------------------------------------------
template <int ACT>
__device__ __forceinline__ float act_value(float x) {
    if (ACT == EPI_GELU) return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
    if (ACT == EPI_TANH) return tanhf(x);
    return x / (1.0f + expf(-x));
}
template <int ACT>
__device__ __forceinline__ float act_slope(float x) {
    if (ACT == EPI_GELU) return 0.5f * (1.0f + erff(x * 0.70710678118654752f)) + x * 0.39894228040143268f * expf(-0.5f * x * x);
    if (ACT == EPI_TANH) {
        const float t = tanhf(x);
        return 1.0f - t * t;
    }
    const float s = 1.0f / (1.0f + expf(-x));
    return s * (1.0f + x * (1.0f - s));
}
template <int ACT, bool BWD>
__global__ void __launch_bounds__(256) act_kernel(const bf16* __restrict__ u, const bf16* __restrict__ dh, bf16* __restrict__ out,
                                                  size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i * 8 + 8 <= n) {
        float v[8], d[8];
        unpack8(reinterpret_cast<const uint4*>(u)[i], v);
        if (BWD) unpack8(reinterpret_cast<const uint4*>(dh)[i], d);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = BWD ? d[j] * act_slope<ACT>(v[j]) : act_value<ACT>(v[j]);
        reinterpret_cast<uint4*>(out)[i] = pack8(v);
    } else {
        for (size_t e = i * 8; e < n; ++e) {
            const float x = __bfloat162float(u[e]);
            out[e] = __float2bfloat16(BWD ? __bfloat162float(dh[e]) * act_slope<ACT>(x) : act_value<ACT>(x));
        }
    }
}
template <int ACT>
static const char* act_launch_t(cudaStream_t st, const bf16* u, const bf16* dh, bf16* out, size_t n) {
    const unsigned grid = (unsigned)((n + 8 * 256 - 1) / (8 * 256));
    return dh ? launch<act_kernel<ACT, true>>(grid, 256, 0, st, u, dh, out, n) : launch<act_kernel<ACT, false>>(grid, 256, 0, st, u, dh, out, n);
}
const char* act_launch(cudaStream_t st, int act, const bf16* u, const bf16* dh, bf16* out, size_t n) {
    if (((reinterpret_cast<uintptr_t>(u) | reinterpret_cast<uintptr_t>(dh) | reinterpret_cast<uintptr_t>(out)) & 15))
        return "act: operands must be 16-byte aligned";
    switch (act) {
        case EPI_GELU: return act_launch_t<EPI_GELU>(st, u, dh, out, n);
        case EPI_TANH: return act_launch_t<EPI_TANH>(st, u, dh, out, n);
        case EPI_SWISH: return act_launch_t<EPI_SWISH>(st, u, dh, out, n);
    }
    return "act: the activation must be gelu, tanh or swish (OTB_EPI_GELU / TANH / SWISH)";
}

// ------------------------------------------------------------------------------------------------
// ReLU backward through the OUTPUT (conv.py:64): dx = dy where y > 0 else 0; bf16, n multiple of 8; dx may alias dy.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) relu_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ y, bf16* __restrict__ dx, size_t n8) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n8) return;
    float d[8], v[8];
    unpack8(reinterpret_cast<const uint4*>(dy)[i], d);
    unpack8(reinterpret_cast<const uint4*>(y)[i], v);
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] = v[j] > 0.f ? d[j] : 0.f;
    reinterpret_cast<uint4*>(dx)[i] = pack8(d);
}
// Backward of the residual dropout (and the mask export for tests): out[m,n] = dy[m,n] * keep(seed, site, m, n) / (1-p);
// mask (optional, u8 [M,N]) receives keep.  Same pure function as the forward GEMM epilogue (dropout.cuh): nothing was stored.
// TWO: a second mask keep(seed, site2, m, n) on the same element (attention-output dropout under the residual dropout,
// EPI_RESID_DROP2); scale is then 1 / ((1 - p) (1 - p2)).
template <bool TWO>
__global__ void __launch_bounds__(256) dropout_bwd_kernel(const bf16* __restrict__ dy, int lddy, bf16* __restrict__ out, int ldo,
                                                          unsigned char* __restrict__ mask, int M, int N, unsigned thresh, float scale,
                                                          const unsigned* __restrict__ seed_ptr, unsigned site, unsigned thresh2,
                                                          unsigned site2) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int row = (int)(i / (N / 2)), cp = (int)(i % (N / 2));
    if (row >= M) return;
    const unsigned seed = *seed_ptr;
    bool k0 = drop_keep(seed, site, (uint32_t)row, (uint32_t)(2 * cp), thresh);
    bool k1 = drop_keep(seed, site, (uint32_t)row, (uint32_t)(2 * cp + 1), thresh);
    if (TWO) {
        k0 = k0 && drop_keep(seed, site2, (uint32_t)row, (uint32_t)(2 * cp), thresh2);
        k1 = k1 && drop_keep(seed, site2, (uint32_t)row, (uint32_t)(2 * cp + 1), thresh2);
    }
    if (mask) {
        mask[(size_t)row * N + 2 * cp] = k0 ? 1 : 0;
        mask[(size_t)row * N + 2 * cp + 1] = k1 ? 1 : 0;
    }
    if (dy) {
        const float2 v = unpack_bf16(*reinterpret_cast<const uint32_t*>(dy + (size_t)row * lddy + 2 * cp));
        *reinterpret_cast<uint32_t*>(out + (size_t)row * ldo + 2 * cp) = pack_bf16(k0 ? v.x * scale : 0.f, k1 ? v.y * scale : 0.f);
    }
}
const char* dropout_bwd_launch(cudaStream_t st, const bf16* dy, int lddy, bf16* out, int ldo, unsigned char* mask, int M, int N, float p,
                               const unsigned* seed, unsigned site, float p2, unsigned site2) {
    if (M < 1 || N < 2 || (N & 1) || (lddy & 1) || (ldo & 1)) return "dropout: N and the row pitches must be even";
    if (!(p >= 0.f && p < 1.f) || !(p2 >= 0.f && p2 < 1.f)) return "dropout: p must be in [0, 1)";
    if (!seed) return "dropout: null seed";
    const size_t n = (size_t)M * (N / 2);
    const unsigned grid = (unsigned)((n + 255) / 256);
    // as otb_linear_dropout_resid: two masks only when both rates are non-zero, else the one with a rate (or p's)
    if (p > 0.f && p2 > 0.f)
        return launch<dropout_bwd_kernel<true>>(grid, 256, 0, st, dy, lddy, out, ldo, mask, M, N, drop_threshold(p),
                                                drop_scale2(p, p2), seed, site, drop_threshold(p2), site2);
    if (p == 0.f && p2 > 0.f) { p = p2; site = site2; }
    return launch<dropout_bwd_kernel<false>>(grid, 256, 0, st, dy, lddy, out, ldo, mask, M, N, drop_threshold(p), 1.0f / (1.0f - p),
                                             seed, site, 0u, 0u);
}

// out = resid + alpha * dropout_p(rowmask(x)) without a GEMM in front (rel-pos attention has no output projection; the
// Conformer's conv module masks its output before the dropout, module/conformer.py:55).  Same keep(seed, site, row, col) as
// the GEMM epilogue and dropout_bwd_kernel.  resid null: out = alpha * dropout_p(rowmask(x)), which is also the backward of
// such a site (the mask and scale are the forward's); p = 0 without row_len: a plain sum.  Rows with
// row % row_period >= row_len[row / row_period] read x as zero.  Thread = 8 columns of one row.
__global__ void __launch_bounds__(256) dropout_add_kernel(const bf16* __restrict__ x, int ldx, const bf16* __restrict__ resid, int ldr,
                                                          bf16* __restrict__ out, int ldo, int M, int N, float alpha, unsigned thresh,
                                                          float scale, const unsigned* __restrict__ seed_ptr, unsigned site,
                                                          const int* __restrict__ row_len, int row_period) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int cg = N / 8;
    const int row = (int)(i / cg), c0 = (int)(i % cg) * 8;
    if (row >= M) return;
    float v[8], r[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    unpack8(*reinterpret_cast<const uint4*>(x + (size_t)row * ldx + c0), v);
    if (resid) unpack8(*reinterpret_cast<const uint4*>(resid + (size_t)row * ldr + c0), r);
    const bool live = !row_len || row % row_period < row_len[row / row_period];
    const unsigned seed = seed_ptr ? *seed_ptr : 0u;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const bool keep = live && (thresh == 0u || drop_keep(seed, site, (uint32_t)row, (uint32_t)(c0 + j), thresh));
        r[j] += keep ? alpha * (v[j] * scale) : 0.f;
    }
    *reinterpret_cast<uint4*>(out + (size_t)row * ldo + c0) = pack8(r);
}
const char* dropout_add_launch(cudaStream_t st, const bf16* x, int ldx, const bf16* resid, int ldr, bf16* out, int ldo, int M, int N,
                               float alpha, float p, const unsigned* seed, unsigned site, const int* row_len, int row_period) {
    if (M < 1 || N < 8 || N % 8 || ldx % 8 || ldo % 8 || (resid && ldr % 8)) return "dropout_add: N and the row pitches must be multiples of 8";
    if (!(p >= 0.f && p < 1.f)) return "dropout: p must be in [0, 1)";
    if (p > 0.f && !seed) return "dropout: null seed";
    if (row_len && row_period < 1) return "dropout_add: row_len without row_period";
    const size_t n = (size_t)M * (N / 8);
    return launch<dropout_add_kernel>((unsigned)((n + 255) / 256), 256, 0, st, x, ldx, resid, ldr, out, ldo, M, N, alpha,
                                      drop_threshold(p), 1.0f / (1.0f - p), seed, site, row_len, row_period);
}

const char* relu_bwd_launch(cudaStream_t st, const bf16* dy, const bf16* y, bf16* dx, size_t n) {
    if (n % 8) return "relu_bwd: n must be a multiple of 8";
    return launch<relu_bwd_kernel>((unsigned)((n / 8 + 255) / 256), 256, 0, st, dy, y, dx, n / 8);
}

// ------------------------------------------------------------------------------------------------
// Embedding backward (decoder/transformer.py:163,169: x = embedding(tok) * sqrt(d) + PE):
//   dE[tok[n], :] += scale * dx[n, :]   fp32 atomics into the (already initialised) gradient of the tied weight
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) embed_bwd_kernel(const long long* __restrict__ tok, const bf16* __restrict__ dx,
                                                        float* __restrict__ dE, int N, int d, int vocab, float scale) {
    const int n = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (n >= N) return;
    const long long t = tok[n];
    if (t < 0 || t >= vocab) return;
    for (int c = lane * 8; c < d; c += 256) {
        float v[8];
        unpack8(*reinterpret_cast<const uint4*>(dx + (size_t)n * d + c), v);
#pragma unroll
        for (int j = 0; j < 8; ++j) atomicAdd(dE + (size_t)t * d + c + j, v[j] * scale);
    }
}
const char* embed_bwd_launch(cudaStream_t st, const long long* tok, const bf16* dx, float* dE, int N, int d, int vocab, float scale) {
    if (d % 8) return "embed_bwd: d must be a multiple of 8";
    return launch<embed_bwd_kernel>((N + 7) / 8, 256, 0, st, tok, dx, dE, N, d, vocab, scale);
}

// ------------------------------------------------------------------------------------------------
// Optimizer (otrans/train/trainer.py:221-234 + torch.optim.Adam as configured by conf/transformer_baseline.yaml:82-93):
//   total_norm = ||g||_2 over ALL parameters; coef = min(1, max_norm / (total_norm + 1e-6))  (clip_grad_norm_);
//   a non-finite norm skips the update (trainer.py:229-230);  g' = coef * g + wd * p (Adam's L2 weight decay);
//   m = b1 m + (1-b1) g' ; v = b2 v + (1-b2) g'^2 ; p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
// All parameters / gradients / moments live in flat fp32 buffers; everything stays on the device (no host sync).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ g, size_t n, float* __restrict__ out) {
    __shared__ float red[8];
    float s = 0.f;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float v = g[i];
        s += v * v;
    }
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += red[i];
        atomicAdd(out, t);
    }
}
// hyper (device f32 [4] = {lr, 1 - b1^t, 1 - b2^t, apply}) is written by adam_prepare_kernel, which owns the step counters
// on the device so that a skipped (non-finite) step advances neither the LR schedule nor Adam's bias-correction count --
// exactly what trainer.py:229-233 does on the host.
// NOISE (trainer.py:223-227, gradient noise): the clipped gradient gets noise * z before the weight decay, z a standard
// normal drawn from (*noise_seed, Adam step t = counters[0], element index) (counter_rng.cuh) on the elements whose bit is
// set in noise_mask (the parameters: the alignment gaps of the flat buffer stay zero).  noise = sigma / accum_steps.
template <bool NOISE>
__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                   float* __restrict__ v, size_t n, const float* __restrict__ sumsq,
                                                   float max_norm, float b1, float b2, float eps, float wd,
                                                   const float* __restrict__ hyper, float noise, const int* __restrict__ noise_seed,
                                                   const int* __restrict__ counters, const uint8_t* __restrict__ noise_mask) {
    const float total = sqrtf(*sumsq);
    if (!isfinite(total)) return;                      // NaN / Inf gradients: skip the step (trainer.py:229-230)
    const float lr = hyper[0], bc1 = hyper[1], bc2 = hyper[2];
    float coef = 1.0f;
    if (max_norm > 0.f) coef = fminf(1.0f, max_norm / (total + 1e-6f));
    const float step = lr / bc1, rs2 = rsqrtf(bc2);
    uint32_t key = 0;
    if constexpr (NOISE) key = rng_key((uint32_t)*noise_seed, (uint32_t)counters[0]);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float pi = p[i];
        float gi;
        if constexpr (NOISE) {
            float gc = g[i] * coef;
            if ((noise_mask[i >> 3] >> (i & 7)) & 1) gc = __fadd_rn(gc, __fmul_rn(noise, normal_at(key, i)));
            gi = gc + wd * pi;
        } else {
            gi = g[i] * coef + wd * pi;
        }
        const float mi = b1 * m[i] + (1.0f - b1) * gi;
        const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
        m[i] = mi;
        v[i] = vi;
        p[i] = pi - step * mi / (sqrtf(vi) * rs2 + eps);
    }
}
// counters i32 [3] = {optimizer steps taken, scheduler global_step, skipped steps}.  One thread: advance them only when
// the gradient norm is finite, then evaluate TransformerScheduler.get_step_lr (scheduler.py:137-138; warmup <= 0: constant
// base_lr) and Adam's bias corrections for the step about to be taken.
__global__ void adam_prepare_kernel(const float* __restrict__ sumsq, int* __restrict__ counters, float* __restrict__ hyper,
                                    float base_lr, float model_size, float warmup, float factor, float b1, float b2) {
    const float total = sqrtf(*sumsq);
    if (!isfinite(total)) {
        counters[2] += 1;
        hyper[3] = 0.f;
        return;
    }
    const int t = counters[0] + 1, s = counters[1] + 1;
    counters[0] = t;
    counters[1] = s;
    double lr = (double)base_lr;
    if (warmup > 0.f) lr = (double)factor * pow((double)model_size, -0.5) * fmin(pow((double)s, -0.5), (double)s * pow((double)warmup, -1.5));
    hyper[0] = (float)lr;
    hyper[1] = (float)(1.0 - pow((double)b1, (double)t));
    hyper[2] = (float)(1.0 - pow((double)b2, (double)t));
    hyper[3] = 1.f;
}
const char* sumsq_launch(cudaStream_t st, const float* g, size_t n, float* out, int zero_first) {
    if (zero_first) {
        cudaError_t e = cudaMemsetAsync(out, 0, 4, st);
        if (e != cudaSuccess) return cudaGetErrorString(e);
    }
    size_t blocks = (n + 2047) / 2048;
    if (blocks > (size_t)(8 * num_sms())) blocks = 8 * num_sms();
    if (blocks < 1) blocks = 1;
    return launch<sumsq_kernel>((unsigned)blocks, 256, 0, st, g, n, out);
}
const char* adam_sched_launch(cudaStream_t st, float* p, const float* g, float* m, float* v, size_t n, const float* sumsq,
                              float max_norm, float base_lr, float model_size, float warmup, float factor, float b1, float b2,
                              float eps, float wd, int* counters, float* hyper, float noise, const int* noise_seed,
                              const uint8_t* noise_mask) {
    const char* err = launch<adam_prepare_kernel>(1, 1, 0, st, sumsq, counters, hyper, base_lr, model_size, warmup, factor, b1, b2);
    if (err) return err;
    size_t blocks = (n + 1023) / 1024;
    if (blocks > (size_t)(8 * num_sms())) blocks = 8 * num_sms();
    if (blocks < 1) blocks = 1;
    if (noise > 0.f)
        return launch<adam_kernel<true>>((unsigned)blocks, 256, 0, st, p, g, m, v, n, sumsq, max_norm, b1, b2, eps, wd, hyper, noise,
                                         noise_seed, counters, noise_mask);
    return launch<adam_kernel<false>>((unsigned)blocks, 256, 0, st, p, g, m, v, n, sumsq, max_norm, b1, b2, eps, wd, hyper, 0.f,
                                      nullptr, nullptr, nullptr);
}

}  // namespace otb

namespace otb {

// ------------------------------------------------------------------------------------------------
// Conv2d subsampling front end, backward (frontend/conv.py:50-76 under autograd).
// Layouts as in the forward (ConvGeom): conv1 activation h1 = NHWC bf16 [B, T1p = st2*T1s, F1p = sf2*F1s, C]; conv2 output
// rows are (b, t2, f2) with C2 channels.  conv2's weight / input gradients are GEMMs over the explicit im2col matrix
//   col[(b,t2,f2), (kh*kf2+kw)*C + c] = h1[b, st2*t2+kh, sf2*f2+kw-pf2, c]      (f outside [0, F1) is the zero padding)
// (wgrad: dW2 = dpre2^T col on the TN wgmma kernel; dgrad: dcol = dpre2 W2, then the gather below).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) im2col_kernel(const bf16* __restrict__ h1, bf16* __restrict__ col, int B, int T2,
                                                     int F2, int C, int T1p, int F1p, int F1, int kt, int kf, int st, int sf) {
    const int cg = C / 8, ntap = kt * kf;
    const size_t total = (size_t)B * T2 * F2 * ntap * cg;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c8 = (int)(i % cg);
    size_t r = i / cg;
    const int tap = (int)(r % ntap);
    r /= ntap;
    const int f2 = (int)(r % F2);
    r /= F2;
    const int t2 = (int)(r % T2), b = (int)(r / T2);
    const int kh = tap / kf, kw = tap % kf;
    const int t = st * t2 + kh, f = sf * f2 + kw - kf / 2;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (f >= 0 && f < F1) v = *reinterpret_cast<const uint4*>(h1 + (((size_t)b * T1p + t) * F1p + f) * C + c8 * 8);
    *reinterpret_cast<uint4*>(col + (((size_t)(b * T2 + t2) * F2 + f2) * ntap + tap) * C + c8 * 8) = v;
}

// dpre1[b,t1,f1,c] = relu'(h1) * sum over the (kh,kw) taps that read this input position of dcol[(b,t2,f2),(kh,kw,c)],
// t2 = (t1-kh)/st2, f2 = (f1+pf2-kw)/sf2 (both must be integral and in range).  Output in the h1 layout (positions outside
// [0,T1) x [0,F1) are written as zero so that the buffer is fully defined).
__global__ void __launch_bounds__(256) col2im_relu_kernel(const bf16* __restrict__ dcol, const bf16* __restrict__ h1,
                                                          bf16* __restrict__ dpre1, int B, int T1, int F1, int T2, int F2,
                                                          int C, int T1p, int F1p, int kt, int kf, int st, int sf) {
    const int cg = C / 8, ntap = kt * kf;
    const size_t total = (size_t)B * T1p * F1p * cg;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c8 = (int)(i % cg);
    size_t r = i / cg;
    const int f1 = (int)(r % F1p);
    r /= F1p;
    const int t1 = (int)(r % T1p), b = (int)(r / T1p);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (t1 < T1 && f1 < F1) {
        for (int kh = 0; kh < kt; ++kh) {
            const int tt = t1 - kh;
            if (tt < 0 || tt % st) continue;
            const int t2 = tt / st;
            if (t2 >= T2) continue;
            for (int kw = 0; kw < kf; ++kw) {
                const int ff = f1 + kf / 2 - kw;
                if (ff < 0 || ff % sf) continue;
                const int f2 = ff / sf;
                if (f2 >= F2) continue;
                float v[8];
                unpack8(*reinterpret_cast<const uint4*>(dcol + (((size_t)(b * T2 + t2) * F2 + f2) * ntap + kh * kf + kw) * C + c8 * 8), v);
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] += v[j];
            }
        }
        float hv[8];
        unpack8(*reinterpret_cast<const uint4*>(h1 + i * 8), hv);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = hv[j] > 0.f ? acc[j] : 0.f;
    }
    *reinterpret_cast<uint4*>(dpre1 + i * 8) = pack8(acc);
}

// conv1 (C_in = 1) weight / bias gradient: dW1[c, kh*kf+kw] = sum dpre1[b,t1,f1,c] * x[b, st*t1+kh, sf*f1+kw-pf], db1[c] =
// sum dpre1.  out f32 [C, kt*kf + 1] (taps + bias), zeroed by the launcher.  CTA = (b, 8 rows of t1); thread = (channel,
// position lane).  KMAX bounds kt and kf: the per-thread sums are registers indexed at compile time.
template <int KMAX>
__global__ void __launch_bounds__(256) conv1_wgrad_kernel(const bf16* __restrict__ dpre1, const float* __restrict__ x,
                                                          float* __restrict__ out, int B, int T, int F, int T1, int F1,
                                                          int T1p, int F1p, int C, int kt, int kf, int st, int sf) {
    extern __shared__ float sx[];   // [st*7 + kt][F + 2*pf], then red [256][kt*kf + 1]
    constexpr int ROWS = 8;
    const int pf = kf / 2, ntap = kt * kf, nout = ntap + 1;
    const int chunks = (T1 + ROWS - 1) / ROWS;
    const int b = blockIdx.x / chunks, t1_0 = (blockIdx.x % chunks) * ROWS;
    const int nrows = min(ROWS, T1 - t1_0);
    const int W2 = F + 2 * pf;
    float* red = sx + (st * (ROWS - 1) + kt) * W2;
    for (int i = threadIdx.x; i < (st * (nrows - 1) + kt) * W2; i += blockDim.x) {
        const int r = i / W2, f = i % W2 - pf;
        sx[i] = (f >= 0 && f < F) ? x[((size_t)b * T + st * t1_0 + r) * F + f] : 0.f;
    }
    __syncthreads();
    const int lanes = blockDim.x / C;
    const int c = threadIdx.x % C, pl = threadIdx.x / C;
    float acc[KMAX * KMAX + 1];
#pragma unroll
    for (int j = 0; j < KMAX * KMAX + 1; ++j) acc[j] = 0.f;
    if (pl < lanes) {
        for (int pos = pl; pos < nrows * F1; pos += lanes) {
            const int r = pos / F1, f1 = pos % F1;
            const float g = __bfloat162float(dpre1[(((size_t)b * T1p + t1_0 + r) * F1p + f1) * C + c]);
#pragma unroll
            for (int kh = 0; kh < KMAX; ++kh) {
                if (kh >= kt) break;
#pragma unroll
                for (int kw = 0; kw < KMAX; ++kw) {
                    if (kw >= kf) break;
                    acc[kh * KMAX + kw] = fmaf(g, sx[(st * r + kh) * W2 + sf * f1 + kw], acc[kh * KMAX + kw]);
                }
            }
            acc[KMAX * KMAX] += g;
        }
    }
#pragma unroll
    for (int kh = 0; kh < KMAX; ++kh)
#pragma unroll
        for (int kw = 0; kw < KMAX; ++kw)
            if (kh < kt && kw < kf) red[threadIdx.x * nout + kh * kf + kw] = acc[kh * KMAX + kw];
    red[threadIdx.x * nout + ntap] = acc[KMAX * KMAX];
    __syncthreads();
    for (int i = threadIdx.x; i < C * nout; i += blockDim.x) {
        const int cc = i / nout, j = i % nout;
        float s = 0.f;
        for (int l = 0; l < lanes; ++l) s += red[(l * C + cc) * nout + j];
        atomicAdd(out + cc * nout + j, s);
    }
}

const char* im2col_launch(cudaStream_t st, const bf16* h1, bf16* col, int B, const ConvGeom& g, int C) {
    if (C % 8) return "im2col: C must be a multiple of 8";
    const size_t total = (size_t)B * g.T2 * g.F2 * g.kt2 * g.kf2 * (C / 8);
    return launch<im2col_kernel>((unsigned)((total + 255) / 256), 256, 0, st, h1, col, B, g.T2, g.F2, C, g.st2 * g.T1s,
                                 g.sf2 * g.F1s, g.F1, g.kt2, g.kf2, g.st2, g.sf2);
}
const char* col2im_relu_launch(cudaStream_t st, const bf16* dcol, const bf16* h1, bf16* dpre1, int B, const ConvGeom& g, int C) {
    if (C % 8) return "col2im: C must be a multiple of 8";
    const size_t total = (size_t)B * g.st2 * g.T1s * g.sf2 * g.F1s * (C / 8);
    return launch<col2im_relu_kernel>((unsigned)((total + 255) / 256), 256, 0, st, dcol, h1, dpre1, B, g.T1, g.F1, g.T2, g.F2, C,
                                      g.st2 * g.T1s, g.sf2 * g.F1s, g.kt2, g.kf2, g.st2, g.sf2);
}
const char* conv1_wgrad_launch(cudaStream_t st, const bf16* dpre1, const float* x, float* out, int B, int T, int F,
                               const ConvGeom& g, int C) {
    // one thread per (channel, position lane): C <= 256 leaves at least one lane per channel (threads past the last full
    // lane idle, e.g. C = 192); C > 256 would leave none and silently return zeros
    if (C < 8 || C > 256 || C % 8) return "conv1_wgrad: C must be a multiple of 8, at most 256";
    const int nout = g.kt1 * g.kf1 + 1;
    const size_t sx = (size_t)(g.st1 * 7 + g.kt1) * (F + 2 * (g.kf1 / 2)) * sizeof(float);
    if (sx > 40 * 1024) return "conv1_wgrad: F too large";
    const size_t smem = sx + (size_t)256 * nout * sizeof(float);
    cudaError_t e = cudaMemsetAsync(out, 0, (size_t)C * nout * 4, st);
    if (e != cudaSuccess) return cudaGetErrorString(e);
    const int chunks = (g.T1 + 7) / 8;
    const int kmax = max(g.kt1, g.kf1);
#define WGRAD_ARGS B * chunks, 256, smem, st, dpre1, x, out, B, T, F, g.T1, g.F1, g.st2 * g.T1s, g.sf2 * g.F1s, C, g.kt1, g.kf1, g.st1, g.sf1
    if (kmax <= 3) return launch<conv1_wgrad_kernel<3>>(WGRAD_ARGS);
    if (kmax <= 5) return launch<conv1_wgrad_kernel<5>>(WGRAD_ARGS);
    return launch<conv1_wgrad_kernel<7>>(WGRAD_ARGS);
#undef WGRAD_ARGS
}

}  // namespace otb

namespace otb {

// ------------------------------------------------------------------------------------------------
// SpecAugment application (otrans/data/augment.py:9-41): zero `nf` frequency bands and `nt` time bands per utterance.
// The band positions are drawn on the host with the reference's RNG call order (opentransformer_b200/augment.py) and
// replayed here on the device-resident batch: x f32 [B, T, F] in place; bands i32 [B, 2*(nf+nt)] = (f0, f)*nf, (t0, t)*nt.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) spec_augment_kernel(float* __restrict__ x, const int* __restrict__ bands, int B, int T,
                                                           int F, int nf, int nt) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)B * T * F) return;
    const int f = (int)(i % F);
    const int t = (int)((i / F) % T);
    const int b = (int)(i / ((size_t)F * T));
    const int* bd = bands + (size_t)b * 2 * (nf + nt);
    bool kill = false;
    for (int j = 0; j < nf; ++j) kill |= (f >= bd[2 * j] && f < bd[2 * j] + bd[2 * j + 1]);
    for (int j = 0; j < nt; ++j) kill |= (t >= bd[2 * (nf + j)] && t < bd[2 * (nf + j)] + bd[2 * (nf + j) + 1]);
    if (kill) x[i] = 0.f;
}
const char* spec_augment_launch(cudaStream_t st, float* x, const int* bands, int B, int T, int F, int nf, int nt) {
    const size_t n = (size_t)B * T * F;
    return launch<spec_augment_kernel>((unsigned)((n + 255) / 256), 256, 0, st, x, bands, B, T, F, nf, nt);
}

}  // namespace otb
