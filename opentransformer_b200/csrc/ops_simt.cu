// HBM-bound / latency-bound kernels of the hot path (no tensor cores): coalesced, vectorised,
// warp-shuffle reductions.  Each kernel cites the reference lines it replaces.
#include <math.h>

#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

// ------------------------------------------------------------------------------------------------
// conv1: Conv2d(1 -> C1, (kt, kf), stride (st, sf), padding (0, kf/2)) + ReLU      otrans/frontend/conv.py:27-37,63-64
// in : x f32 [B, T, F]
// out: bf16 NHWC [B, st2*T1s, sf2*F1s, C1] (ConvGeom); columns f >= F1 are written as zero (they are the right
//      frequency padding of conv2); rows t >= T1 are never read for valid outputs and left untouched.
// HBM-bound on the output write (82 MB at cfg 2).  One CTA = 24 consecutive output rows of one utterance: their
// st*23 + kt input rows are staged in smem once, each thread keeps the filters + bias of its CPT channels in registers
// and walks over (row, f1) positions, one store per position, fully coalesced along (f1, c).  (With 8 rows per CTA the
// 80 weight loads per thread outnumbered the stores 8:1.)  KMAX bounds kt and kf: the filters of a thread take
// KMAX^2 * CPT registers (72, 100, 98), indexed at compile time by unrolled loops that skip the taps past (kt, kf).
// SHIPPED fixes the shipped geometry (3x3, stride 2) at compile time: the run-time strides and tap bounds cost the
// shipped front end 17 % of conv1's time on H100.
// ------------------------------------------------------------------------------------------------
static constexpr int CONV1_ROWS = 24;

template <int KMAX, int CPT, bool SHIPPED>
__global__ void __launch_bounds__(256) conv1_relu_nhwc_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                              const float* __restrict__ bias, bf16* __restrict__ out,
                                                              int B, int T, int F, int T1, int F1, int T1pad,
                                                              int F1pad, int C1, int kt_, int kf_, int st_, int sf_) {
    const int kt = SHIPPED ? 3 : kt_, kf = SHIPPED ? 3 : kf_, st = SHIPPED ? 2 : st_, sf = SHIPPED ? 2 : sf_;
    extern __shared__ float sx[];  // [st*(CONV1_ROWS-1) + kt][F + 2*pf]  (pf = kf/2 zero columns each side)
    const int pf = kf / 2;
    const int chunks = (T1 + CONV1_ROWS - 1) / CONV1_ROWS;
    const int b = blockIdx.x / chunks, t1_0 = (blockIdx.x % chunks) * CONV1_ROWS;
    const int nrows = min(CONV1_ROWS, T1 - t1_0);
    const int W2 = F + 2 * pf;
    const int in_rows = st * (nrows - 1) + kt;
    for (int i = threadIdx.x; i < in_rows * W2; i += blockDim.x) {
        const int r = i / W2, f = i % W2 - pf;
        sx[i] = (f >= 0 && f < F) ? x[((size_t)b * T + st * t1_0 + r) * F + f] : 0.f;
    }
    const int cgs = C1 / CPT;           // channel groups of CPT
    const int ppp = blockDim.x / cgs;   // positions per pass
    const int cg = threadIdx.x % cgs, pos0 = threadIdx.x / cgs;
    const int ntap = kt * kf;
    float wr[KMAX * KMAX][CPT], br[CPT];
#pragma unroll
    for (int j = 0; j < CPT; ++j) {
        br[j] = bias[cg * CPT + j];
#pragma unroll
        for (int kh = 0; kh < KMAX; ++kh)
#pragma unroll
            for (int kw = 0; kw < KMAX; ++kw)
                if (kh < kt && kw < kf) wr[kh * KMAX + kw][j] = w[(cg * CPT + j) * ntap + kh * kf + kw];
    }
    __syncthreads();
    if (pos0 >= ppp) return;
    const int npos = nrows * F1pad;
    for (int pos = pos0; pos < npos; pos += ppp) {
        const int r = pos / F1pad, f1 = pos % F1pad;
        float v[CPT];
        if (f1 < F1) {
#pragma unroll
            for (int j = 0; j < CPT; ++j) v[j] = br[j];
#pragma unroll
            for (int kh = 0; kh < KMAX; ++kh) {
                if (kh >= kt) break;
#pragma unroll
                for (int kw = 0; kw < KMAX; ++kw) {
                    if (kw >= kf) break;
                    const float xv = sx[(st * r + kh) * W2 + sf * f1 + kw];  // input col sf*f1 + kw - pf, +pf for the halo
#pragma unroll
                    for (int j = 0; j < CPT; ++j) v[j] = fmaf(xv, wr[kh * KMAX + kw][j], v[j]);
                }
            }
#pragma unroll
            for (int j = 0; j < CPT; ++j) v[j] = fmaxf(v[j], 0.f);
        } else {
#pragma unroll
            for (int j = 0; j < CPT; ++j) v[j] = 0.f;
        }
        uint32_t u[CPT / 2];
#pragma unroll
        for (int j = 0; j < CPT / 2; ++j) u[j] = pack_bf16(v[2 * j], v[2 * j + 1]);
        bf16* dst = out + (((size_t)b * T1pad + t1_0 + r) * F1pad + f1) * C1 + cg * CPT;
        if constexpr (CPT == 8) *reinterpret_cast<uint4*>(dst) = make_uint4(u[0], u[1], u[2], u[3]);
        else if constexpr (CPT == 4) *reinterpret_cast<uint2*>(dst) = make_uint2(u[0], u[1]);
        else *reinterpret_cast<uint32_t*>(dst) = u[0];
    }
}

const char* conv1_launch(cudaStream_t st, const float* x, const float* w, const float* bias, bf16* out, int B, int T,
                         int F, const ConvGeom& g, int C1) {
    const int kmax = max(g.kt1, g.kf1);
    const int cpt = kmax <= 3 ? 8 : kmax <= 5 ? 4 : 2;   // channels per thread: the filters fit the registers
    if (C1 % 8 || C1 > 256 * cpt) return "conv1: C1 must be a multiple of 8, at most 2048 (1024 for kernels wider than 3, 512 wider than 5)";
    size_t smem = (size_t)(g.st1 * (CONV1_ROWS - 1) + g.kt1) * (F + 2 * (g.kf1 / 2)) * sizeof(float);
    if (smem > 48 * 1024) return "conv1: F too large";
    const int chunks = (g.T1 + CONV1_ROWS - 1) / CONV1_ROWS;
    const int T1pad = g.st2 * g.T1s, F1pad = g.sf2 * g.F1s;
#define CONV1_ARGS dim3(B * chunks), dim3(256), smem, st, x, w, bias, out, B, T, F, g.T1, g.F1, T1pad, F1pad, C1, g.kt1, g.kf1, g.st1, g.sf1
    if (g.kt1 == 3 && g.kf1 == 3 && g.st1 == 2 && g.sf1 == 2) return launch<conv1_relu_nhwc_kernel<3, 8, true>>(CONV1_ARGS);
    if (cpt == 8) return launch<conv1_relu_nhwc_kernel<3, 8, false>>(CONV1_ARGS);
    if (cpt == 4) return launch<conv1_relu_nhwc_kernel<5, 4, false>>(CONV1_ARGS);
    return launch<conv1_relu_nhwc_kernel<7, 2, false>>(CONV1_ARGS);
#undef CONV1_ARGS
}

// ------------------------------------------------------------------------------------------------
// LayerNorm over the last dim (nn.LayerNorm, eps 1e-5): otrans/encoder/conformer.py:52,57,62,67,87,89
// bf16 in -> bf16 (or f32) out, fp32 statistics, warp per row, 16-byte loads.  An optional second
// affine LayerNorm is applied back to back (Conformer post_ffn_norm -> final_norm, conformer.py:87-89).
// ------------------------------------------------------------------------------------------------
template <int CH>  // CH = 16-byte chunks per lane (N = CH * 256)
__global__ void __launch_bounds__(256) layernorm_kernel(const bf16* __restrict__ x, int ldx, void* __restrict__ out,
                                                        int ldo, int out_f32, const float* __restrict__ g1,
                                                        const float* __restrict__ b1, const float* __restrict__ g2,
                                                        const float* __restrict__ b2, float eps, int M, int N) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= M) return;
    float v[CH * 8];
    const bf16* xr = x + (size_t)row * ldx;
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
        const int col = (c * 32 + lane) * 8;
        if (col < N) {
            uint4 u = *reinterpret_cast<const uint4*>(xr + col);
            float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y), cc = unpack_bf16(u.z), d = unpack_bf16(u.w);
            v[c * 8 + 0] = a.x; v[c * 8 + 1] = a.y; v[c * 8 + 2] = b.x; v[c * 8 + 3] = b.y;
            v[c * 8 + 4] = cc.x; v[c * 8 + 5] = cc.y; v[c * 8 + 6] = d.x; v[c * 8 + 7] = d.y;
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) v[c * 8 + j] = 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[c * 8 + j];
    }
    for (int pass = 0; pass < 2; ++pass) {
        const float* g = pass ? g2 : g1;
        const float* bb = pass ? b2 : b1;
        if (pass == 1) {
            if (g2 == nullptr) break;
            s = 0.f;
#pragma unroll
            for (int i = 0; i < CH * 8; ++i) s += v[i];
        }
        const float mean = warp_sum(s) / N;
        float q = 0.f;
#pragma unroll
        for (int c = 0; c < CH; ++c) {
            const int col = (c * 32 + lane) * 8;
            if (col < N) {
#pragma unroll
                for (int j = 0; j < 8; ++j) { const float d = v[c * 8 + j] - mean; q += d * d; }
            }
        }
        const float rstd = rsqrtf(warp_sum(q) / N + eps);
#pragma unroll
        for (int c = 0; c < CH; ++c) {
            const int col = (c * 32 + lane) * 8;
            if (col < N) {
#pragma unroll
                for (int j = 0; j < 8; ++j) v[c * 8 + j] = (v[c * 8 + j] - mean) * rstd * g[col + j] + bb[col + j];
            }
        }
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
        const int col = (c * 32 + lane) * 8;
        if (col < N) {
            if (out_f32) {
                float* o = reinterpret_cast<float*>(out) + (size_t)row * ldo + col;
                *reinterpret_cast<float4*>(o) = make_float4(v[c * 8], v[c * 8 + 1], v[c * 8 + 2], v[c * 8 + 3]);
                *reinterpret_cast<float4*>(o + 4) = make_float4(v[c * 8 + 4], v[c * 8 + 5], v[c * 8 + 6], v[c * 8 + 7]);
            } else {
                uint4 u;
                u.x = pack_bf16(v[c * 8], v[c * 8 + 1]);
                u.y = pack_bf16(v[c * 8 + 2], v[c * 8 + 3]);
                u.z = pack_bf16(v[c * 8 + 4], v[c * 8 + 5]);
                u.w = pack_bf16(v[c * 8 + 6], v[c * 8 + 7]);
                *reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(out) + (size_t)row * ldo + col) = u;
            }
        }
    }
}

// N <= 256 fast path: one warp normalises 4 rows at a time so that 4 independent 16-byte loads (and 4
// independent reduction chains) are in flight per lane -- the one-row-per-warp version was latency-bound.
__global__ void __launch_bounds__(256) layernorm256_kernel(const bf16* __restrict__ x, int ldx, void* __restrict__ out,
                                                           int ldo, int out_f32, const float* __restrict__ g1,
                                                           const float* __restrict__ b1, const float* __restrict__ g2,
                                                           const float* __restrict__ b2, float eps, int M, int N) {
    constexpr int R = 4;
    const int lane = threadIdx.x & 31;
    const int row0 = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * R;
    if (row0 >= M) return;
    const int col = lane * 8;
    const bool live = col < N;
    float v[R][8];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        uint4 u = make_uint4(0, 0, 0, 0);
        if (live && row0 + r < M) u = *reinterpret_cast<const uint4*>(x + (size_t)(row0 + r) * ldx + col);
        const float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y), c = unpack_bf16(u.z), d = unpack_bf16(u.w);
        v[r][0] = a.x; v[r][1] = a.y; v[r][2] = b.x; v[r][3] = b.y; v[r][4] = c.x; v[r][5] = c.y; v[r][6] = d.x; v[r][7] = d.y;
    }
    float gg[8], bb[8];
    for (int pass = 0; pass < 2; ++pass) {
        const float* g = pass ? g2 : g1;
        const float* be = pass ? b2 : b1;
        if (g == nullptr) break;
#pragma unroll
        for (int j = 0; j < 8; ++j) { gg[j] = live ? g[col + j] : 0.f; bb[j] = live ? be[col + j] : 0.f; }
        float s[R], q[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            s[r] = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) s[r] += v[r][j];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
            for (int r = 0; r < R; ++r) s[r] += __shfl_xor_sync(0xffffffffu, s[r], o);
#pragma unroll
        for (int r = 0; r < R; ++r) {
            s[r] /= N;
            q[r] = 0.f;
            if (live) {
#pragma unroll
                for (int j = 0; j < 8; ++j) { const float d = v[r][j] - s[r]; q[r] += d * d; }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
            for (int r = 0; r < R; ++r) q[r] += __shfl_xor_sync(0xffffffffu, q[r], o);
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const float rstd = rsqrtf(q[r] / N + eps);
#pragma unroll
            for (int j = 0; j < 8; ++j) v[r][j] = live ? (v[r][j] - s[r]) * rstd * gg[j] + bb[j] : 0.f;
        }
    }
    if (!live) return;
#pragma unroll
    for (int r = 0; r < R; ++r) {
        if (row0 + r >= M) break;
        if (out_f32) {
            float* o = reinterpret_cast<float*>(out) + (size_t)(row0 + r) * ldo + col;
            *reinterpret_cast<float4*>(o) = make_float4(v[r][0], v[r][1], v[r][2], v[r][3]);
            *reinterpret_cast<float4*>(o + 4) = make_float4(v[r][4], v[r][5], v[r][6], v[r][7]);
        } else {
            uint4 u;
            u.x = pack_bf16(v[r][0], v[r][1]);
            u.y = pack_bf16(v[r][2], v[r][3]);
            u.z = pack_bf16(v[r][4], v[r][5]);
            u.w = pack_bf16(v[r][6], v[r][7]);
            *reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(out) + (size_t)(row0 + r) * ldo + col) = u;
        }
    }
}

const char* layernorm_launch(cudaStream_t st, const bf16* x, int ldx, void* out, int ldo, int out_f32, const float* g1,
                             const float* b1, const float* g2, const float* b2, float eps, int M, int N) {
    if (N % 8 || ldx % 8 || N > 1024) return "layernorm: N must be a multiple of 8 and <= 1024";
    if ((out_f32 && ldo % 4) || (!out_f32 && ldo % 8)) return "layernorm: bad output stride";
    if (N <= 256) {
        const int rows_per_block = 8 * 4;
        return launch<layernorm256_kernel>(dim3((M + rows_per_block - 1) / rows_per_block), dim3(256), 0, st, x, ldx, out, ldo,
                                           out_f32, g1, b1, g2, b2, eps, M, N);
    }
    const int rows_per_block = 8;
    dim3 grid((M + rows_per_block - 1) / rows_per_block);
    const int ch = (N + 255) / 256;
    switch (ch) {
        case 1: return launch<layernorm_kernel<1>>(grid, dim3(256), 0, st, x, ldx, out, ldo, out_f32, g1, b1, g2, b2, eps, M, N);
        case 2: return launch<layernorm_kernel<2>>(grid, dim3(256), 0, st, x, ldx, out, ldo, out_f32, g1, b1, g2, b2, eps, M, N);
        case 3: return launch<layernorm_kernel<3>>(grid, dim3(256), 0, st, x, ldx, out, ldo, out_f32, g1, b1, g2, b2, eps, M, N);
        default: return launch<layernorm_kernel<4>>(grid, dim3(256), 0, st, x, ldx, out, ldo, out_f32, g1, b1, g2, b2, eps, M, N);
    }
}

// ------------------------------------------------------------------------------------------------
// Sinusoidal table: PE[p,2i] = sin(p*w_i), PE[p,2i+1] = cos(p*w_i), w_i = exp(-2i*ln(1e4)/d)
// otrans/module/pos.py:30-42 (recomputed on every call there; computed once per (first_pos, n, d) here)
// ------------------------------------------------------------------------------------------------
__global__ void sinusoid_table_kernel(float* __restrict__ out, int n_pos, int d, int first_pos) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pos * d) return;
    const int p = i / d + first_pos, c = i % d;
    const float w = expf((float)(c & ~1) * -(logf(10000.0f) / (float)d));
    const float a = (float)p * w;
    out[i] = (c & 1) ? cosf(a) : sinf(a);
}

const char* sinusoid_table_launch(cudaStream_t st, float* out, int n_pos, int d, int first_pos) {
    const int n = n_pos * d;
    return launch<sinusoid_table_kernel>((n + 255) / 256, 256, 0, st, out, n_pos, d, first_pos);
}

// ------------------------------------------------------------------------------------------------
// Embedding gather + positional encoding:  out[n] = emb[tok[n]] * sqrt(d) + PE[pos(n)]
// otrans/decoder/transformer.py:163,169  (+ module/pos.py:56)
// tok index:  tok[n * tok_stride + tok_off]; position: row_pos ? row_pos[n] : step_ptr ? *step_ptr : n % period
// ------------------------------------------------------------------------------------------------
template <bool ROW_POS>
__global__ void embed_posenc_kernel(const long long* __restrict__ tok, int tok_stride, const bf16* __restrict__ emb,
                                    const float* __restrict__ table, bf16* __restrict__ out, int N, int d, int period,
                                    const int* __restrict__ step_ptr, float xscale, int vocab, const int* __restrict__ row_pos) {
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= N) return;
    int pos;
    if constexpr (ROW_POS) pos = max(row_pos[n], 0);      // a row without a position (-1) reads position 0
    else pos = step_ptr ? *step_ptr : (n % period);
    long long t = tok[(size_t)n * tok_stride];
    if (t < 0 || t >= vocab) t = 0;
    const bf16* e = emb + (size_t)t * d;
    const float* pe = table + (size_t)pos * d;
    for (int col = lane * 8; col < d; col += 256) {
        uint4 u = *reinterpret_cast<const uint4*>(e + col);
        float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y), c = unpack_bf16(u.z), dd = unpack_bf16(u.w);
        const float4 p0 = *reinterpret_cast<const float4*>(pe + col);
        const float4 p1 = *reinterpret_cast<const float4*>(pe + col + 4);
        uint4 o;
        o.x = pack_bf16(a.x * xscale + p0.x, a.y * xscale + p0.y);
        o.y = pack_bf16(b.x * xscale + p0.z, b.y * xscale + p0.w);
        o.z = pack_bf16(c.x * xscale + p1.x, c.y * xscale + p1.y);
        o.w = pack_bf16(dd.x * xscale + p1.z, dd.y * xscale + p1.w);
        *reinterpret_cast<uint4*>(out + (size_t)n * d + col) = o;
    }
}

const char* embed_posenc_launch(cudaStream_t st, const long long* tok, int tok_stride, const bf16* emb,
                                const float* table, bf16* out, int N, int d, int period, const int* step_ptr,
                                int vocab, const int* row_pos) {
    if (d % 8) return "embed: d must be a multiple of 8";
    if (row_pos)
        return launch<embed_posenc_kernel<true>>(dim3((N + 7) / 8), dim3(256), 0, st, tok, tok_stride, emb, table, out, N, d,
                                                 period, step_ptr, sqrtf((float)d), vocab, row_pos);
    return launch<embed_posenc_kernel<false>>(dim3((N + 7) / 8), dim3(256), 0, st, tok, tok_stride, emb, table, out, N, d, period,
                                              step_ptr, sqrtf((float)d), vocab, row_pos);
}

// ------------------------------------------------------------------------------------------------
// Row log-softmax, fp32 (F.log_softmax of the last position's logits, decoder/transformer.py:206)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) log_softmax_kernel(const float* __restrict__ x, int ldx, float* __restrict__ out,
                                                          int ldo, int V) {
    __shared__ float red[8];
    __shared__ float bc;
    const float* xr = x + (size_t)blockIdx.x * ldx;
    float* orow = out + (size_t)blockIdx.x * ldo;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float m = -INFINITY;
    for (int i = threadIdx.x; i < V; i += 256) m = fmaxf(m, xr[i]);
    m = warp_max(m);
    if (lane == 0) red[warp] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = red[0];
        for (int i = 1; i < 8; ++i) t = fmaxf(t, red[i]);
        bc = t;
    }
    __syncthreads();
    m = bc;
    float s = 0.f;
    for (int i = threadIdx.x; i < V; i += 256) s += expf(xr[i] - m);
    s = warp_sum(s);
    __syncthreads();
    if (lane == 0) red[warp] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += red[i];
        bc = m + logf(t);
    }
    __syncthreads();
    const float lse = bc;
    for (int i = threadIdx.x; i < V; i += 256) orow[i] = xr[i] - lse;
}

const char* log_softmax_launch(cudaStream_t st, const float* x, int ldx, float* out, int ldo, int rows, int V) {
    return launch<log_softmax_kernel>(dim3(rows), dim3(256), 0, st, x, ldx, out, ldo, V);
}

// Chunk c of a staged K/V row goes to position rot_chunk(c + s) in row s (bank-conflict-free rows); i >= 0.
template <int CH>
__device__ __forceinline__ int rot_chunk(int i) {
    if constexpr (CH == 8) return i & 7;
    else return (int)((unsigned)i % CH);
}

// ------------------------------------------------------------------------------------------------
// Decode-time self-attention with a per-hypothesis KV cache (the `cache` the reference stubbed out,
// decoder/transformer.py:92-126,188-203).  One query (the newest token) per hypothesis; the prefix
// K/V of hypothesis n at position s' < step live in slot anc[n][s'] of step s' (beam reordering
// moves 4-byte ancestry entries, never K/V rows).  Warp = (hypothesis, head), d_k = DK (64 or 96).
// Also appends the current K/V to the cache.
//   qkv   bf16 [N, 3d] (Q | K | V of the current token, attention.py:73 split order)
//   kc,vc bf16 [Lmax, N, d]
//   anc   int32 [2, N, Lmax]  (ping-pong, buffer (step & 1) is current)
// ROW_POS (the LM-fused CTC search, DESIGN.md 4.19): every row has its own position, step_ptr[n] (row_pos), and
// kc / vc are [cache rows, d]: anc int32 [N, Lmax] lists the cache row of each position of row n, the newest included,
// and the newest K/V go to that row.  A row with row_pos -1 computes nothing and gets zeros.
// ------------------------------------------------------------------------------------------------
template <int DK, bool CHUNKED, bool ROW_POS = false>
__global__ void __launch_bounds__(128, DK == 64 ? 6 : 4) decode_self_attn_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ kc,
                                                               bf16* __restrict__ vc, const int* __restrict__ anc,
                                                               const int* __restrict__ step_ptr, bf16* __restrict__ out,
                                                               int N, int H, int Lmax, float scale, int keys_pad) {
    // Lanes run over KEYS: each lane owns up to KPL cached positions, resolves their slots through the
    // ancestry table and pulls the whole K and V rows (DK * 2 bytes) with 16-byte loads -- all loads of a lane are
    // independent, so the kernel costs ~3 dependent memory round trips (anc -> K/V -> out) instead of a
    // serial walk over the prefix.  V rows go through smem so that the P.V reduction is a column sum.
    // CHUNKED (prefixes of 129..1023 positions): the prefix is walked in chunks of 32 KPL keys with an online softmax (running
    // max and sum, P.V accumulators rescaled between chunks), and the V staging holds one chunk.  Without it the one
    // chunk is the whole prefix (at most 128 positions).
    constexpr int KPL = 4;               // keys per lane -> 128 cached positions per chunk
    constexpr int CH = DK / 8;           // 16-byte chunks per K / V row
    extern __shared__ uint4 sv_raw[];    // [warps][keys_pad][CH x 16 B]  V rows (bf16)
    const int n = blockIdx.x;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int nw = blockDim.x >> 5;
    const int d = H * DK;
    const int step = ROW_POS ? step_ptr[n] : *step_ptr;            // ROW_POS: step_ptr holds the row positions
    const int nkeys = step + 1;
    const int* an = ROW_POS ? anc + (size_t)n * Lmax : anc + ((size_t)(step & 1) * N + n) * Lmax;
    if (ROW_POS && step < 0) {
        for (int i = threadIdx.x; i < d / 2; i += blockDim.x) reinterpret_cast<uint32_t*>(out + (size_t)n * d)[i] = 0u;
        return;
    }
    uint4* sv = sv_raw + (size_t)wib * keys_pad * CH;    // [keys_pad][CH x 16 B] per warp
    // q lives in shared memory (every lane needs all DK dims: 64 registers per thread otherwise, which capped the kernel
    // at 3 resident CTAs per SM -- the SM-time of this latency-bound kernel is what concurrent batches compete for)
    float* sq = reinterpret_cast<float*>(sv_raw + (size_t)(blockDim.x >> 5) * keys_pad * CH) + wib * DK;
    for (int h = wib; h < H; h += nw) {
        const bf16* base = qkv + (size_t)n * 3 * d + h * DK;
        // append the newest K/V to the cache (lane owns dims 2*lane, 2*lane+1; at DK 96 lanes 0..15 also own 64+2*lane, +1)
        const uint32_t kcur = *reinterpret_cast<const uint32_t*>(base + d + 2 * lane);
        const uint32_t vcur = *reinterpret_cast<const uint32_t*>(base + 2 * d + 2 * lane);
        const size_t cur_off = (ROW_POS ? (size_t)an[step] * d : ((size_t)step * N + n) * d) + h * DK + 2 * lane;
        *reinterpret_cast<uint32_t*>(kc + cur_off) = kcur;
        *reinterpret_cast<uint32_t*>(vc + cur_off) = vcur;
        if (DK == 96 && lane < 16) {
            *reinterpret_cast<uint32_t*>(kc + cur_off + 64) = *reinterpret_cast<const uint32_t*>(base + d + 64 + 2 * lane);
            *reinterpret_cast<uint32_t*>(vc + cur_off + 64) = *reinterpret_cast<const uint32_t*>(base + 2 * d + 64 + 2 * lane);
        }
        {
            const float2 qq = unpack_bf16(*reinterpret_cast<const uint32_t*>(base + 2 * lane));
            float2 qh = make_float2(0.f, 0.f);
            if (DK == 96 && lane < 16) qh = unpack_bf16(*reinterpret_cast<const uint32_t*>(base + 64 + 2 * lane));
            __syncwarp();
            sq[2 * lane] = qq.x;
            sq[2 * lane + 1] = qq.y;
            if (DK == 96 && lane < 16) {
                sq[64 + 2 * lane] = qh.x;
                sq[64 + 2 * lane + 1] = qh.y;
            }
            __syncwarp();
        }
        float mx = -INFINITY, l = 0.f;
        // P.V accumulators: at DK 64 lane owns output dims 2*lane, 2*lane+1 (acc[0..1]); at DK 96 lanes 0..23 own
        // 4*lane .. 4*lane+3 (acc[0..3])
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        const int c_end = CHUNKED ? nkeys : 1;
        for (int c0 = 0; c0 < c_end; c0 += 32 * KPL) {
            int slot[KPL];
#pragma unroll
            for (int j = 0; j < KPL; ++j) {
                const int s = c0 + lane + 32 * j;
                slot[j] = (s < step) ? an[s] : n;
            }
            float sc[KPL];
            float cmx = -INFINITY;
#pragma unroll
            for (int j = 0; j < KPL; ++j) {
                const int s = c0 + lane + 32 * j, sl = lane + 32 * j;   // position in the prefix / in the chunk
                sc[j] = -INFINITY;
                if (s < nkeys) {   // warp-divergent only in the last group
                    const size_t crow = ROW_POS ? (size_t)slot[j] : (size_t)s * N + slot[j];
                    const bf16* krow = (s == step) ? base + d : kc + crow * d + h * DK;
                    const bf16* vrow = (s == step) ? base + 2 * d : vc + crow * d + h * DK;
                    uint4 ku[CH], vu[CH];
#pragma unroll
                    for (int i = 0; i < CH; ++i) ku[i] = *reinterpret_cast<const uint4*>(krow + 8 * i);
#pragma unroll
                    for (int i = 0; i < CH; ++i) vu[i] = *reinterpret_cast<const uint4*>(vrow + 8 * i);
                    float dot = 0.f;
#pragma unroll
                    for (int i = 0; i < CH; ++i) {
                        const float2 a = unpack_bf16(ku[i].x), b = unpack_bf16(ku[i].y), c = unpack_bf16(ku[i].z),
                                     e = unpack_bf16(ku[i].w);
                        const float4 q0 = *reinterpret_cast<const float4*>(sq + 8 * i);      // broadcast reads
                        const float4 q1 = *reinterpret_cast<const float4*>(sq + 8 * i + 4);
                        dot += q0.x * a.x + q0.y * a.y + q0.z * b.x + q0.w * b.y + q1.x * c.x + q1.y * c.y + q1.z * e.x + q1.w * e.y;
                    }
                    sc[j] = dot * scale;
                    cmx = fmaxf(cmx, sc[j]);
#pragma unroll
                    for (int i = 0; i < CH; ++i) sv[sl * CH + rot_chunk<CH>(i + sl)] = vu[i];   // rotate chunks: conflict-free rows
                }
            }
            cmx = warp_max(cmx);
            float corr = 0.f;   // rescales the previous chunks' sum and accumulators to the new running max
            if constexpr (CHUNKED) {
                const float m = fmaxf(mx, cmx);
                corr = __expf(mx - m);
                mx = m;
            } else {
                mx = cmx;
            }
            float cl = 0.f;
#pragma unroll
            for (int j = 0; j < KPL; ++j) {
                sc[j] = (c0 + lane + 32 * j < nkeys) ? __expf(sc[j] - mx) : 0.f;
                cl += sc[j];
            }
            cl = warp_sum(cl);
            if constexpr (CHUNKED) {
                l = l * corr + cl;
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[i] *= corr;
            } else {
                l = cl;
            }
            __syncwarp();
            if constexpr (DK == 64) {
                // P.V as a column sum over the staged V rows
                const uint32_t* svw = reinterpret_cast<const uint32_t*>(sv);
#pragma unroll
                for (int j = 0; j < KPL; ++j) {
                    const int cnt = min(32, nkeys - c0 - 32 * j);
                    if (cnt <= 0) break;   // warp-uniform
#pragma unroll 4
                    for (int t = 0; t < cnt; ++t) {
                        const int s = t + 32 * j;
                        const float pw = __shfl_sync(0xffffffffu, sc[j], t);
                        // dims 2*lane.. live in 16-byte chunk (lane >> 2), word (lane & 3); chunks were rotated by s
                        const uint32_t vv = svw[(s * 8 + (((lane >> 2) + s) & 7)) * 4 + (lane & 3)];
                        const float2 vf = unpack_bf16(vv);
                        acc[0] = fmaf(pw, vf.x, acc[0]);
                        acc[1] = fmaf(pw, vf.y, acc[1]);
                    }
                }
            } else {
                // P.V as a column sum: 8-byte half (lane & 1) of 16-byte chunk (lane >> 1); lanes 24..31 repeat lane 23's
                // reads and store nothing
                const uint2* svh = reinterpret_cast<const uint2*>(sv);
                const int ln = min(lane, 23);
#pragma unroll
                for (int j = 0; j < KPL; ++j) {
                    const int cnt = min(32, nkeys - c0 - 32 * j);
                    if (cnt <= 0) break;   // warp-uniform
#pragma unroll 4
                    for (int t = 0; t < cnt; ++t) {
                        const int s = t + 32 * j;
                        const float pw = __shfl_sync(0xffffffffu, sc[j], t);
                        const uint2 vv = svh[(s * CH + rot_chunk<CH>((ln >> 1) + s)) * 2 + (ln & 1)];
                        const float2 v01 = unpack_bf16(vv.x), v23 = unpack_bf16(vv.y);
                        acc[0] = fmaf(pw, v01.x, acc[0]);
                        acc[1] = fmaf(pw, v01.y, acc[1]);
                        acc[2] = fmaf(pw, v23.x, acc[2]);
                        acc[3] = fmaf(pw, v23.y, acc[3]);
                    }
                }
            }
            if constexpr (CHUNKED) __syncwarp();   // the next chunk overwrites the staged V rows
        }
        const float inv = 1.0f / l;
        if constexpr (DK == 64) {
            *reinterpret_cast<uint32_t*>(out + (size_t)n * d + h * 64 + 2 * lane) = pack_bf16(acc[0] * inv, acc[1] * inv);
        } else {
            if (lane < 24)
                *reinterpret_cast<uint2*>(out + (size_t)n * d + h * DK + 4 * lane) =
                    make_uint2(pack_bf16(acc[0] * inv, acc[1] * inv), pack_bf16(acc[2] * inv, acc[3] * inv));
        }
        __syncwarp();
    }
}

template <int DK, bool ROW_POS>
static const char* decode_self_attn_launch_dk(cudaStream_t st, const bf16* qkv, bf16* kc, bf16* vc, const int* anc,
                                              const int* step_ptr, bf16* out, int N, int H, int Lmax, const int* row_pos) {
    const int warps = H < 4 ? H : 4;
    // V staging sized by the longest prefix this search can reach, up to one 128-key chunk: at max_len 60 this halves the
    // shared memory per CTA and doubles the resident CTAs of this latency-bound kernel (less SM-time per decode step)
    const bool chunked = Lmax > 128;
    const int keys_pad = chunked ? 128 : (Lmax + 31) / 32 * 32;
    const size_t smem = (size_t)warps * keys_pad * DK * 2 + (size_t)warps * DK * sizeof(float);   // V rows | q per warp
    const float scale = DK == 64 ? 0.125f : 1.0f / sqrtf((float)DK);
    const int* pos = ROW_POS ? row_pos : step_ptr;         // the kernel reads the row positions through step_ptr
    if (chunked)
        return launch<decode_self_attn_kernel<DK, true, ROW_POS>>(dim3(N), dim3(warps * 32), smem, st, qkv, kc, vc, anc, pos, out,
                                                                  N, H, Lmax, scale, keys_pad);
    return launch<decode_self_attn_kernel<DK, false, ROW_POS>>(dim3(N), dim3(warps * 32), smem, st, qkv, kc, vc, anc, pos, out,
                                                               N, H, Lmax, scale, keys_pad);
}

const char* decode_self_attn_launch(cudaStream_t st, const bf16* qkv, bf16* kc, bf16* vc, const int* anc,
                                    const int* step_ptr, bf16* out, int N, int H, int Lmax, int d_k, const int* row_pos) {
    if (Lmax > 1023) return "decode_self_attn: at most 1023 cached positions (max_len <= 1023)";
    if (row_pos) {
        if (d_k == 64) return decode_self_attn_launch_dk<64, true>(st, qkv, kc, vc, anc, step_ptr, out, N, H, Lmax, row_pos);
        if (d_k == 96) return decode_self_attn_launch_dk<96, true>(st, qkv, kc, vc, anc, step_ptr, out, N, H, Lmax, row_pos);
    } else {
        if (d_k == 64) return decode_self_attn_launch_dk<64, false>(st, qkv, kc, vc, anc, step_ptr, out, N, H, Lmax, row_pos);
        if (d_k == 96) return decode_self_attn_launch_dk<96, false>(st, qkv, kc, vc, anc, step_ptr, out, N, H, Lmax, row_pos);
    }
    return "decode_self_attn: head width d_k must be 64 or 96";
}

// ------------------------------------------------------------------------------------------------
// Stand-alone PositionalEncoding.forward: out = x * alpha + table[row % period]   (module/pos.py:56)
// (the fused path does this in the front-end Linear's epilogue; this kernel serves the module-level
// drop-in API where frontend and encoder are called separately).  x f32 or bf16 -> bf16.  alpha_dev (optional): alpha is
// multiplied by this device scalar (a loss-gradient scale known only on the device, e.g. MixSpeech's lambda / accum_steps).
// ------------------------------------------------------------------------------------------------
__global__ void scale_add_table_kernel(const void* __restrict__ x, int ldx, int x_f32, bf16* __restrict__ out, int ldo,
                                       float alpha, const float* __restrict__ table, int period, int M, int N,
                                       const float* __restrict__ alpha_dev) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int row = (int)(i / N), col = (int)(i % N);
    if (row >= M) return;
    const float v = x_f32 ? reinterpret_cast<const float*>(x)[(size_t)row * ldx + col]
                          : __bfloat162float(reinterpret_cast<const bf16*>(x)[(size_t)row * ldx + col]);
    const float t = table ? table[(size_t)(row % period) * N + col] : 0.f;
    const float a = alpha_dev ? alpha * *alpha_dev : alpha;
    out[(size_t)row * ldo + col] = __float2bfloat16(v * a + t);
}

const char* scale_add_table_launch(cudaStream_t st, const void* x, int ldx, int x_f32, bf16* out, int ldo, float alpha,
                                   const float* table, int period, int M, int N, const float* alpha_dev) {
    const size_t n = (size_t)M * N;
    return launch<scale_add_table_kernel>(dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, x, ldx, x_f32, out, ldo, alpha,
                                          table, period, M, N, alpha_dev);
}

// ------------------------------------------------------------------------------------------------
// Conformer convolution-module middle: depthwise Conv1d over time (k taps, zero padding (k-1)/2) +
// eval-mode BatchNorm (folded into w/b by the caller) + swish.   otrans/module/conformer.py:48-52
// x, out bf16 [B*T, d].  HBM-bound: thread = (row, 8 channels), 16-byte loads of the k neighbour rows
// (re-reads hit L1/L2), fp32 math.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) dwconv_swish_kernel(const bf16* __restrict__ x, const float* __restrict__ w,
                                                           const float* __restrict__ b, bf16* __restrict__ out, int B,
                                                           int T, int d, int k) {
    const int cg = d / 8;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)B * T * cg) return;
    const int c0 = (int)(i % cg) * 8;
    const int row = (int)(i / cg);
    const int t = row % T;
    const int pad = (k - 1) / 2;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = b[c0 + j];
    for (int tap = 0; tap < k; ++tap) {
        const int tt = t + tap - pad;
        if (tt < 0 || tt >= T) continue;
        const uint4 u = *reinterpret_cast<const uint4*>(x + (size_t)(row + tap - pad) * d + c0);
        const float2 a = unpack_bf16(u.x), bb = unpack_bf16(u.y), c = unpack_bf16(u.z), e = unpack_bf16(u.w);
        const float xv[8] = {a.x, a.y, bb.x, bb.y, c.x, c.y, e.x, e.y};
        const float4 w0 = *reinterpret_cast<const float4*>(w + (size_t)tap * d + c0);
        const float4 w1 = *reinterpret_cast<const float4*>(w + (size_t)tap * d + c0 + 4);
        const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(xv[j], wv[j], acc[j]);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = acc[j] * __fdividef(1.0f, 1.0f + __expf(-acc[j]));
    uint4 o;
    o.x = pack_bf16(acc[0], acc[1]);
    o.y = pack_bf16(acc[2], acc[3]);
    o.z = pack_bf16(acc[4], acc[5]);
    o.w = pack_bf16(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(out + (size_t)row * d + c0) = o;
}

const char* dwconv_swish_launch(cudaStream_t st, const bf16* x, const float* w, const float* b, bf16* out, int B, int T,
                                int d, int k) {
    if (d % 8 || !(k & 1)) return "dwconv: d must be a multiple of 8 and k odd";
    const size_t n = (size_t)B * T * (d / 8);
    return launch<dwconv_swish_kernel>(dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, x, w, b, out, B, T, d, k);
}

}  // namespace otb
