// Pruned RNN-T (DESIGN.md 4.22): the simple joint, its backward, and the prune ranges.  The simple joint's logits at node
// (b, t, u) are am[b T + t] + lm[b U1 + u] (am = simple_am_proj(memory) f32 [B T, lda], lm = simple_lm_proj(g) f32
// [B U1, ldl]); its normalizer factors through one [T, V] x [V, U1] product per utterance:
//   Z[t,u] = m_t + m_u + log sum_v exp(am[t,v] - m_t) exp(lm[u,v] - m_u),   m_t = max_v am[t,v], m_u = max_v lm[u,v].
//   rnnt_simple_lse_kernel   one CTA per (utterance, 32 frames, 32 label positions): the row maxima of its 64 rows, then
//                            the product over V in chunks of 32 columns through shared memory, fp32 accumulation -> the
//                            node log-probs in rnnt_logprob's layout [lse, log p(blank), log p(y_{u+1})] and m_t, m_u.
//   rnnt_simple_bwd_kernel   one CTA per (utterance, 32 rows of am or of lm, 64 columns): with w = scale (a + c) and
//                            P[t,u] = w exp(m_t + m_u - Z[t,u]),
//                              d am[t,v] = D[t,v] - exp(am[t,v] - m_t) sum_u P[t,u] exp(lm[u,v] - m_u)
//                              d lm[u,v] = D[u,v] - exp(lm[u,v] - m_u) sum_t P[t,u] exp(am[t,v] - m_t)
//                            with D the one-hot part (scale a at column 0, scale c at column y_{u+1}), summed by one thread
//                            per row in ascending order (no atomics); bf16 out, columns >= V zero.  A node whose
//                            factorized sum left the normal fp32 range (SJ_ACC_MIN) has Z from the logits directly,
//                            and the backward subtracts its term w exp(am[t,v] + lm[u,v] - Z) on its own.
//   rnnt_prune_ranges_kernel one CTA per utterance: the window of S label positions with the largest occupancy at every
//                            frame, then the range rule of DESIGN.md 4.22.
#include <math.h>

#include "launch.cuh"
#include "otb_internal.h"

namespace otb {

static constexpr int SJ_ROWS = 32;        // frames and label positions per CTA of the normalizer; rows of the backward
static constexpr int SJ_K = 32;           // reduction chunk (columns of V in the forward, rows in the backward)
static constexpr int SJ_COLS = 64;        // columns of V per CTA of the backward
static constexpr int SJ_THREADS = 256;
static constexpr int PRUNE_THREADS = 256;
// The factorized sum acc = sum_v exp(am[t,v] - m_t) exp(lm[u,v] - m_u) is exact to a few ulps only while its terms are
// normal numbers.  A term below 2^-126 (subnormal factor or product) carries an absolute error up to 2^-149, so the V
// terms together up to V 2^-149; against acc >= 2^-100 that is below V 2^-49, under one f32 ulp for any V < 2^25.  A
// node with acc < 2^-100 (every logit sum at least 69.3 below m_t + m_u; 0 or -inf when it is above 87 or 103) takes
// Z from the logits directly instead.  The backward recognizes those nodes by m_t + m_u - Z > 100 ln 2 and adds their
// exact term, so the factorized product never scales a node by exp(m_t + m_u - Z) > 2^100.
static constexpr float SJ_ACC_MIN = 0x1p-100f;
static constexpr float SJ_GAP_MAX = 69.3147181f;     // 100 ln 2

// Z = max_v (am[v] + lm[v]) + log sum_v exp(am[v] + lm[v] - max), one thread, ascending v in fp32
__device__ __forceinline__ float simple_lse_direct(const float* xa, const float* xl, int V) {
    float m = -INFINITY;
    for (int v = 0; v < V; ++v) m = fmaxf(m, xa[v] + xl[v]);
    float s = 0.f;
    for (int v = 0; v < V; ++v) s += expf((xa[v] + xl[v]) - m);
    return m + logf(s);
}

__device__ __forceinline__ int simple_label(const int* labels, int ldy, int b, int u, int Ub, int V) {
    if (u >= Ub) return -1;
    const int y = labels[(size_t)b * ldy + u];
    return (y < 1 || y >= V) ? -1 : y;
}

__global__ void __launch_bounds__(SJ_THREADS) rnnt_simple_lse_kernel(const float* __restrict__ am, int lda, const float* __restrict__ lm,
                                                                      int ldl, int V, int T, int U1, const int* __restrict__ t_len,
                                                                      const int* __restrict__ u_len, const int* __restrict__ labels,
                                                                      int ldy, float* __restrict__ lp, float* __restrict__ m_am,
                                                                      float* __restrict__ m_lm) {
    __shared__ float ea[SJ_K][SJ_ROWS + 1];      // exp(am - m_t), [v][t]
    __shared__ float el[SJ_K][SJ_ROWS + 1];      // exp(lm - m_u), [v][u]
    __shared__ float mx[2 * SJ_ROWS];            // m_t of the 32 frames, then m_u of the 32 positions
    const int b = blockIdx.z, t0 = blockIdx.y * SJ_ROWS, u0 = blockIdx.x * SJ_ROWS;
    const int Tb = min(t_len[b], T), Ub = min(u_len[b], U1 - 1);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // row r < 32: am row t0 + r; r >= 32: lm row u0 + r - 32; a row outside the lattice is dead (max 0, operands 0)
    const auto row_ptr = [&](int r) -> const float* {
        if (r < SJ_ROWS) return t0 + r < Tb ? am + ((size_t)b * T + t0 + r) * lda : nullptr;
        return u0 + r - SJ_ROWS <= Ub && Tb > 0 ? lm + ((size_t)b * U1 + u0 + r - SJ_ROWS) * ldl : nullptr;
    };
    for (int r = warp; r < 2 * SJ_ROWS; r += SJ_THREADS / 32) {
        const float* x = row_ptr(r);
        float m = -INFINITY;
        if (x)
            for (int v = lane; v < V; v += 32) m = fmaxf(m, x[v]);
#pragma unroll
        for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0) mx[r] = x ? m : 0.f;
    }
    __syncthreads();
    const int ti = threadIdx.x / 8, uj = threadIdx.x % 8;      // frame t0 + ti, positions u0 + uj + 8 q
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int v0 = 0; v0 < V; v0 += SJ_K) {
        for (int e = threadIdx.x; e < 2 * SJ_ROWS * SJ_K; e += SJ_THREADS) {
            const int r = e / SJ_K, v = e % SJ_K;
            const float* x = row_ptr(r);
            const float val = (x && v0 + v < V) ? expf(x[v0 + v] - mx[r]) : 0.f;
            if (r < SJ_ROWS) ea[v][r] = val;
            else el[v][r - SJ_ROWS] = val;
        }
        __syncthreads();
#pragma unroll 8
        for (int v = 0; v < SJ_K; ++v) {
            const float a = ea[v][ti];
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[q] = fmaf(a, el[v][uj + 8 * q], acc[q]);
        }
        __syncthreads();
    }
    if (blockIdx.x == 0 && uj == 0 && t0 + ti < T) m_am[(size_t)b * T + t0 + ti] = mx[ti];
    if (blockIdx.y == 0 && uj == 0 && u0 + ti < U1) m_lm[(size_t)b * U1 + u0 + ti] = mx[SJ_ROWS + ti];
    const int t = t0 + ti;
    if (t >= T) return;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int u = u0 + uj + 8 * q;
        if (u >= U1) continue;
        float* o = lp + (((size_t)b * T + t) * U1 + u) * 3;
        if (t >= Tb || u > Ub) {
            o[0] = o[1] = o[2] = 0.f;
            continue;
        }
        const float* xa = am + ((size_t)b * T + t) * lda;
        const float* xl = lm + ((size_t)b * U1 + u) * ldl;
        const float z = acc[q] < SJ_ACC_MIN ? simple_lse_direct(xa, xl, V) : mx[ti] + mx[SJ_ROWS + uj + 8 * q] + logf(acc[q]);
        const int y = simple_label(labels, ldy, b, u, Ub, V);
        o[0] = z;
        o[1] = (xa[0] + xl[0]) - z;
        o[2] = y < 0 ? -INFINITY : (xa[y] + xl[y]) - z;
    }
}

// grid (column tiles, am row tiles + lm row tiles, B).  side 0: rows t of am, reduction over u; side 1: rows u of lm,
// reduction over t.  grad f32 [B T U1, 2] (otb_rnnt_loss over the simple joint's lp), scale = scale (* *scale_dev).
__global__ void __launch_bounds__(SJ_THREADS) rnnt_simple_bwd_kernel(const float* __restrict__ am, int lda, const float* __restrict__ lm,
                                                                      int ldl, int V, int T, int U1, const int* __restrict__ t_len,
                                                                      const int* __restrict__ u_len, const int* __restrict__ labels,
                                                                      int ldy, const float* __restrict__ lp,
                                                                      const float* __restrict__ m_am, const float* __restrict__ m_lm,
                                                                      const float* __restrict__ grad, float scale,
                                                                      const float* __restrict__ scale_dev, bf16* __restrict__ d_am,
                                                                      bf16* __restrict__ d_lm, int ldd) {
    __shared__ float ps[SJ_ROWS][SJ_K + 1];          // P of the CTA's rows against the chunk's reduction rows
    __shared__ float ey[SJ_K][SJ_COLS + 1];          // exp(other - m) of the chunk's reduction rows
    __shared__ float dsum[SJ_ROWS][SJ_COLS + 1];     // the one-hot part D
    __shared__ float pw[SJ_ROWS][SJ_K + 1];          // w of the nodes whose Z the forward took directly, else 0
    __shared__ int s_exact;                          // some such node with w != 0 seen so far
    const int b = blockIdx.z, v0 = blockIdx.x * SJ_COLS;
    const int n_am = (T + SJ_ROWS - 1) / SJ_ROWS;
    const bool side_am = (int)blockIdx.y < n_am;
    const int r0 = (side_am ? (int)blockIdx.y : (int)blockIdx.y - n_am) * SJ_ROWS;
    const int Tb = min(t_len[b], T), Ub = min(u_len[b], U1 - 1);
    const int n_own = side_am ? Tb : (Tb > 0 ? Ub + 1 : 0);      // live rows of this side
    const int n_red = side_am ? (Tb > 0 ? Ub + 1 : 0) : Tb;      // live rows of the other side
    const float sc = scale_dev ? scale * *scale_dev : scale;
    // node (t, u) of own row i, reduction row j
    const auto node = [&](int i, int j) -> size_t {
        const int t = side_am ? i : j, u = side_am ? j : i;
        return ((size_t)b * T + t) * U1 + u;
    };
    const float* own = side_am ? am : lm;
    const float* oth = side_am ? lm : am;
    const int ld_own = side_am ? lda : ldl, ld_oth = side_am ? ldl : lda;
    const size_t own0 = (size_t)b * (side_am ? T : U1), oth0 = (size_t)b * (side_am ? U1 : T);
    const float* m_own = side_am ? m_am : m_lm;
    const float* m_oth = side_am ? m_lm : m_am;

    const int ri = threadIdx.x / 8, cj = threadIdx.x % 8;       // own row r0 + ri, columns v0 + cj + 8 q
    const float* x = own + (own0 + r0 + ri) * ld_own;
    float acc[8], exact[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q] = exact[q] = 0.f;
    if (threadIdx.x == 0) s_exact = 0;
    __syncthreads();
    for (int j0 = 0; j0 < n_red; j0 += SJ_K) {
        for (int e = threadIdx.x; e < SJ_ROWS * SJ_K; e += SJ_THREADS) {
            const int i = e / SJ_K, j = e % SJ_K;
            float p = 0.f, pe = 0.f;
            if (r0 + i < n_own && j0 + j < n_red) {
                const size_t k = node(r0 + i, j0 + j);
                const float w = sc * (grad[2 * k] + grad[2 * k + 1]);
                const float gap = m_own[own0 + r0 + i] + m_oth[oth0 + j0 + j] - lp[3 * k];
                if (gap > SJ_GAP_MAX) {         // Z came from the logits directly (forward): the node's own term below
                    pe = w;
                    if (w != 0.f) s_exact = 1;
                } else {
                    p = w * expf(gap);
                }
            }
            ps[i][j] = p;
            pw[i][j] = pe;
        }
        for (int e = threadIdx.x; e < SJ_K * SJ_COLS; e += SJ_THREADS) {
            const int j = e / SJ_COLS, v = e % SJ_COLS;
            float x = 0.f;
            if (j0 + j < n_red && v0 + v < V) x = expf(oth[(oth0 + j0 + j) * ld_oth + v0 + v] - m_oth[oth0 + j0 + j]);
            ey[j][v] = x;
        }
        __syncthreads();
#pragma unroll 4
        for (int j = 0; j < SJ_K; ++j) {
            const float p = ps[ri][j];
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] = fmaf(p, ey[j][cj + 8 * q], acc[q]);
        }
        if (s_exact) {      // w exp(own + other - Z) of the nodes left out of ps, ascending j
            for (int j = 0; j < SJ_K; ++j) {
                const float pe = pw[ri][j];
                if (pe == 0.f) continue;
                const float z = lp[3 * node(r0 + ri, j0 + j)];
                const float* y = oth + (oth0 + j0 + j) * ld_oth;
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int v = v0 + cj + 8 * q;
                    if (v < V) exact[q] += pe * expf((x[v] + y[v]) - z);
                }
            }
        }
        __syncthreads();
    }
    // the one-hot part: thread i < 32 owns row r0 + i and adds its terms in ascending order of the reduction index
    for (int e = threadIdx.x; e < SJ_ROWS * SJ_COLS; e += SJ_THREADS) dsum[e / SJ_COLS][e % SJ_COLS] = 0.f;
    __syncthreads();
    if (threadIdx.x < SJ_ROWS && r0 + (int)threadIdx.x < n_own) {
        const int i = r0 + threadIdx.x;
        if (side_am) {
            for (int u = 0; u <= Ub; ++u) {
                const size_t k = node(i, u);
                const int y = simple_label(labels, ldy, b, u, Ub, V);
                if (v0 == 0) dsum[threadIdx.x][0] += sc * grad[2 * k];
                if (y >= v0 && y < v0 + SJ_COLS) dsum[threadIdx.x][y - v0] += sc * grad[2 * k + 1];
            }
        } else {
            const int y = simple_label(labels, ldy, b, i, Ub, V);
            const bool has_y = y >= v0 && y < v0 + SJ_COLS;
            if (v0 == 0 || has_y) {
                float sa = 0.f, sy = 0.f;
                for (int t = 0; t < Tb; ++t) {
                    const size_t k = node(i, t);
                    sa += sc * grad[2 * k];
                    sy += sc * grad[2 * k + 1];
                }
                if (v0 == 0) dsum[threadIdx.x][0] += sa;
                if (has_y) dsum[threadIdx.x][y - v0] += sy;
            }
        }
    }
    __syncthreads();
    const int i = r0 + ri;
    if (i >= (side_am ? T : U1)) return;
    bf16* out = (side_am ? d_am : d_lm) + (own0 + i) * ldd;
    const bool live = i < n_own, with_exact = s_exact;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const int v = v0 + cj + 8 * q;
        if (v >= ldd) continue;
        float d = 0.f;
        if (live && v < V) d = dsum[ri][cj + 8 * q] - expf(x[v] - m_own[own0 + i]) * acc[q];
        if (with_exact) d -= exact[q];
        out[v] = __float2bfloat16_rn(d);
    }
}

// One CTA per utterance.  occupancy(t, u) = -(g_blank + g_label) of the simple loss's node gradients (f32); the window at
// frame t starting at s sums occupancy(t, s .. s + S - 1) in ascending u in f32; s_t = the arg-max over s in [0, s_max],
// s_max = max(0, U_b + 1 - S), the lowest s on a tie.  Then, in order: s_0 = 0; for t ascending s_t = min(max(s_t,
// s_{t-1}), s_{t-1} + S - 1); s_t = min(s_t, s_max); for t descending from T_b - 1 with lo = U_b - S + 1: s_t = max(s_t,
// lo), lo = s_t - (S - 1).  Frames t >= T_b get 0.
__global__ void __launch_bounds__(PRUNE_THREADS) rnnt_prune_ranges_kernel(const float* __restrict__ grad, int T, int U1,
                                                                          const int* __restrict__ t_len, const int* __restrict__ u_len,
                                                                          int S, int* __restrict__ s_begin) {
    const int b = blockIdx.x;
    const int Tb = max(0, min(t_len[b], T)), Ub = min(u_len[b], U1 - 1);
    const int s_max = max(0, Ub + 1 - S);
    int* sb = s_begin + (size_t)b * T;
    for (int t = threadIdx.x; t < T; t += PRUNE_THREADS) {
        int best_s = 0;
        if (t < Tb) {
            const float* g = grad + ((size_t)b * T + t) * U1 * 2;
            float best = -INFINITY;
            for (int s = 0; s <= s_max; ++s) {
                float w = 0.f;
                for (int u = s; u < s + S && u <= Ub; ++u) w += -(g[2 * u] + g[2 * u + 1]);
                if (w > best) {
                    best = w;
                    best_s = s;
                }
            }
        }
        sb[t] = best_s;
    }
    __syncthreads();
    if (threadIdx.x != 0 || Tb < 1) return;
    sb[0] = 0;
    for (int t = 1; t < Tb; ++t) sb[t] = min(max(sb[t], sb[t - 1]), sb[t - 1] + S - 1);
    for (int t = 0; t < Tb; ++t) sb[t] = min(sb[t], s_max);
    int lo = Ub - S + 1;
    for (int t = Tb - 1; t >= 0; --t) {
        sb[t] = max(sb[t], lo);
        lo = sb[t] - (S - 1);
    }
}

static const char* simple_check(int lda, int ldl, int V, int B, int T, int U1, int ldy) {
    if (B < 1 || T < 1 || U1 < 1) return "empty lattice";
    if (U1 > 1024) return "transcripts of at most 1023 labels";
    if (V < 2 || lda < V || ldl < V) return "need V >= 2 and row strides >= V";
    if (ldy < U1 - 1) return "labels narrower than the lattice";
    return nullptr;
}

const char* rnnt_simple_lse_launch(cudaStream_t st, const float* am, int lda, const float* lm, int ldl, int V, int B, int T, int U1,
                                   const int* t_len, const int* u_len, const int* labels, int ldy, float* lp, float* m_am,
                                   float* m_lm) {
    if (const char* e = simple_check(lda, ldl, V, B, T, U1, ldy)) return e;
    const dim3 grid((U1 + SJ_ROWS - 1) / SJ_ROWS, (T + SJ_ROWS - 1) / SJ_ROWS, B);
    return launch<rnnt_simple_lse_kernel>(grid, SJ_THREADS, 0, st, am, lda, lm, ldl, V, T, U1, t_len, u_len, labels, ldy, lp, m_am,
                                          m_lm);
}

const char* rnnt_simple_bwd_launch(cudaStream_t st, const float* am, int lda, const float* lm, int ldl, int V, int B, int T, int U1,
                                   const int* t_len, const int* u_len, const int* labels, int ldy, const float* lp, const float* m_am,
                                   const float* m_lm, const float* grad, float scale, const float* scale_dev, bf16* d_am,
                                   bf16* d_lm, int ldd) {
    if (const char* e = simple_check(lda, ldl, V, B, T, U1, ldy)) return e;
    if (ldd < V) return "gradient rows narrower than V";
    const dim3 grid((ldd + SJ_COLS - 1) / SJ_COLS, (T + SJ_ROWS - 1) / SJ_ROWS + (U1 + SJ_ROWS - 1) / SJ_ROWS, B);
    return launch<rnnt_simple_bwd_kernel>(grid, SJ_THREADS, 0, st, am, lda, lm, ldl, V, T, U1, t_len, u_len, labels, ldy, lp, m_am,
                                          m_lm, grad, scale, scale_dev, d_am, d_lm, ldd);
}

const char* rnnt_prune_ranges_launch(cudaStream_t st, const float* grad, int B, int T, int U1, const int* t_len, const int* u_len,
                                     int S, int* s_begin) {
    if (B < 1 || T < 1 || U1 < 1) return "empty lattice";
    if (S < 2 || S > 1024) return "the band width S must be in [2, 1024]";
    return launch<rnnt_prune_ranges_kernel>(B, PRUNE_THREADS, 0, st, grad, T, U1, t_len, u_len, S, s_begin);
}

}  // namespace otb
