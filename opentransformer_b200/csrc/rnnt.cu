// Transducer (RNN-T) joint network and loss (DESIGN.md 4.22).  The lattice of utterance b has the nodes (t, u),
// t < T_b frames and u <= U_b emitted labels, stored padded as [B, T, U1] with u fastest (U1 = U_max + 1); every kernel
// skips the nodes past T_b or U_b and writes zeros for them.  Blank is token 0.
// Pruned lattice (s_begin non-null, pruned RNN-T): frame t keeps the S label positions u = s_begin[b T + t] + k, k < S,
// stored [B, T, S] with k fastest; a node outside every frame's band does not exist.  A null s_begin is the full lattice.
//   rnnt_joint_kernel      Hj[b,t,u] = tanh(Ep[b,t] + Pp[b,u]), bf16 in and out, 8 columns per thread.
//   rnnt_joint_bwd_kernel  dZ = dHj (1 - Hj^2), summed over u into dEp[b,t] and over t into dPp[b,u]: one CTA per output
//                          row, each column summed by one thread in ascending order (no atomics: repeated runs are
//                          bit-identical, eager or captured).
//   rnnt_logprob_kernel    one warp per fp32 logits row (otb_token_logprob's row reduction, row_lse.cuh) -> [lse,
//                          log p(blank), log p(y_{u+1})], the last -inf at u = U_b.
//   rnnt_loss_kernel       one CTA per utterance, thread u: alpha over the anti-diagonals t + u ascending (stored), then
//                          beta descending (kept in shared memory only) and, at each node, the gradient of the loss with
//                          respect to its two log-probs.  log-space in fp64: over 1023 labels alpha reaches thousands in
//                          magnitude, where an fp32 ulp would already be a 1e-4 relative error of exp(alpha + beta - log P).
//   rnnt_dlogits_kernel    one warp per recomputed logits row: dz_k = [k = 0] a + [k = y] c - p_k (a + c), bf16.
//   The pruned loss's simple joint and its prune ranges are in rnnt_pruned.cu.
//   rnnt_greedy_step_kernel  one CTA per utterance: the decision of one step of greedy search, and the copy of the
//                          predictor state forward for the rows that emitted.
#include <math.h>

#include "launch.cuh"
#include "otb_internal.h"
#include "row_lse.cuh"

namespace otb {

static constexpr int RNNT_MAX_U1 = 1024;      // U_b <= 1023 labels: one thread per u of the loss CTA
static constexpr int RNNT_WARPS = 8;          // rows per CTA of the per-row kernels
static constexpr int RNNT_BWD_THREADS = 128;

struct LatticeNode {
    int b, t, u;
    bool valid;
};

// Row width of the stored lattice: S label positions per frame when banded, else U1.
__device__ __forceinline__ int lattice_width(int U1, const int* s_begin, int S) { return s_begin ? S : U1; }

// node index -> (b, t, u), valid when t < T_b and u <= U_b (null length arrays: every node is valid); banded: the row
// (b, t) holds u = s_begin[b T + t] + k
__device__ __forceinline__ LatticeNode lattice_node(long long node, int T, int U1, const int* t_len, const int* u_len,
                                                    const int* s_begin, int S) {
    const int W = lattice_width(U1, s_begin, S);
    LatticeNode n;
    n.b = (int)(node / ((long long)T * W));
    const int rem = (int)(node - (long long)n.b * T * W);
    n.t = rem / W;
    n.u = rem - n.t * W + (s_begin ? s_begin[(size_t)n.b * T + n.t] : 0);
    n.valid = n.u < U1 && (!t_len || n.t < t_len[n.b]) && (!u_len || n.u <= u_len[n.b]);
    return n;
}

__device__ __forceinline__ double log_add(double a, double b) {
    const double m = fmax(a, b);
    if (m == -INFINITY) return m;
    return m + log1p(exp(-fabs(a - b)));
}

__global__ void __launch_bounds__(256) rnnt_joint_kernel(const bf16* __restrict__ ep, const bf16* __restrict__ pp, int D, int T,
                                                         int U1, const int* __restrict__ t_len, const int* __restrict__ u_len,
                                                         const int* __restrict__ s_begin, int S, bf16* __restrict__ out,
                                                         long long n_vec) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_vec) return;
    const int nv = D >> 3;
    const long long node = i / nv;
    const int c = (int)(i - node * nv) * 8;
    const LatticeNode n = lattice_node(node, T, U1, t_len, u_len, s_begin, S);
    uint4 r = make_uint4(0, 0, 0, 0);
    if (n.valid) {
        const uint4 e = *reinterpret_cast<const uint4*>(ep + ((size_t)n.b * T + n.t) * D + c);
        const uint4 p = *reinterpret_cast<const uint4*>(pp + ((size_t)n.b * U1 + n.u) * D + c);
        const __nv_bfloat162* e2 = reinterpret_cast<const __nv_bfloat162*>(&e);
        const __nv_bfloat162* p2 = reinterpret_cast<const __nv_bfloat162*>(&p);
        __nv_bfloat162* r2 = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 a = __bfloat1622float2(e2[j]), b = __bfloat1622float2(p2[j]);
            r2[j] = __floats2bfloat162_rn(tanhf(a.x + b.x), tanhf(a.y + b.y));
        }
    }
    *reinterpret_cast<uint4*>(out + node * D + c) = r;
}

// CTAs [0, B T): dEp row (b, t) = sum_{u <= U_b} dZ[b,t,u]; CTAs [B T, B T + B U1): dPp row (b, u) = sum_{t < T_b} dZ[b,t,u],
// both over the nodes that exist (banded: the frame's S positions; the frames whose band holds u), in ascending order
__global__ void __launch_bounds__(RNNT_BWD_THREADS) rnnt_joint_bwd_kernel(const bf16* __restrict__ dh, const bf16* __restrict__ h, int D,
                                                                          int B, int T, int U1, const int* __restrict__ t_len,
                                                                          const int* __restrict__ u_len, const int* __restrict__ s_begin,
                                                                          int S, bf16* __restrict__ dep, bf16* __restrict__ dpp) {
    const int row = blockIdx.x;
    const bool enc = row < B * T;
    const int r = enc ? row : row - B * T;
    const int b = enc ? r / T : r / U1, i = enc ? r % T : r % U1;
    const int Tb = min(t_len[b], T), Ub = min(u_len[b], U1 - 1);
    const int W = lattice_width(U1, s_begin, S);
    const int* sb = s_begin ? s_begin + (size_t)b * T : nullptr;
    const bool live = enc ? i < Tb : (i <= Ub && Tb > 0);
    const int n = enc ? min(W, Ub + 1 - (sb ? sb[i] : 0)) : Tb;         // terms of the sum
    const size_t base = enc ? ((size_t)b * T + i) * W * D : ((size_t)b * T * W + i) * D;
    const size_t stride = enc ? (size_t)D : (size_t)W * D;              // from one term to the next (full lattice)
    bf16* out = (enc ? dep : dpp) + (size_t)r * D;
    const auto term = [&](size_t o, float& sx, float& sy) {
        const float2 g = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(dh + o));
        const float2 y = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(h + o));
        sx += g.x * (1.f - y.x * y.x);
        sy += g.y * (1.f - y.y * y.y);
    };
    for (int c = 2 * threadIdx.x; c < D; c += 2 * RNNT_BWD_THREADS) {
        float sx = 0.f, sy = 0.f;
        if (live && (!sb || enc)) {
            for (int k = 0; k < n; ++k) term(base + k * stride + c, sx, sy);
        } else if (live) {
            // dPp row i of a band: frame k holds u = i at position i - s_k when that is inside [0, S)
            for (int k = 0; k < n; ++k) {
                const int pos = i - sb[k];
                if (pos >= 0 && pos < W) term((((size_t)b * T + k) * W + pos) * D + c, sx, sy);
            }
        }
        *reinterpret_cast<__nv_bfloat162*>(out + c) = __floats2bfloat162_rn(sx, sy);
    }
}

__device__ __forceinline__ int rnnt_label(const int* labels, int ldy, int b, int u, int Ub, int V) {
    if (u >= Ub) return -1;
    const int y = labels[(size_t)b * ldy + u];
    return (y < 1 || y >= V) ? -1 : y;                  // blank or out of range: no label arc
}

__global__ void __launch_bounds__(RNNT_WARPS * 32) rnnt_logprob_kernel(const float* __restrict__ logits, int ld, int rows,
                                                                       long long row0, int V, int T, int U1,
                                                                       const int* __restrict__ t_len, const int* __restrict__ u_len,
                                                                       const int* __restrict__ labels, int ldy,
                                                                       const int* __restrict__ s_begin, int S,
                                                                       float* __restrict__ lp) {
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * RNNT_WARPS + (threadIdx.x >> 5);
    if (r >= rows) return;
    const long long node = row0 + r;
    const LatticeNode n = lattice_node(node, T, U1, t_len, u_len, s_begin, S);
    float* o = lp + node * 3;
    if (!n.valid) {
        if (lane == 0) o[0] = o[1] = o[2] = 0.f;
        return;
    }
    const float* x = logits + (size_t)r * ld;
    float m, s;
    warp_row_lse(x, V, lane, m, s);
    if (lane == 0) {
        const int y = rnnt_label(labels, ldy, n.b, n.u, min(u_len[n.b], U1 - 1), V);
        const float ls = logf(s);
        o[0] = m + ls;
        o[1] = (x[0] - m) - ls;
        o[2] = y < 0 ? -INFINITY : (x[y] - m) - ls;
    }
}

// lp f32 [B T W, 3] (rnnt_logprob), alpha f64 [B T W] scratch; nll f32 [B]; grad f32 [B T W, 2] = scale * d loss / d
// (log p(blank), log p(y_{u+1})) of every node, scale = grad_scale (* *scale_dev) / B ('mean' over the batch).  W = U1, or
// S when banded: node (t, u) exists only when s_t <= u < s_t + S and is stored at (t, u - s_t); alpha and beta are -inf
// at every other node.  When no alignment stays inside the bands, nll is +inf and every gradient of the utterance is zero.
__global__ void __launch_bounds__(RNNT_MAX_U1) rnnt_loss_kernel(const float* __restrict__ lp, int B, int T, int U1,
                                                                const int* __restrict__ t_len, const int* __restrict__ u_len,
                                                                const int* __restrict__ s_begin, int S,
                                                                double* __restrict__ alpha, float* __restrict__ nll,
                                                                float* __restrict__ grad, float grad_scale,
                                                                const float* __restrict__ scale_dev) {
    __shared__ double buf[2][RNNT_MAX_U1];
    __shared__ double s_logp;
    const int b = blockIdx.x, u = threadIdx.x;
    const int Tb = min(t_len[b], T), Ub = min(u_len[b], U1 - 1);
    const int W = lattice_width(U1, s_begin, S);
    const int* sb = s_begin ? s_begin + (size_t)b * T : nullptr;
    const size_t n0 = (size_t)b * T * W;
    float* g = grad + n0 * 2;
    for (int i = threadIdx.x; i < T * W; i += blockDim.x) {      // nodes past T_b or U_b
        if (i / W >= Tb || i % W + (sb ? sb[i / W] : 0) > Ub) g[2 * i] = g[2 * i + 1] = 0.f;
    }
    if (Tb < 1 || Ub < 0) {     // no frame, or a negative label count: no node, no alignment
        if (threadIdx.x == 0) nll[b] = INFINITY;
        return;
    }
    // the stored node of (t, uu), or -1 outside the frame's band
    const auto at = [&](int t, int uu) -> long long {
        const int k = sb ? uu - sb[t] : uu;
        return (k >= 0 && k < W) ? (long long)(n0 + (size_t)t * W + k) : -1;
    };
    const int last = Tb - 1 + Ub;
    int cur = 0;
    for (int d = 0; d <= last; ++d) {
        const int t = d - u;
        if (u <= Ub && t >= 0 && t < Tb) {
            const long long k = at(t, u);
            double a = -INFINITY;
            if (k >= 0) {
                a = d == 0 ? 0.0 : -INFINITY;
                const long long kb = t > 0 ? at(t - 1, u) : -1, ky = u > 0 ? at(t, u - 1) : -1;
                if (kb >= 0) a = buf[cur][u] + (double)lp[kb * 3 + 1];
                if (ky >= 0) a = log_add(a, buf[cur][u - 1] + (double)lp[ky * 3 + 2]);
                alpha[k] = a;
            }
            buf[cur ^ 1][u] = a;
            if (d == last) s_logp = k >= 0 ? a + (double)lp[k * 3 + 1] : -INFINITY;
        }
        __syncthreads();
        cur ^= 1;
    }
    const double logp = s_logp;
    if (threadIdx.x == 0) nll[b] = (float)-logp;
    const float gs = (scale_dev ? grad_scale * *scale_dev : grad_scale) / (float)B;
    const bool dead = logp == -INFINITY;        // no alignment: zero gradients
    for (int d = last; d >= 0; --d) {
        const int t = d - u;
        if (u <= Ub && t >= 0 && t < Tb) {
            const long long k = at(t, u);
            double beta = -INFINITY;
            if (k >= 0) {
                const double lb = lp[k * 3 + 1], ly = lp[k * 3 + 2];
                const double bt = t + 1 < Tb ? buf[cur][u] : (u == Ub ? 0.0 : -INFINITY);    // beta(t + 1, u)
                const double bu = u < Ub ? buf[cur][u + 1] : -INFINITY;                       // beta(t, u + 1)
                const double a = alpha[k];
                beta = log_add(bt + lb, bu + ly);
                const double eb = a + lb + bt - logp, ey = a + ly + bu - logp;
                g[2 * (k - n0)] = (dead || eb == -INFINITY) ? 0.f : -gs * (float)exp(eb);
                g[2 * (k - n0) + 1] = (dead || ey == -INFINITY) ? 0.f : -gs * (float)exp(ey);
            }
            buf[cur ^ 1][u] = beta;
        }
        __syncthreads();
        cur ^= 1;
    }
}

// loss = sum_b nll_b / B, in ascending b (single thread: B is a batch size)
__global__ void rnnt_mean_kernel(const float* __restrict__ nll, int B, float* __restrict__ loss) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += nll[b];
    *loss = s / (float)B;
}

__global__ void __launch_bounds__(RNNT_WARPS * 32) rnnt_dlogits_kernel(const float* __restrict__ logits, int ld, int rows,
                                                                       long long row0, int V, int T, int U1,
                                                                       const int* __restrict__ t_len, const int* __restrict__ u_len,
                                                                       const int* __restrict__ labels, int ldy,
                                                                       const float* __restrict__ lp, const float* __restrict__ grad,
                                                                       const int* __restrict__ s_begin, int S,
                                                                       bf16* __restrict__ dz, int ldd) {
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * RNNT_WARPS + (threadIdx.x >> 5);
    if (r >= rows) return;
    const long long node = row0 + r;
    const LatticeNode n = lattice_node(node, T, U1, t_len, u_len, s_begin, S);
    const float a = n.valid ? grad[node * 2] : 0.f, c = n.valid ? grad[node * 2 + 1] : 0.f;
    const int y = n.valid ? rnnt_label(labels, ldy, n.b, n.u, min(u_len[n.b], U1 - 1), V) : -1;
    const float lse = lp[node * 3], ac = a + c;
    const float* x = logits + (size_t)r * ld;
    __nv_bfloat162* o = reinterpret_cast<__nv_bfloat162*>(dz + (size_t)r * ldd);
    const bool zero = a == 0.f && c == 0.f;
    for (int k = 2 * lane; k < ldd; k += 64) {
        float v[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int kk = k + j;
            v[j] = 0.f;
            if (!zero && kk < V) v[j] = (kk == 0 ? a : 0.f) + (kk == y ? c : 0.f) - expf(x[kk] - lse) * ac;
        }
        o[k >> 1] = __floats2bfloat162_rn(v[0], v[1]);
    }
}

// One step of greedy search for utterance b = blockIdx.x (DESIGN.md 4.22).  tok = the arg-max of the joint's log-probs
// (otb_logsoftmax_topk, k = 1), or blank when the row may not emit (max_sym emissions at this frame, or max_len tokens
// out); its log-prob is added to the score.  A label is appended to ids and the predictor state computed from it (h_new,
// c_new [layers, B, H] f32, pp_new [B, D] bf16) replaces the row's (h, c, pp); a blank moves the row to its next frame and
// copies that frame's encoder projection into ep_cur, or ends the row (active -= 1).  Ended rows are left as they are.
// LM fusion (val non-null): val [B] is the fused value of the arg-max (otb_logsoftmax_topk with blank exempt), and a
// label adds it to the score in place of its log-prob; emit [B] (optional) gets 1 where the row emitted and 0 elsewhere,
// lm_pos [B] (optional) the label's LM position n_out (1 .. max_len) where it emitted and -1 elsewhere.
__global__ void __launch_bounds__(128) rnnt_greedy_step_kernel(const int* __restrict__ idx, const float* __restrict__ logp, int ldlp,
                                                               const float* __restrict__ h_new, const float* __restrict__ c_new,
                                                               const bf16* __restrict__ pp_new, float* __restrict__ h,
                                                               float* __restrict__ c, bf16* __restrict__ pp, int layers, int B,
                                                               int H, int D, const bf16* __restrict__ ep, int T,
                                                               bf16* __restrict__ ep_cur, const int* __restrict__ t_len,
                                                               int* __restrict__ frame, int* __restrict__ n_sym,
                                                               int* __restrict__ n_out, int* __restrict__ ids, int max_len,
                                                               int max_sym, float* __restrict__ score, int* __restrict__ active,
                                                               const float* __restrict__ val, int* __restrict__ emit,
                                                               int* __restrict__ lm_pos) {
    __shared__ int s_act;      // 0: ended, 1: emitted, 2: moved to the next frame
    __shared__ int s_t;
    const int b = blockIdx.x;
    if (threadIdx.x == 0) {
        const int t = frame[b], Tb = min(t_len[b], T);
        int act = 0;
        if (t < Tb) {
            const int k = n_out[b];
            const int tok = (n_sym[b] < max_sym && k < max_len) ? idx[b] : 0;
            score[b] += (val != nullptr && tok != 0) ? val[b] : logp[(size_t)b * ldlp + tok];
            if (tok != 0) {
                ids[(size_t)b * max_len + k] = tok;
                n_out[b] = k + 1;
                n_sym[b] += 1;
                act = 1;
            } else {
                frame[b] = t + 1;
                n_sym[b] = 0;
                act = 2;
                if (t + 1 >= Tb) {
                    atomicSub(active, 1);
                    act = 0;
                }
                s_t = t + 1;
            }
        }
        s_act = act;
        if (emit) emit[b] = act == 1;
        if (lm_pos) lm_pos[b] = act == 1 ? n_out[b] : -1;
    }
    __syncthreads();
    if (s_act == 1) {
        for (int l = 0; l < layers; ++l) {
            const size_t o = ((size_t)l * B + b) * H;
            for (int i = threadIdx.x; i < H; i += blockDim.x) {
                h[o + i] = h_new[o + i];
                c[o + i] = c_new[o + i];
            }
        }
        for (int i = threadIdx.x; i < D; i += blockDim.x) pp[(size_t)b * D + i] = pp_new[(size_t)b * D + i];
    } else if (s_act == 2) {
        const bf16* src = ep + ((size_t)b * T + s_t) * D;
        for (int i = threadIdx.x; i < D; i += blockDim.x) ep_cur[(size_t)b * D + i] = src[i];
    }
}

static const char* rnnt_band_check(const int* s_begin, int S, const int* t_len) {
    if (s_begin && (S < 2 || S > RNNT_MAX_U1)) return "the band width S must be in [2, 1024]";
    if (s_begin && !t_len) return "a banded lattice needs t_len and u_len";
    return nullptr;
}

const char* rnnt_joint_launch(cudaStream_t st, const bf16* ep, const bf16* pp, int B, int T, int U1, int D, const int* t_len,
                              const int* u_len, const int* s_begin, int S, bf16* out) {
    if (B < 1 || T < 1 || U1 < 1) return "rnnt_joint: empty lattice";
    if (D < 8 || D % 8) return "rnnt_joint: inner size must be a positive multiple of 8";
    if (const char* e = rnnt_band_check(s_begin, S, t_len)) return e;
    const long long n_vec = (long long)B * T * (s_begin ? S : U1) * (D / 8);
    return launch<rnnt_joint_kernel>((unsigned)((n_vec + 255) / 256), 256, 0, st, ep, pp, D, T, U1, t_len, u_len, s_begin, S, out,
                                     n_vec);
}

const char* rnnt_joint_bwd_launch(cudaStream_t st, const bf16* dh, const bf16* h, int B, int T, int U1, int D, const int* t_len,
                                  const int* u_len, const int* s_begin, int S, bf16* dep, bf16* dpp) {
    if (B < 1 || T < 1 || U1 < 1) return "rnnt_joint_bwd: empty lattice";
    if (D < 2 || D % 2) return "rnnt_joint_bwd: inner size must be a positive even number";
    if (const char* e = rnnt_band_check(s_begin, S, t_len)) return e;
    return launch<rnnt_joint_bwd_kernel>(B * T + B * U1, RNNT_BWD_THREADS, 0, st, dh, h, D, B, T, U1, t_len, u_len, s_begin, S, dep,
                                         dpp);
}

static const char* rnnt_rows_check(int ld, int rows, int V, int ldy, int U1, const float* logits) {
    if (rows < 0 || V < 2 || ld < V) return "need rows >= 0, V >= 2 and ld >= V";
    if (ld % 4 || reinterpret_cast<uintptr_t>(logits) % 16) return "logits rows must be 16-byte aligned (ld % 4 == 0)";
    if (U1 < 1 || ldy < U1 - 1) return "labels narrower than the lattice";
    return nullptr;
}

const char* rnnt_logprob_launch(cudaStream_t st, const float* logits, int ld, int rows, long long row0, int V, int T, int U1,
                                const int* t_len, const int* u_len, const int* labels, int ldy, const int* s_begin, int S, float* lp) {
    if (const char* e = rnnt_rows_check(ld, rows, V, ldy, U1, logits)) return e;
    if (const char* e = rnnt_band_check(s_begin, S, t_len)) return e;
    if (rows == 0) return nullptr;
    return launch<rnnt_logprob_kernel>((rows + RNNT_WARPS - 1) / RNNT_WARPS, RNNT_WARPS * 32, 0, st, logits, ld, rows, row0, V, T,
                                       U1, t_len, u_len, labels, ldy, s_begin, S, lp);
}

const char* rnnt_loss_launch(cudaStream_t st, const float* lp, int B, int T, int U1, const int* t_len, const int* u_len,
                             const int* s_begin, int S, double* alpha, float* nll, float* loss, float* grad, float grad_scale,
                             const float* scale_dev) {
    if (B < 1 || T < 1) return "rnnt_loss: empty lattice";
    if (U1 < 1 || U1 > RNNT_MAX_U1) return "rnnt_loss: transcripts of at most 1023 labels";
    if (const char* e = rnnt_band_check(s_begin, S, t_len)) return e;
    const int threads = (U1 + 31) / 32 * 32;
    if (const char* e = launch<rnnt_loss_kernel>(B, threads, 0, st, lp, B, T, U1, t_len, u_len, s_begin, S, alpha, nll, grad, grad_scale,
                                                 scale_dev))
        return e;
    return launch<rnnt_mean_kernel>(1, 1, 0, st, nll, B, loss);
}

const char* rnnt_dlogits_launch(cudaStream_t st, const float* logits, int ld, int rows, long long row0, int V, int T, int U1,
                                const int* t_len, const int* u_len, const int* labels, int ldy, const float* lp, const float* grad,
                                const int* s_begin, int S, bf16* dz, int ldd) {
    if (const char* e = rnnt_rows_check(ld, rows, V, ldy, U1, logits)) return e;
    if (ldd < V || ldd % 2) return "rnnt_dlogits: need an even ldd >= V";
    if (const char* e = rnnt_band_check(s_begin, S, t_len)) return e;
    if (rows == 0) return nullptr;
    return launch<rnnt_dlogits_kernel>((rows + RNNT_WARPS - 1) / RNNT_WARPS, RNNT_WARPS * 32, 0, st, logits, ld, rows, row0, V, T,
                                       U1, t_len, u_len, labels, ldy, lp, grad, s_begin, S, dz, ldd);
}

const char* rnnt_greedy_step_launch(cudaStream_t st, const int* idx, const float* logp, int ldlp, const float* h_new,
                                    const float* c_new, const bf16* pp_new, float* h, float* c, bf16* pp, int layers, int B, int H,
                                    int D, const bf16* ep, int T, bf16* ep_cur, const int* t_len, int* frame, int* n_sym, int* n_out,
                                    int* ids, int max_len, int max_sym, float* score, int* active, const float* val, int* emit,
                                    int* lm_pos) {
    if (B < 1 || T < 1 || layers < 1 || H < 1 || D < 1) return "rnnt_greedy_step: empty problem";
    if (max_len < 1 || max_sym < 1) return "rnnt_greedy_step: need max_len >= 1 and max_sym >= 1";
    return launch<rnnt_greedy_step_kernel>(B, 128, 0, st, idx, logp, ldlp, h_new, c_new, pp_new, h, c, pp, layers, B, H, D, ep, T,
                                           ep_cur, t_len, frame, n_sym, n_out, ids, max_len, max_sym, score, active, val, emit,
                                           lm_pos);
}

}  // namespace otb
