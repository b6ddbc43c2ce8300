// Minimum word error rate training (DESIGN.md 4.11): the edit distances of an n-best and the gradient of its expected risk.
//   edit_distance_kernel   one warp per (hypothesis i, reference i / K) pair: the Levenshtein DP row by row over the
//                          hypothesis tokens, the row over the reference columns in chunks of 32.  With X[0] = a and
//                          X[j] = min(D[a-1][j] + 1, D[a-1][j-1] + (h_a != r_j)), the insertion chain along the row is a
//                          prefix minimum, D[a][j] = j + min_{k <= j} (X[k] - k): one warp min-scan per chunk, carried from
//                          chunk to chunk.  Integer arithmetic, so the result is exact.
//   mwer_coeff_kernel      one warp per utterance, lane k = hypothesis k (K <= 32): the duplicate test against lower lanes,
//                          l_k = sum of its token log-probs in position order, P_k = softmax over the kept l, the loss
//                          sum_k P_k (W_k - mean W) and the coefficient c_k = dL/dl_k * scale of the row gradient.
//   mwer_sample_coeff_kernel  the sampled estimator: one warp per utterance, lane k = sample k (K <= 32).  Samples are
//                          drawn with replacement, so every one counts (no duplicate rule) and there is no softmax: the
//                          loss is W^_b = mean W and c_k = (W_k - W^_b) / K * scale, exactly 0 when all W are equal.
//   mwer_grad_kernel       one warp per logits row: dlogits = c_k (onehot(target) - softmax(x)) as bf16, zero in padding
//                          columns and in rows without a target or with c_k = 0 (those rows are not read).  The row's
//                          log-sum-exp is the one otb_token_logprob formed: lse = x[target] - logprob, so the row is read
//                          once here and no second reduction runs; the target column takes 1 - p = -expm1(logprob).
#include <limits.h>
#include <math.h>

#include "launch.cuh"
#include "otb_internal.h"

namespace otb {

static constexpr int ED_WARPS = 4;
static constexpr int ED_MAX_LEN = 1023;       // a DP row of ED_MAX_LEN + 1 ints, two rows per warp in shared memory
static constexpr int MWER_KMAX = 32;          // one lane per hypothesis
static constexpr int MG_WARPS = 8;

__global__ void __launch_bounds__(ED_WARPS * 32) edit_distance_kernel(const int* __restrict__ hyp, int ldh,
                                                                      const int* __restrict__ hyp_len,
                                                                      const int* __restrict__ ref, int ldr,
                                                                      const int* __restrict__ ref_len, int N, int K, int max_h,
                                                                      int max_r, int* __restrict__ out) {
    __shared__ int rows[ED_WARPS][2][ED_MAX_LEN + 1];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int i = blockIdx.x * ED_WARPS + w;
    if (i >= N) return;
    const int b = i / K;
    const int n = min(max(hyp_len[i], 0), max_h);
    const int m = min(max(ref_len[b], 0), max_r);
    const int* h = hyp + (size_t)i * ldh;
    const int* r = ref + (size_t)b * ldr;
    int* prev = rows[w][0];
    int* cur = rows[w][1];
    for (int j = lane; j <= m; j += 32) prev[j] = j;
    __syncwarp();
    for (int a = 1; a <= n; ++a) {
        const int ha = h[a - 1];
        int carry = INT_MAX;                      // min of X[k] - k over the chunks before this one
        for (int j0 = 0; j0 <= m; j0 += 32) {
            const int j = j0 + lane;
            int y = INT_MAX;
            if (j == 0) {
                y = a;
            } else if (j <= m) {
                y = min(prev[j] + 1, prev[j - 1] + (ha != __ldg(r + j - 1))) - j;
            }
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, y, o);
                if (lane >= o) y = min(y, v);
            }
            y = min(y, carry);
            if (j <= m) cur[j] = j + y;
            carry = __shfl_sync(0xffffffffu, y, 31);
        }
        __syncwarp();
        int* t = prev;
        prev = cur;
        cur = t;
    }
    if (lane == 0) out[i] = prev[m];
}

__global__ void __launch_bounds__(32) mwer_coeff_kernel(const int* __restrict__ len, const int* __restrict__ err,
                                                        const float* __restrict__ tok_lp, int Lp, const int* __restrict__ tgt,
                                                        int K, float scale, const float* __restrict__ scale_dev,
                                                        float* __restrict__ coeff, float* __restrict__ loss) {
    const int b = blockIdx.x, k = threadIdx.x;
    const bool live = k < K;
    const size_t h = (size_t)b * K + k;
    // a length is clamped to [0, Lp - 1]: y <S/E> fills at most the Lp positions of its row
    const int n = live ? min(max(len[h], 0), Lp - 1) : 0;
    bool kept = live;
    for (int j = 0; j < k && kept && live; ++j) {       // the rescoring rule: a copy of a higher-ranked hypothesis is dropped
        const size_t hj = (size_t)b * K + j;
        if (min(max(len[hj], 0), Lp - 1) != n) continue;
        bool same = true;
        for (int t = 0; t < n && same; ++t) same = tgt[hj * Lp + t] == tgt[h * Lp + t];
        kept = !same;
    }
    // no contraction into FMAs: plain left-to-right float sums, as a host restatement forms them
    float l = -INFINITY;
    if (kept) {
        l = 0.f;
        for (int t = 0; t <= n; ++t) l = __fadd_rn(l, tok_lp[h * Lp + t]);
    }
    const float W = kept ? (float)err[h] : 0.f;
    float mx = l, nk = kept ? 1.f : 0.f, sw = W;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        nk += __shfl_xor_sync(0xffffffffu, nk, o);
        sw += __shfl_xor_sync(0xffffffffu, sw, o);
    }
    const float e = kept ? expf(l - mx) : 0.f;
    float z = e;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
    const float p = e / z;
    const float dw = kept ? W - sw / nk : 0.f;          // W_k - mean W: exactly 0 when all kept W are equal
    float risk = p * dw;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) risk += __shfl_xor_sync(0xffffffffu, risk, o);
    // dL/dl_k = P_k (W_k - sum_j P_j W_j) = P_k ((W_k - mean W) - sum_j P_j (W_j - mean W))
    const float s = scale_dev != nullptr ? scale * *scale_dev : scale;
    if (live) coeff[h] = kept ? p * (dw - risk) * s : 0.f;
    if (k == 0) loss[b] = risk;
}

__global__ void __launch_bounds__(32) mwer_sample_coeff_kernel(const int* __restrict__ err, int K, float scale,
                                                               const float* __restrict__ scale_dev, float* __restrict__ coeff,
                                                               float* __restrict__ loss) {
    const int b = blockIdx.x, k = threadIdx.x;
    const bool live = k < K;
    const size_t h = (size_t)b * K + k;
    const float W = live ? (float)err[h] : 0.f;
    float sw = W;                       // integer-valued: the sum is exact below 2^24
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sw += __shfl_xor_sync(0xffffffffu, sw, o);
    const float mean = sw / (float)K;
    const float s = scale_dev != nullptr ? scale * *scale_dev : scale;
    if (live) coeff[h] = (W - mean) / (float)K * s;
    if (k == 0) loss[b] = mean;
}

__global__ void __launch_bounds__(MG_WARPS * 32) mwer_grad_kernel(const float* __restrict__ logits, int ld, int rows, int V,
                                                                  const int* __restrict__ target, const float* __restrict__ tok_lp,
                                                                  const float* __restrict__ coeff, int Lp, bf16* __restrict__ dlogits) {
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * MG_WARPS + (threadIdx.x >> 5);
    if (r >= rows) return;
    const int tgt = target[r];
    const float c = coeff[r / Lp];
    uint2* d = reinterpret_cast<uint2*>(dlogits + (size_t)r * ld);       // 4 bf16 per store
    const int nv = ld >> 2;
    if (tgt < 0 || tgt >= V || c == 0.f) {
        for (int i = lane; i < nv; i += 32) d[i] = make_uint2(0u, 0u);
        return;
    }
    const float* x = logits + (size_t)r * ld;
    const float lp_t = tok_lp[r];
    const float lse = x[tgt] - lp_t;
    // the target's 1 - p as -expm1(log p): exact where the row is saturated (p -> 1), where 1 - exp(x - lse) cancels
    const float g_t = c * -expm1f(lp_t);
    const float4* x4 = reinterpret_cast<const float4*>(x);
    for (int i = lane; i < nv; i += 32) {
        const float4 v = __ldcs(x4 + i);
        const float xs[4] = {v.x, v.y, v.z, v.w};
        float g[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int col = 4 * i + q;
            g[q] = col == tgt ? g_t : col < V ? -c * expf(xs[q] - lse) : 0.f;
        }
        const __nv_bfloat162 lo = __floats2bfloat162_rn(g[0], g[1]), hi = __floats2bfloat162_rn(g[2], g[3]);
        d[i] = make_uint2(*reinterpret_cast<const unsigned*>(&lo), *reinterpret_cast<const unsigned*>(&hi));
    }
}

const char* edit_distance_launch(cudaStream_t stream, const int* hyp, int ldh, const int* hyp_len, const int* ref, int ldr,
                                 const int* ref_len, int N, int K, int max_h, int max_r, int* out) {
    if (N < 0 || K < 1) return "edit_distance: need N >= 0 and K >= 1";
    if (max_h < 0 || max_r < 0 || max_h > ED_MAX_LEN || max_r > ED_MAX_LEN)
        return "edit_distance: sequences of up to 1023 tokens are supported";
    if (ldh < max_h || ldr < max_r) return "edit_distance: row pitch shorter than the longest sequence";
    if (N == 0) return nullptr;
    return launch<edit_distance_kernel>((N + ED_WARPS - 1) / ED_WARPS, ED_WARPS * 32, 0, stream, hyp, ldh, hyp_len, ref, ldr, ref_len,
                                        N, K, max_h, max_r, out);
}

const char* mwer_coeff_launch(cudaStream_t stream, const int* len, const int* err, const float* tok_lp, int Lp, const int* tgt, int B,
                              int K, float scale, const float* scale_dev, float* coeff, float* loss) {
    if (B < 1 || K < 1 || K > MWER_KMAX) return "mwer_coeff: need B >= 1 and 1 <= K <= 32";
    if (Lp < 1) return "mwer_coeff: need Lp >= 1";
    return launch<mwer_coeff_kernel>(B, 32, 0, stream, len, err, tok_lp, Lp, tgt, K, scale, scale_dev, coeff, loss);
}

const char* mwer_sample_coeff_launch(cudaStream_t stream, const int* err, int B, int K, float scale, const float* scale_dev,
                                     float* coeff, float* loss) {
    if (B < 1 || K < 1 || K > MWER_KMAX) return "mwer_sample_coeff: need B >= 1 and 1 <= K <= 32";
    return launch<mwer_sample_coeff_kernel>(B, 32, 0, stream, err, K, scale, scale_dev, coeff, loss);
}

const char* mwer_grad_launch(cudaStream_t stream, const float* logits, int ld, int rows, int V, const int* target, const float* tok_lp,
                             const float* coeff, int Lp, bf16* dlogits) {
    if (rows < 0 || V < 1 || ld < V || Lp < 1) return "mwer_grad: need rows >= 0, V >= 1, ld >= V and Lp >= 1";
    if (ld % 4 || reinterpret_cast<uintptr_t>(logits) % 16 || reinterpret_cast<uintptr_t>(dlogits) % 8)
        return "mwer_grad: rows must be 16-byte aligned (ld % 4 == 0)";
    if (rows == 0) return nullptr;
    return launch<mwer_grad_kernel>((rows + MG_WARPS - 1) / MG_WARPS, MG_WARPS * 32, 0, stream, logits, ld, rows, V, target, tok_lp,
                                    coeff, Lp, dlogits);
}

}  // namespace otb
