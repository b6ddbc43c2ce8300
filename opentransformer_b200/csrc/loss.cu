// Label-smoothed cross entropy, forward (+ optional dlogits) in one pass over the logits.
// Replaces LabelSmoothingLoss.forward (otrans/module/loss.py:21-48): the reference clones a [B*L, V]
// "confidence" tensor, runs log_softmax and an element-wise kl_div; here one CTA per token row computes
//   loss_tok = sum_v conf_v (log conf_v - logp_v),  conf_v = eps/(V-1) (v != t), 1-eps (v == t)
//            = C - eps/(V-1) * (sum_v x_v - V*lse) - (1 - eps - eps/(V-1)) * (x_t - lse)
// from the row maximum, the log-sum-exp and the plain sum of the logits; PAD(0) targets give 0
// (loss.py:31,46) and the mean is taken over the non-PAD tokens (:44-46).  A target outside [0, V) is scored like PAD
// and not counted either.
#include <math.h>

#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

__device__ __forceinline__ float block_reduce(float v, float* red, bool is_max) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    v = is_max ? warp_max(v) : warp_sum(v);
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = red[0];
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) t = is_max ? fmaxf(t, red[i]) : t + red[i];
    return t;
}

__global__ void __launch_bounds__(256) ls_ce_kernel(const float* __restrict__ logits, int ldl, const long long* __restrict__ tgt,
                                                    int V, float eps, int pad_id, float* __restrict__ tok_loss,
                                                    float* __restrict__ dlogits, int ldd, const int* __restrict__ n_valid_ptr,
                                                    bf16* __restrict__ dlogits_bf16) {
    __shared__ float red[8];
    const int row = blockIdx.x;
    const float* x = logits + (size_t)row * ldl;
    long long t = tgt[row];
    // a target outside [0, V) has no logit to read: treat the row like PAD (contributes nothing) instead of reading out of bounds
    const bool is_pad = (t == pad_id) || t < 0 || t >= V;
    if (t < 0 || t >= V) t = 0;
    float m = -INFINITY, s = 0.f;
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
        const float v = x[i];
        m = fmaxf(m, v);
        s += v;
    }
    m = block_reduce(m, red, true);
    s = block_reduce(s, red, false);
    float e = 0.f;
    for (int i = threadIdx.x; i < V; i += blockDim.x) e += expf(x[i] - m);
    e = block_reduce(e, red, false);
    const float lse = m + logf(e);
    const float lo = eps / (float)(V - 1), hi = 1.0f - eps;
    if (threadIdx.x == 0) {
        float l = 0.f;
        if (!is_pad) {
            // sum_v conf_v log conf_v with xlogy semantics (0 log 0 = 0, what F.kl_div does): smoothing 0 or 1 stay finite
            const float c = (lo > 0.f ? (float)(V - 1) * lo * logf(lo) : 0.f) + (hi > 0.f ? hi * logf(hi) : 0.f);
            l = c - lo * (s - (float)V * lse) - (hi - lo) * (x[t] - lse);
        }
        tok_loss[row] = l;
    }
    if (dlogits != nullptr) {  // d(mean loss)/dlogits = (softmax - conf) / n_valid   (0 for PAD rows)
        const float inv = is_pad ? 0.f : 1.0f / (float)max(*n_valid_ptr, 1);
        float* d = dlogits + (size_t)row * ldd;
        for (int i = threadIdx.x; i < V; i += blockDim.x) {
            const float p = expf(x[i] - lse);
            d[i] = (p - ((i == t) ? hi : lo)) * inv;
        }
    }
    if (dlogits_bf16 != nullptr) {   // bf16 copy for the backward GEMMs (columns [V, ldd) are zero padding)
        const float inv = is_pad ? 0.f : 1.0f / (float)max(*n_valid_ptr, 1);
        bf16* d = dlogits_bf16 + (size_t)row * ldd;
        for (int i = threadIdx.x; i < ldd; i += blockDim.x) {
            float gv = 0.f;
            if (i < V) gv = (expf(x[i] - lse) - ((i == t) ? hi : lo)) * inv;
            d[i] = __float2bfloat16(gv);
        }
    }
}

// n_valid = #(target != PAD and in [0, V)): exactly the rows ls_ce_kernel scores; loss = sum(tok_loss) / n_valid
// (single CTA, deterministic order)
__global__ void __launch_bounds__(256) ls_count_kernel(const long long* __restrict__ tgt, int rows, int V, int pad_id,
                                                       int* n_valid) {
    __shared__ float red[8];
    float c = 0.f;
    for (int i = threadIdx.x; i < rows; i += blockDim.x) {
        const long long t = tgt[i];
        c += (t != pad_id && t >= 0 && t < V) ? 1.f : 0.f;
    }
    c = block_reduce(c, red, false);
    if (threadIdx.x == 0) *n_valid = (int)(c + 0.5f);
}
__global__ void __launch_bounds__(256) ls_mean_kernel(const float* __restrict__ tok_loss, int rows, const int* n_valid,
                                                      float* loss) {
    __shared__ float red[8];
    float c = 0.f;
    for (int i = threadIdx.x; i < rows; i += blockDim.x) c += tok_loss[i];
    c = block_reduce(c, red, false);
    if (threadIdx.x == 0) *loss = c / (float)max(*n_valid, 1);
}

const char* ls_ce_launch(cudaStream_t st, const float* logits, int ldl, const long long* tgt, int rows, int V, float eps,
                         int pad_id, float* tok_loss, float* loss, int* n_valid, float* dlogits, int ldd, bf16* dlogits_bf16) {
    if (rows < 1 || V < 2) return "ls_ce: empty problem";
    const char* err;
    if ((err = launch<ls_count_kernel>(1, 256, 0, st, tgt, rows, V, pad_id, n_valid))) return err;
    if ((err = launch<ls_ce_kernel>(rows, 256, 0, st, logits, ldl, tgt, V, eps, pad_id, tok_loss, dlogits_bf16 ? nullptr : dlogits,
                                    ldd, n_valid, dlogits_bf16)))
        return err;
    return launch<ls_mean_kernel>(1, 256, 0, st, tok_loss, rows, n_valid, loss);
}

}  // namespace otb
