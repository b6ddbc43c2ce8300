// Joint-CTC branch of SpeechToText.forward (otrans/model/speech2text.py:30-36,60-64 -> CTCAssistor, model/ctc.py:12-52):
//   loss_ctc = nn.CTCLoss(blank = 0, reduction 'mean', zero_infinity = True)(log_softmax(output_layer(memory)).transpose(0,1),
//                                                                              targets_out, memory_length, targets_length)
// Forward AND gradient with respect to the logits in two kernels (the reference differentiates F.ctc_loss by autograd):
//   ctc_alpha_beta_kernel  one CTA per utterance, thread = state of the blank-extended label sequence (S = 2 L + 1 <= 129):
//                          forward variables alpha_t(s) over the valid frames (log domain, fp32), the utterance's negative
//                          log-likelihood, then the backward variables; ws[b,t,s] <- alpha_t(s) + beta_t(s)
//   ctc_grad_kernel        one CTA per (utterance, frame): d loss / d logit[k] = scale_b (softmax[k] - sum_{s: l_s = k}
//                          exp(alpha_t(s) + beta_t(s) - logp[k] + nll_b)), scale_b = 1 / (B max(target_len_b, 1)) ('mean'
//                          divides every utterance by its target length, then averages), zero for padded frames and for
//                          infeasible utterances (zero_infinity).  bf16 output for the wgmma backward GEMMs.
// HBM-bound integer/float work: the [B T', V] log-prob matrix is read once by each kernel.
#include <math.h>

#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

static constexpr int CTC_SMAX = 129;   // 2 * 64 + 1 states

__device__ __forceinline__ float log_add(float a, float b) {
    if (a == -INFINITY) return b;
    if (b == -INFINITY) return a;
    const float m = fmaxf(a, b);
    return m + log1pf(expf(fminf(a, b) - m));
}

__global__ void __launch_bounds__(160) ctc_alpha_beta_kernel(const float* __restrict__ logp, int ldl, int T, const int* __restrict__ in_len,
                                                             const long long* __restrict__ targets, int ldt,
                                                             const int* __restrict__ tgt_len, int blank, int V, float* __restrict__ nll,
                                                             float* __restrict__ ws, int S_ws) {
    __shared__ int lab[CTC_SMAX + 2];
    __shared__ float buf[2][CTC_SMAX + 2];
    const int b = blockIdx.x, s = threadIdx.x;
    const int L = min(tgt_len[b], (CTC_SMAX - 1) / 2);
    const int S = 2 * L + 1;
    const int Tb = min(in_len[b], T);
    if (s < S + 2) {
        int l = blank;
        if (s < S && (s & 1)) {
            long long v = targets[(size_t)b * ldt + (s >> 1)];
            l = (v < 0 || v >= V) ? blank : (int)v;
        }
        lab[s] = l;
    }
    __syncthreads();
    const float* lp = logp + (size_t)b * T * ldl;
    float* w = ws + (size_t)b * T * S_ws;
    if (Tb < 1) {   // no frames: infeasible unless the target is empty too (PyTorch: inf -> 0 with zero_infinity)
        if (s == 0) nll[b] = INFINITY;
        return;
    }
    const int my = (s < S) ? lab[s] : blank;
    const bool skip_ok = (s >= 2 && s < S && my != blank && my != lab[s - 2]);
    // ---- forward variables
    float a = -INFINITY;
    if (s == 0) a = lp[blank];
    if (s == 1 && S > 1) a = lp[my];
    if (s < S) { buf[0][s] = a; w[s] = a; }
    __syncthreads();
    int cur = 0;
    for (int t = 1; t < Tb; ++t) {
        if (s < S) {
            float v = buf[cur][s];
            if (s >= 1) v = log_add(v, buf[cur][s - 1]);
            if (skip_ok) v = log_add(v, buf[cur][s - 2]);
            a = (v == -INFINITY) ? -INFINITY : v + lp[(size_t)t * ldl + my];
            buf[cur ^ 1][s] = a;
            w[(size_t)t * S_ws + s] = a;
        }
        cur ^= 1;
        __syncthreads();
    }
    float total = buf[cur][S - 1];
    if (S > 1) total = log_add(total, buf[cur][S - 2]);
    __syncthreads();
    if (s == 0) nll[b] = -total;          // +inf when no alignment exists
    // ---- backward variables; ws <- alpha + beta
    const bool skip_fw = (s + 2 < S && lab[s + 2] != blank && lab[s + 2] != my);
    float be = -INFINITY;
    if (s == S - 1) be = lp[(size_t)(Tb - 1) * ldl + blank];
    if (s == S - 2 && S > 1) be = lp[(size_t)(Tb - 1) * ldl + my];
    if (s < S) {
        buf[0][s] = be;
        w[(size_t)(Tb - 1) * S_ws + s] += be;
    }
    __syncthreads();
    cur = 0;
    for (int t = Tb - 2; t >= 0; --t) {
        if (s < S) {
            float v = buf[cur][s];
            if (s + 1 < S) v = log_add(v, buf[cur][s + 1]);
            if (skip_fw) v = log_add(v, buf[cur][s + 2]);
            be = (v == -INFINITY) ? -INFINITY : v + lp[(size_t)t * ldl + my];
            buf[cur ^ 1][s] = be;
            w[(size_t)t * S_ws + s] += be;
        }
        cur ^= 1;
        __syncthreads();
    }
}

// loss = mean_b (finite nll_b ? nll_b / max(tgt_len_b, 1) : 0)   (single CTA)
__global__ void ctc_mean_kernel(const float* __restrict__ nll, const int* __restrict__ tgt_len, int B, float* loss) {
    __shared__ float red[32];
    float c = 0.f;
    for (int i = threadIdx.x; i < B; i += blockDim.x) {
        const float v = nll[i];
        if (isfinite(v)) c += v / (float)max(tgt_len[i], 1);
    }
    c = warp_sum(c);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
        *loss = t / (float)B;
    }
}

__global__ void __launch_bounds__(256) ctc_grad_kernel(const float* __restrict__ logp, int ldl, int T, int V, const int* __restrict__ in_len,
                                                       const long long* __restrict__ targets, int ldt,
                                                       const int* __restrict__ tgt_len, int blank, const float* __restrict__ nll,
                                                       const float* __restrict__ ws, int S_ws, int B, float grad_scale,
                                                       bf16* __restrict__ dlogits, int ldd) {
    __shared__ int lab[CTC_SMAX];
    __shared__ float occ[CTC_SMAX];
    const int row = blockIdx.x, b = row / T, t = row % T;
    const int L = min(tgt_len[b], (CTC_SMAX - 1) / 2);
    const int S = 2 * L + 1;
    const float nl = nll[b];
    bf16* d = dlogits + (size_t)row * ldd;
    const bool live = (t < min(in_len[b], T)) && isfinite(nl);
    if (!live) {
        for (int k = threadIdx.x; k < ldd; k += blockDim.x) d[k] = __float2bfloat16(0.f);
        return;
    }
    const float* lp = logp + (size_t)row * ldl;
    const float scale = grad_scale / ((float)B * (float)max(tgt_len[b], 1));
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
        int l = blank;
        if (s & 1) {
            long long v = targets[(size_t)b * ldt + (s >> 1)];
            l = (v < 0 || v >= V) ? blank : (int)v;
        }
        lab[s] = l;
        const float ab = ws[((size_t)b * T + t) * S_ws + s];
        occ[s] = (ab == -INFINITY) ? 0.f : expf(ab - lp[l] + nl);
    }
    for (int k = threadIdx.x; k < ldd; k += blockDim.x) d[k] = __float2bfloat16(k < V ? scale * expf(lp[k]) : 0.f);
    __syncthreads();
    // first occurrence of every label owns the combined entry (same-CTA global writes after the barrier: the later write wins)
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
        const int l = lab[s];
        bool first = true;
        float tot = 0.f;
        for (int s2 = 0; s2 < S; ++s2) {
            if (lab[s2] == l) {
                if (s2 < s) { first = false; break; }
                tot += occ[s2];
            }
        }
        if (first) d[l] = __float2bfloat16(scale * (expf(lp[l]) - tot));
    }
}

const char* ctc_launch(cudaStream_t st, const float* logp, int ldl, int B, int T, int V, const int* in_len, const long long* targets,
                       int ldt, const int* tgt_len, int max_tgt, int blank, float* nll, float* loss, float* ws, bf16* dlogits, int ldd,
                       float grad_scale) {
    if (B < 1 || T < 1 || V < 2) return "ctc: empty problem";
    if (max_tgt < 0 || 2 * max_tgt + 1 > CTC_SMAX) return "ctc: targets longer than 64 labels are not supported";
    if (blank < 0 || blank >= V) return "ctc: bad blank id";
    const int S_ws = 2 * max_tgt + 1;
    ctc_alpha_beta_kernel<<<B, 160, 0, st>>>(logp, ldl, T, in_len, targets, ldt, tgt_len, blank, V, nll, ws, S_ws);
    ctc_mean_kernel<<<1, 256, 0, st>>>(nll, tgt_len, B, loss);
    if (dlogits) ctc_grad_kernel<<<B * T, 256, 0, st>>>(logp, ldl, T, V, in_len, targets, ldt, tgt_len, blank, nll, ws, S_ws, B, grad_scale, dlogits, ldd);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace otb
