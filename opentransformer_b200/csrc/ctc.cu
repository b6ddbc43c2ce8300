// Joint-CTC branch of SpeechToText.forward (otrans/model/speech2text.py:30-36,60-64 -> CTCAssistor, model/ctc.py:12-52):
//   loss_ctc = nn.CTCLoss(blank = 0, reduction 'mean', zero_infinity = True)(log_softmax(output_layer(memory)).transpose(0,1),
//                                                                              targets_out, memory_length, targets_length)
// Forward AND gradient with respect to the logits in two kernels (the reference differentiates F.ctc_loss by autograd):
//   ctc_alpha_beta_kernel  one CTA per utterance over the S = 2 L + 1 states of the trellis (ctc_trellis.cuh): one
//                          state per thread up to 64 labels (<129, 160>), two per thread up to 1023 (<2047, 1024>):
//                          forward variables alpha_t(s) over the valid frames (log domain, fp32), the utterance's negative
//                          log-likelihood, then the backward variables; ws[b,t,s] <- alpha_t(s) + beta_t(s)
//   ctc_grad_kernel        one CTA per (utterance, frame): d loss / d logit[k] = scale_b (softmax[k] - sum_{s: l_s = k}
//                          exp(alpha_t(s) + beta_t(s) - logp[k] + nll_b)), scale_b = 1 / (B max(target_len_b, 1)) ('mean'
//                          divides every utterance by its target length, then averages), zero for padded frames and for
//                          infeasible utterances (zero_infinity).  bf16 output for the wgmma backward GEMMs.
// HBM-bound integer/float work: the [B T', V] log-prob matrix is read once by each kernel.
#include <math.h>

#include "ctc_trellis.cuh"
#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

static constexpr int CTC_SMAX = 129;        // 2 * 64 + 1 states: targets of up to 64 labels
static constexpr int CTC_SMAX_LONG = 2047;  // 2 * 1023 + 1 states: targets of up to 1023 labels

template <int SMAX, int NT>
__global__ void __launch_bounds__(NT) ctc_alpha_beta_kernel(const float* __restrict__ logp, int ldl, int T, const int* __restrict__ in_len,
                                                            const long long* __restrict__ targets, int ldt,
                                                            const int* __restrict__ tgt_len, int blank, int V, float* __restrict__ nll,
                                                            float* __restrict__ ws, int S_ws) {
    constexpr int SPT = (SMAX + NT - 1) / NT;
    __shared__ float buf[2][SMAX];
    const int b = blockIdx.x;
    const int L = min(tgt_len[b], (SMAX - 1) / 2);
    const int S = 2 * L + 1;
    const int Tb = min(in_len[b], T);
    if (Tb < 1) {   // no frames: infeasible unless the target is empty too (PyTorch: inf -> 0 with zero_infinity)
        if (threadIdx.x == 0) nll[b] = INFINITY;
        return;
    }
    const long long* tg = targets + (size_t)b * ldt;
    const auto label = [&](int i) {     // an out-of-range label counts as the blank
        const long long v = tg[i];
        return (v < 0 || v >= V) ? blank : (int)v;
    };
    const float* lp = logp + (size_t)b * T * ldl;
    float* w = ws + (size_t)b * T * S_ws;
    unsigned col[SPT];
    bool skip[SPT];
    // ---- forward variables, from frame -1
#pragma unroll
    for (int j = 0; j < SPT; ++j) {
        const int s = trellis_state(j, NT);
        col[j] = trellis_col(s, S, blank, label);
        skip[j] = trellis_skip(s, S, blank, label);
        if (s < S) buf[0][s] = s == 0 ? 0.f : -INFINITY;
    }
    __syncthreads();
    int cur = 0;
    for (int t = 0; t < Tb; ++t)
        trellis_step<TrellisLogAdd>(
            buf, cur, NT, S, skip, [&](int j) { return lp[(size_t)t * ldl + col[j]]; },
            [&](int, int s, TrellisLogAdd, float v) { w[(size_t)t * S_ws + s] = v; });
    if (threadIdx.x == 0) nll[b] = -trellis_log_total(buf[cur], S);          // +inf when no alignment exists
    __syncthreads();
    // ---- backward variables, from frame Tb; ws <- alpha + beta
#pragma unroll
    for (int j = 0; j < SPT; ++j) {
        const int s = trellis_state(j, NT);
        skip[j] = trellis_skip(s + 2, S, blank, label);
        if (s < S) buf[0][s] = s == S - 1 ? 0.f : -INFINITY;
    }
    __syncthreads();
    cur = 0;
    for (int t = Tb - 1; t >= 0; --t)
        trellis_step<TrellisLogAdd, true>(
            buf, cur, NT, S, skip, [&](int j) { return lp[(size_t)t * ldl + col[j]]; },
            [&](int, int s, TrellisLogAdd, float v) { w[(size_t)t * S_ws + s] += v; });
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

// Each label's occupancies are summed in ascending state order by the label's first state, which writes d[label].
// SORT false (targets <= 64 labels): every state scans the states before it for its label, O(S^2) per frame.
// SORT true (up to 1023 labels): the (label, state) pairs are sorted in shared memory (bitonic, O(S log^2 S) work in
// O(log^2 S) barriers), so each label's states form one ascending run that its first state walks.
template <int SMAX, bool SORT>
__global__ void __launch_bounds__(256) ctc_grad_kernel(const float* __restrict__ logp, int ldl, int T, int V, const int* __restrict__ in_len,
                                                       const long long* __restrict__ targets, int ldt,
                                                       const int* __restrict__ tgt_len, int blank, const float* __restrict__ nll,
                                                       const float* __restrict__ ws, int S_ws, int B, float grad_scale,
                                                       bf16* __restrict__ dlogits, int ldd, const float* __restrict__ scale_dev) {
    __shared__ int lab[SMAX];
    __shared__ float occ[SMAX];
    const int row = blockIdx.x, b = row / T, t = row % T;
    const int L = min(tgt_len[b], (SMAX - 1) / 2);
    const int S = 2 * L + 1;
    const float nl = nll[b];
    bf16* d = dlogits + (size_t)row * ldd;
    const bool live = (t < min(in_len[b], T)) && isfinite(nl);
    if (!live) {
        for (int k = threadIdx.x; k < ldd; k += blockDim.x) d[k] = __float2bfloat16(0.f);
        return;
    }
    const float* lp = logp + (size_t)row * ldl;
    // scale_dev (optional, read on the device): a loss weight known only on the device (MixSpeech's lambda / accum_steps)
    const float gs = scale_dev ? grad_scale * *scale_dev : grad_scale;
    const float scale = gs / ((float)B * (float)max(tgt_len[b], 1));
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
    if constexpr (!SORT) {
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
    } else {
        constexpr int NK = 2048;                      // power of two >= SMAX
        static_assert(SMAX <= NK, "sort width");
        __shared__ unsigned long long key[NK];        // label << 32 | state; padding sorts last
        const int n = S <= 1 ? 1 : 1 << (32 - __clz(S - 1));
        for (int i = threadIdx.x; i < n; i += blockDim.x)
            key[i] = i < S ? ((unsigned long long)(unsigned)lab[i] << 32 | (unsigned)i) : ~0ull;
        __syncthreads();
        for (int k = 2; k <= n; k <<= 1) {
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int i = threadIdx.x; i < n; i += blockDim.x) {
                    const int p = i ^ j;
                    if (p > i) {
                        const unsigned long long x = key[i], y = key[p];
                        if (((i & k) == 0) == (x > y)) {
                            key[i] = y;
                            key[p] = x;
                        }
                    }
                }
                __syncthreads();
            }
        }
        for (int i = threadIdx.x; i < S; i += blockDim.x) {
            const unsigned l = (unsigned)(key[i] >> 32);
            if (i > 0 && (unsigned)(key[i - 1] >> 32) == l) continue;
            float tot = 0.f;
            for (int r = i; r < S && (unsigned)(key[r] >> 32) == l; ++r) tot += occ[(unsigned)key[r]];
            d[l] = __float2bfloat16(scale * (expf(lp[l]) - tot));
        }
    }
}

const char* ctc_launch(cudaStream_t st, const float* logp, int ldl, int B, int T, int V, const int* in_len, const long long* targets,
                       int ldt, const int* tgt_len, int max_tgt, int blank, float* nll, float* loss, float* ws, bf16* dlogits, int ldd,
                       float grad_scale, const float* scale_dev) {
    if (B < 1 || T < 1 || V < 2) return "ctc: empty problem";
    if (max_tgt < 0 || 2 * max_tgt + 1 > CTC_SMAX_LONG) return "ctc: targets longer than 1023 labels are not supported";
    if (blank < 0 || blank >= V) return "ctc: bad blank id";
    const int S_ws = 2 * max_tgt + 1;
    const bool lng = S_ws > CTC_SMAX;
    const char* err;
    if ((err = lng ? launch<ctc_alpha_beta_kernel<CTC_SMAX_LONG, 1024>>(B, 1024, 0, st, logp, ldl, T, in_len, targets, ldt, tgt_len,
                                                                        blank, V, nll, ws, S_ws)
                   : launch<ctc_alpha_beta_kernel<CTC_SMAX, 160>>(B, 160, 0, st, logp, ldl, T, in_len, targets, ldt, tgt_len, blank,
                                                                  V, nll, ws, S_ws)))
        return err;
    if ((err = launch<ctc_mean_kernel>(1, 256, 0, st, nll, tgt_len, B, loss))) return err;
    if (!dlogits) return nullptr;
    return lng ? launch<ctc_grad_kernel<CTC_SMAX_LONG, true>>(B * T, 256, 0, st, logp, ldl, T, V, in_len, targets, ldt, tgt_len, blank,
                                                              nll, ws, S_ws, B, grad_scale, dlogits, ldd, scale_dev)
               : launch<ctc_grad_kernel<CTC_SMAX, false>>(B * T, 256, 0, st, logp, ldl, T, V, in_len, targets, ldt, tgt_len, blank,
                                                          nll, ws, S_ws, B, grad_scale, dlogits, ldd, scale_dev);
}

}  // namespace otb
