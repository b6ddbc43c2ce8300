// CTC rescoring of an attention n-best (DESIGN.md 4.18): out[r] = log p_ctc(target_r | x_b), b = r / K, of B*K target rows
// over the utterance's shared log-prob matrix (no per-row copy of it).
//   ctc_nbest_score_kernel  one CTA per target row, the K rows of an utterance in adjacent CTAs (they read the same frames,
//                           so the per-frame label gather is served by L2): the forward pass over the trellis
//                           (ctc_trellis.cuh) in the log domain and in fp32.  Each thread keeps the emission log-probs of
//                           its states for the next PF frames in flight, so the gather's L2 latency is not paid at every
//                           barrier.  Forward only: no beta, no [rows, T, S] scratch.
// L is the number of labels before the row's first negative entry.  A row gets -inf when no alignment exists: a label equal
// to the blank or outside [0, V), an utterance with no frames, or too few frames for the labels and their repeats.
#include <math.h>

#include "ctc_trellis.cuh"
#include "launch.cuh"
#include "otb_internal.h"

namespace otb {

static constexpr int CTC_SCORE_MAX_LABELS = 1024;   // max_len 1023 tokens + the closing <S/E>: S <= 2049
static constexpr int CTC_SCORE_PF = 4;              // frames of emission log-probs in flight per state

template <int NT, int SPT>
__global__ void __launch_bounds__(NT) ctc_nbest_score_kernel(const float* __restrict__ logp, int ld, int T, int V,
                                                             const int* __restrict__ in_len, const int* __restrict__ targets,
                                                             int K, int Lp, int blank, float* __restrict__ out) {
    constexpr int SMAX = NT * SPT;
    __shared__ float buf[2][SMAX];
    __shared__ int len;
    const int r = blockIdx.x, b = r / K;
    const int* y = targets + (size_t)r * Lp;
    if (threadIdx.x == 0) len = Lp;
    __syncthreads();
    for (int i = threadIdx.x; i < Lp; i += NT)
        if (y[i] < 0) atomicMin(&len, i);
    __syncthreads();
    const int L = len;
    bool bad = false;
    for (int i = threadIdx.x; i < L; i += NT) bad |= (y[i] == blank || y[i] >= V);
    const int Tb = min(in_len[b], T);
    if (__syncthreads_or(bad) || Tb < 1) {
        if (threadIdx.x == 0) out[r] = -INFINITY;
        return;
    }
    const int S = 2 * L + 1;
    const float* lp = logp + (size_t)b * T * ld;
    const auto label = [&](int i) { return y[i]; };
    unsigned col[SPT];
    bool skip[SPT];
    float e[CTC_SCORE_PF][SPT];     // e[d][j]: emission of state j at the frame the d-th step of an unrolled round reads
#pragma unroll
    for (int j = 0; j < SPT; ++j) {
        const int s = trellis_state(j, NT);
        col[j] = trellis_col(s, S, blank, label);
        skip[j] = trellis_skip(s, S, blank, label);
        if (s < S) buf[0][s] = s == 0 ? 0.f : -INFINITY;      // frame -1
#pragma unroll
        for (int d = 0; d < CTC_SCORE_PF; ++d) e[d][j] = (s < S && d < Tb) ? lp[(size_t)d * ld + col[j]] : 0.f;
    }
    __syncthreads();
    int cur = 0;
    for (int t0 = 0; t0 < Tb; t0 += CTC_SCORE_PF) {
#pragma unroll
        for (int d = 0; d < CTC_SCORE_PF; ++d) {
            const int t = t0 + d;
            if (t >= Tb) break;        // uniform over the CTA
            trellis_step<TrellisLogAdd>(buf, cur, NT, S, skip, [&](int j) {
                const float em = e[d][j];
                if (t + CTC_SCORE_PF < Tb) e[d][j] = lp[(size_t)(t + CTC_SCORE_PF) * ld + col[j]];
                return em;
            }, [](int, int, TrellisLogAdd, float) {});
        }
    }
    if (threadIdx.x == 0) out[r] = trellis_log_total(buf[cur], S);
}

const char* ctc_nbest_score_launch(cudaStream_t st, const float* logp, int ld, int B, int T, int V, const int* in_len,
                                   const int* targets, int K, int Lp, int blank, float* out) {
    if (B < 1 || T < 1 || V < 1 || K < 1) return "ctc_nbest_score: need B, T, V, K >= 1";
    if (ld < V) return "ctc_nbest_score: row pitch < V";
    if (Lp < 1 || Lp > CTC_SCORE_MAX_LABELS) return "ctc_nbest_score: target rows must be 1..1024 labels wide";
    if (blank < 0 || blank >= V) return "ctc_nbest_score: bad blank id";
    const int S = 2 * Lp + 1;
    const int rows = B * K;
    if (S <= 128)
        return launch<ctc_nbest_score_kernel<128, 1>>(rows, 128, 0, st, logp, ld, T, V, in_len, targets, K, Lp, blank, out);
    if (S <= 320)
        return launch<ctc_nbest_score_kernel<320, 1>>(rows, 320, 0, st, logp, ld, T, V, in_len, targets, K, Lp, blank, out);
    return launch<ctc_nbest_score_kernel<704, 3>>(rows, 704, 0, st, logp, ld, T, V, in_len, targets, K, Lp, blank, out);
}

}  // namespace otb
