// N-best rescoring (DESIGN.md 4.10): the second pass that re-ranks a first pass's n-best by a teacher-forced model.
//   token_logprob_kernel   one warp per row of fp32 logits: out[r] = logits[r, target[r]] - logsumexp(logits[r, :V]), 0 where
//                          target[r] < 0 (such rows are not read).  The HBM-bound pass: each row is read once, as float4,
//                          with an online max / sum-exp, and no [rows, V] log-softmax is ever written.  Lane i folds the
//                          float4s i, i + 32, ... in that order and the lanes combine by a fixed xor tree, so the result
//                          does not depend on scheduling: two calls are bit-identical.
//   nbest_rescore_kernel   one warp per utterance, lane k = first-pass hypothesis k (K <= 32): the sum of each model's
//                          token log-probs in position order, duplicates of a better first-pass hypothesis dropped,
//                          s = s1 + weight * sum over models, a stable sort (dropped last, then descending s, then first-pass
//                          order) and the gather of the nbest ids, lengths and scores.
#include <math.h>

#include "launch.cuh"
#include "otb_internal.h"
#include "row_lse.cuh"

namespace otb {

static constexpr int TLP_WARPS = 8;
static constexpr int RESCORE_KMAX = 32;       // one lane per first-pass hypothesis

__global__ void __launch_bounds__(TLP_WARPS * 32) token_logprob_kernel(const float* __restrict__ logits, int ld, int rows, int V,
                                                                       const int* __restrict__ target, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * TLP_WARPS + (threadIdx.x >> 5);
    if (r >= rows) return;
    const int tgt = target[r];
    if (tgt < 0) {
        if (lane == 0) out[r] = 0.f;
        return;
    }
    const float* x = logits + (size_t)r * ld;
    float m, s;
    warp_row_lse(x, V, lane, m, s);
    if (lane == 0) out[r] = tgt < V ? (x[tgt] - m) - logf(s) : NAN;
}

__global__ void __launch_bounds__(32) nbest_rescore_kernel(const int* __restrict__ tgt, int Lp, const int* __restrict__ len,
                                                           const float* __restrict__ s1, const float* __restrict__ tok_lp, int M,
                                                           int B, int K, float weight, int nbest, int Lout, long long pad_id,
                                                           long long* __restrict__ ids, int* __restrict__ out_len,
                                                           float* __restrict__ out_score) {
    const int b = blockIdx.x, k = threadIdx.x;
    const bool live = k < K;
    const size_t h = (size_t)b * K + k;
    const int n = live ? len[h] : 0;
    bool dropped = !live;
    float s = -INFINITY;
    if (live) {
        for (int j = 0; j < k && !dropped; ++j) {
            const size_t hj = (size_t)b * K + j;
            if (len[hj] != n) continue;
            bool same = true;
            for (int t = 0; t < n && same; ++t) same = tgt[hj * Lp + t] == tgt[h * Lp + t];
            dropped = same;
        }
        if (!dropped) {
            // no contraction into FMAs: the sums are the plain left-to-right float sums a host restatement forms
            float total = 0.f;
            for (int mdl = 0; mdl < M; ++mdl) {
                const float* p = tok_lp + ((size_t)mdl * B * K + h) * Lp;
                float sm = 0.f;
                for (int t = 0; t <= n; ++t) sm = __fadd_rn(sm, p[t]);
                total = __fadd_rn(total, sm);
            }
            s = __fadd_rn(s1[h], __fmul_rn(weight, total));
        }
    }
    const float key = s != s ? -INFINITY : s;        // a NaN score ranks as -inf
    int rank = 0;
    for (int j = 0; j < K; ++j) {
        const float kj = __shfl_sync(0xffffffffu, key, j);
        const bool dj = __shfl_sync(0xffffffffu, dropped, j);
        rank += (dj != dropped) ? !dj : (kj > key || (kj == key && j < k));
    }
    if (live && rank < nbest) {
        const size_t o = (size_t)b * nbest + rank;
        const int keep = dropped ? 0 : min(n, Lout);
        out_score[o] = s;
        out_len[o] = keep;
        long long* row = ids + o * Lout;
        for (int t = 0; t < Lout; ++t) row[t] = t < keep ? (long long)tgt[h * Lp + t] : pad_id;
    }
}

const char* token_logprob_launch(cudaStream_t stream, const float* logits, int ld, int rows, int V, const int* target, float* out) {
    if (rows < 0 || V < 1 || ld < V) return "token_logprob: need rows >= 0, V >= 1 and ld >= V";
    if (ld % 4 || reinterpret_cast<uintptr_t>(logits) % 16) return "token_logprob: rows must be 16-byte aligned (ld % 4 == 0)";
    if (rows == 0) return nullptr;
    return launch<token_logprob_kernel>((rows + TLP_WARPS - 1) / TLP_WARPS, TLP_WARPS * 32, 0, stream, logits, ld, rows, V, target,
                                        out);
}

const char* nbest_rescore_launch(cudaStream_t stream, const int* tgt, int Lp, const int* len, const float* s1, const float* tok_lp,
                                 int M, int B, int K, float weight, int nbest, int Lout, long long pad_id, long long* ids,
                                 int* out_len, float* out_score) {
    if (B < 1 || K < 1 || K > RESCORE_KMAX) return "nbest_rescore: need B >= 1 and 1 <= K <= 32";
    if (nbest < 1 || nbest > K) return "nbest_rescore: need 1 <= nbest <= K";
    if (Lp < 1 || Lout < 1 || M < 0) return "nbest_rescore: need Lp >= 1, Lout >= 1 and M >= 0";
    return launch<nbest_rescore_kernel>(B, 32, 0, stream, tgt, Lp, len, s1, tok_lp, M, B, K, weight, nbest, Lout, pad_id, ids,
                                        out_len, out_score);
}

}  // namespace otb
