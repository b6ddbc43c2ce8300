// CTC forced alignment: the best (Viterbi) path of each utterance through the CTC trellis of its target, on fp32 log-probs
// (or logits with a per-frame log-sum-exp).  One CTA per utterance; DESIGN.md 4.8 states the layout, tie-break and limits.
//
//   delta_t(s) = the best of s's predecessors in the trellis (ctc_trellis.cuh) at frame t - 1, + lp_t(l'_s)
//   end = S-1 unless delta(S-2) > delta(S-1); the path is walked back through the choices (0, 1 or 2 back) in bp.
#include <math.h>
#include <stdint.h>

#include "ctc_trellis.cuh"
#include "launch.cuh"
#include "otb_internal.h"

namespace otb {

static constexpr int ALIGN_LMAX = 1023;
static constexpr int ALIGN_SMAX = 2 * ALIGN_LMAX + 1;
static constexpr int ALIGN_PER_THREAD = 2;           // states per thread: 2047 states on 1024 threads
static constexpr int ALIGN_THREADS_MAX = 1024;

__global__ void __launch_bounds__(ALIGN_THREADS_MAX, 1) ctc_align_kernel(
    const float* __restrict__ rows, int ld, int T, int V, const float* __restrict__ lse, const int* __restrict__ in_len,
    const long long* __restrict__ targets, int ldt, const int* __restrict__ tgt_len, int max_tgt, int blank,
    uint8_t* bp_all, int* labels_all, float* __restrict__ frame_scores, int* __restrict__ spans, float* __restrict__ path_score) {
    __shared__ float delta[2][ALIGN_SMAX];
    __shared__ int end_state;
    const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const int L = tgt_len[b];
    const int Tb = max(0, min(in_len[b], T));
    const bool Lok = L >= 0 && L <= max_tgt && (L == 0 || Tb > 0);
    const int S = Lok ? 2 * L + 1 : 0, S_ws = 2 * max_tgt + 1;
    const long long* tg = targets + (size_t)b * ldt;
    const float* x = rows + (size_t)b * T * ld;
    const float* ls = lse ? lse + (size_t)b * T : nullptr;
    uint8_t* bp = bp_all + (size_t)b * T * S_ws;
    int* labels = labels_all + (size_t)b * T;       // holds the path's states until the last pass turns them into labels
    float* fsc = frame_scores + (size_t)b * T;
    int* sp = spans + (size_t)b * max_tgt * 2;

    bool bad = !Lok;
    for (int i = tid; i < (S >> 1); i += nt) {
        const long long v = tg[i];
        bad |= v < 0 || v >= V || v == blank;       // a blank or out-of-range token: no alignment exists
    }
    const auto label = [&](int i) { return (int)tg[i]; };
    unsigned col[ALIGN_PER_THREAD];
    bool skip[ALIGN_PER_THREAD];
#pragma unroll
    for (int k = 0; k < ALIGN_PER_THREAD; ++k) {
        const int s = trellis_state(k, nt);
        col[k] = trellis_col(s, S, blank, label);
        skip[k] = trellis_skip(s, S, blank, label);
        if (s < S) delta[0][s] = s == 0 ? 0.f : -INFINITY;       // frame -1
    }
    const bool ok = !__syncthreads_or(bad);
    int cur = 0;
    if (ok && Tb > 0) {
        float v[ALIGN_PER_THREAD], nv[ALIGN_PER_THREAD];
        float m = ls ? ls[0] : 0.f, nm = 0.f;
#pragma unroll
        for (int k = 0; k < ALIGN_PER_THREAD; ++k) v[k] = trellis_state(k, nt) < S ? x[col[k]] : 0.f;
        for (int t = 0; t < Tb; ++t) {
            // the gather of frame t + 1: only the columns of this thread's states, in flight across this frame's barrier
            if (t + 1 < Tb) {
                const float* xn = x + (size_t)(t + 1) * ld;
#pragma unroll
                for (int k = 0; k < ALIGN_PER_THREAD; ++k) nv[k] = trellis_state(k, nt) < S ? xn[col[k]] : 0.f;
                if (ls) nm = ls[t + 1];
            }
            trellis_step<TrellisMax>(delta, cur, nt, S, skip, [&](int k) { return v[k] - m; },
                                     [&](int, int s, TrellisMax c, float) { bp[(size_t)t * S_ws + s] = (uint8_t)c.c; });
#pragma unroll
            for (int k = 0; k < ALIGN_PER_THREAD; ++k) v[k] = nv[k];
            m = nm;
        }
    }
    // ---- the end state and the walk back (one thread: T_b dependent byte loads); spans of the odd states on the way
    if (tid == 0) {
        float score = ok && Tb == 0 ? 0.f : -INFINITY;      // L == 0 and no frames: the empty path
        int e = -1;
        if (ok && Tb > 0) {
            e = S - 1;
            if (S > 1 && delta[cur][S - 2] > delta[cur][S - 1]) e = S - 2;
            score = delta[cur][e];
            if (!(score > -INFINITY)) { score = -INFINITY; e = -1; }   // no alignment has a finite log-probability (or NaN)
        }
        path_score[b] = score;
        end_state = e;
        int s = e;
        for (int t = Tb - 1; t >= 0 && s >= 0; --t) {
            labels[t] = s;
            const int prev = t > 0 ? s - bp[(size_t)t * S_ws + s] : -1;
            if (s & 1) {
                if (t == Tb - 1 || labels[t + 1] != s) sp[(s >> 1) * 2 + 1] = t + 1;
                if (prev != s) sp[(s >> 1) * 2] = t;
            }
            s = prev;
        }
    }
    __syncthreads();
    // ---- states -> labels and frame scores; frames past the path and span slots past the target: -1 (-inf)
    const bool found = end_state >= 0;
    for (int t = tid; t < T; t += nt) {
        int lab = -1;
        float sc = -INFINITY;
        if (found && t < Tb) {
            const int s = labels[t];
            lab = (s & 1) ? (int)tg[s >> 1] : blank;
            sc = x[(size_t)t * ld + lab] - (ls ? ls[t] : 0.f);
        }
        labels[t] = lab;
        fsc[t] = sc;
    }
    for (int i = tid; i < max_tgt; i += nt)
        if (!found || i >= L) { sp[2 * i] = -1; sp[2 * i + 1] = -1; }
}

const char* ctc_align_launch(cudaStream_t st, const float* rows, int ld, int B, int T, int V, const float* lse, const int* in_len,
                             const long long* targets, int ldt, const int* tgt_len, int max_tgt, int blank, uint8_t* bp, int* labels,
                             float* frame_scores, int* spans, float* path_score) {
    if (B < 1 || T < 1 || V < 1) return "empty problem";
    if (max_tgt < 0 || max_tgt > ALIGN_LMAX) return "targets longer than 1023 tokens are not supported";
    if (blank < 0 || blank >= V) return "bad blank id";
    const int S = 2 * max_tgt + 1;
    const int threads = ((S + ALIGN_PER_THREAD - 1) / ALIGN_PER_THREAD + 31) / 32 * 32;
    return launch<ctc_align_kernel>(B, threads, 0, st, rows, ld, T, V, lse, in_len, targets, ldt, tgt_len, max_tgt, blank, bp, labels,
                                    frame_scores, spans, path_score);
}

}  // namespace otb
