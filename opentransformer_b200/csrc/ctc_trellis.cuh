// The CTC trellis that the loss (csrc/ctc.cu), the n-best score (csrc/ctc_score.cu) and forced alignment
// (csrc/ctc_align.cu) run over: the S = 2 L + 1 states of the blank-extended label sequence, blank at even s and label s / 2
// at odd s.  State s comes from s and s - 1, and from s - 2 when its label is not the blank and differs from the label
// before it; the backward pass mirrors this (s, s + 1, and s + 2 when s + 2 may skip).
//
// One CTA per sequence; thread threadIdx.x owns the states s = threadIdx.x + j nt, j < SPT.  A frame's values live in one
// row of a double-buffered shared array: one barrier per frame.  Every recursion starts from a row one frame outside the
// sequence, 0 at the state the paths start from (0 forward, S - 1 backward) and -inf elsewhere, so its first frame is an
// ordinary step: log_add(-inf, 0) = max(-inf, 0) = 0 and 0 + x = x.
//
// The caller checks the labels; each kernel has its own policy for a bad one.
#pragma once

#include <math.h>

#include "ptx.cuh"

namespace otb {

__device__ __forceinline__ int trellis_state(int j, int nt) { return threadIdx.x + j * nt; }

// The column of the emissions that state s reads: its label at odd s, else (and past the last state) the blank.  Unsigned,
// so that adding it to a 64-bit row offset needs no sign-extended copy: the kernels that keep emissions in flight have no
// register to spare for one.
template <class Label>
__device__ __forceinline__ unsigned trellis_col(int s, int S, int blank, Label label) {
    return (unsigned)((s < S && (s & 1)) ? label(s >> 1) : blank);
}

// Whether state s may also come from s - 2 (never past the last state).
template <class Label>
__device__ __forceinline__ bool trellis_skip(int s, int S, int blank, Label label) {
    if (s >= S || !(s & 1) || s < 3) return false;
    const int l = label(s >> 1);
    return l != blank && l != label((s >> 1) - 1);
}

// The sum over paths (loss, score).  A state no path reaches stays -inf whatever its emission.
struct TrellisLogAdd {
    float v;
    __device__ __forceinline__ void take(float x, int) { v = log_add(v, x); }
    __device__ __forceinline__ float plus(float em) const { return v == -INFINITY ? -INFINITY : v + em; }
};

// The best path (alignment), and which predecessor gave it (0, 1 or 2 states back).  Ties prefer staying, then one back:
// a later predecessor must be strictly better.
struct TrellisMax {
    float v;
    int c = 0;
    __device__ __forceinline__ void take(float x, int k) {
        if (x > v) { v = x; c = k; }
    }
    __device__ __forceinline__ float plus(float em) const { return v + em; }
};

// One frame.  Each state s < S of this thread combines its value in the row buf[cur] with those of its predecessors there
// and adds its emission, emission(j), read first so that a load behind it overlaps the combine.  The new value goes to
// buf[cur ^ 1], and done(j, s, combined, value) may record more.  skip[j] says whether the state two back (two ahead when
// BACK) is a predecessor.  Then the rows swap behind one barrier.
template <class Combine, bool BACK = false, int SPT, int N, class Emission, class Done>
__device__ __forceinline__ void trellis_step(float (&buf)[2][N], int& cur, int nt, int S, const bool (&skip)[SPT],
                                             Emission emission, Done done) {
#pragma unroll
    for (int j = 0; j < SPT; ++j) {
        const int s = trellis_state(j, nt);
        if (s < S) {
            const float em = emission(j);
            Combine c{buf[cur][s]};
            if (BACK ? s + 1 < S : s >= 1) c.take(buf[cur][BACK ? s + 1 : s - 1], 1);
            if (skip[j]) c.take(buf[cur][BACK ? s + 2 : s - 2], 2);
            const float v = c.plus(em);
            buf[cur ^ 1][s] = v;
            done(j, s, c, v);
        }
    }
    cur ^= 1;
    __syncthreads();
}

// log p of all paths that end in the last label or the final blank, from the last frame's row.
__device__ __forceinline__ float trellis_log_total(const float* row, int S) {
    return S > 1 ? log_add(row[S - 1], row[S - 2]) : row[0];
}

}  // namespace otb
