// CTC decoding of CTCRecognizer (otrans/recognize/ctc.py) on the head's fp32 logits [B T', ld]:
//   ctc_frame_topk_kernel    one CTA per frame: log-sum-exp of the row and its K best tokens as log-probs (ties to the lower
//                            index); frames past the utterance's length, and ranks a row of NaN logits cannot fill, get
//                            id -1 / -inf.  The HBM-bound pass: the logits are read once, into shared memory, where each
//                            thread owns the columns i = tid (mod blockDim).
//   ctc_greedy_kernel        one CTA per utterance: recognize_greedy (recognize/ctc.py:38-58) on the top-1 ids -- a frame
//                            is kept unless its token is blank / PAD or equals the previous frame's token -- compacted with
//                            a ballot prefix sum; the score is the best path's log-prob.
//   ctc_prefix_beam_kernel   one CTA per utterance, the whole search in one launch: the CTC prefix beam search of ctcdecode
//                            without a scorer, over each frame's top-K tokens.  DESIGN.md 4.7 states the rules.
//   ctc_prefix_beam_step_kernel  one CTA per utterance, ONE frame of the same search with a neural LM as ctcdecode's scorer
//                            (DESIGN.md 4.19): the frame index comes from a device counter and the slots live in global
//                            memory between launches, so the frame and the LM step after it replay as one CUDA graph.
//   ctc_lm_carry_kernel      the LM rows and state of the fused search follow its slots (gather by source slot / select).
#include <math.h>
#include <stdint.h>

#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

static constexpr int TOPK_THREADS = 256;
static constexpr int BEAM_THREADS = 256;
static constexpr int CTC_TOPK_MAX = 64;
static constexpr int CTC_BEAM_MAX = 16;
static constexpr int CTC_CAND_MAX = CTC_BEAM_MAX * (CTC_TOPK_MAX + 1);
static constexpr int CTC_V_MAX = 50000;      // the frame row is staged in shared memory

// (v, i) beats (bv, bi): the larger value, the lower index on ties.  NaN (a removed entry) never wins.
__device__ __forceinline__ bool beats(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

__device__ __forceinline__ void warp_argmax(float& v, int& i) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float v2 = __shfl_xor_sync(0xffffffffu, v, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, i, o);
        if (beats(v2, i2, v, i)) { v = v2; i = i2; }
    }
}

// Block-wide argmax of every thread's (v, i); red_v / red_i [NW] are this round's slots (the caller alternates two sets,
// so one barrier per round suffices).  Every thread returns the winner.
template <int NW>
__device__ __forceinline__ void block_argmax(float& v, int& i, float* red_v, int* red_i) {
    warp_argmax(v, i);
    if ((threadIdx.x & 31) == 0) { red_v[threadIdx.x >> 5] = v; red_i[threadIdx.x >> 5] = i; }
    __syncthreads();
    v = red_v[0];
    i = red_i[0];
#pragma unroll
    for (int w = 1; w < NW; ++w)
        if (beats(red_v[w], red_i[w], v, i)) { v = red_v[w]; i = red_i[w]; }
}

template <int NW>
__device__ __forceinline__ float block_reduce(float v, float* red, bool is_max) {
    v = is_max ? warp_max(v) : warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = red[0];
#pragma unroll
    for (int w = 1; w < NW; ++w) r = is_max ? fmaxf(r, red[w]) : r + red[w];
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(TOPK_THREADS) ctc_frame_topk_kernel(const float* __restrict__ logits, int ld, int V, int T,
                                                                      const int* __restrict__ in_len, int K,
                                                                      float* __restrict__ top_lp, int* __restrict__ top_id) {
    constexpr int NW = TOPK_THREADS / 32;
    extern __shared__ float row[];
    __shared__ float red[NW];
    __shared__ float red_v[2][NW];
    __shared__ int red_i[2][NW];
    const int r = blockIdx.x, tid = threadIdx.x;
    float* olp = top_lp + (size_t)r * K;
    int* oid = top_id + (size_t)r * K;
    if (r % T >= in_len[r / T]) {
        for (int k = tid; k < K; k += TOPK_THREADS) { olp[k] = -INFINITY; oid[k] = -1; }
        return;
    }
    const float* x = logits + (size_t)r * ld;
    float m = -INFINITY;
    for (int i = tid; i < V; i += TOPK_THREADS) {
        const float v = x[i];
        row[i] = v;                   // only this thread reads row[i] again: no barrier needed for the row
        m = fmaxf(m, v);
    }
    m = block_reduce<NW>(m, red, true);
    float s = 0.f;
    for (int i = tid; i < V; i += TOPK_THREADS) s += expf(row[i] - m);
    const float lse = m + logf(block_reduce<NW>(s, red, false));
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < V; i += TOPK_THREADS)
        if (beats(row[i], i, bv, bi)) { bv = row[i]; bi = i; }
    for (int k = 0; k < K; ++k) {
        float v = bv;
        int i = bi;
        block_argmax<NW>(v, i, red_v[k & 1], red_i[k & 1]);
        const bool found = i < V;            // false once only NaN columns are left (a row with fewer than K numbers)
        if (tid == 0) { olp[k] = found ? v - lse : -INFINITY; oid[k] = found ? i : -1; }
        if (found && i % TOPK_THREADS == tid) {       // the owner removes the winner and rescans its columns
            row[i] = NAN;
            bv = -INFINITY;
            bi = 0x7fffffff;
            for (int j = tid; j < V; j += TOPK_THREADS)
                if (beats(row[j], j, bv, bi)) { bv = row[j]; bi = j; }
        }
    }
}

__global__ void __launch_bounds__(256) ctc_greedy_kernel(const float* __restrict__ top_lp, const int* __restrict__ top_id, int ldk,
                                                         int T, const int* __restrict__ in_len, int blank, int* __restrict__ ids,
                                                         int* __restrict__ lengths, float* __restrict__ scores) {
    constexpr int NW = 256 / 32;
    __shared__ int cnt[NW];
    __shared__ float red[NW];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = min(in_len[b], T);
    const size_t row0 = (size_t)b * T;
    int* out = ids + row0;
    int base = 0;
    float s = 0.f;
    for (int t0 = 0; t0 < n; t0 += 256) {
        const int t = t0 + tid;
        int k = 0;
        bool keep = false;
        if (t < n) {
            k = top_id[(row0 + t) * ldk];
            const int prev = t == 0 ? 0 : top_id[(row0 + t - 1) * ldk];      // last_k starts at PAD (0)
            keep = k != prev && k > 0 && k != blank;          // k < 0: no token (a row without numbers)
            s += top_lp[(row0 + t) * ldk];
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) cnt[warp] = __popc(bal);
        __syncthreads();
        int off = base, tot = 0;
#pragma unroll
        for (int w = 0; w < NW; ++w) {
            off += w < warp ? cnt[w] : 0;
            tot += cnt[w];
        }
        if (keep) out[off + __popc(bal & ((1u << lane) - 1u))] = k;
        base += tot;
        __syncthreads();
    }
    for (int t = base + tid; t < T; t += 256) out[t] = 0;
    s = block_reduce<NW>(s, red, false);
    if (tid == 0) {
        lengths[b] = base;
        scores[b] = s;
    }
}

// Node table of the search: nodes[b][id] = (parent id, token); id 0 is the empty prefix, a prefix that enters the beam at
// frame t in slot s gets id 1 + t * beam + s.  Written and read by the same CTA: plain (coherent) loads, no __restrict__.
// Two prefixes of equal length are the same string when their chains agree token by token.
__device__ bool same_prefix(const int2* nodes, int a, int c) {
    while (a != c) {
        const int2 na = nodes[a], nc = nodes[c];
        if (na.y != nc.y) return false;
        a = na.x;
        c = nc.x;
    }
    return true;
}

struct BeamSlots {
    int node[CTC_BEAM_MAX], par[CTC_BEAM_MAX], last[CTC_BEAM_MAX], len[CTC_BEAM_MAX];
    float pb[CTC_BEAM_MAX], pnb[CTC_BEAM_MAX], tot[CTC_BEAM_MAX];
    float lml[CTC_BEAM_MAX];     // LM-fused search: log p_lm(last | prefix minus last), stored when the prefix is created
};

// Shared scratch of one frame of the search.
struct FrameScratch {
    int s_id[CTC_TOPK_MAX];
    float s_lp[CTC_TOPK_MAX];
    unsigned char eq[CTC_BEAM_MAX][CTC_BEAM_MAX];     // eq[q][i]: slot q's prefix minus its last token == slot i's
    float rep_lp[CTC_BEAM_MAX], stay_pb[CTC_BEAM_MAX], stay_pnb[CTC_BEAM_MAX];
    float cand[CTC_CAND_MAX];
    int sel[CTC_BEAM_MAX];
    float sel_score[CTC_BEAM_MAX];
    float red_v[2][BEAM_THREADS / 32];
    int red_i[2][BEAM_THREADS / 32];
    float blank_lp;
    int n_sel;
};

// The LM term of a fused search (DESIGN.md 4.19): lm_w * lm + beta, two separately rounded operations; with lm_w 0 the
// LM row is not read, so the term is beta exactly (0 * -inf would be NaN).
__device__ __forceinline__ float lm_term(float lm_w, float beta, float lm) {
    return lm_w == 0.f ? beta : __fadd_rn(__fmul_rn(lm_w, lm), beta);
}

// One frame t of the prefix beam search of utterance b (DESIGN.md 4.7): slots c (n of them) -> slots nx, in selection
// order; returns their number.  sm.sel[s] = i * (K + 1) + r names where new slot s came from (r = 0: kept slot i, else
// slot i extended by the frame's top-K token r - 1).  LM: the fused search of DESIGN.md 4.19, lm the LM rows of the
// utterance's slots (row i at lm + i * ld_lm).  Every thread returns after a barrier.
template <bool LM>
__device__ int prefix_beam_frame(const BeamSlots& c, BeamSlots& nx, int n, const float* __restrict__ lp_row,
                                 const int* __restrict__ id_row, int K, int blank, int W, int t, int2* nodes, FrameScratch& sm,
                                 const float* __restrict__ lm, int ld_lm, float lm_w, float beta) {
    constexpr int NW = BEAM_THREADS / 32;
    const int tid = threadIdx.x;
    const int S = K + 1;                      // candidate j = slot * (K + 1) + r: r = 0 keeps the slot, r = 1 + k extends it by top-K k
    if (tid < K) { sm.s_id[tid] = id_row[tid]; sm.s_lp[tid] = lp_row[tid]; }
    __syncthreads();
    // ---- which slot is which slot's parent; the blank's and each slot's last token's log-prob this frame
    for (int p = tid; p < n * n; p += BEAM_THREADS) {
        const int q = p / n, i = p % n;
        sm.eq[q][i] = c.len[q] == c.len[i] + 1 && same_prefix(nodes, c.par[q], c.node[i]);
    }
    if (tid < n) {
        float v = -INFINITY;
        for (int k = 0; k < K; ++k) if (sm.s_id[k] == c.last[tid]) v = sm.s_lp[k];
        sm.rep_lp[tid] = v;
    }
    if (tid == BEAM_THREADS - 1) {
        float v = -INFINITY;
        for (int k = 0; k < K; ++k) if (sm.s_id[k] == blank) v = sm.s_lp[k];
        sm.blank_lp = v;
    }
    __syncthreads();
    // ---- candidates: every slot kept, every slot extended by every top-K token
    for (int j = tid; j < n * S; j += BEAM_THREADS) {
        const int i = j / S, r = j % S;
        float sc = -INFINITY;
        if (r == 0) {
            // blank keeps the prefix (p_b); repeating its last token keeps it (p_nb, from p_nb only); and the prefix
            // may also be reached by extending its parent slot (merge; with an LM it adds the term of the last token)
            const float pb = sm.blank_lp == -INFINITY ? -INFINITY : c.tot[i] + sm.blank_lp;
            float pnb = (sm.rep_lp[i] == -INFINITY || c.pnb[i] == -INFINITY) ? -INFINITY : c.pnb[i] + sm.rep_lp[i];
            for (int p = 0; p < n; ++p) {
                if (!sm.eq[i][p] || sm.rep_lp[i] == -INFINITY) continue;
                const float from = c.last[i] == c.last[p] ? c.pb[p] : c.tot[p];
                if (from == -INFINITY) continue;
                if constexpr (LM) pnb = log_add(pnb, (from + sm.rep_lp[i]) + lm_term(lm_w, beta, c.lml[i]));
                else pnb = log_add(pnb, from + sm.rep_lp[i]);
            }
            sm.stay_pb[i] = pb;
            sm.stay_pnb[i] = pnb;
            sc = log_add(pb, pnb);
        } else {
            const int tok = sm.s_id[r - 1];
            bool merged = tok == blank || tok < 0;
            for (int q = 0; q < n && !merged; ++q) merged = sm.eq[q][i] && c.last[q] == tok;
            if (!merged) {
                // repeating the last token reaches a new prefix through a blank only (p_b)
                const float from = tok == c.last[i] ? c.pb[i] : c.tot[i];
                sc = from == -INFINITY ? -INFINITY : from + sm.s_lp[r - 1];
                if constexpr (LM)
                    if (sc != -INFINITY) sc = sc + lm_term(lm_w, beta, lm_w == 0.f ? 0.f : lm[(size_t)i * ld_lm + tok]);
            }
        }
        sm.cand[j] = sc;
    }
    __syncthreads();
    // ---- keep the W best by (score desc, candidate index asc); -inf never enters the beam
    float bv = -INFINITY;
    int bj = 0x7fffffff;
    for (int j = tid; j < n * S; j += BEAM_THREADS)
        if (beats(sm.cand[j], j, bv, bj)) { bv = sm.cand[j]; bj = j; }
    int ns = 0;
    for (; ns < W; ++ns) {
        float v = bv;
        int j = bj;
        block_argmax<NW>(v, j, sm.red_v[ns & 1], sm.red_i[ns & 1]);
        if (v == -INFINITY) break;
        if (tid == 0) { sm.sel[ns] = j; sm.sel_score[ns] = v; }
        if (j % BEAM_THREADS == tid) {
            sm.cand[j] = NAN;
            bv = -INFINITY;
            bj = 0x7fffffff;
            for (int jj = tid; jj < n * S; jj += BEAM_THREADS)
                if (beats(sm.cand[jj], jj, bv, bj)) { bv = sm.cand[jj]; bj = jj; }
        }
    }
    if (tid == 0) sm.n_sel = ns;
    __syncthreads();
    // ---- the next beam, in selection order
    const int n_sel = sm.n_sel;
    if (tid < n_sel) {
        const int j = sm.sel[tid], i = j / S, r = j % S;
        if (r == 0) {
            nx.node[tid] = c.node[i]; nx.par[tid] = c.par[i]; nx.last[tid] = c.last[i]; nx.len[tid] = c.len[i];
            nx.pb[tid] = sm.stay_pb[i]; nx.pnb[tid] = sm.stay_pnb[i];
            if constexpr (LM) nx.lml[tid] = c.lml[i];
        } else {
            const int id = 1 + t * W + tid, tok = sm.s_id[r - 1];
            nodes[id] = make_int2(c.node[i], tok);
            nx.node[tid] = id; nx.par[tid] = c.node[i]; nx.last[tid] = tok; nx.len[tid] = c.len[i] + 1;
            nx.pb[tid] = -INFINITY; nx.pnb[tid] = sm.sel_score[tid];
            if constexpr (LM) nx.lml[tid] = lm_w == 0.f ? 0.f : lm[(size_t)i * ld_lm + tok];
        }
        nx.tot[tid] = sm.sel_score[tid];
    }
    __syncthreads();
    return n_sel;
}

// The n-best of utterance b from its final slots c (n of them): slot s's tokens by walking its chain back; unused slots
// are empty with score -inf.
__device__ void prefix_beam_write_nbest(const BeamSlots& c, int n, int b, int W, int T, const int2* nodes, int* __restrict__ ids,
                                        int* __restrict__ lengths, float* __restrict__ scores) {
    const int tid = threadIdx.x;
    for (int s = tid; s < W; s += BEAM_THREADS) {
        int* out = ids + ((size_t)b * W + s) * T;
        const int L = s < n ? c.len[s] : 0;
        int id = s < n ? c.node[s] : 0;
        for (int p = L - 1; p >= 0; --p) {
            const int2 nd = nodes[id];
            out[p] = nd.y;
            id = nd.x;
        }
        lengths[b * W + s] = L;
        scores[b * W + s] = s < n ? c.tot[s] : -INFINITY;
    }
    for (int s = 0; s < W; ++s) {
        const int L = s < n ? c.len[s] : 0;
        int* out = ids + ((size_t)b * W + s) * T;
        for (int p = L + tid; p < T; p += BEAM_THREADS) out[p] = 0;
    }
}

__device__ __forceinline__ void empty_beam(BeamSlots& c, int2* nodes) {
    nodes[0] = make_int2(-1, -1);
    c.node[0] = 0; c.par[0] = -1; c.last[0] = -1; c.len[0] = 0;
    c.pb[0] = 0.f; c.pnb[0] = -INFINITY; c.tot[0] = 0.f; c.lml[0] = 0.f;
}

__global__ void __launch_bounds__(BEAM_THREADS) ctc_prefix_beam_kernel(const float* __restrict__ top_lp, const int* __restrict__ top_id,
                                                                       int K, int T, const int* __restrict__ in_len, int blank, int W,
                                                                       int2* nodes_all, int* __restrict__ ids, int* __restrict__ lengths,
                                                                       float* __restrict__ scores) {
    __shared__ BeamSlots bs[2];
    __shared__ FrameScratch sm;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int Tb = min(in_len[b], T);
    int2* nodes = nodes_all + (size_t)b * (1 + (size_t)T * W);
    int cur = 0, n = 1;
    if (tid == 0) empty_beam(bs[0], nodes);
    __syncthreads();                          // the empty prefix is read by every thread, also when Tb == 0 skips the loop
    for (int t = 0; t < Tb; ++t) {
        const size_t row = (size_t)b * T + t;
        n = prefix_beam_frame<false>(bs[cur], bs[cur ^ 1], n, top_lp + row * K, top_id + row * K, K, blank, W, t, nodes, sm,
                                     nullptr, 0, 0.f, 0.f);
        cur ^= 1;
    }
    prefix_beam_write_nbest(bs[cur], n, b, W, T, nodes, ids, lengths, scores);
}

// ---- the LM-fused search, one frame per launch (DESIGN.md 4.19) -------------------------------------------------------

// Slot state of one utterance between frames, in global memory.
struct GlobalSlots {
    BeamSlots s;
    int n;
};

__global__ void __launch_bounds__(BEAM_THREADS, 1) ctc_prefix_beam_step_kernel(const __grid_constant__ CtcStepArgs a) {
    __shared__ BeamSlots bs[2];
    __shared__ FrameScratch sm;
    __shared__ int s_t, s_n, s_src[CTC_BEAM_MAX], s_ext[CTC_BEAM_MAX], s_len[CTC_BEAM_MAX];
    const int b = blockIdx.x, tid = threadIdx.x, W = a.beam, T = a.T;
    if (tid == 0) s_t = *a.ctl;
    __syncthreads();
    const int t = s_t;
    const int Tb = min(a.in_len[b], T);
    const size_t n_nodes = 1 + (size_t)T * W;
    int2* nodes = reinterpret_cast<int2*>(a.nodes) + (size_t)b * n_nodes;
    GlobalSlots* gs = reinterpret_cast<GlobalSlots*>(a.slots);
    // ---- this frame's slots: the empty prefix at frame 0, else what the previous frame left (buffer t & 1)
    if (t == 0) {
        if (tid == 0) { empty_beam(bs[0], nodes); s_n = 1; }
    } else {
        const GlobalSlots& g = gs[(size_t)(t & 1) * gridDim.x + b];
        const int* src = reinterpret_cast<const int*>(&g.s);
        int* dst = reinterpret_cast<int*>(&bs[0]);
        for (int i = tid; i < (int)(sizeof(BeamSlots) / 4); i += BEAM_THREADS) dst[i] = src[i];
        if (tid == 0) s_n = g.n;
    }
    __syncthreads();
    int n = s_n;
    const int row0 = b * W;
    if (t < Tb) {
        const size_t row = (size_t)b * T + t;
        const int n_old = n;
        n = prefix_beam_frame<true>(bs[0], bs[1], n, a.top_lp + row * a.K, a.top_id + row * a.K, a.K, a.blank, W, t, nodes, sm,
                                    a.lm + (size_t)row0 * a.ld_lm, a.ld_lm, a.lm_w, a.beta);
        if (tid < W) {
            int i = tid, ext = 0, tok = bs[0].last[0];
            if (tid < n) {
                const int j = sm.sel[tid];
                i = j / (a.K + 1);
                ext = j % (a.K + 1) != 0;
                tok = bs[1].last[tid];
            } else if (tid < n_old) {
                tok = bs[0].last[tid];
            }
            s_src[tid] = i; s_ext[tid] = ext; s_len[tid] = tid < n_old || tid < n ? bs[0].len[i] : 0;
            a.src[row0 + tid] = row0 + i;
            a.ext[row0 + tid] = ext;
            a.tok[row0 + tid] = tok >= 0 ? tok : CTC_LM_BOS;
        }
    } else {
        // past the utterance's frames: every slot carries over unchanged
        for (int i = tid; i < (int)(sizeof(BeamSlots) / 4); i += BEAM_THREADS)
            reinterpret_cast<int*>(&bs[1])[i] = reinterpret_cast<const int*>(&bs[0])[i];
        if (tid < W) {
            s_src[tid] = tid; s_ext[tid] = 0; s_len[tid] = tid < n ? bs[0].len[tid] : 0;
            a.src[row0 + tid] = row0 + tid;
            a.ext[row0 + tid] = 0;
            a.tok[row0 + tid] = tid < n && bs[0].last[tid] >= 0 ? bs[0].last[tid] : CTC_LM_BOS;
        }
        __syncthreads();
    }
    // ---- the next frame's slots (buffer (t + 1) & 1)
    GlobalSlots& g = gs[(size_t)((t + 1) & 1) * gridDim.x + b];
    for (int i = tid; i < (int)(sizeof(BeamSlots) / 4); i += BEAM_THREADS)
        reinterpret_cast<int*>(&g.s)[i] = reinterpret_cast<const int*>(&bs[1])[i];
    if (tid == 0) g.n = n;
    __syncthreads();
    // ---- Transformer LM: each new slot's ancestry row (cache rows of its prefix's nodes, BOS at position 0) is its source
    // slot's, plus the new node when it extended; the row's query position is the new token's, -1 when there is nothing
    // to compute (kept prefix, or a position past the table)
    if (a.anc != nullptr) {
        const int L = a.Lpos;
        for (int s = 0; s < W; ++s) {
            if (s_src[s] == s) continue;                       // the row already holds its prefix
            const int* from = a.anc + (size_t)(row0 + s_src[s]) * L;
            int* to = a.anc_tmp + (size_t)(row0 + s) * L;
            for (int p = tid; p <= s_len[s] && p < L; p += BEAM_THREADS) to[p] = from[p];
        }
        __syncthreads();
        for (int s = 0; s < W; ++s) {
            if (s_src[s] == s) continue;
            const int* from = a.anc_tmp + (size_t)(row0 + s) * L;
            int* to = a.anc + (size_t)(row0 + s) * L;
            for (int p = tid; p <= s_len[s] && p < L; p += BEAM_THREADS) to[p] = from[p];
        }
        if (tid < W) {
            const int len = s_len[tid] + 1;
            const bool run = s_ext[tid] && len < L;
            if (run) a.anc[(size_t)(row0 + tid) * L + len] = (int)((size_t)b * n_nodes) + bs[1].node[tid];
            a.pos[row0 + tid] = run ? len : -1;
        }
    }
    if (t == T - 1) prefix_beam_write_nbest(bs[1], n, b, W, T, nodes, a.ids, a.lengths, a.scores);
    // ---- the last CTA to finish moves the frame counter on (every CTA has read it by then)
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        if (atomicAdd(a.ctl + 1, 1) == (int)gridDim.x - 1) {
            a.ctl[1] = 0;
            a.ctl[0] = t + 1;
        }
    }
}

// The LM rows and state of the fused search follow its slots: dst[n] = a[n] where ext[n] (rows left as they are when a is
// null), else b[idx[n]] (b[n] without idx).  4-byte words, one CTA per row.
__global__ void __launch_bounds__(256) ctc_lm_carry_kernel(uint32_t* dst, int ldd, const uint32_t* a, int lda, const uint32_t* b,
                                                           int ldb, const int* __restrict__ idx, const int* __restrict__ ext,
                                                           int width) {
    const int n = blockIdx.x;
    const bool from_a = ext != nullptr && ext[n] != 0;
    if (from_a && a == nullptr) return;
    const uint32_t* src = from_a ? a + (size_t)n * lda : b + (size_t)(idx != nullptr ? idx[n] : n) * ldb;
    uint32_t* out = dst + (size_t)n * ldd;
    if (((ldd | (from_a ? lda : ldb) | width) & 3) == 0 && ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(out)) & 15) == 0) {
        for (int i = threadIdx.x * 4; i < width; i += 1024)
            *reinterpret_cast<uint4*>(out + i) = *reinterpret_cast<const uint4*>(src + i);
        return;
    }
    for (int i = threadIdx.x; i < width; i += 256) out[i] = src[i];
}

const char* ctc_frame_topk_launch(cudaStream_t st, const float* logits, int ld, int B, int T, int V, const int* in_len, int K,
                                  float* top_lp, int* top_id) {
    if (B < 1 || T < 1 || V < 1) return "empty problem";
    if (K < 1 || K > CTC_TOPK_MAX || K > V) return "K must be in 1..min(64, V)";
    if (V > CTC_V_MAX) return "vocabularies above 50000 tokens are not supported";
    return launch<ctc_frame_topk_kernel>(B * T, TOPK_THREADS, (size_t)V * sizeof(float), st, logits, ld, V, T, in_len, K, top_lp,
                                         top_id);
}

const char* ctc_greedy_launch(cudaStream_t st, const float* top_lp, const int* top_id, int ldk, int B, int T, const int* in_len,
                              int blank, int* ids, int* lengths, float* scores) {
    if (B < 1 || T < 1 || ldk < 1) return "empty problem";
    return launch<ctc_greedy_kernel>(B, 256, 0, st, top_lp, top_id, ldk, T, in_len, blank, ids, lengths, scores);
}

const char* ctc_prefix_beam_step_launch(cudaStream_t st, const CtcStepArgs& a, int B) {
    if (B < 1 || a.T < 1) return "empty problem";
    if (a.K < 1 || a.K > CTC_TOPK_MAX) return "K must be in 1..64";
    if (a.beam < 1 || a.beam > CTC_BEAM_MAX) return "beam width must be in 1..16";
    if (a.anc != nullptr && (a.anc_tmp == nullptr || a.pos == nullptr || a.Lpos < 1)) return "anc needs anc_tmp, pos and Lpos";
    return launch<ctc_prefix_beam_step_kernel>(B, BEAM_THREADS, 0, st, a);
}

const char* ctc_lm_carry_launch(cudaStream_t st, void* dst, int ldd, const void* a, int lda, const void* b, int ldb, const int* idx,
                                const int* ext, int rows, int width) {
    if (rows < 1 || width < 1) return "empty problem";
    return launch<ctc_lm_carry_kernel>(rows, 256, 0, st, static_cast<uint32_t*>(dst), ldd, static_cast<const uint32_t*>(a), lda,
                                       static_cast<const uint32_t*>(b), ldb, idx, ext, width);
}

int ctc_prefix_beam_slots_bytes(int B) { return 2 * B * (int)sizeof(GlobalSlots); }

const char* ctc_prefix_beam_launch(cudaStream_t st, const float* top_lp, const int* top_id, int K, int B, int T, const int* in_len,
                                   int blank, int beam, int* nodes, int* ids, int* lengths, float* scores) {
    if (B < 1 || T < 1) return "empty problem";
    if (K < 1 || K > CTC_TOPK_MAX) return "K must be in 1..64";
    if (beam < 1 || beam > CTC_BEAM_MAX) return "beam width must be in 1..16";
    return launch<ctc_prefix_beam_kernel>(B, BEAM_THREADS, 0, st, top_lp, top_id, K, T, in_len, blank, beam,
                                          reinterpret_cast<int2*>(nodes), ids, lengths, scores);
}

}  // namespace otb
