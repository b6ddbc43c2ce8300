// Transducer beam search: alignment-length synchronous decoding (ALSD, Saon et al. 2020), DESIGN.md 4.22.  Utterance b
// holds K hypothesis slots, rows b K .. b K + K - 1 of every [B K, ...] array.  At search step i every live hypothesis
// (score > -inf) with u labels sits at frame t = i - u < T_b and takes exactly one lattice step: blank (frame t + 1) or one
// of its K' = min(K, V - 1) best labels (u + 1, same frame).
//   rnnt_beam_step_kernel    one CTA per utterance over its K (K' + 1) candidates: merging, the K best, the n-best F, the
//                            node table, termination and the n-best output.
//   rnnt_beam_gather_kernel  each new slot's predictor state (h, c, Pp) from its parent slot, and its current Ep row.
//   rnnt_beam_commit_kernel  the predictor's output where the slot took a label, the gathered state where it took blank.
#include <math.h>

#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

static constexpr int RNNT_BEAM_KMAX = 15;        // K + 1 <= otb_logsoftmax_topk's 16
static constexpr int RNNT_BEAM_THREADS = 256;    // >= K (K' + 1) = 240 candidates, one per thread

// Do the node chains a and c (of equal depth) spell the same labels?  Equal strings can sit on different nodes: a prefix
// that drops out of the beam and is formed again later gets a new node.
__device__ __forceinline__ bool same_chain(const int* __restrict__ par, const int* __restrict__ tok, int a, int c) {
    while (a != c) {
        if (tok[a] != tok[c]) return false;
        a = par[a];
        c = par[c];
    }
    return true;
}

// The end rule's bound of kept candidate c: its score, plus beta per label it may still take when beta > 0
__device__ __forceinline__ float end_bound(const float* c_sc, const int* s_u, int c, int KL, float beta, int max_len) {
    if (!(beta > 0.f)) return c_sc[c];
    const int a = c / (KL + 1), u = s_u[a] + (c - a * (KL + 1) > 0);
    return c_sc[c] + beta * (float)(max_len - u);
}

// Candidate c = j (K' + 1) + q of slot j: q = 0 blank, q >= 1 the q-th best label.  That index is the formation order the
// tie rule uses (parent slot ascending, blank before labels, labels in top-k order).
// LM fusion (DESIGN.md 4.22) changes no decision here: val already holds the fused label values.  beta > 0 (a bonus per
// label) only loosens the end bound to logsumexp(s + beta (max_len - u)).  lm_src / lm_ext (optional, i32 [B K]) tell the
// LM carry each new slot's parent row b K + par and whether it took a label; anc (optional, i32 [B K, Lpos], with anc_tmp
// the same size of scratch and lm_pos i32 [B K]) lists the LM cache rows b n_cap + node of each slot's labels from
// position 0 (<S/E>, node 0), and lm_pos is the new label's position u where the slot took one, -1 elsewhere.
__global__ void __launch_bounds__(RNNT_BEAM_THREADS, 1)
    rnnt_beam_step_kernel(const float* __restrict__ logp, int ldlp, const float* __restrict__ val, const int* __restrict__ idx,
                          int k1, int K, int W, int V, int T, int max_len, const int* __restrict__ t_len, float* __restrict__ score,
                          int* __restrict__ slot_u, int* __restrict__ frame, int* __restrict__ node, int* __restrict__ par,
                          long long* __restrict__ tok, int* __restrict__ node_par, int* __restrict__ node_tok, int n_cap,
                          int* __restrict__ n_nodes, float* __restrict__ f_score, int* __restrict__ f_node, int* __restrict__ f_u,
                          int* __restrict__ f_n, int* __restrict__ done, int* __restrict__ active, int* __restrict__ ids,
                          int* __restrict__ lengths, float* __restrict__ out_score, float beta, int* __restrict__ lm_src,
                          int* __restrict__ lm_ext, int* __restrict__ anc, int* __restrict__ anc_tmp, int* __restrict__ lm_pos,
                          int Lpos) {
    __shared__ float s_sc[RNNT_BEAM_KMAX], s_final[RNNT_BEAM_KMAX], s_merge[RNNT_BEAM_KMAX];
    __shared__ int s_u[RNNT_BEAM_KMAX], s_fr[RNNT_BEAM_KMAX], s_nd[RNNT_BEAM_KMAX], s_partner[RNNT_BEAM_KMAX];
    __shared__ int s_sel[RNNT_BEAM_KMAX], s_new_node[RNNT_BEAM_KMAX], s_from[RNNT_BEAM_KMAX], s_lab[RNNT_BEAM_KMAX];
    __shared__ float c_sc[RNNT_BEAM_THREADS];
    __shared__ int c_tok[RNNT_BEAM_THREADS];
    __shared__ int s_end;
    const int b = blockIdx.x, tid = threadIdx.x, row0 = b * K;
    if (done[b]) {              // ended: its slots keep their state (the carry kernels copy each slot onto itself)
        if (tid < K) {
            par[row0 + tid] = tid;
            tok[row0 + tid] = 0;
            if (lm_src) {
                lm_src[row0 + tid] = row0 + tid;
                lm_ext[row0 + tid] = 0;
            }
            if (anc) lm_pos[row0 + tid] = -1;
        }
        return;
    }
    const int Tb = min(t_len[b], T);
    const int KL = min(K, V - 1), n_cand = K * (KL + 1);
    int* const npar = node_par + (size_t)b * n_cap;
    int* const ntok = node_tok + (size_t)b * n_cap;
    if (tid < K) {
        s_sc[tid] = score[row0 + tid];
        s_u[tid] = slot_u[row0 + tid];
        s_fr[tid] = frame[row0 + tid];
        s_nd[tid] = node[row0 + tid];
        s_partner[tid] = -1;
        s_final[tid] = -INFINITY;
    }
    __syncthreads();

    // candidates: c_sc = -inf for none (an empty slot, a label past max_len, a final)
    const int j = tid / (KL + 1), q = tid - j * (KL + 1);
    const bool mine = tid < n_cand;
    float sc = -INFINITY;
    int ct = 0;
    if (mine && s_sc[j] > -INFINITY) {
        const size_t r = (size_t)row0 + j;
        if (q == 0) {
            sc = s_sc[j] + logp[r * ldlp];
            if (s_fr[j] + 1 == Tb) {            // blank at the last frame: a final, offered to F
                s_final[j] = sc;
                sc = -INFINITY;
            }
        } else if (s_u[j] < max_len) {
            int n = 0;
            for (int e = 0; e < k1; ++e) {
                const int id = idx[r * k1 + e];
                if (id != 0 && ++n == q) {
                    sc = s_sc[j] + val[r * k1 + e];
                    ct = id;
                    break;
                }
            }
        }
    }
    if (mine) {
        c_sc[tid] = sc;
        c_tok[tid] = ct;
    }
    __syncthreads();

    // merge: label candidate (j, ct) onto the live blank candidate of the slot a whose sequence is y_j + [ct].  Live
    // hypotheses are distinct strings, so each blank meets at most one label candidate and each label at most one blank.
    bool merged = false;
    if (mine && q > 0 && sc > -INFINITY) {
        for (int a = 0; a < K && !merged; ++a) {
            if (c_sc[a * (KL + 1)] > -INFINITY && s_u[a] == s_u[j] + 1 && ntok[s_nd[a]] == ct &&
                same_chain(npar, ntok, npar[s_nd[a]], s_nd[j])) {
                s_partner[a] = tid;
                merged = true;
            }
        }
    }
    __syncthreads();
    // the merged candidate takes the blank's place in the order: log-add in fp32, m + log1p(exp(-|a - b|))
    if (tid < K && s_partner[tid] >= 0) s_merge[tid] = log_add(c_sc[tid * (KL + 1)], c_sc[s_partner[tid]]);
    __syncthreads();
    if (mine && q == 0 && s_partner[j] >= 0) sc = s_merge[j];
    if (merged) sc = -INFINITY;
    __syncthreads();
    if (mine) c_sc[tid] = sc;
    __syncthreads();

    // the K best live candidates: rank = number of candidates ahead in (score descending, formation order)
    const bool live = mine && sc > -INFINITY;
    const int n_live = __syncthreads_count(live);
    if (live) {
        int rank = 0;
        for (int o = 0; o < n_cand; ++o) {
            const float v = c_sc[o];
            rank += (v > sc) || (v == sc && o < tid);
        }
        if (rank < K) s_sel[rank] = tid;
    }
    __syncthreads();
    const int n_sel = min(n_live, K);
    if (tid == 0) {
        // F: this step's finals in slot order, each after every entry of F it does not beat (earlier steps win ties)
        int nf = f_n[b];
        float* fs = f_score + (size_t)b * W;
        int* fn = f_node + (size_t)b * W;
        int* fu = f_u + (size_t)b * W;
        for (int a = 0; a < K; ++a) {
            const float v = s_final[a];
            if (v == -INFINITY) continue;
            int p = nf;
            while (p > 0 && fs[p - 1] < v) --p;
            if (p >= W) continue;
            for (int e = min(nf, W - 1); e > p; --e) {
                fs[e] = fs[e - 1];
                fn[e] = fn[e - 1];
                fu[e] = fu[e - 1];
            }
            fs[p] = v;
            fn[p] = s_nd[a];
            fu[p] = s_u[a];
            nf = min(nf + 1, W);
        }
        f_n[b] = nf;
        // a node for each kept label candidate, in rank order
        int nn = n_nodes[b];
        for (int r = 0; r < n_sel; ++r) {
            const int c = s_sel[r], a = c / (KL + 1);
            if (c - a * (KL + 1) == 0) {
                s_new_node[r] = s_nd[a];
            } else {
                npar[nn] = s_nd[a];
                ntok[nn] = c_tok[c];
                s_new_node[r] = nn++;
            }
        }
        n_nodes[b] = nn;
        // end: no live hypothesis, or F full and the live set's total probability no more than F's worst.  With a label
        // bonus beta > 0 a hypothesis can gain up to beta (max_len - u): the bound adds it (beta <= 0: the plain scores).
        bool end = n_sel == 0;
        if (!end && nf == W) {
            float m = -INFINITY, s = 0.f;
            for (int r = 0; r < n_sel; ++r) m = fmaxf(m, end_bound(c_sc, s_u, s_sel[r], KL, beta, max_len));
            for (int r = 0; r < n_sel; ++r) s += expf(end_bound(c_sc, s_u, s_sel[r], KL, beta, max_len) - m);
            end = m + logf(s) <= fs[W - 1];
        }
        s_end = end;
        if (end) {
            done[b] = 1;
            atomicSub(active, 1);
        }
    }
    __syncthreads();
    if (tid < K) {
        const size_t r = (size_t)row0 + tid;
        int a = tid, lab = 0;
        if (tid < n_sel) {
            const int c = s_sel[tid], qq = c - c / (KL + 1) * (KL + 1);
            a = c / (KL + 1);
            lab = qq > 0;
            score[r] = c_sc[c];
            slot_u[r] = s_u[a] + lab;
            frame[r] = s_fr[a] + (qq == 0);
            node[r] = s_new_node[tid];
            par[r] = a;
            tok[r] = lab ? c_tok[c] : 0;
        } else {            // empty: keeps its own (finite) predictor state and frame
            score[r] = -INFINITY;
            par[r] = tid;
            tok[r] = 0;
        }
        if (lm_src) {
            lm_src[r] = row0 + a;
            lm_ext[r] = lab;
        }
        s_from[tid] = a;
        s_lab[tid] = lab;
    }
    // Transformer LM: a slot's cache rows are its parent's (positions 0 .. u_parent), plus its new node's at u where it took a
    // label; copied through anc_tmp, since a parent's row can be a child's destination
    if (anc != nullptr) {
        __syncthreads();
        for (int s = 0; s < K; ++s) {
            const int a = s_from[s];
            if (a == s) continue;
            const int* from = anc + (size_t)(row0 + a) * Lpos;
            int* to = anc_tmp + (size_t)(row0 + s) * Lpos;
            for (int p = tid; p <= s_u[a]; p += RNNT_BEAM_THREADS) to[p] = from[p];
        }
        __syncthreads();
        for (int s = 0; s < K; ++s) {
            const int a = s_from[s];
            if (a == s) continue;
            const int* from = anc_tmp + (size_t)(row0 + s) * Lpos;
            int* to = anc + (size_t)(row0 + s) * Lpos;
            for (int p = tid; p <= s_u[a]; p += RNNT_BEAM_THREADS) to[p] = from[p];
        }
        if (tid < K) {
            const int u = s_u[s_from[tid]] + 1;
            const bool lab = s_lab[tid];
            if (lab) anc[(size_t)(row0 + tid) * Lpos + u] = b * n_cap + s_new_node[tid];
            lm_pos[row0 + tid] = lab ? u : -1;
        }
    }
    if (s_end) {            // the n-best, best first: ids padded with 0, unfilled entries length 0 and score -inf
        const int nf = f_n[b];
        for (int i = tid; i < W * max_len; i += RNNT_BEAM_THREADS) {
            const int w = i / max_len;
            if (w >= nf || i - w * max_len >= f_u[(size_t)b * W + w]) ids[(size_t)b * W * max_len + i] = 0;
        }
        if (tid < W) {
            const size_t o = (size_t)b * W + tid;
            lengths[o] = tid < nf ? f_u[o] : 0;
            out_score[o] = tid < nf ? f_score[o] : -INFINITY;
            if (tid < nf) {
                int nd = f_node[o];
                for (int p = f_u[o] - 1; p >= 0; --p) {
                    ids[o * max_len + p] = ntok[nd];
                    nd = npar[nd];
                }
            }
        }
    }
}

// One CTA per slot row r of utterance b = r / K: (h, c) [layers, B K, H] f32 and pp [B K, D] bf16 of row b K + par[r] into
// (hg, cg, ppg) row r; ep bf16 [B T, D] row b T + frame[r] into ep_cur row r.
__global__ void __launch_bounds__(128) rnnt_beam_gather_kernel(const int* __restrict__ par, const int* __restrict__ frame, int K,
                                                               int layers, int BK, int H, int D, int T, const float* __restrict__ h,
                                                               const float* __restrict__ c, const bf16* __restrict__ pp,
                                                               const bf16* __restrict__ ep, float* __restrict__ hg,
                                                               float* __restrict__ cg, bf16* __restrict__ ppg,
                                                               bf16* __restrict__ ep_cur) {
    const int r = blockIdx.x, b = r / K;
    const int src = b * K + par[r];
    for (int l = 0; l < layers; ++l) {
        const size_t o = ((size_t)l * BK + r) * H, s = ((size_t)l * BK + src) * H;
        for (int i = threadIdx.x; i < H; i += blockDim.x) {
            hg[o + i] = h[s + i];
            cg[o + i] = c[s + i];
        }
    }
    const int t = frame[r];
    const bf16* e = ep + ((size_t)b * T + t) * D;
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
        ppg[(size_t)r * D + i] = pp[(size_t)src * D + i];
        ep_cur[(size_t)r * D + i] = e[i];
    }
}

// (h, c, pp) row r = the predictor's output (hn, cn, ppn) where tok[r] is a label, else the gathered (hg, cg, ppg)
__global__ void __launch_bounds__(128) rnnt_beam_commit_kernel(const long long* __restrict__ tok, int layers, int BK, int H, int D,
                                                               const float* __restrict__ hg, const float* __restrict__ cg,
                                                               const bf16* __restrict__ ppg, const float* __restrict__ hn,
                                                               const float* __restrict__ cn, const bf16* __restrict__ ppn,
                                                               float* __restrict__ h, float* __restrict__ c, bf16* __restrict__ pp) {
    const int r = blockIdx.x;
    const bool label = tok[r] > 0;
    const float* hs = label ? hn : hg;
    const float* cs = label ? cn : cg;
    const bf16* ps = label ? ppn : ppg;
    for (int l = 0; l < layers; ++l) {
        const size_t o = ((size_t)l * BK + r) * H;
        for (int i = threadIdx.x; i < H; i += blockDim.x) {
            h[o + i] = hs[o + i];
            c[o + i] = cs[o + i];
        }
    }
    for (int i = threadIdx.x; i < D; i += blockDim.x) pp[(size_t)r * D + i] = ps[(size_t)r * D + i];
}

const char* rnnt_beam_step_launch(cudaStream_t st, const float* logp, int ldlp, const float* val, const int* idx, int k1, int B, int K,
                                  int W, int V, int T, int max_len, const int* t_len, float* score, int* slot_u, int* frame, int* node,
                                  int* par, long long* tok, int* node_par, int* node_tok, int n_cap, int* n_nodes, float* f_score,
                                  int* f_node, int* f_u, int* f_n, int* done, int* active, int* ids, int* lengths, float* out_score,
                                  float beta, int* lm_src, int* lm_ext, int* anc, int* anc_tmp, int* lm_pos, int Lpos) {
    if (B < 1 || T < 1) return "rnnt_beam_step: empty batch";
    if (K < 1 || K > RNNT_BEAM_KMAX) return "rnnt_beam_step: beam width K must be in [1, 15]";
    if (W < 1 || W > K) return "rnnt_beam_step: nbest W must be in [1, K]";
    if (V < 2) return "rnnt_beam_step: need V >= 2 (blank and a label)";
    if (k1 != min(K + 1, V)) return "rnnt_beam_step: the top-k list must hold min(K + 1, V) entries";
    if (ldlp < V) return "rnnt_beam_step: log-prob rows narrower than V";
    if (max_len < 1 || max_len > 1023) return "rnnt_beam_step: max_len must be in [1, 1023]";
    if ((long long)n_cap < (long long)K * (T + max_len) + 1) return "rnnt_beam_step: node table narrower than K (T + max_len) + 1";
    if ((lm_src == nullptr) != (lm_ext == nullptr)) return "rnnt_beam_step: lm_src and lm_ext go together";
    if (anc != nullptr && (anc_tmp == nullptr || lm_pos == nullptr || Lpos < max_len + 1))
        return "rnnt_beam_step: anc needs anc_tmp, lm_pos and Lpos >= max_len + 1";
    if ((long long)B * n_cap > 0x7fffffffLL) return "rnnt_beam_step: B n_cap must fit in 32 bits";
    return launch<rnnt_beam_step_kernel>(B, RNNT_BEAM_THREADS, 0, st, logp, ldlp, val, idx, k1, K, W, V, T, max_len, t_len, score,
                                         slot_u, frame, node, par, tok, node_par, node_tok, n_cap, n_nodes, f_score, f_node, f_u, f_n,
                                         done, active, ids, lengths, out_score, beta, lm_src, lm_ext, anc, anc_tmp, lm_pos, Lpos);
}

const char* rnnt_beam_gather_launch(cudaStream_t st, const int* par, const int* frame, int B, int K, int layers, int H, int D, int T,
                                    const float* h, const float* c, const bf16* pp, const bf16* ep, float* hg, float* cg, bf16* ppg,
                                    bf16* ep_cur) {
    if (B < 1 || K < 1 || layers < 1 || H < 1 || D < 1 || T < 1) return "rnnt_beam_gather: empty problem";
    return launch<rnnt_beam_gather_kernel>(B * K, 128, 0, st, par, frame, K, layers, B * K, H, D, T, h, c, pp, ep, hg, cg, ppg, ep_cur);
}

const char* rnnt_beam_commit_launch(cudaStream_t st, const long long* tok, int rows, int layers, int H, int D, const float* hg,
                                    const float* cg, const bf16* ppg, const float* hn, const float* cn, const bf16* ppn, float* h,
                                    float* c, bf16* pp) {
    if (rows < 1 || layers < 1 || H < 1 || D < 1) return "rnnt_beam_commit: empty problem";
    return launch<rnnt_beam_commit_kernel>(rows, 128, 0, st, tok, layers, rows, H, D, hg, cg, ppg, hn, cn, ppn, h, c, pp);
}

}  // namespace otb
