// Batched beam-search step and finalisation on the device.
// Replaces the ~10 ATen launches + host sync per step of SpeechToTextRecognizer.decode_step
//   otrans/recognize/speech2text.py:102-153 (LM add, top-k per hypothesis, finished masking :156-192,
//   score add, top-k over beam^2, gather tokens/parents, EOS flags)
// and the tail of recognize() (:70-91: lengths, length penalty applied once, sort, n-best gather).
//
// Integer outputs (token ids, parent rows, top-k offsets) are bit-exact with the reference on
// tie-free inputs; ties are broken towards the LOWER index (torch.topk's tie order is
// implementation-defined).  Scores are fp32 and use the same additions as the reference.
//
// Device-resident search state (N = B * beam hypotheses):
//   tok_hist  i32 [Lmax, N]   token chosen at step s for (post-reorder) hypothesis n
//   par_hist  i32 [Lmax, N]   its parent row (global, pre-reorder) at step s
//   last_tok  i64 [N]         newest token of every hypothesis (decoder input of the next step)
//   scores    f32 [N], flag u8 [N]
//   anc       i32 [2, N, Lmax] ping-pong ancestry table used by the KV-cache attention
//   ctrl      i32 [4]: {step, done, ended_now, unused}
#include <math.h>

#include "beam_common.cuh"
#include "counter_rng.cuh"
#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

// one CTA per utterance, `beam` warps
__global__ void __launch_bounds__(KMAX * 32) beam_step_kernel(const float* __restrict__ logp, int ldl, int V,
                                                              const float* __restrict__ lm_logp, int ld_lm,
                                                              float lm_weight, BeamState st, long long* dbg_ktok,
                                                              int* dbg_offs, const float* __restrict__ pre_val,
                                                              const int* __restrict__ pre_idx) {
    __shared__ float c_val[KMAX * KMAX];
    __shared__ int c_tok[KMAX * KMAX];
    __shared__ float sel_v[KMAX];
    __shared__ int sel_i[KMAX];
    __shared__ float row_v[KMAX][KMAX];
    __shared__ int row_i[KMAX][KMAX];
    const int beam = st.beam;
    const int u = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (st.ctrl[1] || st.ctrl[0] >= st.Lmax) return;  // search already ended: state stays frozen (reference breaks out, speech2text.py:67)
    const int step = st.ctrl[0];

    // ---- phase 1: per-hypothesis top-k over the vocabulary (speech2text.py:112), finished masking (:114-115)
    if (warp < beam) {
        const int n = u * beam + warp;
        const bool fin = st.flag[n] != 0;
        if (fin) {
            if (lane < beam) {
                row_v[warp][lane] = (lane == 0) ? 0.f : -INFINITY;
                row_i[warp][lane] = (int)EOS_ID;
            }
        } else if (pre_val != nullptr) {
            if (lane < beam) {
                row_v[warp][lane] = pre_val[(size_t)n * beam + lane];
                row_i[warp][lane] = pre_idx[(size_t)n * beam + lane];
            }
        } else {
            const float* lp = logp + (size_t)n * ldl;
            const float* lm = lm_logp ? lm_logp + (size_t)n * ld_lm : nullptr;
            warp_topk([&](int idx) { return lm ? lp[idx] + lm_weight * lm[idx] : lp[idx]; }, V, beam, row_v[warp],
                      row_i[warp]);
        }
        __syncwarp();
        const float base = st.scores[n];
        if (lane < beam) {
            c_val[warp * beam + lane] = base + row_v[warp][lane];  // scores + last_k_scores (:118)
            c_tok[warp * beam + lane] = row_i[warp][lane];
            if (dbg_ktok) dbg_ktok[(size_t)n * beam + lane] = row_i[warp][lane];
        }
    }
    __syncthreads();
    // ---- phase 2: top-k over the beam*beam candidates of this utterance (:119-122)
    if (warp == 0) {
        warp_topk([&](int idx) { return c_val[idx]; }, beam * beam, beam, sel_v, sel_i);
    }
    __syncthreads();
    // ---- phase 3: gather tokens / parents, update state (:126-146)
    const int cur = step & 1, nxt = cur ^ 1;
    int ended = 0;
    for (int r = warp; r < beam; r += (blockDim.x >> 5)) {
        const int off = sel_i[r];
        const int parent = u * beam + off / beam;
        const int tok = c_tok[off];
        const int nn = u * beam + r;
        const int* a_old = st.anc + ((size_t)cur * st.N + parent) * st.Lmax;
        int* a_new = st.anc + ((size_t)nxt * st.N + nn) * st.Lmax;
        for (int s = lane; s < step; s += 32) a_new[s] = a_old[s];
        if (lane == 0) {
            a_new[step] = parent;
            st.tok_hist[(size_t)step * st.N + nn] = tok;
            st.par_hist[(size_t)step * st.N + nn] = parent;
            if (dbg_offs) dbg_offs[nn] = off;
        }
    }
    __syncthreads();  // every read of the old scores / flags of this utterance happened in phase 1
    if (threadIdx.x < beam) {
        const int r = threadIdx.x;
        const int nn = u * beam + r;
        const int tok = c_tok[sel_i[r]];
        st.scores[nn] = sel_v[r];
        st.last_tok[nn] = tok;
        st.flag[nn] = (tok == (int)EOS_ID) ? 1 : 0;
        ended = (tok == (int)EOS_ID) ? 1 : 0;
    }
    if (threadIdx.x < 32) {
        ended = (int)warp_sum((float)ended);
        if (threadIdx.x == 0) {
            if (ended) atomicAdd(&st.ctrl[2], ended);
            __threadfence();
            // last CTA of this step advances {step, done}: replaces a separate 1-thread kernel per step
            if (atomicAdd(&st.ctrl[3], 1) == (int)gridDim.x - 1) {
                const int total = atomicAdd(&st.ctrl[2], 0);
                st.ctrl[2] = 0;
                st.ctrl[3] = 0;
                __threadfence();
                if (total == st.N) st.ctrl[1] = 1;      // every hypothesis ended (speech2text.py:66-67)
                st.ctrl[0] = step + 1;
            }
        }
    }
}

const char* beam_step_launch(cudaStream_t stream, const float* logp, int ldl, int V, const float* lm_logp, int ld_lm,
                             float lm_weight, BeamState st, long long* dbg_ktok, int* dbg_offs, const float* pre_val,
                             const int* pre_idx) {
    if (st.beam < 1 || st.beam > KMAX) return "beam_step: beam must be in [1,16]";
    if (st.N % st.beam) return "beam_step: N must be a multiple of beam";
    if (!logp && !pre_val) return "beam_step: need log-probs or a precomputed top-k";
    if ((pre_val == nullptr) != (pre_idx == nullptr)) return "beam_step: pre_val / pre_idx must both be given";
    return launch<beam_step_kernel>(dim3(st.N / st.beam), dim3(st.beam * 32), 0, stream, logp, ldl, V, lm_logp, ld_lm,
                                    lm_weight, st, dbg_ktok, dbg_offs, pre_val, pre_idx);
}

// ------------------------------------------------------------------------------------------------
// Ancestral sampling step (DESIGN.md 4.11): every live row n draws token = argmax_v (x_v + g_v), v < V, ties to the lower
// id, with g_v = -log(-log u) the Gumbel noise of the uniform
//     u(seed, step, n, v) = rng_u01(rng_key(rng_key(rng_key(seed, step), n), v))          (counter_rng.cuh)
// so the token is distributed as softmax(x).  The row adds x_token - logsumexp(x[:V]) to its score; drawing <S/E> ends it,
// and an ended row emits <S/E> at no cost.  Rows are never reordered (each row's parent is itself), and the search state
// moves under otb_beam_step's conventions (tok_hist, par_hist, anc ping-pong, last_tok, flag, ctrl), so reconstruction
// and the KV-cached decoder's ancestry addressing work unchanged.  One CTA per row, one pass over its logits: an online
// log-sum-exp (running max m and sum s of exp(x - m)) and the perturbed arg-max, both merged over warps and then the CTA.
// ------------------------------------------------------------------------------------------------
static constexpr int SAMPLE_MAX_V = 48 * 1024;

// (m, s) <- the log-sum-exp state of both halves; -inf entries contribute nothing
__device__ __forceinline__ void lse_merge(float& m, float& s, float om, float os) {
    const float M = fmaxf(m, om);
    if (M == -INFINITY) return;                    // both empty
    s = s * expf(m - M) + os * expf(om - M);
    m = M;
}

// THREADS threads per row (a multiple of 32).  The launch takes 512 while the rows fit one CTA per SM and 256 past that,
// as the sweep of 32 .. 512 (tools/sample_step_sweep.cu, DESIGN.md 4.11) favours
template <int THREADS>
__global__ void __launch_bounds__(THREADS) sample_step_kernel(const float* __restrict__ logits, int ldl, int V, BeamState st,
                                                              const int* __restrict__ seed) {
    constexpr int WARPS = THREADS / 32;
    __shared__ float r_m[WARPS], r_s[WARPS], r_z[WARPS];
    __shared__ int r_i[WARPS];
    __shared__ int s_tok, s_step, s_live, s_fin;
    __shared__ float s_inc;
    const int n = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // ctrl and the row's flag are read once, by thread 0, before any thread can reach the atomics below: the last CTA of
    // the step rewrites ctrl[0] / ctrl[1] and this CTA's thread 0 rewrites flag[n], and a warp of this CTA that started
    // late must not see either
    if (tid == 0) {
        s_step = st.ctrl[0];
        s_live = !st.ctrl[1] && s_step < st.Lmax;
        s_fin = st.flag[n] != 0;
    }
    __syncthreads();
    if (!s_live) return;                            // the search has ended: the state stays frozen, as in beam_step
    const int step = s_step;
    const bool fin = s_fin;
    if (!fin) {
        const uint32_t hrow = mix32(rng_key(rng_key((uint32_t)*seed, (uint32_t)step), (uint32_t)n));
        const float* x = logits + (size_t)n * ldl;
        float m = -INFINITY, s = 0.f, bz = -INFINITY;
        int bi = 0x7fffffff;
        for (int v = tid; v < V; v += THREADS) {
            const float xv = __ldg(x + v);
            if (xv == -INFINITY) continue;          // probability 0: neither in the sum nor drawable
            if (xv > m) {
                s = s * expf(m - xv) + 1.f;
                m = xv;
            } else {
                s += expf(xv - m);
            }
            const float u = rng_u01(mix32(hrow ^ (uint32_t)v));      // rng_key(row key, v)
            const float z = xv - logf(-logf(u));
            if (better(z, v, bz, bi)) { bz = z; bi = v; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
            lse_merge(m, s, om, os);
        }
        warp_best(bz, bi);
        if (lane == 0) { r_m[warp] = m; r_s[warp] = s; r_z[warp] = bz; r_i[warp] = bi; }
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < WARPS; ++w) {       // fixed order: repeated calls are bit-identical
                lse_merge(m, s, r_m[w], r_s[w]);
                if (better(r_z[w], r_i[w], bz, bi)) { bz = r_z[w]; bi = r_i[w]; }
            }
            // a row without a finite logit has nothing to draw: token 0 (the lowest id) and score -inf
            if (m == -INFINITY) {
                s_tok = 0;
                s_inc = -INFINITY;
            } else {
                s_tok = bi;
                s_inc = x[bi] - (m + logf(s));
            }
        }
        __syncthreads();
    }
    const int tok = fin ? (int)EOS_ID : s_tok;
    const int cur = step & 1, nxt = cur ^ 1;
    const int* a_old = st.anc + ((size_t)cur * st.N + n) * st.Lmax;
    int* a_new = st.anc + ((size_t)nxt * st.N + n) * st.Lmax;
    for (int t = tid; t < step; t += THREADS) a_new[t] = a_old[t];
    if (tid == 0) {
        a_new[step] = n;
        st.tok_hist[(size_t)step * st.N + n] = tok;
        st.par_hist[(size_t)step * st.N + n] = n;
        if (!fin) st.scores[n] += s_inc;            // an ended row keeps its score
        st.last_tok[n] = tok;
        st.flag[n] = tok == (int)EOS_ID ? 1 : 0;
        const int ended = tok == (int)EOS_ID ? 1 : 0;
        if (ended) atomicAdd(&st.ctrl[2], 1);
        __threadfence();
        // the last CTA of this step advances {step, done}, as beam_step's does
        if (atomicAdd(&st.ctrl[3], 1) == (int)gridDim.x - 1) {
            const int total = atomicAdd(&st.ctrl[2], 0);
            st.ctrl[2] = 0;
            st.ctrl[3] = 0;
            __threadfence();
            if (total == st.N) st.ctrl[1] = 1;
            st.ctrl[0] = step + 1;
        }
    }
}

static const char* sample_step_check(int ldl, int V, const BeamState& st) {
    if (V < 1 || V > SAMPLE_MAX_V) return "sample_step: V must be in [1, 49152]";
    if (ldl < V) return "sample_step: ldl < V";
    if (st.N < 1 || st.Lmax < 1) return "sample_step: empty problem (need N >= 1 and Lmax >= 1)";
    return nullptr;
}

const char* sample_step_launch(cudaStream_t stream, const float* logits, int ldl, int V, BeamState st, const int* seed) {
    if (const char* e = sample_step_check(ldl, V, st)) return e;
    if (st.N <= num_sms()) return launch<sample_step_kernel<512>>(dim3(st.N), dim3(512), 0, stream, logits, ldl, V, st, seed);
    return launch<sample_step_kernel<256>>(dim3(st.N), dim3(256), 0, stream, logits, ldl, V, st, seed);
}

// ------------------------------------------------------------------------------------------------
// preds reconstruction: walk the (token, parent) back-pointers.  preds [N, ld] i64, column 0 = BOS.
// ------------------------------------------------------------------------------------------------
__global__ void beam_reconstruct_kernel(BeamState st, long long* preds, int ld, int steps) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= st.N) return;
    long long* row = preds + (size_t)n * ld;
    row[0] = 1;  // BOS
    int cur = n;
    for (int s = steps - 1; s >= 0; --s) {
        row[s + 1] = st.tok_hist[(size_t)s * st.N + cur];
        cur = st.par_hist[(size_t)s * st.N + cur];
    }
}

const char* beam_reconstruct_launch(cudaStream_t stream, BeamState st, long long* preds, int ld, int steps) {
    if (steps < 0 || steps > st.Lmax || ld < steps + 1) return "beam_reconstruct: bad steps / ld";
    return launch<beam_reconstruct_kernel>((st.N + 127) / 128, 128, 0, stream, st, preds, ld, steps);
}

// ------------------------------------------------------------------------------------------------
// finalisation (speech2text.py:70-91): lengths = #(tok != EOS) (BOS == EOS so BOS is not counted),
// scores /= ((lamda + len)/(lamda + 1))^penalty, sort descending, gather, strip BOS, take nbest.
// One CTA per utterance; thread r < beam handles hypothesis r.  steps is read from ctrl[0].
//   out_preds i64 [B, nbest, Lmax]  (columns >= steps are filled with EOS), out_scores f32 [B, nbest]
// ------------------------------------------------------------------------------------------------
__global__ void beam_finalize_kernel(BeamState st, float penalty, float lamda, int nbest, long long* out_preds,
                                     float* out_scores) {
    __shared__ float s_score[KMAX];
    __shared__ int s_rank[KMAX];
    const int u = blockIdx.x, r = threadIdx.x, beam = st.beam;
    const int steps = st.ctrl[0];
    const int n = u * beam + r;
    float sc = -INFINITY;
    if (r < beam) {
        int cur = n, len = 0;
        for (int s = steps - 1; s >= 0; --s) {
            len += (st.tok_hist[(size_t)s * st.N + cur] != (int)EOS_ID) ? 1 : 0;
            cur = st.par_hist[(size_t)s * st.N + cur];
        }
        sc = st.scores[n];
        if (penalty != 0.f) sc = sc / powf((lamda + (float)len) / (lamda + 1.0f), penalty);
        s_score[r] = sc;
    }
    __syncthreads();
    if (r < beam) {
        int rank = 0;
        for (int j = 0; j < beam; ++j)
            if (better(s_score[j], j, sc, r)) ++rank;
        s_rank[rank] = r;
    }
    __syncthreads();
    if (r < nbest && r < beam) {
        const int src = u * beam + s_rank[r];
        out_scores[(size_t)u * nbest + r] = s_score[s_rank[r]];
        long long* row = out_preds + ((size_t)u * nbest + r) * st.Lmax;
        for (int s = steps; s < st.Lmax; ++s) row[s] = EOS_ID;
        int cur = src;
        for (int s = steps - 1; s >= 0; --s) {
            row[s] = st.tok_hist[(size_t)s * st.N + cur];
            cur = st.par_hist[(size_t)s * st.N + cur];
        }
    }
}

const char* beam_finalize_launch(cudaStream_t stream, BeamState st, float penalty, float lamda, int nbest,
                                 long long* out_preds, float* out_scores) {
    if (nbest < 1) return "beam_finalize: nbest < 1";
    return launch<beam_finalize_kernel>(st.N / st.beam, 32, 0, stream, st, penalty, lamda, nbest, out_preds, out_scores);
}

// initial state (speech2text.py:54-58): preds = BOS, scores = [0, -inf, ...] per utterance, flags = 0
__global__ void beam_init_kernel(BeamState st) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n < 4) st.ctrl[n] = 0;
    if (n >= st.N) return;
    st.last_tok[n] = 1;
    st.scores[n] = (n % st.beam == 0) ? 0.f : -INFINITY;
    st.flag[n] = 0;
}

const char* beam_init_launch(cudaStream_t stream, BeamState st) {
    int n = st.N < 4 ? 4 : st.N;
    return launch<beam_init_kernel>((n + 127) / 128, 128, 0, stream, st);
}

// ------------------------------------------------------------------------------------------------
// Fused  log_softmax(logits[row]) (+ lm_weight * lm_logp[row])  ->  top-k (values, vocabulary ids)
// With lm_exempt >= 0 (the transducer's fusion, DESIGN.md 4.22) column lm_exempt (blank) keeps its plain log-prob and every
// other column gets  + (lm_weight * lm_logp + lm_beta)  (+ lm_beta alone without lm_logp); out_logp then holds the plain
// log-probs.  lm_exempt < 0 is the attention decoder's fusion, unchanged.
// decoder/transformer.py:206 + recognize/speech2text.py:102-112 in ONE pass over the logits: the row is
// staged in smem once (coalesced), so the [N,V] log-prob matrix is never written or re-read.  Values are
// formed exactly as the stand-alone log-softmax kernel does (x - (max + log sum exp(x - max))) before the
// top-k, so the selected ids equal top-k over the materialised log-probs (ties -> lower index).
// One CTA per hypothesis row, 8 warps; per-warp top-k over a slice, then one warp merges 8*k candidates.
// ------------------------------------------------------------------------------------------------
static constexpr int TOPK_THREADS = 256;

__global__ void __launch_bounds__(TOPK_THREADS) logsoftmax_topk_kernel(const float* __restrict__ logits, int ldl, int V,
                                                                       const float* __restrict__ lm_logp, int ld_lm,
                                                                       float lm_weight, float lm_beta, int lm_exempt, int k,
                                                                       float* __restrict__ out_val,
                                                                       int* __restrict__ out_idx,
                                                                       float* __restrict__ out_logp, int ld_logp) {
    extern __shared__ float srow[];   // [V]
    __shared__ float red[8];
    __shared__ float bc;
    __shared__ float cand_v[8 * KMAX];
    __shared__ int cand_i[8 * KMAX];
    const int row = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const float* x = logits + (size_t)row * ldl;
    float m = -INFINITY;
    for (int i = tid; i < V; i += TOPK_THREADS) {
        const float v = x[i];
        srow[i] = v;
        m = fmaxf(m, v);
    }
    m = warp_max(m);
    if (lane == 0) red[warp] = m;
    __syncthreads();
    if (tid == 0) {
        float t = red[0];
        for (int i = 1; i < 8; ++i) t = fmaxf(t, red[i]);
        bc = t;
    }
    __syncthreads();
    m = bc;
    float sum = 0.f;
    for (int i = tid; i < V; i += TOPK_THREADS) sum += expf(srow[i] - m);
    sum = warp_sum(sum);
    __syncthreads();
    if (lane == 0) red[warp] = sum;
    __syncthreads();
    if (tid == 0) {
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += red[i];
        bc = m + logf(t);
    }
    __syncthreads();
    const float lse = bc;
    const float* lm = lm_logp ? lm_logp + (size_t)row * ld_lm : nullptr;
    for (int i = tid; i < V; i += TOPK_THREADS) {
        const float p = srow[i] - lse;
        float v = p;
        if (lm_exempt < 0) {
            if (lm) v = v + lm_weight * lm[i];
        } else if (i != lm_exempt) {
            v = lm ? v + (lm_weight * lm[i] + lm_beta) : v + lm_beta;
        }
        srow[i] = v;
        if (out_logp) out_logp[(size_t)row * ld_logp + i] = lm_exempt < 0 ? v : p;
    }
    __syncthreads();
    // per-warp top-k over a contiguous slice: k rounds of (lane-local scan of smem, warp arg-max), round r taking the best
    // element ranked after round r-1's pick in the order (value descending, index ascending).  Elements equal to -inf are
    // ranked like any other value, so a row with fewer than k finite values still yields real token ids, as torch.topk and
    // warp_topk do.  (Knocking the pick out by overwriting it with -inf made picked elements and real -inf ones look alike,
    // and a scan that skipped -inf returned index 0x7fffffff for them: found by tests/test_gpu_beam_ties.py, an LM that
    // rules tokens out with lm_logp = -inf.)
    const int per = (V + 7) / 8;
    const int lo = warp * per, hi = min(V, lo + per);
    float pv = INFINITY;
    int pi = -1;
    for (int r = 0; r < k; ++r) {
        float bv = -INFINITY;
        int bi = 0x7fffffff;
        for (int idx = lo + lane; idx < hi; idx += 32) {
            const float v = srow[idx];
            const bool after = (v < pv) || (v == pv && idx > pi);
            if (after && better(v, idx, bv, bi)) { bv = v; bi = idx; }
        }
        warp_best(bv, bi);
        pv = bv;
        pi = bi;
        if (lane == 0) { cand_v[warp * KMAX + r] = bv; cand_i[warp * KMAX + r] = bi; }
    }
    __syncthreads();
    if (warp == 0) {
        // merge: 8 sorted lists of k -> global top-k (lane w < 8 walks list w)
        int pos = 0;
        for (int r = 0; r < k; ++r) {
            float bv = (lane < 8 && pos < k) ? cand_v[lane * KMAX + pos] : -INFINITY;
            int bi = (lane < 8 && pos < k) ? cand_i[lane * KMAX + pos] : 0x7fffffff;
            const float mv = bv;
            const int mi = bi;
            warp_best(bv, bi);
            if (mi == bi && mv == bv && lane < 8) ++pos;
            if (lane == 0) { out_val[(size_t)row * k + r] = bv; out_idx[(size_t)row * k + r] = bi; }
        }
    }
}

const char* logsoftmax_topk_launch(cudaStream_t stream, const float* logits, int ldl, int V, const float* lm_logp,
                                   int ld_lm, float lm_weight, float lm_beta, int lm_exempt, int k, int rows, float* out_val,
                                   int* out_idx, float* out_logp, int ld_logp) {
    if (k < 1 || k > KMAX) return "logsoftmax_topk: k must be in [1,16]";
    if (lm_exempt >= V) return "logsoftmax_topk: the LM-exempt column must be below V";
    if (lm_exempt < 0 && lm_beta != 0.f) return "logsoftmax_topk: lm_beta needs an LM-exempt column";
    if (V < 1 || V > 48 * 1024) return "logsoftmax_topk: vocabulary too large for one CTA's shared memory";
    // past V the scan has nothing left to pick and would return its sentinel (-inf, id 0x7fffffff) as a token
    if (k > V) return "logsoftmax_topk: k must not exceed the vocabulary size V";
    const size_t smem = (size_t)V * sizeof(float);
    return launch<logsoftmax_topk_kernel>(dim3(rows), dim3(TOPK_THREADS), smem, stream, logits, ldl, V, lm_logp, ld_lm,
                                          lm_weight, lm_beta, lm_exempt, k, out_val, out_idx, out_logp, ld_logp);
}

}  // namespace otb
