// CTC prefix scoring for joint CTC/attention decoding (Watanabe et al. 2017): the CTC term of the beam search's step score.
// DESIGN.md 4.9 gives the definition; in short, per utterance with log-probs lp[t, v] of its T_b frames, for a hypothesis
// g (its tokens after <S/E>) and a candidate token c, h = g c:
//
//   gn(h, t) / gb(h, t)  log-probability that frames 0..t emit exactly h, ending in a non-blank / a blank
//   phi(t) = gb(g, t) if c is g's last token, else logaddexp(gn(g, t), gb(g, t));   phi(-1) = 0 for empty g, else -inf
//   gn(h, t) = logaddexp(gn(h, t-1), phi(t-1)) + lp[t, c]             gn(h, -1) = gb(h, -1) = -inf
//   gb(h, t) = logaddexp(gn(h, t-1), gb(h, t-1)) + lp[t, blank]
//   psi(h)   = logsumexp_t(phi(t-1) + lp[t, c])                       the probability that the labels START with h
//   psi(h)   = logaddexp(gn(h, T_b-1), gb(h, T_b-1)) for c = <S/E>:   the closing <S/E> is a label the head was trained
//                                                                     on, so a complete hypothesis scores as the whole sequence
//
// State of the N live hypotheses: gamma f32 [2, N, T, 2] ({gn, gb} per frame) and psi f32 [2, N]; the half in use is the
// parity of the search's step counter, as for the ancestry table of the KV cache.  Three kernels:
//   init     gamma(empty prefix) = running sum of the blank column, psi = 0, in half 0
//   score    one warp per hypothesis, one lane per candidate: the recursion over T_b frames into the candidate scratch,
//            then the joint step score of each candidate and the hypothesis' `beam` best, in otb_beam_step's top-k layout
//   advance  after the beam step: every new row takes its (parent, token)'s candidate state into the other half
// score and advance read {step, done} of the search state on the device and do nothing once the search has ended.
#include <math.h>

#include "beam_common.cuh"
#include "launch.cuh"
#include "otb_internal.h"

namespace otb {

static constexpr int PREFIX_CHUNK = 8;        // frames whose lp[t, c] gathers are in flight ahead of the recursion
static constexpr int PREFIX_TMAX = 16 * 1024; // 3 T floats of shared memory per hypothesis

__device__ __forceinline__ float logaddexp(float a, float b) {
    const float m = fmaxf(a, b);
    if (m == -INFINITY) return m;
    return m + log1pf(expf(fminf(a, b) - m));
}

// one warp per utterance: inclusive scan of the blank column, 32 frames per round
__global__ void __launch_bounds__(32) ctc_prefix_init_kernel(const float* __restrict__ lp, int ld, int T,
                                                             const int* __restrict__ in_len, int blank, int beam,
                                                             float* __restrict__ gamma, float* __restrict__ psi) {
    const int u = blockIdx.x, lane = threadIdx.x;
    const int Tb = max(0, min(in_len[u], T));
    const float* x = lp + (size_t)u * T * ld + blank;
    float carry = 0.f;
    for (int t0 = 0; t0 < Tb; t0 += 32) {
        const int t = t0 + lane;
        float v = t < Tb ? x[(size_t)t * ld] : 0.f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float w = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += w;
        }
        v += carry;
        carry = __shfl_sync(0xffffffffu, v, 31);
        if (t < Tb)
            for (int r = 0; r < beam; ++r)
                reinterpret_cast<float2*>(gamma)[(size_t)(u * beam + r) * T + t] = make_float2(-INFINITY, v);
    }
    if (lane < beam) psi[u * beam + lane] = 0.f;
}

__global__ void __launch_bounds__(32) ctc_prefix_score_kernel(
    const float* __restrict__ lp, int ld, int T, const int* __restrict__ in_len, int blank, const float* __restrict__ gamma,
    const float* __restrict__ psi, const float* __restrict__ cand_val, const int* __restrict__ cand_id, int P,
    const float* __restrict__ lm_logp, int ld_lm, float lm_weight, float ctc_weight, BeamState st, float* __restrict__ gamma_cand,
    float* __restrict__ psi_cand, float* __restrict__ out_val, int* __restrict__ out_idx) {
    extern __shared__ float sm[];   // [3, T]: phi for a candidate that repeats g's last token, phi for any other, lp[t, blank]
    if (st.ctrl[1] || st.ctrl[0] >= st.Lmax) return;
    const int step = st.ctrl[0];
    const int n = blockIdx.x, lane = threadIdx.x, beam = st.beam;
    if (st.flag[n]) return;         // a finished hypothesis: the beam step masks its candidates itself
    const int u = n / beam;
    const int Tb = max(0, min(in_len[u], T));
    const float* x = lp + (size_t)u * T * ld;
    float* phi_same = sm;
    float* phi_diff = sm + T;
    float* lpb = sm + 2 * T;
    const float2* g = reinterpret_cast<const float2*>(gamma) + ((size_t)(step & 1) * st.N + n) * T;
    for (int t = lane; t < Tb; t += 32) {
        const float2 v = g[t];
        phi_same[t] = v.y;
        phi_diff[t] = logaddexp(v.x, v.y);
        lpb[t] = x[(size_t)t * ld + blank];
    }
    __syncwarp();
    const bool live = lane < P;
    const int c = live ? cand_id[(size_t)n * P + lane] : 0;
    // at step 0 last_tok is the opening <S/E>, not a label: gn of the empty prefix is -inf, so both phi agree anyway
    const float* phi = (step > 0 && (long long)c == st.last_tok[n]) ? phi_same : phi_diff;
    float psi_c = -INFINITY;
    if (live) {
        // the blank is not a label: a candidate that names it reads -inf log-probs, and no hypothesis continues with it
        const bool is_blank = c == blank;
        const float* xc = x + c;
        float2* gc = reinterpret_cast<float2*>(gamma_cand) + ((size_t)n * P + lane) * T;
        float gn = -INFINITY, gb = -INFINITY, ph = step == 0 ? 0.f : -INFINITY;
        float pm = -INFINITY, ps = 0.f;           // psi as max + log(sum): one exp per frame instead of a logaddexp
        float cur[PREFIX_CHUNK], nxt[PREFIX_CHUNK];
#pragma unroll
        for (int j = 0; j < PREFIX_CHUNK; ++j) cur[j] = is_blank ? -INFINITY : j < Tb ? xc[(size_t)j * ld] : 0.f;
        for (int t0 = 0; t0 < Tb; t0 += PREFIX_CHUNK) {
#pragma unroll
            for (int j = 0; j < PREFIX_CHUNK; ++j) {
                const int t = t0 + PREFIX_CHUNK + j;
                nxt[j] = is_blank ? -INFINITY : t < Tb ? xc[(size_t)t * ld] : 0.f;
            }
#pragma unroll
            for (int j = 0; j < PREFIX_CHUNK; ++j) {
                const int t = t0 + j;
                if (t < Tb) {
                    const float term = ph + cur[j];
                    const float ngn = logaddexp(gn, ph) + cur[j];
                    gb = logaddexp(gn, gb) + lpb[t];
                    gn = ngn;
                    if (term > pm) {
                        ps = ps * expf(pm - term) + 1.f;
                        pm = term;
                    } else if (term > -INFINITY) {
                        ps += expf(term - pm);
                    }
                    ph = phi[t];
                    gc[t] = make_float2(gn, gb);
                }
            }
#pragma unroll
            for (int j = 0; j < PREFIX_CHUNK; ++j) cur[j] = nxt[j];
        }
        psi_c = c == (int)EOS_ID ? logaddexp(gn, gb) : (pm == -INFINITY ? pm : pm + logf(ps));
        psi_cand[(size_t)n * P + lane] = psi_c;
    }
    // ---- joint step score (1 - w) logp_att + w (psi(g c) - psi(g)) + lm_weight lm, then the `beam` best of the P
    float v = -INFINITY;
    int id = 0x7fffffff;
    if (live) {
        const float lm = lm_logp ? lm_weight * lm_logp[(size_t)n * ld_lm + c] : 0.f;
        const float att = cand_val[(size_t)n * P + lane] - lm;
        const float d = psi_c == -INFINITY ? psi_c : psi_c - psi[(size_t)(step & 1) * st.N + n];
        v = d == -INFINITY ? d : (1.f - ctc_weight) * att + ctc_weight * d + lm;
        id = c;
    }
    int rank = 0;
    for (int j = 0; j < P; ++j) {
        const float vj = __shfl_sync(0xffffffffu, v, j);
        const int ij = __shfl_sync(0xffffffffu, id, j);
        rank += better(vj, ij, v, id) ? 1 : 0;
    }
    if (live && rank < beam) {
        out_val[(size_t)n * beam + rank] = v;
        out_idx[(size_t)n * beam + rank] = id;
    }
}

__global__ void __launch_bounds__(64) ctc_prefix_advance_kernel(BeamState st, const int* __restrict__ cand_id, int P, int T,
                                                                const int* __restrict__ in_len,
                                                                const float* __restrict__ gamma_cand,
                                                                const float* __restrict__ psi_cand, float* gamma, float* psi) {
    // the beam step has advanced the counter; when it also ended the search, no state is read again
    if (st.ctrl[1] || st.ctrl[0] < 1) return;
    const int step = st.ctrl[0] - 1;
    const int nn = blockIdx.x;
    const int parent = st.par_hist[(size_t)step * st.N + nn];
    const int tok = st.tok_hist[(size_t)step * st.N + nn];
    const int Tb = max(0, min(in_len[nn / st.beam], T));
    const int cur = step & 1, nxt = cur ^ 1;
    const float2* src = reinterpret_cast<const float2*>(gamma) + ((size_t)cur * st.N + parent) * T;
    float ps = psi[(size_t)cur * st.N + parent];
    if (tok != (int)EOS_ID) {        // <S/E> ends the hypothesis (a finished parent emits nothing else): it keeps the parent's state
        int slot = 0;
        for (int j = 0; j < P; ++j)
            if (cand_id[(size_t)parent * P + j] == tok) slot = j;
        src = reinterpret_cast<const float2*>(gamma_cand) + ((size_t)parent * P + slot) * T;
        ps = psi_cand[(size_t)parent * P + slot];
    }
    float2* dst = reinterpret_cast<float2*>(gamma) + ((size_t)nxt * st.N + nn) * T;
    for (int t = threadIdx.x; t < Tb; t += blockDim.x) dst[t] = src[t];
    if (threadIdx.x == 0) psi[(size_t)nxt * st.N + nn] = ps;
}

const char* ctc_prefix_init_launch(cudaStream_t stream, const float* lp, int ld, int B, int T, const int* in_len, int blank,
                                   int beam, float* gamma, float* psi) {
    if (B < 1 || T < 1) return "ctc_prefix_init: empty problem";
    if (beam < 1 || beam > KMAX) return "ctc_prefix_init: beam must be in [1,16]";
    return launch<ctc_prefix_init_kernel>(B, 32, 0, stream, lp, ld, T, in_len, blank, beam, gamma, psi);
}

const char* ctc_prefix_score_launch(cudaStream_t stream, const float* lp, int ld, int T, int V, const int* in_len, int blank,
                                    const float* gamma, const float* psi, const float* cand_val, const int* cand_id, int P,
                                    const float* lm_logp, int ld_lm, float lm_weight, float ctc_weight, BeamState st,
                                    float* gamma_cand, float* psi_cand, float* out_val, int* out_idx) {
    if (st.beam < 1 || P < st.beam || P > KMAX) return "ctc_prefix_score: need 1 <= beam <= P <= 16";
    if (st.N % st.beam) return "ctc_prefix_score: N must be a multiple of beam";
    if (T < 1 || T > PREFIX_TMAX) return "ctc_prefix_score: T must be in [1, 16384]";
    if (blank < 0 || blank >= V || ld < V) return "ctc_prefix_score: bad blank id or row pitch";
    if (!(ctc_weight >= 0.f && ctc_weight <= 1.f)) return "ctc_prefix_score: ctc_weight must be in [0, 1]";
    return launch<ctc_prefix_score_kernel>(st.N, 32, 3 * (size_t)T * sizeof(float), stream, lp, ld, T, in_len, blank, gamma, psi,
                                           cand_val, cand_id, P, lm_logp, ld_lm, lm_weight, ctc_weight, st, gamma_cand, psi_cand,
                                           out_val, out_idx);
}

const char* ctc_prefix_advance_launch(cudaStream_t stream, BeamState st, const int* cand_id, int P, int T, const int* in_len,
                                      const float* gamma_cand, const float* psi_cand, float* gamma, float* psi) {
    if (st.beam < 1 || P < st.beam || P > KMAX) return "ctc_prefix_advance: need 1 <= beam <= P <= 16";
    if (T < 1) return "ctc_prefix_advance: T < 1";
    return launch<ctc_prefix_advance_kernel>(st.N, 64, 0, stream, st, cand_id, P, T, in_len, gamma_cand, psi_cand, gamma, psi);
}

}  // namespace otb
