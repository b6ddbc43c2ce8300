// Fused masked multi-head attention for sm_90a (d_k = 64 or 96):  softmax(Q K^T / sqrt(d_k) + mask) V
// Both contractions run on wgmma tensor cores with the score tile and the output tile in registers;
// the key-padding mask comes from lengths[b] (masks are always contiguous prefixes, SURVEY.md 8a),
// the causal mask from row/column indices, so no [B,h,T,T] tensor is ever materialised.
//
// Replaces BasedAttention.compute_context + the QK^T matmul:
//   otrans/module/attention.py:80 (scores), :34 (masked_fill -inf), :36 (softmax), :37 (weights @ V),
//   :41 (merge heads).  The reference also returns the [B,h,T1,T2] weights.  This kernel never forms them; the modules'
//   return_attn_weights switch has them written by a separate kernel over the same operands (attn_probs.cu).
//
// One CTA = 128 query rows of one (batch, head); 256 threads = two warpgroups, warpgroup w owns query rows
// [64 w, 64 w + 64).  Keys are consumed in blocks of 128 with an online softmax:
//   TMA: Q tile [128x64], K block [128x64] (K-major) and V block [128 keys x 64] (MN-major B operand)
//   S  = Q K^T      : 4 x wgmma 64x128x16 per warpgroup (registers)
//   P  = exp2(S*c - m) as bf16 written to smem in the canonical K-major SWIZZLE_128B layout
//   O  = O*alpha + P V : 8 x wgmma 64x64x16 per warpgroup, accumulated in registers
//
// d_k = 96 (the Conformer configuration, d_model 384 / 4 heads): a SWIZZLE_128B box is at most 64 bf16 wide, so
// every Q, K and V tile is two 64-column boxes, at columns h*96 and h*96 + 64 of the head.  The upper 32 columns of
// the second box belong to the next head (or are TMA zero-fill past the matrix edge).  S = QK^T takes 6 k16 steps,
// 4 from the first box and 2 from the second, so those columns are never read.  O = PV runs two 64-wide wgmma chains,
// one per V box, into o[64]; the upper 32 columns of the second chain are computed and dropped.  That does 4/3 of the
// needed PV work, but keeps the operand layout and descriptors of the 64-wide kernel exactly (an n96 MN-major chain
// would need a partial 64-element swizzle atom in N).
#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

// per head width: Q, K, V tiles of DK / 64 rounded up boxes of 16 KB each, P (32 KB), barriers, alignment slack
template <int DK>
struct AttnCfg {
    static constexpr int BOXES = (DK + 63) / 64;
    static constexpr int TILE = 16384 * BOXES;
    static constexpr int SMEM = TILE * 3 + 32768 + 128 + 1024;
};

template <int DK, bool HAS_BD>
__global__ void __launch_bounds__(256, 1)
attn_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
               const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    constexpr int NB = AttnCfg<DK>::BOXES, TILE = AttnCfg<DK>::TILE;
    uint8_t* sQ = smem;
    uint8_t* sK = smem + TILE;
    uint8_t* sV = smem + 2 * TILE;
    uint8_t* sP = smem + 3 * TILE;  // 2 k-blocks x [128 rows x 128 B]
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 3 * TILE + 32768);  // q, k, v

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wg = warp >> 2;
    const int q0 = blockIdx.x * 128, h = blockIdx.y, b = blockIdx.z;
    const int kv_len = p.kv_len ? min(p.kv_len[b], p.Tk) : p.Tk;
    int kv_end = kv_len;
    if (p.causal) kv_end = min(kv_end, q0 + 128);
    const int nblk = (kv_end + 127) / 128;

    if (tid == 0) {
        for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
        fence_barrier_init();
        tma_prefetch_desc(&tmQ);
        tma_prefetch_desc(&tmK);
        tma_prefetch_desc(&tmV);
        // a row block with no visible key (kv_len 0) reads nothing: a Q load nobody waits for would still be landing in
        // shared memory after the CTA has exited
        if (nblk > 0) {
            mbar_arrive_expect_tx(&bar[0], TILE);
#pragma unroll
            for (int x = 0; x < NB; ++x) tma_load_2d(sQ + x * 16384, &tmQ, &bar[0], p.q_col0 + h * DK + x * 64, b * p.Tq + q0);
            mbar_arrive_expect_tx(&bar[1], TILE);
#pragma unroll
            for (int x = 0; x < NB; ++x) tma_load_2d(sK + x * 16384, &tmK, &bar[1], p.k_col0 + h * DK + x * 64, b * p.Tk);
            mbar_arrive_expect_tx(&bar[2], TILE);
#pragma unroll
            for (int x = 0; x < NB; ++x) tma_load_2d(sV + x * 16384, &tmV, &bar[2], p.v_col0 + h * DK + x * 64, b * p.Tk);
        }
    }
    __syncthreads();

    // this thread's two tile rows (accumulator fragment rows) and its column offset inside every 8-column group
    const int rl0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    int lim[2];
    const float* bd_row[2] = {nullptr, nullptr};
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int qi = q0 + rl0 + 8 * hh;
        lim[hh] = p.causal ? min(kv_len, qi + 1) : kv_len;  // keys [0, lim) are visible to this row
        if (HAS_BD) {
            const int qc = min(qi, p.Tq - 1);
            bd_row[hh] = p.bd + (((size_t)h * p.B + b) * p.Tq + qc) * p.ldbd + (p.Tq - 1 - qc);
        }
    }
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    float o[32 * NB];   // o[32 x + i]: chain x, output columns [64 x, 64 x + 64)
#pragma unroll
    for (int i = 0; i < 32 * NB; ++i) o[i] = 0.f;
    const uint32_t qa = smem_u32(sQ) + wg * 8192, ka = smem_u32(sK), va = smem_u32(sV);
    const uint32_t pa = smem_u32(sP) + wg * 8192;

    for (int blk = 0; blk < nblk; ++blk) {
        const uint32_t ph = blk & 1;
        const int key0 = blk * 128;
        if (blk == 0) mbar_wait(&bar[0], 0);
        mbar_wait(&bar[1], ph);
        float s[64];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < DK / 16; ++k)   // k16 step k lives in box k / 4 at byte column (k % 4) * 32
            wgmma_n128<0, 0>(s, gmma_desc_sw128(qa + (k >> 2) * 16384 + (k & 3) * 32), gmma_desc_sw128(ka + (k >> 2) * 16384 + (k & 3) * 32),
                             (uint32_t)(k != 0));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(s);
        __syncthreads();
        if (tid == 0 && blk + 1 < nblk) {   // S = QK^T has consumed the K block: prefetch the next one
            mbar_arrive_expect_tx(&bar[1], TILE);
#pragma unroll
            for (int x = 0; x < NB; ++x) tma_load_2d(sK + x * 16384, &tmK, &bar[1], p.k_col0 + h * DK + x * 64, b * p.Tk + key0 + 128);
        }

        // ---- row maximum of the visible raw scores (the positive scale is applied afterwards); a row is spread over 4 lanes
        float m_blk[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int key = key0 + jj * 8 + cq + e;
                    float sv = s[4 * jj + 2 * hh + e];
                    if (HAS_BD && key < lim[hh]) sv += bd_row[hh][key];
                    sv = (key < lim[hh]) ? sv : -INFINITY;
                    s[4 * jj + 2 * hh + e] = sv;
                    m_blk[hh] = fmaxf(m_blk[hh], sv);
                }
            }
        }
        float alpha[2], m_use[2], l_blk[2] = {0.f, 0.f};
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            m_blk[hh] = fmaxf(m_blk[hh], __shfl_xor_sync(0xffffffffu, m_blk[hh], 1));
            m_blk[hh] = fmaxf(m_blk[hh], __shfl_xor_sync(0xffffffffu, m_blk[hh], 2));
            m_blk[hh] *= p.scale_log2;  // -inf stays -inf
            const float m_new = fmaxf(m_run[hh], m_blk[hh]);
            m_use[hh] = (m_new == -INFINITY) ? 0.f : m_new;
            alpha[hh] = (m_run[hh] == -INFINITY) ? 0.f : ex2_approx(m_run[hh] - m_use[hh]);
            m_run[hh] = m_new;
        }
        // ---- probabilities -> bf16 -> smem (K-major, 128B swizzle)
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const float sv0 = s[4 * jj + 2 * hh], sv1 = s[4 * jj + 2 * hh + 1];
                const float p0 = (sv0 == -INFINITY) ? 0.f : ex2_approx(fmaf(sv0, p.scale_log2, -m_use[hh]));
                const float p1 = (sv1 == -INFINITY) ? 0.f : ex2_approx(fmaf(sv1, p.scale_log2, -m_use[hh]));
                l_blk[hh] += p0 + p1;
                const int row = rl0 + 8 * hh;
                const int kc = jj * 8 + cq;
                *reinterpret_cast<uint32_t*>(sP + (kc >> 6) * 16384 + row * 128 + (((((kc & 63) >> 3) ^ (row & 7))) << 4) + (kc & 7) * 2) =
                    pack_bf16(p0, p1);
            }
        }
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            l_blk[hh] += __shfl_xor_sync(0xffffffffu, l_blk[hh], 1);
            l_blk[hh] += __shfl_xor_sync(0xffffffffu, l_blk[hh], 2);
            l_run[hh] = l_run[hh] * alpha[hh] + l_blk[hh];
        }
#pragma unroll
        for (int i = 0; i < 32 * NB; ++i) o[i] *= alpha[(i >> 1) & 1];
        fence_proxy_async_smem();  // P (generic-proxy stores) -> visible to the tensor core's async proxy
        __syncthreads();

        mbar_wait(&bar[2], ph);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
            for (int x = 0; x < NB; ++x)
                wgmma_n64<0, 1>(*reinterpret_cast<float(*)[32]>(o + 32 * x), gmma_desc_sw128(pa + (kk >> 2) * 16384 + (kk & 3) * 32),
                                gmma_desc_sw128(va + x * 16384 + kk * 2048, 1024, 8192), 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        __syncthreads();  // K/V/P smem may now be overwritten by the next block
        if (tid == 0 && blk + 1 < nblk) {   // PV has consumed the V block: prefetch the next one
            mbar_arrive_expect_tx(&bar[2], TILE);
#pragma unroll
            for (int x = 0; x < NB; ++x) tma_load_2d(sV + x * 16384, &tmV, &bar[2], p.v_col0 + h * DK + x * 64, b * p.Tk + key0 + 128);
        }
    }

#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int qi = q0 + rl0 + 8 * hh;
        if (qi >= p.Tq) continue;
        if (p.lse && (lane & 3) == 0) p.lse[((size_t)b * p.H + h) * p.Tq + qi] = (l_run[hh] > 0.f) ? m_run[hh] + log2f(l_run[hh]) : INFINITY;
        const float inv = (l_run[hh] > 0.f) ? 1.0f / l_run[hh] : 0.f;
        bf16* orow = p.out + (size_t)(b * p.Tq + qi) * p.ldo + h * DK;
        const bf16* rrow = p.resid ? p.resid + (size_t)(b * p.Tq + qi) * p.ldr + h * DK : nullptr;
#pragma unroll
        for (int jj = 0; jj < DK / 8; ++jj) {   // o[4 jj + ..] is column 8 jj + cq of the head (chain jj / 8)
            const int c = jj * 8 + cq;
            float v0 = o[4 * jj + 2 * hh] * inv, v1 = o[4 * jj + 2 * hh + 1] * inv;
            if (rrow) {
                const float2 r = unpack_bf16(*reinterpret_cast<const uint32_t*>(rrow + c));
                v0 += r.x;
                v1 += r.y;
            }
            *reinterpret_cast<uint32_t*>(orow + c) = pack_bf16(v0, v1);
        }
    }
}

template <int DK>
static const char* attn_launch_dk(cudaStream_t st, const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
                                  const AttnParams& p) {
    constexpr int SMEM = AttnCfg<DK>::SMEM;
    dim3 grid((p.Tq + 127) / 128, p.H, p.B);
    return p.bd ? launch<attn_tc_kernel<DK, true>>(grid, dim3(256), SMEM, st, tq, tk, tv, p)
                : launch<attn_tc_kernel<DK, false>>(grid, dim3(256), SMEM, st, tq, tk, tv, p);
}

const char* attn_launch(cudaStream_t st, const void* q, int ldq, int q_rows, const void* k, int ldk, int k_rows,
                        const void* v, int ldv, const AttnParams& p, int d_k) {
    if (p.B <= 0 || p.H <= 0 || p.Tq <= 0 || p.Tk <= 0) return "attention: empty problem";
    if (d_k != 64 && d_k != 96) return "attention: head width d_k must be 64 or 96";
    CUtensorMap tq, tk, tv;
    const char* err;
    if ((err = encode_tmap_2d(&tq, q, (uint64_t)ldq, (uint64_t)q_rows, (uint64_t)ldq, 64, 128))) return err;
    if ((err = encode_tmap_2d(&tk, k, (uint64_t)ldk, (uint64_t)k_rows, (uint64_t)ldk, 64, 128))) return err;
    if ((err = encode_tmap_2d(&tv, v, (uint64_t)ldv, (uint64_t)k_rows, (uint64_t)ldv, 64, 128))) return err;
    return d_k == 64 ? attn_launch_dk<64>(st, tq, tk, tv, p) : attn_launch_dk<96>(st, tq, tk, tv, p);
}

}  // namespace otb
