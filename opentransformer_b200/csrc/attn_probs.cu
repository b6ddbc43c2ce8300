// Attention weights for sm_90a (d_k = 64 or 96):  P = softmax(Q K^T / sqrt(d_k) (+ BD) + mask), fp32 [B, H, Tq, Tk]
//
// The [B,h,T1,T2] weights BasedAttention.compute_context returns (otrans/module/attention.py:34-37), which the fused
// forward (attn_tc.cu) never forms.  The operands, masks and band are those of otb_attention, minus V and the residual:
// keys j >= kv_len[b] and, when causal, j > i are exactly 0; a row with no visible key (kv_len[b] == 0) is NaN, as torch's
// softmax over all -inf gives; the band is added to the raw scores before the 1/sqrt(d_k) scale.
//
// One CTA = 128 query rows of one (batch, head); 256 threads = two warpgroups, warpgroup w owns rows [64 w, 64 w + 64).
// The Q tile and each K block are TMA loads with the layout of attn_tc.cu (two 64-column boxes at d_k 96), and
// S = Q K^T is the same 64x128x16 wgmma chain.  The key blocks are swept twice:
//   sweep 1: exact row max m and sum-exp l in fp32 (the online update of attn_tc.cu, no P V);
//   sweep 2: S again, P = exp2(S c - m) / l, staged per warp in shared memory (16 rows x 64 columns at a time) and written
//            as streaming 16-byte stores along the output row, with 4-byte stores only where the row pitch leaves a head
//            or a tail unaligned.
// Key blocks no row of the CTA can see (past kv_len, or past the causal diagonal of its last row) are not computed: their
// columns are filled with 0 (NaN when kv_len is 0).  Recomputing S costs one extra Q K^T per block, small next to writing
// 128 x 128 x 4 bytes per block, so the kernel is bound by the HBM writes; it needs no lse from the forward and so has
// one code path for both head widths.
#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

constexpr int PROBS_PITCH = 72;   // staging row pitch in floats: 8-word skew makes the fragment's float2 stores conflict-free

template <int DK>
struct ProbsCfg {
    static constexpr int BOXES = (DK + 63) / 64;
    static constexpr int TILE = 16384 * BOXES;
    static constexpr int STAGE = 8 * 16 * PROBS_PITCH * 4;   // 8 warps x [16 rows x 64 columns]
    static constexpr int SMEM = TILE * 2 + STAGE + 64 + 1024;
};

// n floats of one output row starting at g, from the staging row s (16-byte aligned) or, with s null, the constant fill,
// by the 16 lanes i = 0..15 of a half warp: full 16-byte stores from the first aligned column on, 4-byte head and tail
__device__ __forceinline__ void put_row(float* g, const float* s, float fill, int n, int i) {
    const int head = min(n, (int)((0u - (uint32_t)(uintptr_t)g) >> 2 & 3u));
    const int nv = (n - head) >> 2;
    if (i < nv) {
        const int c = head + 4 * i;
        float4 v = make_float4(fill, fill, fill, fill);
        if (s) v = head ? make_float4(s[c], s[c + 1], s[c + 2], s[c + 3]) : *reinterpret_cast<const float4*>(s + c);
        __stcs(reinterpret_cast<float4*>(g + c), v);
    }
    if (i < head) __stcs(g + i, s ? s[i] : fill);
    const int t0 = head + 4 * nv;
    if (i < n - t0) __stcs(g + t0 + i, s ? s[t0 + i] : fill);
}

template <int DK, bool HAS_BD>
__global__ void __launch_bounds__(256, 2)
attn_probs_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const AttnProbsParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    constexpr int NB = ProbsCfg<DK>::BOXES, TILE = ProbsCfg<DK>::TILE;
    uint8_t* sQ = smem;
    uint8_t* sK = smem + TILE;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wg = warp >> 2;
    float* stage = reinterpret_cast<float*>(smem + 2 * TILE) + warp * 16 * PROBS_PITCH;
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 2 * TILE + ProbsCfg<DK>::STAGE);   // q, k

    const int q0 = blockIdx.x * 128, h = blockIdx.y, b = blockIdx.z;
    const int kv_len = p.kv_len ? max(min(p.kv_len[b], p.Tk), 0) : p.Tk;
    const int kv_end = p.causal ? min(kv_len, q0 + 128) : kv_len;
    const int nblk = (kv_end + 127) / 128;   // key blocks some row of this CTA sees; 0 only when kv_len is 0

    if (tid == 0) {
        for (int i = 0; i < 2; ++i) mbar_init(&bar[i], 1);
        fence_barrier_init();
        tma_prefetch_desc(&tmQ);
        tma_prefetch_desc(&tmK);
        if (nblk > 0) {   // nothing is loaded for a CTA that only fills: no copy may still be landing after it exits
            mbar_arrive_expect_tx(&bar[0], TILE);
#pragma unroll
            for (int x = 0; x < NB; ++x) tma_load_2d(sQ + x * 16384, &tmQ, &bar[0], p.q_col0 + h * DK + x * 64, b * p.Tq + q0);
            mbar_arrive_expect_tx(&bar[1], TILE);
#pragma unroll
            for (int x = 0; x < NB; ++x) tma_load_2d(sK + x * 16384, &tmK, &bar[1], p.k_col0 + h * DK + x * 64, b * p.Tk);
        }
    }
    __syncthreads();

    // this thread's two tile rows (accumulator fragment rows) and its column offset inside every 8-column group
    const int rw0 = (warp & 3) * 16;                  // the warp's first row inside its warpgroup
    const int rl0 = wg * 64 + rw0 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    int lim[2];
    const float* bd_row[2] = {nullptr, nullptr};
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int qi = q0 + rl0 + 8 * hh;
        lim[hh] = p.causal ? min(kv_len, qi + 1) : kv_len;   // keys [0, lim) are visible to this row
        if (HAS_BD) {
            const int qc = min(qi, p.Tq - 1);
            bd_row[hh] = p.bd + (((size_t)h * p.B + b) * p.Tq + qc) * p.ldbd + (p.Tq - 1 - qc);
        }
    }
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f}, inv[2] = {0.f, 0.f};
    const uint32_t qa = smem_u32(sQ) + wg * 8192, ka = smem_u32(sK);
    // the half warp's output rows: lanes 0-15 store row 2 it, lanes 16-31 row 2 it + 1 of the warp's 16
    const int hl = lane & 15;
    const size_t out_row0 = ((size_t)b * p.H + h) * p.Tq + q0 + wg * 64 + rw0;

    for (int it = 0; it < 2 * nblk; ++it) {
        const bool sweep2 = it >= nblk;
        const int key0 = (sweep2 ? it - nblk : it) * 128;
        if (it == 0) mbar_wait(&bar[0], 0);
        mbar_wait(&bar[1], it & 1);
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
        if (tid == 0 && it + 1 < 2 * nblk) {   // both warpgroups have consumed the K block: fetch the next one
            const int nxt = (it + 1 < nblk ? it + 1 : it + 1 - nblk) * 128;
            mbar_arrive_expect_tx(&bar[1], TILE);
#pragma unroll
            for (int x = 0; x < NB; ++x) tma_load_2d(sK + x * 16384, &tmK, &bar[1], p.k_col0 + h * DK + x * 64, b * p.Tk + nxt);
        }

        // visible raw scores (+ band); everything else -inf
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int key = key0 + jj * 8 + cq + e;
                    float sv = s[4 * jj + 2 * hh + e];
                    if (HAS_BD && key < lim[hh]) sv += bd_row[hh][key];
                    s[4 * jj + 2 * hh + e] = (key < lim[hh]) ? sv : -INFINITY;
                }
            }
        }

        if (!sweep2) {
            // ---- sweep 1: running row max (log2 units, scale applied after the max) and sum-exp; a row spans 4 lanes
            float m_blk[2] = {-INFINITY, -INFINITY}, l_blk[2] = {0.f, 0.f};
#pragma unroll
            for (int i = 0; i < 64; ++i) m_blk[(i >> 1) & 1] = fmaxf(m_blk[(i >> 1) & 1], s[i]);
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                m_blk[hh] = fmaxf(m_blk[hh], __shfl_xor_sync(0xffffffffu, m_blk[hh], 1));
                m_blk[hh] = fmaxf(m_blk[hh], __shfl_xor_sync(0xffffffffu, m_blk[hh], 2));
                m_blk[hh] *= p.scale_log2;   // -inf stays -inf
                const float m_new = fmaxf(m_run[hh], m_blk[hh]);
                const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
                const float alpha = (m_run[hh] == -INFINITY) ? 0.f : ex2_approx(m_run[hh] - m_use);
#pragma unroll
                for (int jj = 0; jj < 16; ++jj)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float sv = s[4 * jj + 2 * hh + e];
                        l_blk[hh] += (sv == -INFINITY) ? 0.f : ex2_approx(fmaf(sv, p.scale_log2, -m_use));
                    }
                l_blk[hh] += __shfl_xor_sync(0xffffffffu, l_blk[hh], 1);
                l_blk[hh] += __shfl_xor_sync(0xffffffffu, l_blk[hh], 2);
                l_run[hh] = l_run[hh] * alpha + l_blk[hh];
                m_run[hh] = m_new;
            }
            if (it + 1 == nblk)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) inv[hh] = 1.0f / l_run[hh];   // every row sees key 0: l > 0
            continue;
        }

        // ---- sweep 2: P = exp2(S c - m) / l, 64 columns at a time through the warp's staging rows
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int jj = hf * 8 + j;
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const float sv0 = s[4 * jj + 2 * hh], sv1 = s[4 * jj + 2 * hh + 1];
                    float2 pv;
                    pv.x = (sv0 == -INFINITY) ? 0.f : ex2_approx(fmaf(sv0, p.scale_log2, -m_run[hh])) * inv[hh];
                    pv.y = (sv1 == -INFINITY) ? 0.f : ex2_approx(fmaf(sv1, p.scale_log2, -m_run[hh])) * inv[hh];
                    *reinterpret_cast<float2*>(stage + ((lane >> 2) + 8 * hh) * PROBS_PITCH + j * 8 + cq) = pv;
                }
            }
            __syncwarp();
            const int c0 = key0 + hf * 64;
            const int n = min(64, p.Tk - c0);
            if (n > 0) {
#pragma unroll 2
                for (int r2 = 0; r2 < 8; ++r2) {
                    const int r = 2 * r2 + (lane >> 4);
                    if (q0 + wg * 64 + rw0 + r < p.Tq) put_row(p.out + (out_row0 + r) * p.Tk + c0, stage + r * PROBS_PITCH, 0.f, n, hl);
                }
            }
            __syncwarp();
        }
    }

    // ---- columns of the key blocks no row of the CTA sees: 0, or NaN for a batch entry without a visible key
    const float fill = nblk ? 0.f : __int_as_float(0x7fc00000);
    for (int c0 = nblk * 128; c0 < p.Tk; c0 += 64) {
        const int n = min(64, p.Tk - c0);
        for (int r2 = 0; r2 < 8; ++r2) {
            const int r = 2 * r2 + (lane >> 4);
            if (q0 + wg * 64 + rw0 + r < p.Tq) put_row(p.out + (out_row0 + r) * p.Tk + c0, nullptr, fill, n, hl);
        }
    }
}

template <int DK>
static const char* attn_probs_launch_dk(cudaStream_t st, const CUtensorMap& tq, const CUtensorMap& tk, const AttnProbsParams& p) {
    dim3 grid((p.Tq + 127) / 128, p.H, p.B);
    return p.bd ? launch<attn_probs_kernel<DK, true>>(grid, dim3(256), ProbsCfg<DK>::SMEM, st, tq, tk, p)
                : launch<attn_probs_kernel<DK, false>>(grid, dim3(256), ProbsCfg<DK>::SMEM, st, tq, tk, p);
}

const char* attn_probs_launch(cudaStream_t st, const void* q, int ldq, int q_rows, const void* k, int ldk, int k_rows,
                              const AttnProbsParams& p, int d_k) {
    if (p.B <= 0 || p.H <= 0 || p.Tq <= 0 || p.Tk <= 0) return "attention probs: empty problem";
    if (d_k != 64 && d_k != 96) return "head width d_k must be 64 or 96";
    CUtensorMap tq, tk;
    const char* err;
    if ((err = encode_tmap_2d(&tq, q, (uint64_t)ldq, (uint64_t)q_rows, (uint64_t)ldq, 64, 128))) return err;
    if ((err = encode_tmap_2d(&tk, k, (uint64_t)ldk, (uint64_t)k_rows, (uint64_t)ldk, 64, 128))) return err;
    return d_k == 64 ? attn_probs_launch_dk<64>(st, tq, tk, p) : attn_probs_launch_dk<96>(st, tq, tk, p);
}

}  // namespace otb
