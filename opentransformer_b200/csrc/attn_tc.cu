// Fused masked multi-head attention for sm_90a (d_k = 64):  softmax(Q K^T / sqrt(d_k) + mask) V
// Both contractions run on wgmma tensor cores with the score tile and the output tile in registers;
// the key-padding mask comes from lengths[b] (masks are always contiguous prefixes, SURVEY.md 8a),
// the causal mask from row/column indices, so no [B,h,T,T] tensor is ever materialised.
//
// Replaces BasedAttention.compute_context + the QK^T matmul:
//   otrans/module/attention.py:80 (scores), :34 (masked_fill -inf), :36 (softmax), :37 (weights @ V),
//   :41 (merge heads).  The reference also returns the [B,h,T1,T2] weights; no caller reads them
//   (model/speech2text.py:50,54), so they are not produced here.
//
// One CTA = 128 query rows of one (batch, head); 256 threads = two warpgroups, warpgroup w owns query rows
// [64 w, 64 w + 64).  Keys are consumed in blocks of 128 with an online softmax:
//   TMA: Q tile [128x64], K block [128x64] (K-major) and V block [128 keys x 64] (MN-major B operand)
//   S  = Q K^T      : 4 x wgmma 64x128x16 per warpgroup (registers)
//   P  = exp2(S*c - m) as bf16 written to smem in the canonical K-major SWIZZLE_128B layout
//   O  = O*alpha + P V : 8 x wgmma 64x64x16 per warpgroup, accumulated in registers
#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

static constexpr int ATT_SMEM = 16384 * 3 + 32768 + 128 + 1024;

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

template <bool HAS_BD>
__global__ void __launch_bounds__(256, 1)
attn_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
               const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
    PDL_TRIGGER();
    PDL_WAIT();   // before the first global read (kv_len) -- launch latency and CTA scheduling still overlap the predecessor
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;
    uint8_t* sK = smem + 16384;
    uint8_t* sV = smem + 32768;
    uint8_t* sP = smem + 49152;  // 2 k-blocks x [128 rows x 128 B]
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 49152 + 32768);  // q, k, v

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
        mbar_arrive_expect_tx(&bar[0], 16384);
        tma_load_2d(sQ, &tmQ, &bar[0], p.q_col0 + h * 64, b * p.Tq + q0);
        if (nblk > 0) {
            mbar_arrive_expect_tx(&bar[1], 16384);
            tma_load_2d(sK, &tmK, &bar[1], p.k_col0 + h * 64, b * p.Tk);
            mbar_arrive_expect_tx(&bar[2], 16384);
            tma_load_2d(sV, &tmV, &bar[2], p.v_col0 + h * 64, b * p.Tk);
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
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
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
        for (int k = 0; k < 4; ++k) wgmma_n128<0, 0>(s, gmma_desc_sw128(qa + k * 32), gmma_desc_sw128(ka + k * 32), (uint32_t)(k != 0));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(s);
        __syncthreads();
        if (tid == 0 && blk + 1 < nblk) {   // S = QK^T has consumed the K block: prefetch the next one
            mbar_arrive_expect_tx(&bar[1], 16384);
            tma_load_2d(sK, &tmK, &bar[1], p.k_col0 + h * 64, b * p.Tk + key0 + 128);
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
        for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
        fence_proxy_async_smem();  // P (generic-proxy stores) -> visible to the tensor core's async proxy
        __syncthreads();

        mbar_wait(&bar[2], ph);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)
            wgmma_n64<0, 1>(o, gmma_desc_sw128(pa + (kk >> 2) * 16384 + (kk & 3) * 32), gmma_desc_sw128(va + kk * 2048, 1024, 8192), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        __syncthreads();  // K/V/P smem may now be overwritten by the next block
        if (tid == 0 && blk + 1 < nblk) {   // PV has consumed the V block: prefetch the next one
            mbar_arrive_expect_tx(&bar[2], 16384);
            tma_load_2d(sV, &tmV, &bar[2], p.v_col0 + h * 64, b * p.Tk + key0 + 128);
        }
    }

#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int qi = q0 + rl0 + 8 * hh;
        if (qi >= p.Tq) continue;
        if (p.lse && (lane & 3) == 0) p.lse[((size_t)b * p.H + h) * p.Tq + qi] = (l_run[hh] > 0.f) ? m_run[hh] + log2f(l_run[hh]) : INFINITY;
        const float inv = (l_run[hh] > 0.f) ? 1.0f / l_run[hh] : 0.f;
        bf16* orow = p.out + (size_t)(b * p.Tq + qi) * p.ldo + h * 64;
        const bf16* rrow = p.resid ? p.resid + (size_t)(b * p.Tq + qi) * p.ldr + h * 64 : nullptr;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
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

const char* attn_launch(cudaStream_t st, const void* q, int ldq, int q_rows, const void* k, int ldk, int k_rows,
                        const void* v, int ldv, const AttnParams& p) {
    if (p.B <= 0 || p.H <= 0 || p.Tq <= 0 || p.Tk <= 0) return "attention: empty problem";
    CUtensorMap tq, tk, tv;
    const char* err;
    if ((err = encode_tmap_2d(&tq, q, (uint64_t)ldq, (uint64_t)q_rows, (uint64_t)ldq, 64, 128))) return err;
    if ((err = encode_tmap_2d(&tk, k, (uint64_t)ldk, (uint64_t)k_rows, (uint64_t)ldk, 64, 128))) return err;
    if ((err = encode_tmap_2d(&tv, v, (uint64_t)ldv, (uint64_t)k_rows, (uint64_t)ldv, 64, 128))) return err;
    static bool attr_set = false;
    if (!attr_set) {
        if (cudaFuncSetAttribute(attn_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM) != cudaSuccess ||
            cudaFuncSetAttribute(attn_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM) != cudaSuccess)
            return "cudaFuncSetAttribute(attn smem) failed";
        attr_set = true;
    }
    dim3 grid((p.Tq + 127) / 128, p.H, p.B);
    cudaError_t e = p.bd ? launch_pdl(attn_tc_kernel<true>, grid, dim3(256), ATT_SMEM, st, tq, tk, tv, p)
                         : launch_pdl(attn_tc_kernel<false>, grid, dim3(256), ATT_SMEM, st, tq, tk, tv, p);
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace otb
