// Backward of the fused masked multi-head attention (attn_tc.cu), d_k = 64, on wgmma tensor cores.
// Differentiates BasedAttention.compute_context + the QK^T product (otrans/module/attention.py:80,34-41), which the
// reference leaves to torch autograd.  Flash-attention style: nothing of size [B,h,T,T] is stored by the forward
// (only the per-row log-sum-exp), scores are recomputed here.
//
//   S = Q K^T ; P = exp2(S*c - L)  (c = log2(e)/sqrt(d_k), L = row log-sum-exp in log2 units from the forward)
//   dP = dO V^T ; D_i = sum_d dO_id O_id ; dS = P * (dP - D) / sqrt(d_k)
//   dQ = dS K ; dK = dS^T Q ; dV = P^T dO
//
// Two kernels so that every accumulation stays inside one CTA (no atomics):
//   attn_bwd_dq_kernel : CTA = 128 query rows of one (batch, head); loops over key blocks;  writes dQ and D
//   attn_bwd_dkv_kernel: CTA = 128 key rows   of one (batch, head); loops over query blocks; writes dK and dV
// 256 threads = two warpgroups, warpgroup w owns tile rows [64 w, 64 w + 64); every contraction is a wgmma 64xNx16 per
// warpgroup with operands staged by TMA (K-major tiles; the [rows x 64] tile that is contracted over its rows is read as
// an MN-major B operand, exactly like V in the forward); dS / P^T tiles are written by the threads as bf16 in the
// canonical 128B-swizzled layout.  Score tiles are formed in two 64-column halves to bound the register footprint.
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

static constexpr int ABW_SMEM_DQ = 16384 * 4 + 32768 + 256 + 1024 + 1024;           // Q, dO, K, V, dS, barriers, L/D
static constexpr int ABW_SMEM_DKV = 16384 * 4 + 32768 * 2 + 1024 + 256 + 1024;      // K, V, Q, dO, P^T, dS^T, L/D

__device__ __forceinline__ float ex2a(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// bf16 pair (row, col), (row, col + 1) of a [128 rows x 128] tile in the K-major SW128 layout (two 64-column k-blocks)
__device__ __forceinline__ void put_pair(uint8_t* tile, int row, int col, float a, float b) {
    *reinterpret_cast<uint32_t*>(tile + (col >> 6) * 16384 + row * 128 + ((((col & 63) >> 3) ^ (row & 7)) << 4) + (col & 7) * 2) =
        pack_bf16(a, b);
}

// 64 x 64 fp32 fragment (wgmma n64 accumulator) of rows rl0, rl0 + 8 -> bf16 rows of dst (zeros for rows that are not ok)
__device__ __forceinline__ void store_rows64(const float (&acc)[32], bf16* base, size_t ld, int row0_global, int rl0, int cq,
                                             bool ok0, bool ok1) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        if (!(hh ? ok1 : ok0)) continue;
        bf16* o = base + (size_t)(row0_global + rl0 + 8 * hh) * ld;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
            *reinterpret_cast<uint32_t*>(o + jj * 8 + cq) = pack_bf16(acc[4 * jj + 2 * hh], acc[4 * jj + 2 * hh + 1]);
    }
}

// ------------------------------------------------------------------------------------------------ dQ
__global__ void __launch_bounds__(256, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                   const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO, const AttnBwdParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;
    uint8_t* sdO = smem + 16384;
    uint8_t* sK = smem + 32768;
    uint8_t* sV = smem + 49152;
    uint8_t* sdS = smem + 65536;                                   // 2 k-blocks x [128 rows x 128 B]
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 65536 + 32768);   // 0: Q+dO, 1: K+V
    float* sL = reinterpret_cast<float*>(smem + 65536 + 32768 + 256);    // [128] log-sum-exp of the query rows
    float* sD = sL + 128;                                                // [128] D of the query rows

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int q0 = blockIdx.x * 128, h = blockIdx.y, b = blockIdx.z;
    const int kv_len = p.kv_len ? min(p.kv_len[b], p.Tk) : p.Tk;
    int kv_end = kv_len;
    if (p.causal) kv_end = min(kv_end, q0 + 128);
    const int nblk = (kv_end + 127) / 128;

    if (tid == 0) {
        for (int i = 0; i < 2; ++i) mbar_init(&bar[i], 1);
        fence_barrier_init();
        tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmdO);
        mbar_arrive_expect_tx(&bar[0], 32768);
        tma_load_2d(sQ, &tmQ, &bar[0], p.q_col0 + h * 64, b * p.Tq + q0);
        tma_load_2d(sdO, &tmdO, &bar[0], h * 64, b * p.Tq + q0);
        if (nblk > 0) {
            mbar_arrive_expect_tx(&bar[1], 32768);
            tma_load_2d(sK, &tmK, &bar[1], p.k_col0 + h * 64, b * p.Tk);
            tma_load_2d(sV, &tmV, &bar[1], p.v_col0 + h * 64, b * p.Tk);
        }
    }
    if (tid < 128) {   // D_i = dO_i . O_i and the row's log-sum-exp
        const int qi = q0 + tid;
        float Dv = 0.f, Lv = 0.f;
        if (qi < p.Tq) {
            const bf16* orow = p.o + (size_t)(b * p.Tq + qi) * p.ldo + h * 64;
            const bf16* drow = p.dout + (size_t)(b * p.Tq + qi) * p.lddo + h * 64;
#pragma unroll
            for (int i = 0; i < 64; i += 8) {
                const uint4 uo = *reinterpret_cast<const uint4*>(orow + i), ud = *reinterpret_cast<const uint4*>(drow + i);
                const float2 o0 = unpack_bf16(uo.x), o1 = unpack_bf16(uo.y), o2 = unpack_bf16(uo.z), o3 = unpack_bf16(uo.w);
                const float2 d0 = unpack_bf16(ud.x), d1 = unpack_bf16(ud.y), d2 = unpack_bf16(ud.z), d3 = unpack_bf16(ud.w);
                Dv += o0.x * d0.x + o0.y * d0.y + o1.x * d1.x + o1.y * d1.y + o2.x * d2.x + o2.y * d2.y + o3.x * d3.x + o3.y * d3.y;
            }
            Lv = p.lse[((size_t)b * p.H + h) * p.Tq + qi];
            p.dsum[((size_t)b * p.H + h) * p.Tq + qi] = Dv;
        }
        sL[tid] = Lv;
        sD[tid] = Dv;
    }
    __syncthreads();

    const int rl0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), cq = 2 * (lane & 3);
    bool q_ok[2];
    int lim[2];
    float Lr[2], Dr[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int qi = q0 + rl0 + 8 * hh;
        q_ok[hh] = qi < p.Tq;
        lim[hh] = p.causal ? min(kv_len, qi + 1) : kv_len;
        Lr[hh] = sL[rl0 + 8 * hh];
        Dr[hh] = sD[rl0 + 8 * hh];
    }
    const uint32_t qa = smem_u32(sQ) + wg * 8192, da = smem_u32(sdO) + wg * 8192, ka = smem_u32(sK), va = smem_u32(sV);
    const uint32_t sa = smem_u32(sdS) + wg * 8192;
    const float scale = 0.125f;
    float dq[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) dq[i] = 0.f;

    for (int blk = 0; blk < nblk; ++blk) {
        const uint32_t ph = blk & 1;
        const int key0 = blk * 128;
        if (blk == 0) mbar_wait(&bar[0], 0);
        mbar_wait(&bar[1], ph);
#pragma unroll 1
        for (int kh = 0; kh < 2; ++kh) {     // keys [64 kh, 64 kh + 64) of the block
            float sc[32], dp[32];
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)      // S = Q K^T
                wgmma_n64<0, 0>(sc, gmma_desc_sw128(qa + k * 32), gmma_desc_sw128(ka + kh * 8192 + k * 32), (uint32_t)(k != 0));
#pragma unroll
            for (int k = 0; k < 4; ++k)      // dP = dO V^T
                wgmma_n64<0, 0>(dp, gmma_desc_sw128(da + k * 32), gmma_desc_sw128(va + kh * 8192 + k * 32), (uint32_t)(k != 0));
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(sc);
            wgmma_fence_regs(dp);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float ds[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int i = 4 * jj + 2 * hh + e;
                        const int key = key0 + kh * 64 + jj * 8 + cq + e;
                        const float pv = ex2a(fmaf(sc[i], p.scale_log2, -Lr[hh]));
                        const float v = pv * (dp[i] - Dr[hh]) * scale;
                        ds[e] = (q_ok[hh] && key < lim[hh]) ? v : 0.f;
                    }
                    put_pair(sdS, rl0 + 8 * hh, kh * 64 + jj * 8 + cq, ds[0], ds[1]);
                }
            }
        }
        fence_proxy_async_smem();
        __syncthreads();
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)   // dQ += dS K   (K block read as an MN-major B operand: N = 64 dims, K = keys)
            wgmma_n64<0, 1>(dq, gmma_desc_sw128(sa + (kk >> 2) * 16384 + (kk & 3) * 32), gmma_desc_sw128(ka + kk * 2048, 1024, 8192), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(dq);
        __syncthreads();                     // K, V, dS tiles are free again
        if (tid == 0 && blk + 1 < nblk) {
            mbar_arrive_expect_tx(&bar[1], 32768);
            tma_load_2d(sK, &tmK, &bar[1], p.k_col0 + h * 64, b * p.Tk + key0 + 128);
            tma_load_2d(sV, &tmV, &bar[1], p.v_col0 + h * 64, b * p.Tk + key0 + 128);
        }
    }
    store_rows64(dq, p.dq + p.dq_col0 + h * 64, (size_t)p.lddq, b * p.Tq + q0, rl0, cq, q_ok[0], q_ok[1]);
}

// ------------------------------------------------------------------------------------------------ dK, dV
__global__ void __launch_bounds__(256, 1)
attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO, const AttnBwdParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sK = smem;
    uint8_t* sV = smem + 16384;
    uint8_t* sQ = smem + 32768;
    uint8_t* sdO = smem + 49152;
    uint8_t* sPt = smem + 65536;
    uint8_t* sdSt = smem + 98304;
    float* sL = reinterpret_cast<float*>(smem + 131072);           // [128] log-sum-exp of the query block
    float* sD = sL + 128;                                          // [128] D of the query block
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 131072 + 1024);   // 0: K+V, 1: Q+dO

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int j0 = blockIdx.x * 128, h = blockIdx.y, b = blockIdx.z;
    const int kv_len = p.kv_len ? min(p.kv_len[b], p.Tk) : p.Tk;
    // query blocks that can see this key tile: causal -> queries i >= j0
    const int iblk0 = p.causal ? j0 / 128 : 0;
    const int nq = (p.Tq + 127) / 128;
    const bool tile_live = j0 < kv_len;        // a fully masked key tile gets zero gradients
    const bool any = tile_live && iblk0 < nq;

    if (tid == 0) {
        for (int i = 0; i < 2; ++i) mbar_init(&bar[i], 1);
        fence_barrier_init();
        tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmdO);
        if (any) {
            mbar_arrive_expect_tx(&bar[0], 32768);
            tma_load_2d(sK, &tmK, &bar[0], p.k_col0 + h * 64, b * p.Tk + j0);
            tma_load_2d(sV, &tmV, &bar[0], p.v_col0 + h * 64, b * p.Tk + j0);
            mbar_arrive_expect_tx(&bar[1], 32768);
            tma_load_2d(sQ, &tmQ, &bar[1], p.q_col0 + h * 64, b * p.Tq + iblk0 * 128);
            tma_load_2d(sdO, &tmdO, &bar[1], h * 64, b * p.Tq + iblk0 * 128);
        }
    }
    __syncthreads();

    const int rl0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), cq = 2 * (lane & 3);
    int kj[2];
    bool k_ok[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        kj[hh] = j0 + rl0 + 8 * hh;            // this thread's keys
        k_ok[hh] = kj[hh] < kv_len;
    }
    const uint32_t ka = smem_u32(sK) + wg * 8192, va = smem_u32(sV) + wg * 8192, qa = smem_u32(sQ), da = smem_u32(sdO);
    const uint32_t pa = smem_u32(sPt) + wg * 8192, sa = smem_u32(sdSt) + wg * 8192;
    const float scale = 0.125f;
    float dv[32], dk[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { dv[i] = 0.f; dk[i] = 0.f; }

    if (any) {
        int it = 0;
        for (int ib = iblk0; ib < nq; ++ib, ++it) {
            const uint32_t ph = it & 1;
            const int i0 = ib * 128;
            if (tid < 128) {   // statistics of this query block
                const int qi = i0 + tid;
                const bool ok = qi < p.Tq;
                sL[tid] = ok ? p.lse[((size_t)b * p.H + h) * p.Tq + qi] : 0.f;
                sD[tid] = ok ? p.dsum[((size_t)b * p.H + h) * p.Tq + qi] : 0.f;
            }
            if (it == 0) mbar_wait(&bar[0], 0);
            mbar_wait(&bar[1], ph);
            __syncthreads();                     // sL / sD visible
#pragma unroll 1
            for (int qh = 0; qh < 2; ++qh) {     // queries [64 qh, 64 qh + 64) of the block
                float st[32], dpt[32];
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k)      // S^T = K Q^T
                    wgmma_n64<0, 0>(st, gmma_desc_sw128(ka + k * 32), gmma_desc_sw128(qa + qh * 8192 + k * 32), (uint32_t)(k != 0));
#pragma unroll
                for (int k = 0; k < 4; ++k)      // dP^T = V dO^T
                    wgmma_n64<0, 0>(dpt, gmma_desc_sw128(va + k * 32), gmma_desc_sw128(da + qh * 8192 + k * 32), (uint32_t)(k != 0));
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_regs(st);
                wgmma_fence_regs(dpt);
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        float pt[2], ds[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int i = 4 * jj + 2 * hh + e;
                            const int c = qh * 64 + jj * 8 + cq + e;
                            const int qi = i0 + c;
                            const bool vis = k_ok[hh] && qi < p.Tq && (!p.causal || kj[hh] <= qi);
                            const float pv = ex2a(fmaf(st[i], p.scale_log2, -sL[c]));
                            const float dvv = pv * (dpt[i] - sD[c]) * scale;
                            pt[e] = vis ? pv : 0.f;
                            ds[e] = vis ? dvv : 0.f;
                        }
                        put_pair(sPt, rl0 + 8 * hh, qh * 64 + jj * 8 + cq, pt[0], pt[1]);
                        put_pair(sdSt, rl0 + 8 * hh, qh * 64 + jj * 8 + cq, ds[0], ds[1]);
                    }
                }
            }
            fence_proxy_async_smem();
            __syncthreads();
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 8; ++kk)   // dV += P^T dO   (dO block as MN-major B: N = 64 dims, K = queries)
                wgmma_n64<0, 1>(dv, gmma_desc_sw128(pa + (kk >> 2) * 16384 + (kk & 3) * 32), gmma_desc_sw128(da + kk * 2048, 1024, 8192), 1u);
#pragma unroll
            for (int kk = 0; kk < 8; ++kk)   // dK += dS^T Q
                wgmma_n64<0, 1>(dk, gmma_desc_sw128(sa + (kk >> 2) * 16384 + (kk & 3) * 32), gmma_desc_sw128(qa + kk * 2048, 1024, 8192), 1u);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(dv);
            wgmma_fence_regs(dk);
            __syncthreads();                     // Q, dO, P^T, dS^T and the statistics may be overwritten
            if (tid == 0 && ib + 1 < nq) {
                mbar_arrive_expect_tx(&bar[1], 32768);
                tma_load_2d(sQ, &tmQ, &bar[1], p.q_col0 + h * 64, b * p.Tq + i0 + 128);
                tma_load_2d(sdO, &tmdO, &bar[1], h * 64, b * p.Tq + i0 + 128);
            }
        }
    }

    // ---- write dV / dK rows (zeros for masked / out-of-range keys so that the caller's buffer is fully defined)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        if (!k_ok[hh]) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                dv[4 * jj + 2 * hh] = dv[4 * jj + 2 * hh + 1] = 0.f;
                dk[4 * jj + 2 * hh] = dk[4 * jj + 2 * hh + 1] = 0.f;
            }
        }
    }
    const bool row_ok0 = kj[0] < p.Tk, row_ok1 = kj[1] < p.Tk;
    store_rows64(dv, p.dv + p.dv_col0 + h * 64, (size_t)p.lddv, b * p.Tk + j0, rl0, cq, row_ok0, row_ok1);
    store_rows64(dk, p.dk + p.dk_col0 + h * 64, (size_t)p.lddk, b * p.Tk + j0, rl0, cq, row_ok0, row_ok1);
}

const char* attn_bwd_launch(cudaStream_t st, const void* q, int ldq, int q_rows, const void* k, int ldk, int k_rows,
                            const void* v, int ldv, const AttnBwdParams& p) {
    if (p.B <= 0 || p.H <= 0 || p.Tq <= 0 || p.Tk <= 0) return "attention_bwd: empty problem";
    CUtensorMap tq, tk, tv, tdo;
    const char* err;
    if ((err = encode_tmap_2d(&tq, q, (uint64_t)ldq, (uint64_t)q_rows, (uint64_t)ldq, 64, 128))) return err;
    if ((err = encode_tmap_2d(&tk, k, (uint64_t)ldk, (uint64_t)k_rows, (uint64_t)ldk, 64, 128))) return err;
    if ((err = encode_tmap_2d(&tv, v, (uint64_t)ldv, (uint64_t)k_rows, (uint64_t)ldv, 64, 128))) return err;
    if ((err = encode_tmap_2d(&tdo, p.dout, (uint64_t)p.lddo, (uint64_t)q_rows, (uint64_t)p.lddo, 64, 128))) return err;
    static bool attr_set = false;
    if (!attr_set) {
        if (cudaFuncSetAttribute(attn_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ABW_SMEM_DQ) != cudaSuccess ||
            cudaFuncSetAttribute(attn_bwd_dkv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ABW_SMEM_DKV) != cudaSuccess)
            return "cudaFuncSetAttribute(attn_bwd smem) failed";
        attr_set = true;
    }
    attn_bwd_dq_kernel<<<dim3((p.Tq + 127) / 128, p.H, p.B), 256, ABW_SMEM_DQ, st>>>(tq, tk, tv, tdo, p);
    attn_bwd_dkv_kernel<<<dim3((p.Tk + 127) / 128, p.H, p.B), 256, ABW_SMEM_DKV, st>>>(tq, tk, tv, tdo, p);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace otb
