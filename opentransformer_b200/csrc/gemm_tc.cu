// wgmma GEMM for sm_90a:  C[M,N] = A[M,K] * W[N,K]^T  (bf16 operands, fp32 accumulate in registers)
// with the fused epilogues the speech-transformer hot path needs (bias / ReLU / GLU / x*sqrt(d)+PE /
// residual / residual+LayerNorm / swish / gelu / tanh) and an implicit-GEMM mode for the 3x3 stride-2
// Conv2d subsampling layer (A gathered by a 5-D TMA tensor map, one 64-channel tap per k-block).
//
// Replaces the cuBLAS/oneDNN calls behind nn.Linear / nn.Conv2d at
//   otrans/module/attention.py:68,128-129,44   otrans/module/ffn.py:39-41
//   otrans/frontend/conv.py:63-64,146          otrans/decoder/transformer.py:181
//
// Structure (persistent, one CTA per SM, NWG consumer warpgroups + one producer warp):
//   last warp, lane 0  : TMA producer (A tile BMx64, B tile BNx64 per k-block, SWIZZLE_128B) into a STAGES-deep
//                        full/empty mbarrier ring
//   warpgroups 0..NWG-1: consumers, warpgroup c owns tile rows [64 c, 64 c + 64): wgmma 64 x BN x 16 per k-block with
//                                one k-block in flight, accumulator in registers; then the fused epilogue on the accumulator
//                                fragment -> staged rows in smem -> coalesced 16-byte global stores (one full output row
//                                segment per warp instruction; the residual tile is fetched the same way, before the main
//                                loop, so its latency overlaps the MMAs).
// Residual + LayerNorm epilogue (N = d_model <= 256): the tile spans the whole row, the row statistics are reduced over
// the four lanes that share an accumulator row.  BN <= 128: two consumer warpgroups, 128-row tiles; BN = 256 (only the
// d_model = 256 LayerNorm GEMM): one consumer warpgroup with 64-row tiles, so that its 128 accumulator registers per
// thread fit (a CTA of 288 threads is allocated registers like one of 384: at most 168 per thread).  Static round-robin tile scheduler; the producer runs ahead into the next
// tile while the consumers drain the current one.
#include <stdlib.h>
#include <string.h>

#include "dropout.cuh"
#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

int g_tile_policy = 0;   // otb_set_tile_policy: 0 = lowest latency of a lone launch, 1 = least SM-time (concurrent batches)

static constexpr int BM = 128;
static constexpr int BK = 64;
static constexpr int STG_PITCH_MAX = 512 + 16;          // bytes per staged row (+16 B pad: conflict-free 16 B accesses)
static constexpr int STG_BYTES = BM * STG_PITCH_MAX;    // 67,584
static constexpr int AUX_BYTES = 6144;                  // barriers, bias / gamma / beta, row map

template <int BN>
struct GemmCfg {
    static constexpr int NWG = (BN == 256) ? 1 : 2;    // consumer warpgroups
    static constexpr int BM = 64 * NWG;                // tile rows
    static constexpr int THREADS = 128 * NWG + 32;
    static constexpr int A_BYTES = BM * BK * 2;
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = (BN == 256) ? 3 : (BN == 128 ? 4 : 6);
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STG_BYTES + AUX_BYTES + 1024;
};
static_assert(GemmCfg<256>::SMEM_BYTES <= 227 * 1024, "gemm_tc_kernel: shared-memory budget (227 KB per CTA)");

template <int NT>
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, %0;" ::"n"(NT) : "memory"); }

// one k16 step of the warpgroup's 64 x BN accumulator
template <int BN, int T>
__device__ __forceinline__ void mma_bn(float (&d)[BN / 2], uint64_t a, uint64_t b, uint32_t acc) {
    if constexpr (BN == 64) wgmma_n64<T, T>(d, a, b, acc);
    else if constexpr (BN == 128) wgmma_n128<T, T>(d, a, b, acc);
    else wgmma_n256<T, T>(d, a, b, acc);
}

// two adjacent output values -> staged row (bf16 pair or two floats)
__device__ __forceinline__ void stage2(uint8_t* row_ptr, int col, int out_f32, float a, float b) {
    if (out_f32) *reinterpret_cast<float2*>(row_ptr + col * 4) = make_float2(a, b);
    else *reinterpret_cast<uint32_t*>(row_ptr + col * 2) = pack_bf16(a, b);
}

// TN = true: weight-gradient mode, C[M,N] = A^T B with A = dY [K rows, M cols] and B = X [K rows, N cols], both row-major,
// i.e. both operands are MN-major in shared memory (64x64 TMA boxes, LBO = 8 KB between 64-wide MN groups, SBO = 1 KB
// between 8-row K groups).  p.splitk > 1 splits the contraction over `splitk` tiles that accumulate with fp32 atomics.
template <int BN, int EPI, bool TN = false>
__global__ void __launch_bounds__(GemmCfg<BN>::THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
    using Cfg = GemmCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int BM = Cfg::BM;
    constexpr int kEpiThreads = 128 * Cfg::NWG;
    constexpr int BN_OUT = (EPI == EPI_GLU) ? BN / 2 : BN;  // output columns per tile
    constexpr bool kResid = EPI == EPI_RESID || EPI == EPI_RESID_DROP2;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* stg = smem + STAGES * Cfg::STAGE_BYTES;
    uint8_t* aux = stg + STG_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(aux);
    uint64_t* empty_bar = full_bar + STAGES;
    float* s_bias = reinterpret_cast<float*>(aux + 256);   // [256]  (GLU: value half | gate half)
    float* s_gamma = s_bias + 256;                          // [256]
    float* s_beta = s_gamma + 256;                          // [256]
    int* s_rowmap = reinterpret_cast<int*>(s_beta + 256);   // [128] output row of each tile row, -1 = skip

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    const int m_tiles = p.conv ? (p.conv_B * p.conv_T1h + p.conv_R - 1) / p.conv_R : (p.M + BM - 1) / BM;
    const int n_tiles = (p.N + BN_OUT - 1) / BN_OUT;
    const int splitk = TN ? max(p.splitk, 1) : 1;
    const int num_tiles = m_tiles * n_tiles * splitk;
    const int num_kb_all = (p.K + BK - 1) / BK;
    // k-blocks of split ks: [ks*num_kb_all/splitk, (ks+1)*num_kb_all/splitk); without split-K: all of them
    auto kb_begin = [&](int tile) { return TN ? (int)(((long long)(tile % splitk) * num_kb_all) / splitk) : 0; };
    auto kb_end = [&](int tile) { return TN ? (int)(((long long)(tile % splitk + 1) * num_kb_all) / splitk) : num_kb_all; };
    const uint32_t a_tx = p.conv ? (uint32_t)(p.conv_R * p.conv_F2 * BK * 2) : (uint32_t)Cfg::A_BYTES;

    // One k-block load of the flat (tile, kb) sequence this CTA walks through.
    auto issue_load = [&](int tile, int kb, int stage) {
        const int mn = TN ? tile / splitk : tile;
        const int m_blk = mn / n_tiles, n_blk = mn % n_tiles;
        uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
        uint8_t* sb = sa + Cfg::A_BYTES;
        if (TN) {
            mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)(Cfg::A_BYTES + Cfg::B_BYTES));
#pragma unroll
            for (int j = 0; j < BM / 64; ++j) tma_load_2d(sa + j * 8192, &tmA, &full_bar[stage], m_blk * BM + j * 64, kb * BK);
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, &tmB, &full_bar[stage], n_blk * BN + j * 64, kb * BK);
            return;
        }
        mbar_arrive_expect_tx(&full_bar[stage], a_tx + (uint32_t)Cfg::B_BYTES);
        if (p.conv) {
            // k-block -> (tap, channel chunk); tap (kh,kw): input row st t'+kh, col sf f'+kw-pf, i.e. stride phase
            // (kh mod st, (kw-pf) mod sf) at offset (kh / st, floor((kw-pf) / sf)); negative columns are TMA zero fill
            const int tap = kb / p.conv_cchunks, cc = kb % p.conv_cchunks;
            const unsigned c = p.conv_tap[tap];
            const int par_f = c & 255, f0 = (int)((c >> 8) & 255) - 8, par_t = (c >> 16) & 255, dt = c >> 24;
            tma_load_5d(sa, &tmA, &full_bar[stage], cc * BK, par_f, f0, par_t, m_blk * p.conv_R + dt);
        } else {
            tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, m_blk * BM);
        }
        if (EPI == EPI_GLU) {
            tma_load_2d(sb, &tmB, &full_bar[stage], kb * BK, n_blk * BN_OUT);
            tma_load_2d(sb + Cfg::B_BYTES / 2, &tmB, &full_bar[stage], kb * BK, p.N + n_blk * BN_OUT);
        } else {
            tma_load_2d(sb, &tmB, &full_bar[stage], kb * BK, n_blk * BN);
        }
    };

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], Cfg::NWG);   // one arrival per consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 4 * Cfg::NWG) {
        // ------------------------------------------------------------------ TMA producer (lane 0)
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                for (int kb = kb_begin(tile), kb1 = kb_end(tile); kb < kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    issue_load(tile, kb, stage);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ------------------------------------------------------------------ consumers (256 threads, 2 warpgroups)
    const int et = threadIdx.x;             // consumer thread
    const int cw = et >> 7;                 // consumer warpgroup: tile rows [64 cw, 64 cw + 64)
    const int ewarp = et >> 5;              // 0..7
    const int rl0 = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's accumulator rows: rl0, rl0 + 8
    const int cq = 2 * (lane & 3);                              // its columns in every 8-column group: cq, cq + 1
    const int esize = p.out_f32 ? 4 : 2;
    const int pitch = BN_OUT * esize + 16;

    if (EPI == EPI_RESID_LN) {  // LayerNorm affine parameters (the tile spans the whole row)
        for (int i = et; i < BN; i += kEpiThreads) {
            s_gamma[i] = p.gamma[i];
            s_beta[i] = p.beta[i];
        }
    }
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
        const int mn_ = TN ? tile / splitk : tile;
        const int m_blk = mn_ / n_tiles, n_blk = mn_ % n_tiles;
        const int col_base = n_blk * BN_OUT;             // first output column of the tile
        const int ncols = min(BN_OUT, p.N - col_base);   // valid output columns

        // ---- (a) per-tile smem setup: bias slice, row map, residual tile (all coalesced, loads batched)
        for (int i = et; i < BN; i += kEpiThreads) {
            int c;
            if (EPI == EPI_GLU) c = (i < BN_OUT) ? col_base + i : p.N + col_base + (i - BN_OUT);
            else c = col_base + i;
            const bool ok = (EPI == EPI_GLU) ? ((i % BN_OUT) < ncols) : (i < ncols);
            s_bias[i] = (p.bias != nullptr && ok) ? p.bias[c] : 0.f;
        }
        if (et < BM) {
            const int rr = et;
            int out_row;
            bool ok;
            if (p.conv) {
                const int r = rr / p.conv_F2, f = rr % p.conv_F2;
                const int bt = m_blk * p.conv_R + r;
                const int b = bt / p.conv_T1h, t = bt % p.conv_T1h;
                ok = (r < p.conv_R) && (b < p.conv_B) && (t < p.conv_T2);
                out_row = (b * p.conv_T2 + t) * p.conv_F2 + f;
            } else {
                out_row = m_blk * BM + rr;
                ok = out_row < p.M;
            }
            s_rowmap[rr] = ok ? out_row : -1;
        }
        if (kResid || EPI == EPI_RESID_LN) {
            // residual rows are contiguous (no conv mode); 16-byte chunks, up to 8 independent loads per thread
            if ((ncols & 7) == 0) {
                const int cpr = ncols >> 3;                        // 16-byte chunks per row
                const int rows_here = min(BM, p.M - m_blk * BM);
                const int total = rows_here * cpr;
                const bf16* rbase = p.resid + (size_t)(m_blk * BM) * p.ldr + col_base;
                for (int q0 = et; q0 < total; q0 += kEpiThreads * 8) {
                    uint4 tmp[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int q = q0 + j * kEpiThreads;
                        if (q < total) tmp[j] = *reinterpret_cast<const uint4*>(rbase + (size_t)(q / cpr) * p.ldr + (q % cpr) * 8);
                    }
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int q = q0 + j * kEpiThreads;
                        if (q < total) *reinterpret_cast<uint4*>(stg + (q / cpr) * pitch + (q % cpr) * 16) = tmp[j];
                    }
                }
            } else {
                for (int r = ewarp; r < BM; r += kEpiThreads / 32) {
                    const int grow = m_blk * BM + r;
                    if (grow >= p.M) continue;
                    const bf16* src = p.resid + (size_t)grow * p.ldr + col_base;
                    for (int c = lane; c < ncols; c += 32) reinterpret_cast<bf16*>(stg + r * pitch)[c] = src[c];
                }
            }
        }

        // ---- (b) main loop: one k-block of wgmmas in flight; the stage of the previous k-block is released behind it
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        const int kb0 = kb_begin(tile), kb1 = kb_end(tile);
        int prev = -1;
        for (int kb = kb0; kb < kb1; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t a_addr = smem_u32(smem + stage * Cfg::STAGE_BYTES);
            const uint32_t b_addr = a_addr + Cfg::A_BYTES;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
                if (TN)   // MN-major operands: one k16 step = 16 rows of 128 B; this warpgroup's 64 M columns = A block cw
                    mma_bn<BN, 1>(acc, gmma_desc_sw128(a_addr + cw * 8192 + k * 2048, 1024, 8192),
                                  gmma_desc_sw128(b_addr + k * 2048, 1024, 8192), (uint32_t)(((kb - kb0) | k) != 0));
                else
                    mma_bn<BN, 0>(acc, gmma_desc_sw128(a_addr + cw * 8192 + k * 32), gmma_desc_sw128(b_addr + k * 32),
                                  (uint32_t)(((kb - kb0) | k) != 0));
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (prev >= 0 && (et & 127) == 0) mbar_arrive(&empty_bar[prev]);   // the k-block before this one has been read
            prev = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if (prev >= 0 && (et & 127) == 0) mbar_arrive(&empty_bar[prev]);
        epi_bar<kEpiThreads>();   // bias, row map and residual tile of this tile are in shared memory

        // ---- (c) fused epilogue on the accumulator fragment: rows rl0 + 8 hh, columns 8 jj + cq + {0, 1}
        int out_row[2];
        bool row_live[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            out_row[hh] = s_rowmap[rl0 + 8 * hh];
            row_live[hh] = true;
            if (p.row_len != nullptr && out_row[hh] >= 0) {
                const int b = out_row[hh] / p.row_period, t = out_row[hh] % p.row_period;
                row_live[hh] = t < p.row_len[b];
            }
        }
        if (EPI == EPI_RESID_LN) {
            float s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
#pragma unroll
            for (int jj = 0; jj < BN / 8; ++jj) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int c = jj * 8 + cq;
                    const float2 r = unpack_bf16(*reinterpret_cast<const uint32_t*>(stg + (rl0 + 8 * hh) * pitch + c * 2));
                    float x0 = acc[4 * jj + 2 * hh] + s_bias[c], x1 = acc[4 * jj + 2 * hh + 1] + s_bias[c + 1];
                    x0 = (row_live[hh] ? x0 : 0.f) + r.x;
                    x1 = (row_live[hh] ? x1 : 0.f) + r.y;
                    acc[4 * jj + 2 * hh] = x0;
                    acc[4 * jj + 2 * hh + 1] = x1;
                    s1[hh] += x0 + x1;
                    s2[hh] += x0 * x0 + x1 * x1;
                }
            }
            const float inv_n = 1.0f / (float)BN;
            float mean[2], var[2];
            bool recentre[2];
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
                for (int o = 1; o < 4; o <<= 1) {
                    s1[hh] += __shfl_xor_sync(0xffffffffu, s1[hh], o);
                    s2[hh] += __shfl_xor_sync(0xffffffffu, s2[hh], o);
                }
                mean[hh] = s1[hh] * inv_n;
                var[hh] = fmaxf(s2[hh] * inv_n - mean[hh] * mean[hh], 0.f);
                // E[x^2] - mean^2 loses about log2(mean^2 / var) bits to cancellation: beyond 6 of them, recompute the
                // variance of the centred values (a second pass over the registers, as layernorm_kernel does)
                recentre[hh] = mean[hh] * mean[hh] > 64.f * var[hh];
            }
            if (__any_sync(0xffffffffu, recentre[0] || recentre[1])) {   // warp-uniform: the whole warp shuffles
                float q[2] = {0.f, 0.f};
#pragma unroll
                for (int jj = 0; jj < BN / 8; ++jj) {
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const float d0 = acc[4 * jj + 2 * hh] - mean[hh], d1 = acc[4 * jj + 2 * hh + 1] - mean[hh];
                        q[hh] = fmaf(d0, d0, fmaf(d1, d1, q[hh]));
                    }
                }
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
                    for (int o = 1; o < 4; o <<= 1) q[hh] += __shfl_xor_sync(0xffffffffu, q[hh], o);
                    if (recentre[hh]) var[hh] = q[hh] * inv_n;
                }
            }
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const float rstd = rsqrtf(var[hh] + p.eps);
                uint8_t* row_ptr = stg + (rl0 + 8 * hh) * pitch;
#pragma unroll
                for (int jj = 0; jj < BN / 8; ++jj) {
                    const int c = jj * 8 + cq;
                    stage2(row_ptr, c, 0, (acc[4 * jj + 2 * hh] - mean[hh]) * rstd * s_gamma[c] + s_beta[c],
                           (acc[4 * jj + 2 * hh + 1] - mean[hh]) * rstd * s_gamma[c + 1] + s_beta[c + 1]);
                }
            }
        } else if (EPI == EPI_GLU) {
#pragma unroll
            for (int jj = 0; jj < BN_OUT / 8; ++jj) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int c = jj * 8 + cq;
                    float v[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float a = acc[4 * jj + 2 * hh + e] + s_bias[c + e];
                        const float g = acc[4 * (jj + BN_OUT / 8) + 2 * hh + e] + s_bias[BN_OUT + c + e];
                        v[e] = row_live[hh] ? a * fast_sigmoid(g) : 0.f;
                    }
                    stage2(stg + (rl0 + 8 * hh) * pitch, c, p.out_f32, v[0], v[1]);
                }
            }
        } else {
            const uint32_t dseed = (kResid && p.drop_seed != nullptr) ? *p.drop_seed : 0u;
#pragma unroll
            for (int jj = 0; jj < BN / 8; ++jj) {
                if (jj * 8 >= ncols) break;
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int c = jj * 8 + cq;
                    uint8_t* row_ptr = stg + (rl0 + 8 * hh) * pitch;
                    float2 res = make_float2(0.f, 0.f);
                    if (kResid) res = unpack_bf16(*reinterpret_cast<const uint32_t*>(row_ptr + c * 2));
                    float v[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float x = acc[4 * jj + 2 * hh + e] + s_bias[c + e];
                        if (EPI == EPI_RELU) x = fmaxf(x, 0.f);
                        if (EPI == EPI_SWISH) x = x * fast_sigmoid(x);
                        if (EPI == EPI_GELU) x = 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
                        if (EPI == EPI_TANH) x = tanhf(x);
                        if (EPI == EPI_TABLE)
                            x = x * p.alpha + ((c + e < ncols) ? __ldg(p.table + (size_t)((out_row[hh] >= 0 ? out_row[hh] : 0) % p.period) * p.N + col_base + c + e) : 0.f);
                        if (!row_live[hh]) x = 0.f;
                        if (EPI == EPI_RESID && p.drop_seed != nullptr)   // nn.Dropout on the sub-layer output (transformer.py:54,61)
                            x = drop_keep(dseed, p.drop_site, (uint32_t)out_row[hh], (uint32_t)(col_base + c + e), p.drop_thresh) ? x * p.drop_scale : 0.f;
                        if (EPI == EPI_RESID_DROP2) {   // and, before it, the attention's own dropout on its output (attention.py:46)
                            const uint32_t r = (uint32_t)out_row[hh], cc = (uint32_t)(col_base + c + e);
                            x = (drop_keep(dseed, p.drop_site, r, cc, p.drop_thresh) && drop_keep(dseed, p.drop_site2, r, cc, p.drop_thresh2))
                                    ? x * p.drop_scale : 0.f;
                        }
                        if (kResid) x = (e ? res.y : res.x) + p.alpha * x;
                        v[e] = x;
                    }
                    stage2(row_ptr, c, p.out_f32, v[0], v[1]);
                }
            }
        }
        epi_bar<kEpiThreads>();

        // ---- (d) coalesced copy-out: consecutive threads write consecutive 16-byte chunks of a row
        const int row_bytes = ncols * esize;
        if ((row_bytes & 15) == 0) {
            const int cpr = row_bytes >> 4;
            const int total = BM * cpr;
            uint8_t* obase = reinterpret_cast<uint8_t*>(p.out) + (size_t)col_base * esize;
            const size_t ld_bytes = (size_t)p.ldc * esize;
            for (int q0 = et; q0 < total; q0 += kEpiThreads * 4) {
                uint4 tmp[4];
                int orow[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int q = q0 + j * kEpiThreads;
                    orow[j] = -1;
                    if (q < total) {
                        const int r = q / cpr;
                        orow[j] = s_rowmap[r];
                        tmp[j] = *reinterpret_cast<const uint4*>(stg + r * pitch + (q % cpr) * 16);
                    }
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int q = q0 + j * kEpiThreads;
                    if (orow[j] < 0) continue;
                    if (TN && (splitk > 1 || p.accum)) {   // partial sums meet in the fp32 output (pre-zeroed, or a running gradient)
                        float* dst = reinterpret_cast<float*>(obase + (size_t)orow[j] * ld_bytes + (q % cpr) * 16);
                        atomicAdd(dst, __uint_as_float(tmp[j].x));
                        atomicAdd(dst + 1, __uint_as_float(tmp[j].y));
                        atomicAdd(dst + 2, __uint_as_float(tmp[j].z));
                        atomicAdd(dst + 3, __uint_as_float(tmp[j].w));
                    } else {
                        *reinterpret_cast<uint4*>(obase + (size_t)orow[j] * ld_bytes + (q % cpr) * 16) = tmp[j];
                    }
                }
            }
        } else {
            for (int r = ewarp; r < BM; r += kEpiThreads / 32) {
                const int orow = s_rowmap[r];
                if (orow < 0) continue;
                const uint8_t* src = stg + r * pitch;
                uint8_t* dst = reinterpret_cast<uint8_t*>(p.out) + ((size_t)orow * p.ldc + col_base) * esize;
                if (TN && (splitk > 1 || p.accum)) {   // as above, one fp32 element at a time (ncols % 4 != 0)
                    for (int c = lane; c < ncols; c += 32)
                        atomicAdd(reinterpret_cast<float*>(dst) + c, reinterpret_cast<const float*>(src)[c]);
                } else {
                    for (int off = lane * 2; off < row_bytes; off += 64)
                        *reinterpret_cast<uint16_t*>(dst + off) = *reinterpret_cast<const uint16_t*>(src + off);
                }
            }
        }
        epi_bar<kEpiThreads>();  // staging / bias smem may be rewritten for the next tile
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    if (fn) return fn;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
        return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(ptr);
    return fn;
}

const char* encode_tmap_2d(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint64_t ld_elems,
                           uint32_t box_cols, uint32_t box_rows) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) return "cuTensorMapEncodeTiled unavailable (no CUDA driver?)";
    if ((reinterpret_cast<uintptr_t>(base) & 15) || (ld_elems & 7)) return "TMA operand must be 16-byte aligned with ld % 8 == 0";
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {ld_elems * 2};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? nullptr : "cuTensorMapEncodeTiled(2d) failed";
}

// fp32, no swizzle: box_cols consecutive floats (a multiple of 4) of box_rows consecutive rows land densely in shared memory
const char* encode_tmap_2d_f32(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint64_t ld_elems,
                               uint32_t box_cols, uint32_t box_rows) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) return "cuTensorMapEncodeTiled unavailable (no CUDA driver?)";
    if ((reinterpret_cast<uintptr_t>(base) & 15) || (ld_elems & 3) || (box_cols & 3) || box_cols > 256 || box_rows > 256)
        return "fp32 TMA operand must be 16-byte aligned with ld % 4 == 0 and a box of <= 256 x 256";
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {ld_elems * 4};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? nullptr : "cuTensorMapEncodeTiled(2d, fp32) failed";
}

// conv1 output buffer [B, st*T1s, sf*F1s, C] bf16 viewed as (c, f mod sf, f / sf, t mod st, b*T1s + t / st)
const char* encode_tmap_conv5d(CUtensorMap* m, const void* base, int C, int sf, int F1s, int st, int T1s_total, uint32_t boxF,
                               uint32_t boxR) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) return "cuTensorMapEncodeTiled unavailable (no CUDA driver?)";
    cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)sf, (cuuint64_t)F1s, (cuuint64_t)st, (cuuint64_t)T1s_total};
    cuuint64_t strides[4] = {(cuuint64_t)C * 2, (cuuint64_t)C * sf * 2, (cuuint64_t)F1s * sf * C * 2,
                             (cuuint64_t)F1s * sf * C * st * 2};
    cuuint32_t box[5] = {64, 1, boxF, 1, boxR};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? nullptr : "cuTensorMapEncodeTiled(5d) failed";
}

int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
    }
    return n;
}

template <int BN, int EPI, bool TN = false>
static const char* launch_inst(cudaStream_t st, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                               int num_tiles) {
    using Cfg = GemmCfg<BN>;
    const int grid = num_tiles < num_sms() ? num_tiles : num_sms();
    return launch<gemm_tc_kernel<BN, EPI, TN>>(dim3(grid), dim3(Cfg::THREADS), Cfg::SMEM_BYTES, st, ta, tb, p);
}

template <int BN>
static const char* launch_bn(cudaStream_t st, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                             int epi, int num_tiles) {
    switch (epi) {
        case EPI_BIAS: return launch_inst<BN, EPI_BIAS>(st, ta, tb, p, num_tiles);
        case EPI_RELU: return launch_inst<BN, EPI_RELU>(st, ta, tb, p, num_tiles);
        case EPI_GLU: return launch_inst<BN, EPI_GLU>(st, ta, tb, p, num_tiles);
        case EPI_TABLE: return launch_inst<BN, EPI_TABLE>(st, ta, tb, p, num_tiles);
        case EPI_RESID: return launch_inst<BN, EPI_RESID>(st, ta, tb, p, num_tiles);
        case EPI_RESID_DROP2: return launch_inst<BN, EPI_RESID_DROP2>(st, ta, tb, p, num_tiles);
        case EPI_RESID_LN: return launch_inst<BN, EPI_RESID_LN>(st, ta, tb, p, num_tiles);
        case EPI_SWISH: return launch_inst<BN, EPI_SWISH>(st, ta, tb, p, num_tiles);
        case EPI_GELU: return launch_inst<BN, EPI_GELU>(st, ta, tb, p, num_tiles);
        case EPI_TANH: return launch_inst<BN, EPI_TANH>(st, ta, tb, p, num_tiles);
    }
    return "unknown epilogue";
}

// Pick the N tile that wastes the fewest MMA cycles across the persistent grid.
static int choose_bn(int m_tiles, int n_cols, int epi, int out_f32) {
    // Decode regime (<= 4 row blocks, M = batch x beam rows): a launch lasts about as long whatever its tiling, and
    // utterance batches running concurrently on other streams are bound by the SM-time the launches occupy.  Under the
    // throughput policy small problems therefore take the WIDEST tile (fewer CTAs for slightly more latency); the serving
    // layer picks the policy (otb_set_tile_policy), latency is the default.
    const bool decode = (m_tiles <= 4) && g_tile_policy == 1;
    // residual + LayerNorm: the tile spans the whole row (N <= 256), so the row statistics never leave the CTA
    if (epi == EPI_RESID_LN) return n_cols;
    const int sms = num_sms();
    int best = 0;
    double best_cost = 1e30;
    const int cands[2] = {128, 64};   // 256-wide tiles run on one warpgroup (64-row tiles): kept for the LayerNorm row only
    for (int i = 0; i < 2; ++i) {
        const int bn = cands[i];
        const int bn_out = (epi == EPI_GLU) ? bn / 2 : bn;
        if (bn_out * (out_f32 ? 4 : 2) > 512) continue;  // staged row must fit the staging pitch
        if (bn_out < 64) continue;                       // at least 128-byte staged row segments for the copy-out
        const int n_tiles = (n_cols + bn_out - 1) / bn_out;
        const long tiles = (long)m_tiles * n_tiles;
        const long waves = (tiles + sms - 1) / sms;
        // large problems: fewest MMA cycles across the persistent grid (+48: per-tile fixed overhead in "column" units);
        // decode regime: least SM-time (+200: the fixed ~8 us of a launch expressed in the same units)
        const double cost = decode ? (double)tiles * (bn + 200) : (double)waves * (bn + 48);
        if (cost < best_cost - 1e-9) { best_cost = cost; best = bn; }
    }
    return best;
}

// The checks of gemm_launch that depend only on the output shape, the epilogue and the output type, and the tile width
// it launches (m_tiles 128-row blocks, current tile policy).  Host only: otb_gemm_config answers with it.
const char* gemm_tile(int m_tiles, int N, int epi, int out_f32, int* bn) {
    if (epi == EPI_RESID_LN && !(N == 64 || N == 128 || N == 256))
        return "gemm: fused residual+LayerNorm epilogue needs N in {64,128,256}";
    if (epi == EPI_RESID_LN && out_f32) return "gemm: fused residual+LayerNorm epilogue writes bf16";
    // the residual tile is staged as bf16 in the rows the fp32 results would overwrite
    if ((epi == EPI_RESID || epi == EPI_RESID_DROP2) && out_f32) return "gemm: residual epilogue writes bf16";
    *bn = choose_bn(m_tiles, N, epi, out_f32);
    return *bn == 0 ? "gemm: no tile configuration" : nullptr;
}

const char* gemm_launch(cudaStream_t st, const void* A, int lda, const void* W, int ldw, int w_rows, int epi,
                        GemmParams p, const CUtensorMap* conv_map) {
    if (p.M <= 0 || p.N <= 0 || p.K <= 0) return "gemm: empty problem";
    if (p.K % 8) return "gemm: K must be a multiple of 8";
    if (p.ldc % (p.out_f32 ? 4 : 8)) return "gemm: ldc must keep rows 16-byte aligned (ldc % 8 == 0 for bf16, % 4 for f32)";
    if (reinterpret_cast<uintptr_t>(p.out) & 15) return "gemm: out must be 16-byte aligned";
    if ((epi == EPI_RESID || epi == EPI_RESID_DROP2 || epi == EPI_RESID_LN) && ((p.ldr % 8) || (reinterpret_cast<uintptr_t>(p.resid) & 15)))
        return "gemm: residual must be 16-byte aligned with ldr % 8 == 0";
    const int m_tiles = p.conv ? (p.conv_B * p.conv_T1h + p.conv_R - 1) / p.conv_R : (p.M + BM - 1) / BM;
    int bn = 0;
    const char* err;
    if ((err = gemm_tile(m_tiles, p.N, epi, p.out_f32, &bn))) return err;
    const int bn_out = (epi == EPI_GLU) ? bn / 2 : bn;
    const int n_tiles = (p.N + bn_out - 1) / bn_out;
    const int bm = (bn == 256) ? GemmCfg<256>::BM : BM;   // rows per tile of the chosen configuration
    if (p.conv && bm != BM) return "gemm: conv mode needs 128-row tiles";
    const int num_tiles = (p.conv ? m_tiles : (p.M + bm - 1) / bm) * n_tiles;

    CUtensorMap ta, tb;
    if (p.conv) {
        if (!conv_map) return "gemm: conv mode needs a conv tensor map";
        ta = *conv_map;
    } else {
        if ((err = encode_tmap_2d(&ta, A, (uint64_t)p.K, (uint64_t)p.M, (uint64_t)lda, BK, (uint32_t)bm))) return err;
    }
    const uint32_t box_rows = (epi == EPI_GLU) ? (uint32_t)(bn / 2) : (uint32_t)bn;
    if ((err = encode_tmap_2d(&tb, W, (uint64_t)p.K, (uint64_t)w_rows, (uint64_t)ldw, BK, box_rows))) return err;

    switch (bn) {
        case 256: return launch_bn<256>(st, ta, tb, p, epi, num_tiles);
        case 128: return launch_bn<128>(st, ta, tb, p, epi, num_tiles);
        case 64: return launch_bn<64>(st, ta, tb, p, epi, num_tiles);
    }
    return "gemm: bad tile";
}

// Weight gradient dW[Nw, Kw] (fp32) = dY[Mact, Nw]^T X[Mact, Kw]  (both bf16 row-major): TN mode of the kernel above.
// The contraction (Mact rows, thousands) is split over enough tiles to fill the SMs; splits meet through fp32 atomics,
// so `out` must be zero on entry when the returned split count is > 1 (the launcher zeroes it with a memset node).
const char* gemm_wgrad_launch(cudaStream_t st, const void* dY, int lddy, const void* X, int ldx, float* out, int ldc,
                              int Mact, int Nw, int Kw, int accumulate) {
    if (Mact <= 0 || Nw <= 0 || Kw <= 0) return "wgrad: empty problem";
    if ((lddy % 8) || (ldx % 8) || (ldc % 4) || (reinterpret_cast<uintptr_t>(out) & 15)) return "wgrad: operands must be 16-byte aligned (ld % 8 bf16, ldc % 4 f32)";
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.M = Nw; p.N = Kw; p.K = Mact;
    p.out = out; p.ldc = ldc; p.out_f32 = 1; p.alpha = 1.f;
    const int bn = (Kw > 64) ? 128 : 64;
    const int m_tiles = (Nw + BM - 1) / BM, n_tiles = (Kw + bn - 1) / bn;
    const int num_kb = (Mact + BK - 1) / BK;
    int splitk = num_sms() / (m_tiles * n_tiles);
    if (splitk > num_kb / 4) splitk = num_kb / 4;      // at least 4 k-blocks per split
    if (splitk < 1) splitk = 1;
    p.splitk = splitk;
    p.accum = accumulate ? 1 : 0;      // out += dY^T X (gradient accumulation): no memset, every tile adds atomically
    if (splitk > 1 && !accumulate) {
        cudaError_t e = cudaMemset2DAsync(out, (size_t)ldc * 4, 0, (size_t)Kw * 4, (size_t)Nw, st);
        if (e != cudaSuccess) return cudaGetErrorString(e);
    }
    CUtensorMap ta, tb;
    const char* err;
    if ((err = encode_tmap_2d(&ta, dY, (uint64_t)Nw, (uint64_t)Mact, (uint64_t)lddy, 64, 64))) return err;
    if ((err = encode_tmap_2d(&tb, X, (uint64_t)Kw, (uint64_t)Mact, (uint64_t)ldx, 64, 64))) return err;
    const int num_tiles = m_tiles * n_tiles * splitk;
    return bn == 128 ? launch_inst<128, EPI_BIAS, true>(st, ta, tb, p, num_tiles)
                     : launch_inst<64, EPI_BIAS, true>(st, ta, tb, p, num_tiles);
}

}  // namespace otb
