// LSTM layer recurrence (nn.LSTM: gates i, f, g, o; c_t = s(f) c_{t-1} + s(i) tanh(g), h_t = s(o) tanh(c_t)) forward and
// backward through time, as two persistent kernels launched cooperatively, plus the embedding gather of the RNN LM.
//
// The input projection G_x = X W_ih^T + (b_ih + b_hh) of all L*B rows is one otb_linear call in front; what is left is
// the sequential part.  Sequences are time-major: row t*B + b.
//
// Forward: CTA j owns hidden units U_j = [j u, j u + u) and keeps the W_hh rows of all four gates of those units resident
// in shared memory (4u x H bf16, 64 KB at u = 8, H = 1024): the weights are read from L2 once per launch, never per step.
// At each step it stages h_{t-1} (bf16, written by every CTA in the step before) in row chunks, forms its 4u x chunk slice
// of W_hh h_{t-1}^T with mma.sync (weight rows = m16 operand, batch rows = n8 operand, the contraction split over the
// warps), adds G_x and updates the cell of its own units -- it owns all four gates of each unit, so no gate crosses CTAs --
// and meets the other CTAs at a grid barrier.  c_{t-1} is read back from the c_n buffer by the thread that wrote it.
//
// Backward: the same CTA owns the W_hh COLUMNS of its units (u x 4H, transposed into shared memory) and forms
// dh_t[:, U_j] = dy_t[:, U_j] + dG_{t+1} W_hh[:, U_j] in reverse time order, carrying dc in a buffer only the owning thread
// touches, and writes dG_t (bf16, the pre-activation gate gradient).  Everything after the loop is otb_linear_wgrad,
// otb_colsum and otb_linear.
//
// Grid barrier: the launch is cooperative, so all CTAs are co-resident (checked against the occupancy first), every CTA
// runs every barrier, and the counter is generation based ({arrivals, generation}: the last arrival resets the count and
// bumps the generation), so it needs no reset between launches.
#include <stdint.h>

#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

namespace {

constexpr int LSTM_THREADS = 256;
constexpr int LSTM_WARPS = LSTM_THREADS / 32;
constexpr int BWD_ROWS = 16;            // batch rows per backward chunk (two n8 blocks)

__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + __expf(-x)); }

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u32(unsigned* p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// All CTAs of the (co-resident) grid have finished the step and their global writes are visible.  bar = {arrivals,
// generation}: the generation is read BEFORE arriving (it cannot advance until this CTA has arrived); the last arrival
// resets the count and publishes generation + 1, the others wait for it.
__device__ __forceinline__ void grid_sync(unsigned* bar) {
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned gen = ld_acquire_u32(bar + 1);
        __threadfence();
        if (atomicAdd(bar, 1u) == gridDim.x - 1) {
            atomicExch(bar, 0u);
            __threadfence();
            st_release_u32(bar + 1, gen + 1);
        } else {
            const long long t0 = clock64();
            uint32_t spins = 0;
            while (ld_acquire_u32(bar + 1) == gen) {
                if (((++spins) & 0x3FF) == 0 && (clock64() - t0) > 20000000000LL) __trap();   // a protocol bug traps instead of hanging
            }
        }
    }
    __syncthreads();
}

// Partial sums of out^T[16 MT x 8 NRB] = W[16 MT x K] . X[8 NRB x K]^T, k16 steps ks = warp, warp + 8, ... (the contraction
// is split over the warps).  Weight row r reads smem row r & wmask (the backward's u = 8 columns fill half an m16 tile: the
// other half repeats them and is discarded).  Warp w's partials land in red[w][n][f], row pitch 16 MT + 1.
template <int MT, int NRB>
__device__ __forceinline__ void slice_product(const bf16* sW, int wmask, const bf16* sX, int ld, int nks, float* red, int warp,
                                              int lane) {
    float acc[MT][NRB][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int rb = 0; rb < NRB; ++rb)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[mt][rb][i] = 0.f;
    const int m = lane >> 3, rr = lane & 7;
#pragma unroll 1
    for (int ks = warp; ks < nks; ks += LSTM_WARPS) {
        uint32_t b[NRB][2];
#pragma unroll
        for (int rb = 0; rb < NRB; ++rb)      // (rows 0-7, k lo) (rows 0-7, k hi); lanes 16-31 repeat valid addresses
            ldmatrix_x2(smem_u32(sX + (rb * 8 + rr) * ld + ks * 16 + (m & 1) * 8), b[rb][0], b[rb][1]);
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
            uint32_t a0, a1, a2, a3;          // (rows 0-7, k lo) (rows 8-15, k lo) (rows 0-7, k hi) (rows 8-15, k hi)
            const int row = (mt * 16 + (m & 1) * 8 + rr) & wmask;
            ldmatrix_x4(smem_u32(sW + row * ld + ks * 16 + (m >> 1) * 8), a0, a1, a2, a3);
#pragma unroll
            for (int rb = 0; rb < NRB; ++rb) mma_m16n8k16_bf16(acc[mt][rb], a0, a1, a2, a3, b[rb][0], b[rb][1]);
        }
    }
    constexpr int RP = 16 * MT + 1;
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int rb = 0; rb < NRB; ++rb)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int f = mt * 16 + (lane >> 2) + 8 * (i >> 1), n = rb * 8 + 2 * (lane & 3) + (i & 1);
                red[(warp * 8 * NRB + n) * RP + f] = acc[mt][rb][i];
            }
}

struct LstmFwd {
    const float* gx;        // [L*B, 4H]
    const bf16* w;          // W_hh [4H, H]
    const float* h0;        // [B, H] or null
    const float* c0;        // [B, H] or null
    bf16* y;                // [L*B, H]
    float* hn;              // [B, H]
    float* cn;              // [B, H], also c_{t-1} between steps
    float* gates;           // [L*B, 4H] post-activation gates, or null
    float* call;            // [L*B, H] c_t, or null
    unsigned* bar;
    int L, B, H, kp;        // kp: H rounded up to 16
};

// U = 4 MT units per CTA; chunks of 64 / MT batch rows so that U x rows = 256 = one cell per thread
template <int MT>
__global__ void __launch_bounds__(LSTM_THREADS, 1) lstm_fwd_kernel(LstmFwd p) {
    constexpr int U = 4 * MT, NRB = 8 / MT, BC = 8 * NRB, RP = 16 * MT + 1;
    extern __shared__ __align__(16) uint8_t smem[];
    const int ld = p.kp + 8;                                  // +16 B per row: conflict-free ldmatrix
    bf16* sW = reinterpret_cast<bf16*>(smem);                 // [4U][ld]: row g U + k = gate g of unit j0 + k
    bf16* sX = sW + 4 * U * ld;                               // [BC][ld]: h_{t-1} rows of the chunk
    float* red = reinterpret_cast<float*>(sX + BC * ld);      // [warps][BC][RP]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int H = p.H, B = p.B, j0 = blockIdx.x * U, cpr = ld / 8, hc = H / 8;
    for (int i = tid; i < 4 * U * cpr; i += LSTM_THREADS) {
        const int r = i / cpr, c = i % cpr, g = r / U, k = r % U;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (c < hc && j0 + k < H) v = *reinterpret_cast<const uint4*>(p.w + (size_t)(g * H + j0 + k) * H + c * 8);
        *reinterpret_cast<uint4*>(sW + r * ld + c * 8) = v;
    }
    for (int i = tid; i < BC * cpr; i += LSTM_THREADS)        // columns past H stay zero
        *reinterpret_cast<uint4*>(sX + (i / cpr) * ld + (i % cpr) * 8) = make_uint4(0, 0, 0, 0);
    __syncthreads();
    const int k = tid % U, r = tid / U, unit = j0 + k;
    const size_t H4 = 4 * (size_t)H;
    for (int t = 0; t < p.L; ++t) {
        for (int b0 = 0; b0 < B; b0 += BC) {
            for (int i = tid; i < BC * hc; i += LSTM_THREADS) {
                const int rr = i / hc, c = i % hc, b = b0 + rr;
                uint4 v = make_uint4(0, 0, 0, 0);
                if (b < B) {
                    if (t > 0) {
                        v = __ldcg(reinterpret_cast<const uint4*>(p.y + ((size_t)(t - 1) * B + b) * H + c * 8));
                    } else if (p.h0) {
                        const float4 lo = *reinterpret_cast<const float4*>(p.h0 + (size_t)b * H + c * 8);
                        const float4 hi = *reinterpret_cast<const float4*>(p.h0 + (size_t)b * H + c * 8 + 4);
                        v = make_uint4(pack_bf16(lo.x, lo.y), pack_bf16(lo.z, lo.w), pack_bf16(hi.x, hi.y), pack_bf16(hi.z, hi.w));
                    }
                }
                *reinterpret_cast<uint4*>(sX + rr * ld + c * 8) = v;
            }
            __syncthreads();
            slice_product<MT, NRB>(sW, 16 * MT - 1, sX, ld, p.kp / 16, red, warp, lane);
            __syncthreads();
            const int b = b0 + r;
            if (b < B && unit < H) {
                const size_t row = (size_t)t * B + b, s = (size_t)b * H + unit;
                float a[4];
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    float acc = p.gx[row * H4 + g * H + unit];
#pragma unroll
                    for (int w = 0; w < LSTM_WARPS; ++w) acc += red[(w * BC + r) * RP + g * U + k];
                    a[g] = acc;
                }
                const float ig = sigmoid_f(a[0]), fg = sigmoid_f(a[1]), gg = tanhf(a[2]), og = sigmoid_f(a[3]);
                const float cprev = t > 0 ? p.cn[s] : (p.c0 ? p.c0[s] : 0.f);
                const float c = fg * cprev + ig * gg;
                const float h = og * tanhf(c);
                p.cn[s] = c;
                p.y[row * H + unit] = __float2bfloat16(h);
                if (p.gates) {
                    float* gr = p.gates + row * H4 + unit;
                    gr[0] = ig; gr[H] = fg; gr[2 * H] = gg; gr[3 * H] = og;
                }
                if (p.call) p.call[row * H + unit] = c;
                if (t == p.L - 1) p.hn[s] = h;
            }
        }
        if (t + 1 < p.L) grid_sync(p.bar);
    }
}

struct LstmBwd {
    const bf16* dy;         // [L*B, H] gradient of y
    const bf16* w;          // W_hh [4H, H]
    const float* gates;     // [L*B, 4H] post-activation gates of the forward
    const float* call;      // [L*B, H] c_t of the forward
    const float* c0;        // [B, H] or null
    bf16* dg;               // [L*B, 4H] gradient of the pre-activation gates
    float* dc;              // [B, H] dc carried to the step before
    unsigned* bar;
    int L, B, H;
};

// U units per CTA (8 or 16): one m16 tile of W_hh columns, chunks of 16 batch rows
template <int U>
__global__ void __launch_bounds__(LSTM_THREADS, 1) lstm_bwd_kernel(LstmBwd p) {
    constexpr int BC = BWD_ROWS, RP = 17;
    extern __shared__ __align__(16) uint8_t smem[];
    const int H = p.H, B = p.B, K = 4 * H, ld = K + 8, j0 = blockIdx.x * U;
    bf16* sW = reinterpret_cast<bf16*>(smem);                 // [U][ld]: sW[k][m] = W_hh[m][j0 + k]
    bf16* sX = sW + U * ld;                                   // [BC][ld]: dG_{t+1} rows of the chunk
    float* red = reinterpret_cast<float*>(sX + BC * ld);      // [warps][BC][RP]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int i = tid; i < K * (U / 8); i += LSTM_THREADS) {
        const int m = i / (U / 8), c = i % (U / 8);
        uint4 v = make_uint4(0, 0, 0, 0);
        if (j0 + c * 8 < H) v = *reinterpret_cast<const uint4*>(p.w + (size_t)m * H + j0 + c * 8);
        const bf16* e = reinterpret_cast<const bf16*>(&v);
#pragma unroll
        for (int q = 0; q < 8; ++q) sW[(c * 8 + q) * ld + m] = e[q];
    }
    __syncthreads();
    const int k = tid % U, r = tid / U, unit = j0 + k;
    const int kc = K / 8;
    for (int t = p.L - 1; t >= 0; --t) {
        const bool rec = t + 1 < p.L;         // dG_{t+1} exists
        for (int b0 = 0; b0 < B; b0 += BC) {
            if (rec) {
                for (int i = tid; i < BC * kc; i += LSTM_THREADS) {
                    const int rr = i / kc, c = i % kc, b = b0 + rr;
                    uint4 v = make_uint4(0, 0, 0, 0);
                    if (b < B) v = __ldcg(reinterpret_cast<const uint4*>(p.dg + ((size_t)(t + 1) * B + b) * K + c * 8));
                    *reinterpret_cast<uint4*>(sX + rr * ld + c * 8) = v;
                }
                __syncthreads();
                slice_product<1, BC / 8>(sW, U - 1, sX, ld, K / 16, red, warp, lane);
                __syncthreads();
            }
            const int b = b0 + r;
            if (r < BC && b < B && unit < H) {
                const size_t row = (size_t)t * B + b, s = (size_t)b * H + unit;
                float dh = __bfloat162float(p.dy[row * H + unit]);
                if (rec) {
#pragma unroll
                    for (int w = 0; w < LSTM_WARPS; ++w) dh += red[(w * BC + r) * RP + k];
                }
                const float* gr = p.gates + row * K + unit;
                const float ig = gr[0], fg = gr[H], gg = gr[2 * H], og = gr[3 * H];
                const float c = p.call[row * H + unit];
                const float cprev = t > 0 ? p.call[(row - B) * H + unit] : (p.c0 ? p.c0[s] : 0.f);
                const float tc = tanhf(c);
                const float dc = (rec ? p.dc[s] : 0.f) + dh * og * (1.f - tc * tc);
                p.dc[s] = dc * fg;
                bf16* d = p.dg + row * K + unit;
                d[0] = __float2bfloat16(dc * gg * ig * (1.f - ig));
                d[H] = __float2bfloat16(dc * cprev * fg * (1.f - fg));
                d[2 * H] = __float2bfloat16(dc * ig * (1.f - gg * gg));
                d[3 * H] = __float2bfloat16(dh * tc * og * (1.f - og));
            }
        }
        if (t > 0) grid_sync(p.bar);
    }
}

__global__ void embedding_kernel(const long long* __restrict__ tok, const bf16* __restrict__ emb, bf16* __restrict__ out, int N,
                                 int d, int vocab) {
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (n >= N) return;
    long long t = tok[n];
    if (t < 0 || t >= vocab) t = 0;
    for (int col = (threadIdx.x & 31) * 8; col < d; col += 256)
        *reinterpret_cast<uint4*>(out + (size_t)n * d + col) = *reinterpret_cast<const uint4*>(emb + (size_t)t * d + col);
}

size_t fwd_smem(int u, int H) {
    const int mt = u / 4, bc = 64 / mt, ld = (H + 15) / 16 * 16 + 8;
    return (size_t)(4 * u + bc) * ld * sizeof(bf16) + (size_t)LSTM_WARPS * bc * (16 * mt + 1) * sizeof(float);
}
size_t bwd_smem(int u, int H) {
    return (size_t)(u + BWD_ROWS) * (4 * H + 8) * sizeof(bf16) + (size_t)LSTM_WARPS * BWD_ROWS * 17 * sizeof(float);
}

// Cooperative launches need every CTA resident at once: refuse (and launch nothing) when the occupancy says otherwise.
template <auto Kern, typename P>
const char* coop_launch(int grid, size_t smem, cudaStream_t st, const P& p) {
    if (const char* e = prepare<Kern>()) return e;
    int per_sm = 0;
    const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, Kern, LSTM_THREADS, smem);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        return cudaGetErrorString(e);
    }
    if (per_sm * num_sms() < grid) return "lstm: the grid cannot be co-resident on this device (occupancy x SMs < CTAs)";
    return launch<Kern, 1, true>(dim3(grid), dim3(LSTM_THREADS), smem, st, p);
}

const char* device_plan(int H, LstmPlan* pl) {
    int dev = 0, optin = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        return cudaGetErrorString(e);
    }
    return lstm_plan(H, num_sms(), optin, pl);
}

}  // namespace

const char* lstm_plan(int H, int sms, int smem_optin, LstmPlan* pl) {
    if (H < 8 || H % 8) return "lstm: the hidden size must be a positive multiple of 8";
    int u = 8;
    while ((H + u - 1) / u > sms) u *= 2;
    if (u > 16) return "lstm: the W_hh slice of a CTA does not fit shared memory (more than 16 units per CTA)";
    pl->units = u;
    pl->grid = (H + u - 1) / u;
    pl->smem_fwd = fwd_smem(u, H);
    pl->smem_bwd = bwd_smem(u, H);
    if (pl->smem_fwd > (size_t)smem_optin || pl->smem_bwd > (size_t)smem_optin)
        return "lstm: the W_hh slice of a CTA does not fit shared memory";
    return nullptr;
}

const char* lstm_fwd_launch(cudaStream_t st, const float* gx, const bf16* w, const float* h0, const float* c0, bf16* y, float* hn,
                            float* cn, float* gates, float* call, unsigned* bar, int L, int B, int H) {
    if (L < 1 || B < 1) return "lstm: empty sequence or batch";
    LstmPlan pl;
    if (const char* e = device_plan(H, &pl)) return e;
    LstmFwd p{gx, w, h0, c0, y, hn, cn, gates, call, bar, L, B, H, (H + 15) / 16 * 16};
    if (pl.units == 8) return coop_launch<lstm_fwd_kernel<2>>(pl.grid, pl.smem_fwd, st, p);
    return coop_launch<lstm_fwd_kernel<4>>(pl.grid, pl.smem_fwd, st, p);
}

const char* lstm_bwd_launch(cudaStream_t st, const bf16* dy, const bf16* w, const float* gates, const float* call, const float* c0,
                            bf16* dg, float* dc, unsigned* bar, int L, int B, int H) {
    if (L < 1 || B < 1) return "lstm: empty sequence or batch";
    LstmPlan pl;
    if (const char* e = device_plan(H, &pl)) return e;
    LstmBwd p{dy, w, gates, call, c0, dg, dc, bar, L, B, H};
    if (pl.units == 8) return coop_launch<lstm_bwd_kernel<8>>(pl.grid, pl.smem_bwd, st, p);
    return coop_launch<lstm_bwd_kernel<16>>(pl.grid, pl.smem_bwd, st, p);
}

const char* embedding_launch(cudaStream_t st, const long long* tok, const bf16* emb, bf16* out, int N, int d, int vocab) {
    if (d % 8) return "embedding: d must be a multiple of 8";
    return launch<embedding_kernel>(dim3((N + 7) / 8), dim3(256), 0, st, tok, emb, out, N, d, vocab);
}

}  // namespace otb
