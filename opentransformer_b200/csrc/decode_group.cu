// Persistent beam-search decode kernel for sm_90a: the WHOLE decode loop of SpeechToTextRecognizer.recognize
// (otrans/recognize/speech2text.py:60-68 -> decode_step :95-153 -> TransformerDecoder.inference,
// otrans/decoder/transformer.py:185-208) in ONE launch, GEMMs on wgmma tensor cores.
//
// Round 1 ran a decode step as 52 dependent kernels (7-13 us each for 2-4 us of work: 0.50 ms per beam step) or as one
// cluster of 4 CTAs per utterance streaming ALL decoder weights through mma.sync for its 10 rows (830 MB of L2 traffic per
// step).  This kernel keeps the rows of up to 12 utterances (beam 10 -> 120 hypotheses) together as ONE 128-row wgmma
// tile and gives each such ROW GROUP to P = 16 co-operating CTAs:
//
//   * the wide projections are split over the group's CTAs by OUTPUT column (QKV: 48 columns per CTA; GLU: 128 hidden
//     features per CTA) or, for w_2, by CONTRACTION slice (the CTA's own 128 hidden features; the 16 fp32 partial products are
//     summed by a row-partitioned pass that also applies the residual and LayerNorm 3): the four warpgroups each form a 64-row x N/2
//     quarter with wgmma, operands by TMA straight into the 128B-swizzled shared-memory layout, accumulators in registers;
//   * the d x d projections between the attention cores (W_o, the cross-attention query projection, the second W_o) run on
//     the OWNER of the rows: CTA j holds rows [8 j, 8 j + 8), streams the whole 128 KB weight matrix by TMA one phase ahead
//     and forms the product transposed with mma.sync (weights = m16 operand, the 8 rows = n8 operand); bias + residual +
//     LayerNorm finish inside that CTA (v1 split them by column too: a barrier + a 128-row fp32 gather per LayerNorm);
//   * self-attention of the owner's 8 rows x 4 heads: one (row, head) problem per half-warp, the cached K / V rows (addressed
//     through the ancestry table; beam reordering never moves K / V) are fetched by 512-byte bulk copies of the TMA engine
//     into shared memory, online softmax per lane group; the context rows stay in shared memory for W_o;
//   * cross-attention of the <= 16 hypotheses of an utterance against its <= 256 encoder frames is one m16 problem per
//     (utterance, head), three per CTA, all three side by side on warp groups of 4: mma.sync on K / V tiles that TMA
//     prefetches during the preceding barrier (wgmma has no M < 64 shape);
//   * activations cross CTAs through L2 at 6 group barriers per layer: QKV | self-attention + W_o + LN1 + W_q |
//     cross-attention | W_o + LN2 | GLU + w_2 partial | reduction + LN3.  The group is launched as ONE thread-block cluster
//     of 16 CTAs (barrier.cluster, release / acquire) or as plain CTAs with a release / acquire counter in L2
//     (otb_set_decode_barrier): ~3 k cycles either way instead of a kernel boundary (7-13 us); weight prefetches are issued
//     between arrive and wait; groups never synchronise with each other, utterances are independent;
//   * the tail -- logits (fp32, stored in accumulator order [column group][row]), then per utterance a TMA gather of its rows,
//     log-softmax + per-row top-k (lane-maxima threshold), finished masking, beam^2 pruning, ancestry update -- follows
//     beam.cu exactly (ties -> lower index), so ids / parents are bit-exact with the oracle's beam_step driven by this
//     kernel's log-probs.
// Design notes: DESIGN.md 4.4.
//
// Supported: post-norm decoder, GLU feed-forward with d_ff = 2048, d_model 256, 4 heads, beam <= 16, memory length <= 256
// frames, max_len <= 128.  Anything else runs on the per-step graph path (recognize.BeamDecoder.step).
#include <string.h>

#include <cuda_fp16.h>

#include "beam_common.cuh"
#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

static constexpr int DG_THREADS = 512;
static constexpr int DG_P = 16;            // CTAs per row group
static constexpr int DG_D = 256;           // d_model
static constexpr int DG_H = 4;
static constexpr int DG_DFF = 2048;
static constexpr int DG_A_BYTES = 65536;   // A operand tile: 4 k-blocks of [128 rows x 64] bf16, SWIZZLE_128B
static constexpr int DG_STAGE = 65536;     // two big stages: weight chunks / cross-attention K|V tiles / logit rows of the beam step
static constexpr int DG_SB = 24576;        // QKV B operand (48 weight rows x 256) | ancestry rows | row-block activations | cross-attention scratch | top-k candidates
static constexpr int DG_MISC = 9728;
static constexpr int DG_SMEM = DG_A_BYTES + 2 * DG_STAGE + DG_SB + DG_MISC + 1024;
static_assert(DG_SMEM <= 227 * 1024, "decode_group_kernel: shared-memory budget (227 KB per CTA)");
static constexpr int DG_PP = 528;          // cross-attention probability row pitch (bytes): 512 + 16 -> conflict-free ldmatrix

unsigned long long* g_dg_dbg = nullptr;
int g_dg_dbg_step = 0;
int g_dg_barrier = -1;      // otb_set_decode_barrier: -1 = clusters when the device grants them, 0 = software, 1 = cluster

// Tensor maps in the workspace: DG_LAYER_MAPS per decoder layer (weights [rows, K] bf16, box = 64 columns x one slice),
// then the DG_SHARED_MAPS ones.  The host encoder and the kernel both index them by these names.
enum DgLayerMap { MAP_WQKV, MAP_WO, MAP_WQ, MAP_WO2, MAP_W1, MAP_W2, DG_LAYER_MAPS };
enum DgSharedMap {
    MAP_WOUT,       // output layer [V, d]
    MAP_KVX,        // encoder K | V of every layer [n_layers * B * T, 2 d]
    MAP_X,          // xbuf: layer input (A operand of the QKV projection and of the output layer)
    MAP_X2,         // x2buf: LayerNorm 2 output (A operand of the feed-forward)
    MAP_LG,         // logits as [G * ldv / 4 column groups][128 rows] x 16 B (gather of an utterance's rows)
    DG_SHARED_MAPS
};

struct DgLayer {
    const float *bqkv, *bo, *bq, *bo2, *b1, *b2;
    const float *g1, *be1, *g2, *be2, *g3, *be3;
};
struct DgParams {
    int n_layers, V, G, utts_per_group;
    int cluster;               // 1: launched as thread-block clusters of 16 (group == cluster, hardware barrier)
    const bf16* emb;
    const float* bout;
    const float* pe;
    DgLayer layers[OTB_MEGA_MAX_LAYERS];
    CUtensorMap* maps;         // device array: n_layers * DG_LAYER_MAPS (DgLayerMap order), then DgSharedMap order
    const int* mem_len;
    bf16* kc;
    bf16* vc;
    BeamState st;
    int B, T, max_steps;
    float eps;
    bf16* qbuf;                // [N, d]   self-attention queries of the newest token
    bf16* ctx;                 // [N, d]   cross-attention context
    bf16* xbuf;                // [N + 128, d] layer input x (embedding / LayerNorm 3 of the previous layer)
    bf16* x2buf;               // [N + 128, d] LayerNorm 2 output (A operand and residual of the feed-forward)
    bf16* q2;                  // [N, d]   cross-attention queries
    float* part;               // [16 slices][groups][64 column groups][128 rows][4] w_2 partial products (fp32)
    float* logits;             // [groups][ldv / 4 column groups][128 rows][4] output-layer logits of the step
    int ldv;
    int* bar;                  // [G, 32]  group barrier counters
    int* gstate;               // [G, Lmax] ended-hypothesis count per step
    float* dbg_logp;
    float* dbg_scores;
    unsigned long long* dbg_clk;
    int dbg_step;
};

struct DgMisc {
    uint64_t kb_full[4];      // small B operand k-blocks landed (TMA, prefetched one phase ahead)
    uint64_t a_full[4];       // A operand k-blocks landed (TMA from xbuf / x2buf)
    uint64_t w1_full[4];      // W1 k-blocks landed
    uint64_t st_full[2];      // big stage landed
    uint64_t pw_full[4];      // k-blocks of the out-projection weights (self-attention W_o, then cross-attention W_o) landed
    uint64_t pq_full[4];      // k-blocks of the cross-attention query projection landed
    uint64_t lg_full;         // logits rows of an utterance landed (TMA gather of the beam phase)
    uint64_t kx_full[3];      // encoder K/V tile of a cross-attention problem landed in stage 0 / stage 1 / the A tile
    uint64_t kv_full[32];     // self-attention: [row of the block][half-buffer] (16 used) -- 8 cached K rows + 8 V rows, all heads, landed (bulk copies)
    int flag;                 // broadcast scratch
    alignas(16) float bias[256];          // per-phase bias slice
    float c_val[KMAX * KMAX];
    int c_tok[KMAX * KMAX];
    float sel_v[KMAX];
    int sel_i[KMAX];
    float row_v[KMAX][KMAX];
    int row_i[KMAX][KMAX];
};
static_assert(sizeof(DgMisc) <= DG_MISC, "DgMisc must fit its shared-memory slot");

// ---------------------------------------------------------------------------------------------- small PTX helpers
__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_gpu_add(int* p, int v) {
    asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}
// contiguous global -> shared bulk copy (TMA engine, no tensor map); bytes % 16 == 0, both addresses 16-byte aligned
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// byte offset of the 16-byte chunk (row r, chunk c of 8) inside a [rows x 64] bf16 k-block in the SWIZZLE_128B K-major layout
__device__ __forceinline__ uint32_t sw128(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }

// ---------------------------------------------------------------------------------------------- the kernel
// kStamps: the clock64 phase stamps of tools/decode_phases.py (otb_debug_decode_timing).  Only that instantiation carries
// their state (stamp counters, the per-barrier slot pointer), which would otherwise be live across every phase and barrier;
// the production instantiation (kStamps = false) has none of it.
template <bool kStamps>
__global__ void __launch_bounds__(DG_THREADS, 1) decode_group_kernel(const __grid_constant__ DgParams p) {
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment by an offset from smem_raw, not by integer arithmetic on its address: the compiler then still knows
    // every pointer below is a shared-memory address (32-bit registers, LDS / STS instead of generic loads and stores)
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    // Shared memory (227 KB per CTA): sA | stage 0 | stage 1 | sSB | DgMisc.  Which phase of a step uses which region (R reads,
    // W writes; "pf" = filled by a TMA prefetch issued at the group barrier IN FRONT of the phase, "tma" = filled by TMA
    // inside the phase once its previous user is done; sA0 = sSB [16 KB, 20 KB), sA1 = sSB [20 KB, 24 KB)):
    //
    //   phase              | sA (64 KB)                  | stage 0 (64 KB)                  | stage 1 (64 KB)            | sSB (24 KB)
    //   -------------------+-----------------------------+----------------------------------+----------------------------+------------------------------
    //   embed              | W x tile                    |                                  |                            |
    //   QKV projection     | R x (layer > 0: tma xbuf)   |                                  |                            | R QKV weight slice (pf, all)
    //   self-attention     | W_o k-blocks 0-1 (pf)       | K/V rows of block rows 0-3       | K/V rows of block rows 4-7 | [0, 8 KB) ancestry; W sA0
    //     (behind it, tma) |                             | W_o k-blocks 2-3                 | W_q k-blocks 0-1           |
    //   W_o + LN1 + W_q    | R W_o; tma W_q k-blocks 2-3 | R W_o                            | R W_q                      | R sA0; W, R sA1 (x1)
    //   cross-attention    | K/V tile, problem 2 (pf)    | K/V tile, problem 0 (pf)         | K/V tile, problem 1 (pf)   | [0, 3 KB) softmax scratch
    //   W_o2 + LN2         | R W_o2 k-blocks 0-1 (pf)    | R W_o2 k-blocks 2-3 (pf); tma W1 | W1 k-blocks 2-3 (pf)       | W sA0 (ctx rows); R sA1
    //   GLU + w_2 partial  | tma x2; W h; R h            | R W1; tma W2 slice; R W2         | R W1                       |
    //   reduce + LN3       |                             | last layer: W_out chunk (pf)     | last layer: W_out chunk (pf) | else next QKV slice (pf)
    //   logits             | tma x; R                    | R W_out; tma chunk i + 2         | R W_out; tma chunk i + 2   |
    //   beam step          | tma: an utterance's logit rows over sA and both stages (192 KB)                            | [0, 16 KB) top-k candidates
    //
    // DgMisc: `bias` is the bias slice of the QKV, GLU and logits phases; `c_val` is the LayerNorm row-sum scratch of the
    // row-block phases and the beam^2 candidate list of the beam step; the rest belongs to the beam step.
    uint8_t* sA = smem;
    uint8_t* sST = smem + DG_A_BYTES;                 // [2][DG_STAGE]
    uint8_t* sSB = sST + 2 * DG_STAGE;
    DgMisc& ms = *reinterpret_cast<DgMisc*>(sSB + DG_SB);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = blockIdx.x / DG_P, j = blockIdx.x % DG_P;
    const int beam = p.st.beam, N = p.st.N, Lmax = p.st.Lmax, V = p.V;
    const int u0 = g * p.utts_per_group;
    const int nutt = min(p.utts_per_group, p.B - u0);
    const int row0 = u0 * beam, nrows = nutt * beam;
    const int nl = p.n_layers;
    // tensor-map addresses are formed from the parameters where they are used, not kept in registers across the step
    auto layer_map = [&](int l, DgLayerMap m) { return p.maps + l * DG_LAYER_MAPS + m; };
    auto shared_map = [&](DgSharedMap m) { return p.maps + p.n_layers * DG_LAYER_MAPS + m; };
    int* bar = p.bar + g * 32;                        // 128-byte separated counters
    const bool is_tma = (warp == 0 && lane == 0);
    // wgmma tiles: the four warpgroups split a 128-row product into 64-row halves (mh) x column halves (nh); accumulator
    // fragment of a thread: rows frow, frow + 8, columns 8 i + fcq + {0, 1} of its quarter
    const int mh = (warp >> 2) & 1, nh = warp >> 3;
    const int frow = mh * 64 + (warp & 3) * 16 + (lane >> 2);
    const int fcq = 2 * (lane & 3);

    if (tid == 0) {
        for (int i = 0; i < 4; ++i) {
            mbar_init(&ms.kb_full[i], 1);
            mbar_init(&ms.a_full[i], 1);
            mbar_init(&ms.w1_full[i], 1);
            mbar_init(&ms.pw_full[i], 1);
            mbar_init(&ms.pq_full[i], 1);
        }
        for (int i = 0; i < 2; ++i) {
            mbar_init(&ms.st_full[i], 1);
        }
        mbar_init(&ms.lg_full, 1);
        for (int i = 0; i < 32; ++i) mbar_init(&ms.kv_full[i], 1);
        for (int i = 0; i < 3; ++i) mbar_init(&ms.kx_full[i], 1);
        ms.flag = 0;
        fence_barrier_init();
    }
    __syncthreads();

    // parity of the NEXT completion of every mbarrier, tracked identically by all threads (every thread walks the same phases):
    // one register for all of them, bit PB_x + i = barrier i of the set x (nine words used to be live across every phase)
    constexpr int PB_KB = 0, PB_A = 4, PB_W1 = 8, PB_PW = 12, PB_PQ = 16, PB_STF = 20, PB_KX = 22, PB_KVW = 25, PB_LG = 27;
    uint32_t par = 0;
    auto pbit = [&](int set, int i) { return (par >> (set + i)) & 1u; };
    int bar_target = 0;

    const bool dbg_cta = kStamps && (p.dbg_clk != nullptr && blockIdx.x < DG_P && tid == 0);     // every CTA of group 0: [cta][256] stamps
    int dbg_n = 0;
    bool dbg_on = false;
#define DG_STAMP() do { if (kStamps && dbg_on) p.dbg_clk[blockIdx.x * 256 + dbg_n++] = clock64(); } while (0)
    // sub-phase stamps of layer 2 in slots 200.. (tools/decode_phases.py prints them)
#define DG_STAMP2(k) do { if (kStamps && dbg_on && l == 2) p.dbg_clk[blockIdx.x * 256 + 200 + (k)] = clock64(); } while (0)
#define DG_STAMP3(k) do { if (kStamps && dbg_on) p.dbg_clk[blockIdx.x * 256 + 200 + (k)] = clock64(); } while (0)

    // Group barrier: every CTA of the group has finished the phase (its global writes are visible).  `pre` runs on the TMA
    // thread between arrive and wait -- prefetches that do not depend on the other CTAs (weights, encoder K/V tiles); the
    // leading CTA barrier guarantees that every warp of THIS CTA is done with the shared memory those prefetches overwrite.
    // Launched as thread-block clusters of 16 (p.cluster) the group IS the cluster: hardware barrier.cluster with release /
    // acquire semantics; otherwise one atomic + an acquire poll on a counter in L2.
    int dbg_b = 0;      // group barriers since the start of the step; the six of layer 2 (12..17) get inner stamps (slots 212..229)
    auto gsync = [&](auto pre) {
        __syncthreads();
        DG_STAMP();
        const bool rec = kStamps && dbg_on && dbg_b >= 12 && dbg_b < 18;
        unsigned long long* slot = p.dbg_clk + blockIdx.x * 256 + 212 + (dbg_b - 12) * 3;
        ++dbg_b;
        if (p.cluster) {
            if (tid == 0) fence_proxy_async_all();
            __syncwarp();
            asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
            if (rec) slot[0] = clock64();
            // the prefetch is issued by ANOTHER thread than the one that executes the proxy fence behind the wait: inner stamps
            // showed barriers with a prefetch taking ~1.5 k cycles longer than those without -- fence.proxy.async of a thread
            // also waits for the bulk copies that thread has in flight, i.e. for the weights it had just asked for
            if (tid == 32) pre();
            if (rec) slot[1] = clock64();
            __syncwarp();
            asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
            if (tid == 0) fence_proxy_async_all();
            if (rec) slot[2] = clock64();
            __syncthreads();
            return;
        }
        bar_target += DG_P;
        if (warp == 1) {      // the prefetch follows the arrival (issued together, the arrival queued behind 100+ KB of TMA requests)
            asm volatile("bar.sync 15, 64;" ::: "memory");
            if (tid == 32) pre();
        }
        if (tid == 0) {
            // red.release.gpu orders every write this thread has observed -- those of the other warps through the CTA barrier
            // above (cumulativity) -- before the arrival: no separate __threadfence (it cost a second MEMBAR round per barrier)
            fence_proxy_async_all();
            red_release_gpu_add(bar, 1);
            if (rec) slot[0] = clock64();
        }
        if (warp == 0) asm volatile("bar.sync 15, 64;" ::: "memory");
        if (tid == 0) {
            if (rec) slot[1] = clock64();
            const long long t0 = clock64();
            uint32_t spins = 0;
            // (relaxed polls + one fence.acq_rel.gpu behind the successful one were tried: the fence also waits for the prefetch
            // in flight -- 16.5 -> 17.4 ms per launch)
            while (ld_acquire_gpu(bar) < bar_target) {
                if (((++spins) & 0x3FF) == 0 && (clock64() - t0) > 20000000000LL) __trap();   // a protocol bug traps instead of hanging
            }
            fence_proxy_async_all();
            if (rec) slot[2] = clock64();
        }
        __syncthreads();
    };
    auto nop = [] {};
    // element offset of (layer l, position s, hypothesis row n) in the self-attention K / V cache [layer][step][hyp][d]
    auto kv_off = [&](int l, int s, int n) -> size_t { return (((size_t)l * Lmax + s) * N + n) * DG_D; };

    // ---- operand loads issued by the TMA thread ------------------------------------------------------------------
    // small B operand: nB weight rows [b_row0, b_row0 + nB) x 256, k-block kb at sSB + kb * nB * 128 (prefetched at the
    // barrier in front of the phase that consumes it)
    auto load_small_b = [&](const CUtensorMap* mb, int b_row0, int nB) {
        for (int kb = 0; kb < 4; ++kb) {
            mbar_arrive_expect_tx(&ms.kb_full[kb], (uint32_t)(nB * 128));
            tma_load_2d_hint(sSB + kb * nB * 128, mb, &ms.kb_full[kb], kb * 64, b_row0, TMA_EVICT_LAST);
        }
    };
    auto load_a = [&](const CUtensorMap* ma) {        // A tile: rows [row0, row0 + 128) of xbuf / x2buf
        for (int kb = 0; kb < 4; ++kb) {
            mbar_arrive_expect_tx(&ms.a_full[kb], 16384);
            tma_load_2d(sA + kb * 16384, ma, &ms.a_full[kb], kb * 64, row0);
        }
    };
    auto load_w1 = [&](int l, int kb0) {   // k-blocks kb0, kb0 + 1 -> stage kb0 / 2: [value rows | gate rows] of this CTA's 128 hidden features
        const CUtensorMap* m = layer_map(l, MAP_W1);
        for (int kb = kb0; kb < kb0 + 2; ++kb) {
            uint8_t* dst = sST + (kb >> 1) * DG_STAGE + (kb & 1) * 32768;
            mbar_arrive_expect_tx(&ms.w1_full[kb], 32768);
            tma_load_2d_hint(dst, m, &ms.w1_full[kb], kb * 64, j * 128, TMA_EVICT_LAST);
            tma_load_2d_hint(dst + 16384, m, &ms.w1_full[kb], kb * 64, DG_DFF + j * 128, TMA_EVICT_LAST);
        }
    };
    // one k-block (all 256 output features x 64 input features, 32 KB, SWIZZLE_128B) of a d x d projection
    auto load_proj_kb = [&](const CUtensorMap* m, uint64_t* full, int kb, uint8_t* dst) {
        mbar_arrive_expect_tx(&full[kb], 32768);
        tma_load_2d_hint(dst, m, &full[kb], kb * 64, 0, TMA_EVICT_LAST);
    };
    auto load_kv = [&](int l, int task, int s) {   // K and V tile of (utterance, head) -> stage s (0, 1: the stages; 2: the A tile)
        const int u = u0 + task / DG_H, h = task % DG_H;
        uint8_t* dst = (s < 2) ? sST + s * DG_STAGE : sA;
        mbar_arrive_expect_tx(&ms.kx_full[s], 65536);
        // the encoder K / V tiles are streamed once per step (49 MB per batch): evict-first, so that they do not push the
        // decoder weights (re-read by every group, every step) out of L2
        tma_load_2d_hint(dst, shared_map(MAP_KVX), &ms.kx_full[s], h * 64, (l * p.B + u) * p.T, TMA_EVICT_FIRST);
        tma_load_2d_hint(dst + 32768, shared_map(MAP_KVX), &ms.kx_full[s], DG_D + h * 64, (l * p.B + u) * p.T, TMA_EVICT_FIRST);
    };
    const int n_vchunks = (V + 127) / 128;
    auto load_wout = [&](int chunk, int s) {
        mbar_arrive_expect_tx(&ms.st_full[s], 65536);
        for (int kb = 0; kb < 4; ++kb) tma_load_2d_hint(sST + s * DG_STAGE + kb * 16384, shared_map(MAP_WOUT), &ms.st_full[s], kb * 64, chunk * 128, TMA_EVICT_LAST);
    };
    const int n_tasks = nutt * DG_H;   // cross-attention problems of this group; CTA j takes j, j + P, ...

    // ---- A operand builders -------------------------------------------------------------------------------------
    // embedding + positional encoding (decoder/transformer.py:163,169; pos.py:56): x = emb[last_tok] * sqrt(d) + PE[step].
    // Every CTA builds the whole tile (the QKV projection of layer 0 reads it from shared memory); rows [8 j, 8 j + 8) are also
    // written to xbuf, where the out-projection epilogues fetch their residual slice.
    auto build_a_embed = [&](int step) {
        for (int r = warp; r < 128; r += 16) {
            uint4 o = make_uint4(0, 0, 0, 0);
            if (r < nrows) {
                long long tok = p.st.last_tok[row0 + r];
                if (tok < 0 || tok >= V) tok = 0;
                const uint4 u = *reinterpret_cast<const uint4*>(p.emb + (size_t)tok * DG_D + lane * 8);
                const float* pe = p.pe + (size_t)step * DG_D + lane * 8;
                const float4 p0 = *reinterpret_cast<const float4*>(pe), p1 = *reinterpret_cast<const float4*>(pe + 4);
                const float2 e0 = unpack_bf16(u.x), e1 = unpack_bf16(u.y), e2 = unpack_bf16(u.z), e3 = unpack_bf16(u.w);
                const float xs = 16.0f;   // sqrt(256)
                o.x = pack_bf16(e0.x * xs + p0.x, e0.y * xs + p0.y);
                o.y = pack_bf16(e1.x * xs + p0.z, e1.y * xs + p0.w);
                o.z = pack_bf16(e2.x * xs + p1.x, e2.y * xs + p1.y);
                o.w = pack_bf16(e3.x * xs + p1.z, e3.y * xs + p1.w);
                if ((r >> 3) == j) *reinterpret_cast<uint4*>(p.xbuf + (size_t)(row0 + r) * DG_D + lane * 8) = o;
            }
            *reinterpret_cast<uint4*>(sA + (lane >> 3) * 16384 + sw128(r, lane & 7)) = o;
        }
        fence_proxy_async_smem();
        __syncthreads();
    };
    // ---- row-block projections (v7) ------------------------------------------------------------------------------
    // The three d x d projections between the attention cores (self-attention W_o, the cross-attention query projection and
    // the cross-attention W_o) are computed by the OWNER of the rows: CTA j holds rows [8 j, 8 j + 8) of the tile and
    // multiplies them by the WHOLE weight matrix (128 KB, streamed by TMA through the idle A tile / stages one phase ahead)
    // with mma.sync m16n8k16 (rows 8..15 of the fragment are zero).  A complete row in one CTA means bias + residual +
    // LayerNorm finish right there: v6 split these projections by output column over the 16 CTAs, which cost a group
    // barrier in front of every LayerNorm plus a 128 KB fp32 gather of ALL rows by EVERY CTA (6 k cycles, twice per layer).
    // Activations: [8 rows][256] bf16 in shared memory, 16-byte chunks XOR-swizzled by the row (conflict-free ldmatrix).
    uint8_t* sA0 = sSB + 16384;                       // attention output rows (A operand of W_o)
    uint8_t* sA1 = sSB + 20480;                       // LayerNorm-1 output rows: A operand of the query projection, residual of W_o #2
    auto a_off = [](int r, int chunk) { return (uint32_t)(r * 512 + ((chunk ^ (r & 7)) << 4)); };
    // v22: the product is formed TRANSPOSED, out^T[256 features x 8 rows] = W[256 x 256] . X^T: the weight tile is the m16
    // operand (16 output features per warp), the 8 activation rows are the n8 operand -- no padding rows: 256 mma.sync per
    // projection and CTA instead of 512 (the m16n8k16 path runs at ~16 cycles per instruction and SM sub-partition, which
    // is what bounded the projections: 2.1 k cycles each).  Accumulator fragment of a thread: features ef0 and ef0 + 8,
    // rows era and era + 1.
    const int ef0 = warp * 16 + (lane >> 2);          // first feature of this thread's accumulator fragment (second: + 8)
    const int era = 2 * (lane & 3);                   // first row of the block (second: + 1)
    const bool live_a = j * 8 + era < nrows, live_b = j * 8 + era + 1 < nrows;
    const size_t grow_a = (size_t)(row0 + j * 8 + era) * DG_D, grow_b = grow_a + DG_D;
    auto a_at = [&](uint8_t* A, int r, int f) { return reinterpret_cast<bf16*>(A + a_off(r, f >> 3) + (f & 7) * 2); };
    auto load_rows = [&](const bf16* src, uint8_t* dstA) {    // this CTA's 8 rows of a [N, 256] bf16 buffer -> swizzled smem
        if (tid < 256) {
            const int r = tid >> 5, ch = tid & 31;
            uint4 v = make_uint4(0, 0, 0, 0);
            if (j * 8 + r < nrows) v = *reinterpret_cast<const uint4*>(src + (size_t)(row0 + j * 8 + r) * DG_D + ch * 8);
            *reinterpret_cast<uint4*>(dstA + a_off(r, ch)) = v;
        }
    };
    // acc[0..1] = out[era + {0,1}][ef0], acc[2..3] = out[era + {0,1}][ef0 + 8]; warp w owns output features [16 w, 16 w + 16)
    auto rowgemm = [&](const uint8_t* A, uint64_t* full, int pset, auto kb_addr, float (&acc)[4]) {   // flips the parities of pset
        float acc2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i] = 0.f;
        const int m = lane >> 3, rr = lane & 7;
        const uint32_t abase = smem_u32(A);
#pragma unroll 1
        for (int kb = 0; kb < 4; ++kb) {
            mbar_wait(&full[kb], pbit(pset, kb));
            const uint32_t wb = smem_u32(kb_addr(kb));
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                uint32_t a0, a1, a2, a3, b0, b1;
                // weight fragment (m16 x k16): (features 0-7, k lo) (features 8-15, k lo) (features 0-7, k hi) (features 8-15, k hi)
                ldmatrix_x4(wb + sw128(warp * 16 + (m & 1) * 8 + rr, 2 * ks + (m >> 1)), a0, a1, a2, a3);
                // activation fragment (k16 x n8): (rows 0-7, k lo) (rows 0-7, k hi); lanes 16-31 pass valid but unused addresses
                ldmatrix_x2(abase + a_off(rr, kb * 8 + ks * 2 + (m & 1)), b0, b1);
                if (ks & 1) mma_m16n8k16_bf16(acc2, a0, a1, a2, a3, b0, b1);      // two independent accumulation chains
                else mma_m16n8k16_bf16(acc, a0, a1, a2, a3, b0, b1);
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i] += acc2[i];
        par ^= 0xFu << pset;
    };
    // LayerNorm of the 8 rows held as v[0..3] = (row a, f0) (row b, f0) (row a, f0 + 8) (row b, f0 + 8) (fp32: projection + bias
    // + residual): statistics over the 8 lane groups of a warp (shuffles) and the 16 warps (shared memory)
    auto row_ln = [&](float (&v)[4], float g0, float g1, float t0, float t1) {
        float* rsum = ms.c_val;                       // [16 warps][8 rows]
        float sa = v[0] + v[2], sb = v[1] + v[3];
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
            sa += __shfl_xor_sync(0xffffffffu, sa, o);
            sb += __shfl_xor_sync(0xffffffffu, sb, o);
        }
        if (lane < 4) {
            rsum[warp * 8 + era] = sa;
            rsum[warp * 8 + era + 1] = sb;
        }
        __syncthreads();
        float ma = 0.f, mb = 0.f;
#pragma unroll
        for (int w = 0; w < 16; ++w) {
            ma += rsum[w * 8 + era];
            mb += rsum[w * 8 + era + 1];
        }
        ma *= (1.0f / DG_D);
        mb *= (1.0f / DG_D);
        v[0] -= ma; v[2] -= ma; v[1] -= mb; v[3] -= mb;
        float qa = v[0] * v[0] + v[2] * v[2], qb = v[1] * v[1] + v[3] * v[3];
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
            qa += __shfl_xor_sync(0xffffffffu, qa, o);
            qb += __shfl_xor_sync(0xffffffffu, qb, o);
        }
        __syncthreads();
        if (lane < 4) {
            rsum[warp * 8 + era] = qa;
            rsum[warp * 8 + era + 1] = qb;
        }
        __syncthreads();
        float va = 0.f, vb = 0.f;
#pragma unroll
        for (int w = 0; w < 16; ++w) {
            va += rsum[w * 8 + era];
            vb += rsum[w * 8 + era + 1];
        }
        const float ra = rsqrtf(va * (1.0f / DG_D) + p.eps), rb = rsqrtf(vb * (1.0f / DG_D) + p.eps);
        v[0] = v[0] * ra * g0 + t0;
        v[1] = v[1] * rb * g0 + t0;
        v[2] = v[2] * ra * g1 + t1;
        v[3] = v[3] * rb * g1 + t1;
    };

    // ---- small GEMM: acc[128 x 48] = A[128 x 256] * Bslice^T, B slice prefetched into sSB (kb_full).  a_map != null: A is fetched
    // here by TMA (a_full), else it was built in shared memory by the CTA.  Each warpgroup forms a 64 x 24 quarter with wgmma;
    // epi(row, col, v0, v1) is called for every pair of adjacent columns of the thread's accumulator fragment.  Ends with a
    // CTA barrier.
    auto gemm_small = [&](const CUtensorMap* a_map, const float* bias, int b_row0, auto epi) {
        constexpr int nB = 48;
        if (tid < nB) ms.bias[tid] = bias[b_row0 + tid];
        if (is_tma && a_map != nullptr) load_a(a_map);
        // every operand wait precedes the wgmma chain: wgmma issued behind a divergent spin loop is serialised by ptxas
        for (int kb = 0; kb < 4; ++kb) {
            mbar_wait(&ms.kb_full[kb], pbit(PB_KB, kb));
            if (a_map != nullptr) mbar_wait(&ms.a_full[kb], pbit(PB_A, kb));
        }
        __syncwarp();
        float acc[12];
        wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < 4; ++kb) {
            const uint32_t a_addr = smem_u32(sA + kb * 16384) + mh * 8192, b_addr = smem_u32(sSB + kb * nB * 128) + nh * 24 * 128;
#pragma unroll
            for (int k = 0; k < 4; ++k)
                wgmma_n24<0, 0>(acc, gmma_desc_sw128(a_addr + k * 32), gmma_desc_sw128(b_addr + k * 32), (uint32_t)((kb | k) != 0));
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        __syncthreads();   // bias slice visible to every thread
#pragma unroll
        for (int i = 0; i < 3; ++i) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) epi(frow + 8 * hh, nh * 24 + i * 8 + fcq, acc[4 * i + 2 * hh], acc[4 * i + 2 * hh + 1]);
        }
        par ^= 0xFu << PB_KB;
        if (a_map != nullptr) par ^= 0xFu << PB_A;
        __syncthreads();
    };
    // Buffers that only this kernel reads back (w_2 partial products, logits) are stored as [column group of 4][row][16 bytes]:
    // the readers gather 16-byte pieces of consecutive rows, which are contiguous.
    const size_t part_slab = (size_t)64 * 128;          // uint4 per (contraction slice, group): 64 column groups x 128 rows
    const int ldv4 = p.ldv >> 2;
    uint4* lg4 = reinterpret_cast<uint4*>(p.logits) + (size_t)g * ldv4 * 128;     // this group's logits, [ldv / 4][128 rows] x 16 B

    // ================================================================================================ the phases of a step
    // ---- self-attention over the cached prefix (the cache the reference stubbed out, transformer.py:92-126)
    // by the OWNER of the rows (the CTA that multiplies them by W_o next): all 8 rows x 4 heads of the CTA at the same
    // time.  Warp w = row w / 2 and two of its heads, one per HALF-warp (v19 ran the 32 problems in two rounds of 16,
    // one warp each: every round paid the whole latency chain ancestry -> copies -> wait -> softmax merge; 11 k cycles
    // at step 5).  Within a half-warp 8 lanes share one key (lane c holds bytes [16 c, 16 c + 16) of the head's K / V
    // slice), 2 keys per instruction, the partial dot products meet through 3 shuffles, each of the 2 lane groups keeps an
    // online softmax (m, l, o[8]) over its keys, merged at the end.
    // The cached K / V rows of the prefix (512 bytes per position: all four heads; scattered by the ancestry table) are
    // fetched by the TMA engine -- ONE bulk copy per row and position, shared by the two warps of the row, 8 positions
    // per half-buffer, two halves in flight -- and the dot products read shared memory.
    // History: v13 gathered with 16-byte LDGs, 16 per lane in flight: 9.5 B/clk per SM at step 50 (44 k cycles per
    // layer) whatever the cache policy.  v14 issued one 128-byte bulk copy per (position, head): the stamps showed the
    // ISSUE as the limit -- an SM starts one bulk copy per ~6.5 cycles (41 k cycles per layer at step 50); 512-byte
    // copies need a quarter of the operations (v15: 26 k).
    auto self_attn = [&](int l, int step) {
        const int nkeys = step + 1;
        const int* an_base = p.st.anc + (size_t)(step & 1) * N * Lmax;
        int* an_s = reinterpret_cast<int*>(sSB) + warp * 128;          // this warp's ancestry row (<= 128 positions)
        const int rl = warp >> 1, wr = warp & 1;                       // row of the block, which of its two warps
        const int hl = lane >> 4, g2 = (lane >> 3) & 1, c8 = lane & 7;
        const int h = wr * 2 + hl;                                     // head of this half-warp
        uint8_t* kvst = sST + rl * 16384;                              // [2 halves][K 8 x 512 B | V 8 x 512 B] per row: 8 rows = both stages
        uint64_t* kvb = &ms.kv_full[rl * 2];
        auto row_sync = [&] { asm volatile("bar.sync %0, 64;" ::"r"(rl + 1) : "memory"); };
        // (the K / V rows of this step were written with ordinary stores by other CTAs; the writer side of gsync executes
        // fence.proxy.async before its release, the copies below read L2: no further proxy fence here -- it cost every warp
        // a MEMBAR-class stall per layer)
        const int r = j * 8 + rl;
        const int n = row0 + r;
        DG_STAMP2(39);
        if (r >= nrows) {      // dead row of the tile (warp-uniform): zeros, so that the projection below stays finite
            if (g2 == 0) *reinterpret_cast<uint4*>(sA0 + a_off(rl, h * 8 + c8)) = make_uint4(0, 0, 0, 0);
        } else {
            for (int s0 = lane; s0 < step; s0 += 32) an_s[s0] = an_base[(size_t)n * Lmax + s0];
            float qf[8];
            {
                const uint4 qu = *reinterpret_cast<const uint4*>(p.qbuf + (size_t)n * DG_D + h * 64 + c8 * 8);
                const float2 q0 = unpack_bf16(qu.x), q1 = unpack_bf16(qu.y), q2 = unpack_bf16(qu.z), q3 = unpack_bf16(qu.w);
                qf[0] = q0.x * 0.125f; qf[1] = q0.y * 0.125f; qf[2] = q1.x * 0.125f; qf[3] = q1.y * 0.125f;
                qf[4] = q2.x * 0.125f; qf[5] = q2.y * 0.125f; qf[6] = q3.x * 0.125f; qf[7] = q3.y * 0.125f;
            }
            __syncwarp();
            float m = -INFINITY, lsum = 0.f;
            float o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            const int nh = (nkeys + 7) >> 3;
            auto issue = [&](int hh) {
                const int kk0 = hh * 8, buf = hh & 1;
                const int nk = min(8, nkeys - kk0);
                if (wr == 0 && lane == 0) mbar_arrive_expect_tx(&kvb[buf], (uint32_t)(nk * 1024));
                if (lane < 8) {
                    const int c = wr * 8 + lane;               // 16 copies per half: 8 K rows, 8 V rows; 8 per warp
                    const int key = c & 7, isv = c >> 3;
                    if (key < nk) {
                        const int sidx = kk0 + key;
                        const int slot = (sidx < step) ? an_s[sidx] : n;
                        const bf16* src = (isv ? p.vc : p.kc) + kv_off(l, sidx, slot);
                        bulk_g2s(kvst + buf * 8192 + isv * 4096 + key * 512, src, 512, &kvb[buf]);
                    }
                }
            };
            DG_STAMP2(40);
            issue(0);
            if (nh > 1) issue(1);
            DG_STAMP2(41);
            for (int hh = 0; hh < nh; ++hh) {
                const int buf = hh & 1, k0 = hh * 8;
                mbar_wait(&kvb[buf], pbit(PB_KVW, buf));
                par ^= 1u << (PB_KVW + buf);
                if (hh < 4) DG_STAMP2(42 + 2 * hh);
                const uint8_t* kb_ = kvst + buf * 8192 + h * 128 + c8 * 16;
                uint4 ku[4], vu[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    ku[u] = *reinterpret_cast<const uint4*>(kb_ + (2 * u + g2) * 512);
                    vu[u] = *reinterpret_cast<const uint4*>(kb_ + 4096 + (2 * u + g2) * 512);
                }
                float sc[4];
                float mb = m;
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const float2 a = unpack_bf16(ku[u].x), b2 = unpack_bf16(ku[u].y), c2 = unpack_bf16(ku[u].z), e = unpack_bf16(ku[u].w);
                    float d = qf[0] * a.x + qf[1] * a.y + qf[2] * b2.x + qf[3] * b2.y + qf[4] * c2.x + qf[5] * c2.y + qf[6] * e.x + qf[7] * e.y;
                    d += __shfl_xor_sync(0xffffffffu, d, 1);
                    d += __shfl_xor_sync(0xffffffffu, d, 2);
                    d += __shfl_xor_sync(0xffffffffu, d, 4);
                    sc[u] = (k0 + 2 * u + g2 < nkeys) ? d : -INFINITY;      // rows beyond the prefix hold stale bytes: masked here
                    mb = fmaxf(mb, sc[u]);
                }
                if (mb != -INFINITY) {
                    const float alpha = (m == -INFINITY) ? 0.f : __expf(m - mb);
                    lsum *= alpha;
#pragma unroll
                    for (int q = 0; q < 8; ++q) o[q] *= alpha;
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const bool live_k = sc[u] != -INFINITY;
                        const float pw = live_k ? __expf(sc[u] - mb) : 0.f;
                        lsum += pw;
                        const float2 a = unpack_bf16(vu[u].x), b2 = unpack_bf16(vu[u].y), c2 = unpack_bf16(vu[u].z), e = unpack_bf16(vu[u].w);
                        if (live_k) {      // stale V bytes may be NaN patterns: never multiply them, not even by zero
                            o[0] = fmaf(pw, a.x, o[0]); o[1] = fmaf(pw, a.y, o[1]); o[2] = fmaf(pw, b2.x, o[2]); o[3] = fmaf(pw, b2.y, o[3]);
                            o[4] = fmaf(pw, c2.x, o[4]); o[5] = fmaf(pw, c2.y, o[5]); o[6] = fmaf(pw, e.x, o[6]); o[7] = fmaf(pw, e.y, o[7]);
                        }
                    }
                    m = mb;
                }
                if (hh + 2 < nh) {
                    row_sync();    // both warps (all four heads) are done with this half
                    issue(hh + 2);
                }
                if (hh < 4) DG_STAMP2(43 + 2 * hh);
            }
            DG_STAMP2(50);
            // merge the 2 lane groups of the half-warp (lanes c8 and c8 + 8 hold the same output dims)
            const float M = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
            const float w = (m == -INFINITY) ? 0.f : __expf(m - M);
            lsum *= w;
            lsum += __shfl_xor_sync(0xffffffffu, lsum, 8);
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                o[q] *= w;
                o[q] += __shfl_xor_sync(0xffffffffu, o[q], 8);
            }
            if (g2 == 0) {
                const float inv = 1.0f / lsum;
                uint4 ou;
                ou.x = pack_bf16(o[0] * inv, o[1] * inv);
                ou.y = pack_bf16(o[2] * inv, o[3] * inv);
                ou.z = pack_bf16(o[4] * inv, o[5] * inv);
                ou.w = pack_bf16(o[6] * inv, o[7] * inv);
                *reinterpret_cast<uint4*>(sA0 + a_off(rl, h * 8 + c8)) = ou;      // context row -> A operand of W_o
            }
            DG_STAMP2(51);
        }
    };
    // ---- rows [8 j, 8 j + 8): W_o + bias + residual (the layer input) -> LayerNorm 1 -> query projection
    // (attention.py:44, transformer.py:54-56, attention.py:128), all inside the owning CTA
    auto wo_ln1_q = [&](int l, const DgLayer& ly) {
        DG_STAMP2(9);
        // parameters of this thread's two features, requested before the GEMM (behind it each was an exposed L2 round trip)
        const float pb0 = ly.bo[ef0], pb1 = ly.bo[ef0 + 8], pg0 = ly.g1[ef0], pg1 = ly.g1[ef0 + 8], pt0 = ly.be1[ef0], pt1 = ly.be1[ef0 + 8];
        const float qb0 = ly.bq[ef0], qb1 = ly.bq[ef0 + 8];
        float xres[4] = {0.f, 0.f, 0.f, 0.f};      // residual = the layer input (own rows, written by this CTA)
        if (live_a) {
            xres[0] = __bfloat162float(p.xbuf[grow_a + ef0]);
            xres[2] = __bfloat162float(p.xbuf[grow_a + ef0 + 8]);
        }
        if (live_b) {
            xres[1] = __bfloat162float(p.xbuf[grow_b + ef0]);
            xres[3] = __bfloat162float(p.xbuf[grow_b + ef0 + 8]);
        }
        __syncthreads();
        DG_STAMP2(10);
        float acc[4];
        rowgemm(sA0, ms.pw_full, PB_PW, [&](int kb) { return kb < 2 ? sA + kb * 32768 : sST + (kb - 2) * 32768; }, acc);
        __syncthreads();      // every warp is done with W_o: its first half makes room for the second half of W_q
        DG_STAMP2(11);
        if (is_tma)
            for (int kb = 2; kb < 4; ++kb) load_proj_kb(layer_map(l, MAP_WQ), ms.pq_full, kb, sA + (kb - 2) * 32768);
        float v[4];
        {
            const float b0 = pb0, b1 = pb1;
            v[0] = acc[0] + b0 + xres[0];
            v[1] = acc[1] + b0 + xres[1];
            v[2] = acc[2] + b1 + xres[2];
            v[3] = acc[3] + b1 + xres[3];
        }
        row_ln(v, pg0, pg1, pt0, pt1);
        *a_at(sA1, era, ef0) = __float2bfloat16(v[0]);
        *a_at(sA1, era + 1, ef0) = __float2bfloat16(v[1]);
        *a_at(sA1, era, ef0 + 8) = __float2bfloat16(v[2]);
        *a_at(sA1, era + 1, ef0 + 8) = __float2bfloat16(v[3]);
        __syncthreads();
        DG_STAMP();   // W_o + LN1
        rowgemm(sA1, ms.pq_full, PB_PQ, [&](int kb) { return kb < 2 ? sST + DG_STAGE + kb * 32768 : sA + (kb - 2) * 32768; }, acc);
        {
            const float b0 = qb0, b1 = qb1;
            if (live_a) {
                p.q2[grow_a + ef0] = __float2bfloat16(acc[0] + b0);
                p.q2[grow_a + ef0 + 8] = __float2bfloat16(acc[2] + b1);
            }
            if (live_b) {
                p.q2[grow_b + ef0] = __float2bfloat16(acc[1] + b0);
                p.q2[grow_b + ef0 + 8] = __float2bfloat16(acc[3] + b1);
            }
        }
    };
    // ---- cross-attention (attention.py:129-141,34-41): one m16 problem per (utterance, head), 3 per CTA at
    // beam 10.  A problem is a chain of short dependent stages (with all 16 warps on one problem: QK^T 1.8 k cycles,
    // exp 1.1 k, PV 1.0 k, normalise 0.7 k -- latency, not throughput), so the CTA works on THREE problems at the same
    // time: warp groups 0..2 (4 warps each, own named barrier and scratch; v18 ran two halves of 8 warps: 16.5 k ->
    // 10.5 k cycles per layer) take problems g, g + 3, ...; the tiles of the first three problems are prefetched into
    // both stages and the idle A tile.  The probabilities of a problem are written over its (dead) K tile.
    auto cross_attn = [&](int l) {
        const int grp = warp >> 2, w4 = warp & 3;
        float* wmax = reinterpret_cast<float*>(sSB + grp * 1024);      // [4 warps][16 rows]
        float* wsum = wmax + 64;
        auto grp_sync = [&] { asm volatile("bar.sync %0, 128;" ::"r"(5 + grp) : "memory"); };
        const int gq = lane >> 2, tq = lane & 3;
        const int n_mine = (n_tasks > j) ? (n_tasks - j + DG_P - 1) / DG_P : 0;      // problems of this CTA
        DG_STAMP2(0);
        for (int i = grp; i < n_mine && grp < 3; i += 3) {
            const int task = j + i * DG_P, st = i % 3;
            const int u = u0 + task / DG_H, h = task % DG_H;
            const int kv_len = min(p.mem_len[u], p.T);
            uint8_t* sK = (st < 2) ? sST + st * DG_STAGE : sA;
            const uint8_t* sV = sK + 32768;
            uint8_t* sP = sK;                                          // [16 rows][DG_PP bytes] probabilities (bf16), after QK^T
            // Q fragments (rows = hypotheses of the utterance) straight from L2
            uint32_t qa[4][4];
            {
                const bf16* qb = p.q2 + (size_t)(u * beam) * DG_D + h * 64;
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) {
                    const int d0 = ks * 16 + 2 * tq;
                    qa[ks][0] = (gq < beam) ? *reinterpret_cast<const uint32_t*>(qb + (size_t)gq * DG_D + d0) : 0u;
                    qa[ks][1] = (gq + 8 < beam) ? *reinterpret_cast<const uint32_t*>(qb + (size_t)(gq + 8) * DG_D + d0) : 0u;
                    qa[ks][2] = (gq < beam) ? *reinterpret_cast<const uint32_t*>(qb + (size_t)gq * DG_D + d0 + 8) : 0u;
                    qa[ks][3] = (gq + 8 < beam) ? *reinterpret_cast<const uint32_t*>(qb + (size_t)(gq + 8) * DG_D + d0 + 8) : 0u;
                }
            }
            mbar_wait(&ms.kx_full[st], pbit(PB_KX, st) ^ (uint32_t)((i / 3) & 1));
            // S = Q K^T for this warp's 64 keys
            float sc[8][4];
#pragma unroll
            for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) sc[nt][e] = 0.f;
            {
                const int m = lane >> 3, rr = lane & 7;
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
                    for (int kq = 0; kq < 4; ++kq) {
                        const int key = w4 * 64 + kq * 16 + (m >> 1) * 8 + rr;
                        uint32_t b0, b1, b2, b3;
                        ldmatrix_x4(smem_u32(sK) + sw128(key, 2 * ks + (m & 1)), b0, b1, b2, b3);
                        mma_m16n8k16_bf16(sc[2 * kq], qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3], b0, b1);
                        mma_m16n8k16_bf16(sc[2 * kq + 1], qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3], b2, b3);
                    }
                }
            }
            const float sl2 = 0.125f * 1.4426950408889634f;
            float mlo = -INFINITY, mhi = -INFINITY;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const int k0 = w4 * 64 + nt * 8 + 2 * tq;
                sc[nt][0] = (k0 < kv_len) ? sc[nt][0] * sl2 : -INFINITY;
                sc[nt][1] = (k0 + 1 < kv_len) ? sc[nt][1] * sl2 : -INFINITY;
                sc[nt][2] = (k0 < kv_len) ? sc[nt][2] * sl2 : -INFINITY;
                sc[nt][3] = (k0 + 1 < kv_len) ? sc[nt][3] * sl2 : -INFINITY;
                mlo = fmaxf(mlo, fmaxf(sc[nt][0], sc[nt][1]));
                mhi = fmaxf(mhi, fmaxf(sc[nt][2], sc[nt][3]));
            }
            mlo = fmaxf(mlo, __shfl_xor_sync(0xffffffffu, mlo, 1));
            mlo = fmaxf(mlo, __shfl_xor_sync(0xffffffffu, mlo, 2));
            mhi = fmaxf(mhi, __shfl_xor_sync(0xffffffffu, mhi, 1));
            mhi = fmaxf(mhi, __shfl_xor_sync(0xffffffffu, mhi, 2));
            if (tq == 0) {
                wmax[w4 * 16 + gq] = mlo;
                wmax[w4 * 16 + gq + 8] = mhi;
            }
            grp_sync();       // every warp of the group is also done reading the K tile
            float Mlo = -INFINITY, Mhi = -INFINITY;
#pragma unroll
            for (int w = 0; w < 4; ++w) {
                Mlo = fmaxf(Mlo, wmax[w * 16 + gq]);
                Mhi = fmaxf(Mhi, wmax[w * 16 + gq + 8]);
            }
            float slo = 0.f, shi = 0.f;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const float p0 = ex2_approx(sc[nt][0] - Mlo), p1 = ex2_approx(sc[nt][1] - Mlo);     // exp2(-inf) = 0 for masked keys
                const float p2 = ex2_approx(sc[nt][2] - Mhi), p3 = ex2_approx(sc[nt][3] - Mhi);
                slo += p0 + p1;
                shi += p2 + p3;
                const int kc = w4 * 64 + nt * 8 + 2 * tq;
                *reinterpret_cast<uint32_t*>(sP + gq * DG_PP + kc * 2) = pack_bf16(p0, p1);
                *reinterpret_cast<uint32_t*>(sP + (gq + 8) * DG_PP + kc * 2) = pack_bf16(p2, p3);
            }
            slo += __shfl_xor_sync(0xffffffffu, slo, 1);
            slo += __shfl_xor_sync(0xffffffffu, slo, 2);
            shi += __shfl_xor_sync(0xffffffffu, shi, 1);
            shi += __shfl_xor_sync(0xffffffffu, shi, 2);
            if (tq == 0) {
                wsum[w4 * 16 + gq] = slo;
                wsum[w4 * 16 + gq + 8] = shi;
            }
            grp_sync();
            // O = P V: warp w4 = output dims [16 w4, 16 w4 + 16) over all 256 keys (no cross-warp reduction)
            float oc[2][4], oc2[2][4];
#pragma unroll
            for (int dn = 0; dn < 2; ++dn)
#pragma unroll
                for (int e = 0; e < 4; ++e) oc[dn][e] = oc2[dn][e] = 0.f;
            {
                const int m = lane >> 3, rr = lane & 7;
#pragma unroll
                for (int kk = 0; kk < 16; kk += 2) {
                    const int key0 = kk * 16;
                    uint32_t a0, a1, a2, a3, c0, c1, c2, c3;
                    ldmatrix_x4(smem_u32(sP) + (uint32_t)(((m & 1) * 8 + rr) * DG_PP + (key0 + (m >> 1) * 8) * 2), a0, a1, a2, a3);
                    ldmatrix_x4(smem_u32(sP) + (uint32_t)(((m & 1) * 8 + rr) * DG_PP + (key0 + 16 + (m >> 1) * 8) * 2), c0, c1, c2, c3);
#pragma unroll
                    for (int dn = 0; dn < 2; ++dn) {
                        uint32_t v0, v1, v2, v3;
                        ldmatrix_x4_trans(smem_u32(sV) + sw128(key0 + m * 8 + rr, w4 * 2 + dn), v0, v1, v2, v3);   // keys key0 .. key0+31
                        mma_m16n8k16_bf16(oc[dn], a0, a1, a2, a3, v0, v1);
                        mma_m16n8k16_bf16(oc2[dn], c0, c1, c2, c3, v2, v3);
                    }
                }
            }
            float Llo = 0.f, Lhi = 0.f;
#pragma unroll
            for (int w = 0; w < 4; ++w) {
                Llo += wsum[w * 16 + gq];
                Lhi += wsum[w * 16 + gq + 8];
            }
            {
                const float ilo = 1.0f / Llo, ihi = 1.0f / Lhi;
#pragma unroll
                for (int dn = 0; dn < 2; ++dn) {
                    bf16* dst = p.ctx + (size_t)(u * beam) * DG_D + h * 64 + (w4 * 2 + dn) * 8 + 2 * tq;
                    if (gq < beam)
                        *reinterpret_cast<uint32_t*>(dst + (size_t)gq * DG_D) = pack_bf16((oc[dn][0] + oc2[dn][0]) * ilo, (oc[dn][1] + oc2[dn][1]) * ilo);
                    if (gq + 8 < beam)
                        *reinterpret_cast<uint32_t*>(dst + (size_t)(gq + 8) * DG_D) = pack_bf16((oc[dn][2] + oc2[dn][2]) * ihi, (oc[dn][3] + oc2[dn][3]) * ihi);
                }
            }
            grp_sync();       // this group is done with its tile and its scratch
            if (w4 == 0 && lane == 0 && i + 3 < n_mine) load_kv(l, j + (i + 3) * DG_P, st);
        }
        // stage s was filled once per problem i = s, s + 3, ...
#pragma unroll
        for (int st = 0; st < 3; ++st) {
            const int uses = (n_mine > st) ? (n_mine - st + 2) / 3 : 0;
            par ^= (uint32_t)(uses & 1) << (PB_KX + st);
        }
    };
    // ---- rows [8 j, 8 j + 8): cross-attention W_o + bias + residual (x1, still in shared memory) -> LayerNorm 2
    // -> x2 (bf16, global: A operand of the feed-forward of every CTA and residual of its reduction)
    auto wo2_ln2 = [&](int l, const DgLayer& ly) {
        load_rows(p.ctx, sA0);
        const float pb0 = ly.bo2[ef0], pb1 = ly.bo2[ef0 + 8], pg0 = ly.g2[ef0], pg1 = ly.g2[ef0 + 8], pt0 = ly.be2[ef0], pt1 = ly.be2[ef0 + 8];
        __syncthreads();
        float acc[4];
        rowgemm(sA0, ms.pw_full, PB_PW, [&](int kb) { return kb < 2 ? sA + kb * 32768 : sST + (kb - 2) * 32768; }, acc);
        __syncthreads();      // stage 0 (second half of W_o) is free: first half of W1
        if (is_tma) load_w1(l, 0);
        float v[4];
        {
            const float b0 = pb0, b1 = pb1;      // residual x1 is still in shared memory
            v[0] = acc[0] + b0 + __bfloat162float(*a_at(sA1, era, ef0));
            v[1] = acc[1] + b0 + __bfloat162float(*a_at(sA1, era + 1, ef0));
            v[2] = acc[2] + b1 + __bfloat162float(*a_at(sA1, era, ef0 + 8));
            v[3] = acc[3] + b1 + __bfloat162float(*a_at(sA1, era + 1, ef0 + 8));
        }
        row_ln(v, pg0, pg1, pt0, pt1);
        if (live_a) {
            p.x2buf[grow_a + ef0] = __float2bfloat16(v[0]);
            p.x2buf[grow_a + ef0 + 8] = __float2bfloat16(v[2]);
        }
        if (live_b) {
            p.x2buf[grow_b + ef0] = __float2bfloat16(v[1]);
            p.x2buf[grow_b + ef0 + 8] = __float2bfloat16(v[3]);
        }
    };
    // ---- GLU feed-forward: hidden features [128 j, 128 j + 128) (ffn.py:18,39-41); A = x2 of all rows by TMA
    auto glu_w2 = [&](int l, const DgLayer& ly) {
        if (is_tma) load_a(shared_map(MAP_X2));
        if (tid < 256) ms.bias[tid] = ly.b1[(tid < 128 ? 0 : DG_DFF - 128) + j * 128 + tid];
        // W1: value and gate features [64 nh, 64 nh + 64) of this CTA's 128, rows [64 mh, +64), two wgmma 64 x 64 chains
        float av[32], ag[32];
        for (int kb = 0; kb < 4; ++kb) {
            mbar_wait(&ms.w1_full[kb], pbit(PB_W1, kb));
            mbar_wait(&ms.a_full[kb], pbit(PB_A, kb));
        }
        __syncwarp();
        wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < 4; ++kb) {
            const uint32_t a_addr = smem_u32(sA + kb * 16384) + mh * 8192;
            const uint32_t b_addr = smem_u32(sST + (kb >> 1) * DG_STAGE + (kb & 1) * 32768) + nh * 8192;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                wgmma_n64<0, 0>(av, gmma_desc_sw128(a_addr + k * 32), gmma_desc_sw128(b_addr + k * 32), (uint32_t)((kb | k) != 0));
                wgmma_n64<0, 0>(ag, gmma_desc_sw128(a_addr + k * 32), gmma_desc_sw128(b_addr + 16384 + k * 32), (uint32_t)((kb | k) != 0));
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(av);
        wgmma_fence_regs(ag);
        __syncthreads();      // every warpgroup is done with x2 (A tile) and W1: both may be overwritten
        if (is_tma) {
            // W2[:, 128 j .. 128 j + 128) (this CTA's contraction slice) follows into stage 0
            mbar_arrive_expect_tx(&ms.st_full[0], 65536);
            tma_load_2d_hint(sST, layer_map(l, MAP_W2), &ms.st_full[0], j * 128, 0, TMA_EVICT_LAST);
            tma_load_2d_hint(sST + 32768, layer_map(l, MAP_W2), &ms.st_full[0], j * 128 + 64, 0, TMA_EVICT_LAST);
        }
        // h = (a + b_a) * sigmoid(g + b_g) -> bf16, written over the (dead) A tile as a [128 x 128] K-major operand
#pragma unroll
        for (int i = 0; i < 8; ++i) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int f = nh * 64 + i * 8 + fcq, r = frow + 8 * hh;
                const float a0 = av[4 * i + 2 * hh] + ms.bias[f], a1 = av[4 * i + 2 * hh + 1] + ms.bias[f + 1];
                const float g0 = ag[4 * i + 2 * hh] + ms.bias[128 + f], g1 = ag[4 * i + 2 * hh + 1] + ms.bias[128 + f + 1];
                *reinterpret_cast<uint32_t*>(sA + (f >> 6) * 16384 + sw128(r, (f & 63) >> 3) + (f & 7) * 2) =
                    pack_bf16(a0 * fast_sigmoid(g0), a1 * fast_sigmoid(g1));
            }
        }
        fence_proxy_async_smem();
        par ^= (0xFu << PB_W1) | (0xFu << PB_A);
        __syncthreads();
        DG_STAMP();   // W1 + GLU
        // w_2 partial: acc2[128 x 256] = h[128 x 128] * W2[:, slice]^T; warpgroup (mh, nh): rows [64 mh, +64) x columns [128 nh, +128)
        {
            mbar_wait(&ms.st_full[0], pbit(PB_STF, 0));
            // fp32 partial products in the [column group of 4][row] order the reduction reads; two 64-column passes
            // keep the accumulator within the register budget of 512 threads
            float* dst = reinterpret_cast<float*>(p.part) + ((size_t)j * p.G + g) * part_slab * 4;
#pragma unroll 1
            for (int hb = 0; hb < 2; ++hb) {
                float pc[32];
                __syncwarp();
                wgmma_fence();
#pragma unroll
                for (int kb = 0; kb < 2; ++kb) {
                    const uint32_t a_addr = smem_u32(sA + kb * 16384) + mh * 8192;
                    const uint32_t b_addr = smem_u32(sST + kb * 32768) + nh * 16384 + hb * 8192;
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        wgmma_n64<0, 0>(pc, gmma_desc_sw128(a_addr + k * 32), gmma_desc_sw128(b_addr + k * 32), (uint32_t)((kb | k) != 0));
                }
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_regs(pc);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const int c = nh * 128 + hb * 64 + i * 8 + fcq, r = frow + 8 * hh;
                        if (r < nrows) *reinterpret_cast<float2*>(dst + ((size_t)(c >> 2) * 128 + r) * 4 + (c & 3)) = make_float2(pc[4 * i + 2 * hh], pc[4 * i + 2 * hh + 1]);
                    }
                }
            }
        }
        par ^= 1u << PB_STF;
    };
    // ---- sum of the 16 partial products + bias + residual (x2) + LayerNorm 3, rows [8 j, 8 j + 8) of the
    // tile: every load is a contiguous 512-byte half row, the row statistics stay inside the CTA, and the result is the
    // bf16 input of the next layer (or of the output layer) in xbuf -- no separate LayerNorm pass, no fp32 round trip
    auto reduce_ln3 = [&](const DgLayer& ly) {
        // thread = (row 8 j + (tid & 7), 4-column group tid >> 3): a warp reads four full 128-byte lines per load (8
        // consecutive rows x 16 bytes), the 16 slices in two batches of 8 loads, summed in slice order
        float* rsum = ms.c_val;                                   // [16 warps][8 rows]
        const int rr = tid & 7, c4 = tid >> 3;
        const int r = j * 8 + rr;
        const bool live = r < nrows;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 gm = *reinterpret_cast<const float4*>(ly.g3 + c4 * 4), bt = *reinterpret_cast<const float4*>(ly.be3 + c4 * 4);
        if (live) {
            const float4* src = reinterpret_cast<const float4*>(p.part) + (size_t)g * part_slab + (size_t)c4 * 128 + r;
#pragma unroll
            for (int h8 = 0; h8 < DG_P; h8 += 8) {
                float4 v[8];
#pragma unroll
                for (int pp = 0; pp < 8; ++pp) v[pp] = src[(size_t)(h8 + pp) * p.G * part_slab];
#pragma unroll
                for (int pp = 0; pp < 8; ++pp) { acc.x += v[pp].x; acc.y += v[pp].y; acc.z += v[pp].z; acc.w += v[pp].w; }
            }
            const float4 b = *reinterpret_cast<const float4*>(ly.b2 + c4 * 4);
            const uint2 xr = *reinterpret_cast<const uint2*>(p.x2buf + (size_t)(row0 + r) * DG_D + c4 * 4);
            const float2 r0 = unpack_bf16(xr.x), r1 = unpack_bf16(xr.y);
            acc.x += b.x + r0.x; acc.y += b.y + r0.y; acc.z += b.z + r1.x; acc.w += b.w + r1.y;
        }
        float s = (acc.x + acc.y) + (acc.z + acc.w);
        s += __shfl_xor_sync(0xffffffffu, s, 8);
        s += __shfl_xor_sync(0xffffffffu, s, 16);
        if (lane < 8) rsum[warp * 8 + lane] = s;
        __syncthreads();
        float mean = 0.f;
#pragma unroll
        for (int w = 0; w < 16; ++w) mean += rsum[w * 8 + rr];
        mean *= (1.0f / DG_D);
        const float a = acc.x - mean, b = acc.y - mean, cc = acc.z - mean, d = acc.w - mean;
        float q = (a * a + b * b) + (cc * cc + d * d);
        q += __shfl_xor_sync(0xffffffffu, q, 8);
        q += __shfl_xor_sync(0xffffffffu, q, 16);
        __syncthreads();
        if (lane < 8) rsum[warp * 8 + lane] = q;
        __syncthreads();
        if (live) {
            float var = 0.f;
#pragma unroll
            for (int w = 0; w < 16; ++w) var += rsum[w * 8 + rr];
            const float rstd = rsqrtf(var * (1.0f / DG_D) + p.eps);
            uint2 o;
            o.x = pack_bf16(a * rstd * gm.x + bt.x, b * rstd * gm.y + bt.y);
            o.y = pack_bf16(cc * rstd * gm.z + bt.z, d * rstd * gm.w + bt.w);
            *reinterpret_cast<uint2*>(p.xbuf + (size_t)(row0 + r) * DG_D + c4 * 4) = o;
        }
    };
    // ---- output layer (decoder/transformer.py:181) in 128-column chunks: logits (+ bias) to global memory with
    // coalesced stores.  (v2 formed the log-softmax statistics and a per-row top-k in registers in this epilogue: one
    // sorted insertion per element per lane with all 32 rows of a warp diverging = 300 k cycles per step.)
    auto logits = [&] {
        int my_chunks = 0;
        for (int c = j; c < n_vchunks; c += DG_P) ++my_chunks;
        if (is_tma) load_a(shared_map(MAP_X));
        __syncwarp();
        for (int kb = 0; kb < 4; ++kb) mbar_wait(&ms.a_full[kb], pbit(PB_A, kb));
        // chunk i: wgmma 64 x 64 per warpgroup (rows [64 mh, +64), columns [64 nh, +64) of the chunk), logits + bias stored in the
        // [column group][row] order (columns [V, ldv) as -inf: no bounds checks in the readers); the weights of chunk i + 2
        // stream into the stage as soon as every warpgroup has multiplied chunk i
        for (int i = 0; i < my_chunks; ++i) {
            const int s = i & 1;
            const int col0 = (j + i * DG_P) * 128;
            if (tid < 128) ms.bias[s * 128 + tid] = (p.bout != nullptr && col0 + tid < V) ? p.bout[col0 + tid] : 0.f;
            mbar_wait(&ms.st_full[s], pbit(PB_STF, s) ^ (uint32_t)((i >> 1) & 1));
            float lc[32];
            __syncwarp();
            wgmma_fence();
#pragma unroll
            for (int kb = 0; kb < 4; ++kb) {
                const uint32_t a_addr = smem_u32(sA + kb * 16384) + mh * 8192, b_addr = smem_u32(sST + s * DG_STAGE + kb * 16384) + nh * 8192;
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    wgmma_n64<0, 0>(lc, gmma_desc_sw128(a_addr + k * 32), gmma_desc_sw128(b_addr + k * 32), (uint32_t)((kb | k) != 0));
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(lc);
            __syncthreads();      // stage s consumed by every warpgroup; bias slice visible
            if (is_tma && i + 2 < my_chunks) load_wout(j + (i + 2) * DG_P, s);
            float* lgf = reinterpret_cast<float*>(lg4);
#pragma unroll
            for (int q = 0; q < 8; ++q) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int cl = nh * 64 + q * 8 + fcq, c = col0 + cl, r = frow + 8 * hh;
                    if (r >= nrows || c >= p.ldv) continue;
                    const float o0 = (c < V) ? lc[4 * q + 2 * hh] + ms.bias[s * 128 + cl] : -INFINITY;
                    const float o1 = (c + 1 < V) ? lc[4 * q + 2 * hh + 1] + ms.bias[s * 128 + cl + 1] : -INFINITY;
                    *reinterpret_cast<float2*>(lgf + ((size_t)(c >> 2) * 128 + r) * 4 + (c & 3)) = make_float2(o0, o1);
                }
            }
        }
        // parity bookkeeping: barrier pair s was used ceil((my_chunks - s) / 2) times
        const uint32_t u0n = (uint32_t)((my_chunks + 1) >> 1), u1n = (uint32_t)(my_chunks >> 1);
        par ^= (0xFu << PB_A) | (((u0n & 1) | ((u1n & 1) << 1)) << PB_STF);
    };
    // ---- per utterance: log-softmax + top-`beam` of every hypothesis row (decoder/transformer.py:206,
    // speech2text.py:112), finished masking, beam^2 pruning, ancestry (speech2text.py:102-153); ties -> lower index
    auto beam_step = [&](int step) {
        int ended_here = 0;
        for (int ul = j; ul < nutt; ul += DG_P) {
            const int u = u0 + ul;
            // One warp per hypothesis row, all rows of the utterance at once, no shared-memory copy of the row:
            //   pass 1: row maximum + each lane's own maximum; T = the beam-th largest of the 32 lane
            //           maxima -- at least `beam` elements are >= T, so every element of the row's top-`beam` is >= T;
            //   pass 2: sum of exp(x - max) and the elements >= T compacted into a candidate list (<= 128;
            //           typically 10-20); the list is ranked by (log-prob, lower token id) exactly like the reference path.
            // A flat row (more than 128 elements >= T) takes the exact fallback: `beam` ordered arg-max scans of the row.
            // (v3 staged each row in shared memory with scalar loads behind dependent stores and spent 30 k cycles per row.)
            // The rows of the utterance are gathered from the [column group][row] logits by TMA: box = (the `beam` consecutive
            // 16-byte pieces of one column group) x 64 column groups, ~17 boxes per utterance, issued by one thread (v8 used
            // 10 k 16-byte cp.async: 11.7 k cycles; the A tile and both weight stages are idle: 192 KB).  In shared memory the
            // piece of (column group c, row r) sits at float4 index c * (beam | 1) + r.  A vocabulary x beam that does not fit is read
            // in place (element stride 128 x 16 bytes).
            const int nbox = (ldv4 + 63) >> 6;
            const int bpad = beam | 1;      // rows fetched per column group: an ODD number of 16-byte pieces keeps the float4 reads of
                                            // a warp (stride bpad x 16 bytes between lanes) free of bank conflicts; the extra row is ignored
            const bool staged = (size_t)nbox * 64 * bpad * 16 <= (size_t)(DG_A_BYTES + 2 * DG_STAGE);
            const int lr0 = ul * beam;                               // first row of the utterance inside the group tile
            if (staged) {
                if (is_tma) {
                    mbar_arrive_expect_tx(&ms.lg_full, (uint32_t)(nbox * 64 * bpad * 16));
                    for (int bx = 0; bx < nbox; ++bx)
                        tma_load_2d(smem + (size_t)bx * 64 * bpad * 16, shared_map(MAP_LG), &ms.lg_full, lr0 * 4, g * ldv4 + bx * 64);
                }
                mbar_wait(&ms.lg_full, pbit(PB_LG, 0));
                par ^= 1u << PB_LG;
            }
            if (ul == j) DG_STAMP();      // rows gathered
            if (warp < beam) {
                const int r = warp, n = u * beam + r;
                const int pf_flag = p.st.flag[n];                    // needed after the ranking: their L2 round trips overlap the passes
                const float pf_score = p.st.scores[n];
                const float4* x4 = staged ? reinterpret_cast<const float4*>(smem) + r : reinterpret_cast<const float4*>(lg4 + lr0 + r);
                const int xs4 = staged ? bpad : 128;                 // float4 stride between consecutive column groups
                auto xel = [&](int c) { return reinterpret_cast<const float*>(x4 + (size_t)(c >> 2) * xs4)[c & 3]; };
                const float4 ninf4 = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
                float2* cand = reinterpret_cast<float2*>(sSB) + warp * 128;      // (logit, token id as float bits) x 128 per row
                float lmax = -INFINITY;
                for (int base = 0; base < ldv4; base += 32 * 8) {
                    const int i0 = base + lane;
                    float4 v[8];
#pragma unroll
                    for (int q = 0; q < 8; ++q) v[q] = (i0 + 32 * q < ldv4) ? x4[(size_t)(i0 + 32 * q) * xs4] : ninf4;
#pragma unroll
                    for (int q = 0; q < 8; ++q) lmax = fmaxf(lmax, fmaxf(fmaxf(v[q].x, v[q].y), fmaxf(v[q].z, v[q].w)));
                }
                if (ul == j) DG_STAMP3(52);
                const float rowmax = warp_max(lmax);
                float T = -INFINITY;
                {
                    float t = lmax;
                    for (int k = 0; k < beam; ++k) {
                        const float mxk = warp_max(t);
                        T = mxk;
                        const unsigned who = __ballot_sync(0xffffffffu, t == mxk);
                        if (mxk == -INFINITY) break;       // fewer than `beam` lanes hold anything: every element is a candidate
                        if (lane == __ffs(who) - 1) t = -INFINITY;
                    }
                }
                // pass 2: sum of exp(x - max) (ex2.approx on a pre-scaled argument: 2 instructions per element, relative error
                // 2^-22 -- the log-sum-exp moves by ~1e-7) and the candidates >= T; one ballot per 128 elements decides whether
                // any lane has to look at its four values at all
                if (ul == j) DG_STAMP3(53);
                const float l2e = 1.4426950408889634f, nm = -rowmax * l2e;
                float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
                int ncand = 0;
                // (a separate, unrolled sum pass in front of the candidate pass was tried: 22.7 k -> 25.5 k cycles; four 32-wide
                // rounds per trip, their loads in flight together and one ballot skipping all four, left it at 9-10 k cycles per row)
                for (int base = 0; base < ldv4; base += 32) {        // warp-uniform trip count: whole warps take part in the ballots
                    const int i0 = base + lane;
                    const float4 v = (i0 < ldv4) ? x4[(size_t)i0 * xs4] : ninf4;
                    s0 += ex2_approx(fmaf(v.x, l2e, nm));                  // ex2(-inf) = 0: padding and masked lanes add nothing
                    s1 += ex2_approx(fmaf(v.y, l2e, nm));
                    s2 += ex2_approx(fmaf(v.z, l2e, nm));
                    s3 += ex2_approx(fmaf(v.w, l2e, nm));
                    const bool any4 = fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)) >= T && T != -INFINITY;
                    const bool all4 = T == -INFINITY && i0 < ldv4;   // degenerate threshold: every real element is a candidate
                    if (__ballot_sync(0xffffffffu, any4 || all4)) {
                        const float xv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const bool hit = (any4 && xv[e] >= T) || (all4 && xv[e] != -INFINITY);
                            const unsigned bm = __ballot_sync(0xffffffffu, hit);
                            if (bm) {
                                const int pos = ncand + __popc(bm & ((1u << lane) - 1));
                                if (hit && pos < 128) cand[pos] = make_float2(xv[e], __int_as_float(i0 * 4 + e));
                                ncand += __popc(bm);
                            }
                        }
                    }
                }
                if (ul == j) DG_STAMP3(54);
                float sum = (s0 + s1) + (s2 + s3);
                sum = warp_sum(sum);
                const float lse = rowmax + logf(sum);
                if (p.dbg_logp) {
                    float* dump = p.dbg_logp + ((size_t)step * N + n) * V;
                    for (int c = lane; c < V; c += 32) dump[c] = xel(c) - lse;
                }
                __syncwarp();
                if (ncand <= 128) {
                    float cv[4];
                    int ci[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int idx = lane + 32 * q;
                        cv[q] = -INFINITY;
                        ci[q] = 0x7fffffff;
                        if (idx < ncand) {
                            const float2 c2 = cand[idx];
                            cv[q] = c2.x - lse;
                            ci[q] = __float_as_int(c2.y);
                        }
                    }
                    for (int k = 0; k < beam; ++k) {
                        float bv = -INFINITY;
                        int bi = 0x7fffffff;
#pragma unroll
                        for (int q = 0; q < 4; ++q)
                            if (better(cv[q], ci[q], bv, bi)) { bv = cv[q]; bi = ci[q]; }
                        warp_best(bv, bi);
#pragma unroll
                        for (int q = 0; q < 4; ++q)
                            if (ci[q] == bi && bi != 0x7fffffff) { cv[q] = -INFINITY; ci[q] = 0x7fffffff; }   // token ids are unique in a row
                        if (lane == 0) { ms.row_v[r][k] = bv; ms.row_i[r][k] = bi; }
                    }
                } else {
                    // exact fallback: the next element after (pv, pi) in the order (log-prob descending, token id ascending)
                    float pv = INFINITY;
                    int pi = -1;
                    for (int k = 0; k < beam; ++k) {
                        float bv = -INFINITY;
                        int bi = 0x7fffffff;
                        for (int c = lane; c < V; c += 32) {
                            const float v = xel(c) - lse;
                            const bool after = (v < pv) || (v == pv && c > pi);
                            if (after && better(v, c, bv, bi)) { bv = v; bi = c; }
                        }
                        warp_best(bv, bi);
                        pv = bv;
                        pi = bi;
                        if (lane == 0) { ms.row_v[r][k] = bv; ms.row_i[r][k] = bi; }
                    }
                }
                if (ul == j) DG_STAMP3(55);
                // finished hypotheses keep emitting EOS at no cost (mask_finished_scores / mask_finished_preds, speech2text.py:156-192);
                // candidate scores = scores + last_k_scores (:118)
                __syncwarp();
                if (lane < beam) {
                    const float rv = pf_flag ? ((lane == 0) ? 0.f : -INFINITY) : ms.row_v[r][lane];
                    const int ri = pf_flag ? (int)EOS_ID : ms.row_i[r][lane];
                    ms.c_val[r * beam + lane] = pf_score + rv;
                    ms.c_tok[r * beam + lane] = ri;
                }
            }
            __syncthreads();
            if (ul == j) DG_STAMP();      // per-row log-softmax statistics + top-`beam`
            if (warp == 0) {      // beam^2 -> beam (:119-122): <= 256 candidates, 8 per lane in registers, `beam` arg-max rounds (ties -> lower
                                  // index).  The generic warp_topk (sorted per-lane insertion lists) spent 11 k cycles here.
                float cv[8];
                int ci[8];
                const int nc = beam * beam;
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int idx = lane + 32 * q;
                    cv[q] = (idx < nc) ? ms.c_val[idx] : -INFINITY;
                    ci[q] = (idx < nc) ? idx : 0x7fffffff;
                }
                for (int k = 0; k < beam; ++k) {
                    float bv = -INFINITY;
                    int bi = 0x7fffffff;
#pragma unroll
                    for (int q = 0; q < 8; ++q)
                        if (better(cv[q], ci[q], bv, bi)) { bv = cv[q]; bi = ci[q]; }
                    warp_best(bv, bi);
#pragma unroll
                    for (int q = 0; q < 8; ++q)
                        if (ci[q] == bi) { cv[q] = -INFINITY; ci[q] = 0x7fffffff; }
                    if (lane == 0) { ms.sel_v[k] = bv; ms.sel_i[k] = bi; }
                }
            }
            if (ul == j) DG_STAMP3(30);
            __syncthreads();
            if (ul == j) DG_STAMP3(31);
            const int cur = step & 1, nxt = cur ^ 1;
            for (int r = warp; r < beam; r += 16) {      // ancestry of the surviving hypotheses (:126-140)
                const int off = ms.sel_i[r];
                const int parent = u * beam + off / beam;
                const int nn = u * beam + r;
                const int* a_old = p.st.anc + ((size_t)cur * N + parent) * Lmax;
                int* a_new = p.st.anc + ((size_t)nxt * N + nn) * Lmax;
                int av[4];                                           // Lmax <= 128: all loads in flight before the first store
#pragma unroll
                for (int q = 0; q < 4; ++q) av[q] = (lane + 32 * q < step) ? a_old[lane + 32 * q] : 0;
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (lane + 32 * q < step) a_new[lane + 32 * q] = av[q];
                if (lane == 0) {
                    a_new[step] = parent;
                    p.st.tok_hist[(size_t)step * N + nn] = ms.c_tok[off];
                    p.st.par_hist[(size_t)step * N + nn] = parent;
                }
            }
            if (ul == j) DG_STAMP3(32);
            __syncthreads();   // every read of the old scores / flags of this utterance is done
            if (ul == j) DG_STAMP3(33);
            if (tid < beam) {
                const int nn = u * beam + tid;
                const int tok = ms.c_tok[ms.sel_i[tid]];
                p.st.scores[nn] = ms.sel_v[tid];
                p.st.last_tok[nn] = tok;
                p.st.flag[nn] = (tok == (int)EOS_ID) ? 1 : 0;
                if (p.dbg_scores) p.dbg_scores[(size_t)step * N + nn] = ms.sel_v[tid];
                if (tok == (int)EOS_ID) atomicAdd(&ms.flag, 1);
            }
            if (ul == j) DG_STAMP3(34);
            __syncthreads();
            if (ul == j) DG_STAMP3(35);
        }
        if (j >= nutt) { DG_STAMP(); DG_STAMP(); }      // keep the stamp count of a CTA without an utterance
        if (tid == 0) {
            ended_here = ms.flag;
            ms.flag = 0;
            if (ended_here) atomicAdd(&p.gstate[(size_t)g * Lmax + step], ended_here);
        }
    };
    // A group that ended early keeps emitting EOS from its (sorted) hypotheses with identity parents while the reference loops
    // on for the other utterances (speech2text.py:62-68): fill the rest of its history so that any global step count >= its own
    // gives the reference's tokens.  Global step count = max over groups (the reference breaks when EVERY hypothesis ended).
    auto fill_history = [&](int steps_done, bool group_done) {
        if (j == 0) {
            for (int i = tid; i < (p.max_steps - steps_done) * nrows; i += DG_THREADS) {
                const int s = steps_done + i / nrows, r = i % nrows;
                p.st.tok_hist[(size_t)s * N + row0 + r] = (int)EOS_ID;
                p.st.par_hist[(size_t)s * N + row0 + r] = row0 + r;
                if (p.dbg_scores) p.dbg_scores[(size_t)s * N + row0 + r] = p.st.scores[row0 + r];
            }
            if (tid == 0) {
                atomicMax(&p.st.ctrl[0], group_done ? steps_done : p.max_steps);
                if (!group_done) atomicAdd(&p.st.ctrl[2], 1);
            }
        }
    };

    // ================================================================================================ the step, as a schedule
    // Each phase is followed by the group barrier that publishes its global writes; the prefetch handed to the barrier
    // fills shared memory that the phase before it has released (see the table at the carve).
    int steps_done = 0;
    bool group_done = false;
    if (is_tma) load_small_b(layer_map(0, MAP_WQKV), j * 48, 48);          // QKV weights of layer 0 for the first step
    for (int step = 0; step < p.max_steps; ++step) {
        dbg_on = dbg_cta && step == p.dbg_step;
        dbg_n = 0;
        dbg_b = 0;
        DG_STAMP();
        build_a_embed(step);
        DG_STAMP();   // 1 embed
        for (int l = 0; l < nl; ++l) {
            const DgLayer& ly = p.layers[l];
            // QKV projection of the newest token (attention.py:68-73): 48 of the 768 columns per CTA; q -> qbuf, k / v -> cache
            gemm_small(l == 0 ? nullptr : shared_map(MAP_X), ly.bqkv, j * 48, [&](int r, int c, float v0, float v1) {
                if (r >= nrows) return;
                const int col = j * 48 + c;               // column pairs never straddle the q | k | v boundaries
                const uint32_t o = pack_bf16(v0 + ms.bias[c], v1 + ms.bias[c + 1]);
                bf16* dst;
                if (col < DG_D) dst = p.qbuf + (size_t)(row0 + r) * DG_D + col;
                else if (col < 2 * DG_D) dst = p.kc + kv_off(l, step, row0 + r) + (col - DG_D);
                else dst = p.vc + kv_off(l, step, row0 + r) + (col - 2 * DG_D);
                *reinterpret_cast<uint32_t*>(dst) = o;
            });
            gsync([&] {      // first half of W_o streams into the A tile behind the self-attention (both stages are its K/V staging area)
                for (int kb = 0; kb < 2; ++kb) load_proj_kb(layer_map(l, MAP_WO), ms.pw_full, kb, sA + kb * 32768);
            });
            DG_STAMP();
            self_attn(l, step);
            __syncthreads();
            if (is_tma) {      // the stages are free again: second half of W_o, first half of W_q
                for (int kb = 2; kb < 4; ++kb) load_proj_kb(layer_map(l, MAP_WO), ms.pw_full, kb, sST + (kb - 2) * 32768);
                for (int kb = 0; kb < 2; ++kb) load_proj_kb(layer_map(l, MAP_WQ), ms.pq_full, kb, sST + DG_STAGE + kb * 32768);
            }
            DG_STAMP();
            wo_ln1_q(l, ly);
            gsync([&] {   // encoder K / V tiles of this CTA's first three (utterance, head) problems: stage 0, stage 1, A tile
                for (int i = 0; i < 3; ++i)
                    if (j + i * DG_P < n_tasks) load_kv(l, j + i * DG_P, i);
            });
            DG_STAMP();
            cross_attn(l);
            gsync([&] {    // cross-attention W_o (A tile + stage 0) and the second half of this CTA's W1 slice (stage 1)
                for (int kb = 0; kb < 4; ++kb) load_proj_kb(layer_map(l, MAP_WO2), ms.pw_full, kb, kb < 2 ? sA + kb * 32768 : sST + (kb - 2) * 32768);
                load_w1(l, 2);
            });
            DG_STAMP();
            wo2_ln2(l, ly);
            gsync(nop);
            DG_STAMP();
            glu_w2(l, ly);
            const bool last_layer = (l + 1 == nl);
            gsync([&] {
                if (last_layer) {   // output-layer chunks of this CTA: the first two stream into the stages during the reduction
                    if (j < n_vchunks) load_wout(j, 0);
                    if (j + DG_P < n_vchunks) load_wout(j + DG_P, 1);
                } else {
                    load_small_b(layer_map(l + 1, MAP_WQKV), j * 48, 48);      // QKV weights of the next layer (sSB)
                }
            });
            DG_STAMP();
            reduce_ln3(ly);
            gsync(nop);
            DG_STAMP();
        }
        logits();
        gsync(nop);
        DG_STAMP();
        beam_step(step);
        gsync([&] { load_small_b(layer_map(0, MAP_WQKV), j * 48, 48); });     // QKV weights of layer 0 for the next step
        DG_STAMP();
        steps_done = step + 1;
        if (tid == 0) ms.flag = (ld_acquire_gpu(&p.gstate[(size_t)g * Lmax + step]) == nrows) ? 1 : 0;
        __syncthreads();
        group_done = ms.flag != 0;
        __syncthreads();
        if (tid == 0) ms.flag = 0;
        if (group_done) break;      // every hypothesis of every utterance of this group ended (uniform across the group)
    }
    // drain the QKV-weight prefetch that was issued for a step that will not run
    if (is_tma)
        for (int kb = 0; kb < 4; ++kb) mbar_wait(&ms.kb_full[kb], pbit(PB_KB, kb));
    fill_history(steps_done, group_done);
#undef DG_STAMP
#undef DG_STAMP2
#undef DG_STAMP3
}

// ---------------------------------------------------------------------------------------------- host side
static int dg_ldv(int V) { return (V + 31) / 32 * 32; }

// The workspace layout, written once: the size query calls it with base == nullptr, the launch with the caller's buffer
// (which then receives p's scratch pointers).  Returns the bytes needed.
static size_t dg_workspace(uint8_t* base, DgParams& p, int N, int n_layers, int Lmax, int G, int V) {
    size_t off = 0;
    auto take = [&](size_t n) { void* r = base ? base + off : nullptr; off += (n + 255) & ~(size_t)255; return r; };
    p.maps = static_cast<CUtensorMap*>(take((size_t)(n_layers * DG_LAYER_MAPS + DG_SHARED_MAPS) * sizeof(CUtensorMap)));
    p.qbuf = static_cast<bf16*>(take((size_t)N * DG_D * 2));
    p.ctx = static_cast<bf16*>(take((size_t)N * DG_D * 2));             // plain loads only: rows < N
    p.xbuf = static_cast<bf16*>(take((size_t)(N + 128) * DG_D * 2));   // + one tile of slack rows for the last group's TMA box
    p.x2buf = static_cast<bf16*>(take((size_t)(N + 128) * DG_D * 2));
    p.q2 = static_cast<bf16*>(take((size_t)N * DG_D * 2));
    p.part = static_cast<float*>(take((size_t)DG_P * G * 128 * DG_D * 4));   // fp32, 128 rows per group
    p.ldv = dg_ldv(V);
    p.logits = static_cast<float*>(take((size_t)G * 128 * p.ldv * 4));      // 128 rows per group
    p.bar = static_cast<int*>(take((size_t)G * 128));
    p.gstate = static_cast<int*>(take((size_t)G * Lmax * 4));
    return off + 1024;
}
static int dg_groups(int B, int beam) { const int upg = 128 / beam; return (B + upg - 1) / upg; }

size_t decode_group_workspace_bytes(int N, int n_layers, int Lmax, int B, int beam, int V) {
    DgParams p;
    return dg_workspace(nullptr, p, N, n_layers, Lmax, dg_groups(B, beam), V);
}

const char* decode_group_launch(cudaStream_t st, const otb_mega_model& m, const bf16* kvx, const int* mem_len, bf16* kc,
                                bf16* vc, const BeamState& bs, int B, int T, int max_steps, float* dbg_logp,
                                float* dbg_scores, void* workspace, size_t workspace_bytes) {
    if (m.d_model != DG_D || m.n_heads != DG_H) return "decode_persistent: needs d_model 256 with 4 heads";
    if (m.d_ff != DG_DFF) return "decode_persistent: d_ff must be 2048 (128 hidden features per CTA of a 16-CTA group)";
    if (bs.beam < 1 || bs.beam > KMAX) return "decode_persistent: beam must be in [1,16]";
    if (bs.Lmax > 128 || max_steps > bs.Lmax || max_steps < 1) return "decode_persistent: max_steps <= Lmax <= 128";
    if (m.n_layers < 1 || m.n_layers > OTB_MEGA_MAX_LAYERS) return "decode_persistent: too many layers";
    if (B < 1 || T < 1 || T > 256 || bs.N != B * bs.beam) return "decode_persistent: bad batch geometry (memory length <= 256)";
    if (m.vocab < 16) return "decode_persistent: vocabulary too small";
    const int beam = bs.beam, N = bs.N, V = m.vocab;
    const int G = dg_groups(B, beam);
    if (G * DG_P > num_sms()) return "decode_persistent: batch needs more co-resident CTAs than the GPU has SMs";
    if (reinterpret_cast<uintptr_t>(workspace) & 255) return "decode_persistent: workspace must be 256-byte aligned";
    DgParams p;
    memset(&p, 0, sizeof(p));
    if (workspace_bytes < dg_workspace(reinterpret_cast<uint8_t*>(workspace), p, N, m.n_layers, bs.Lmax, G, V))
        return "decode_persistent: workspace too small";

    // tensor maps (host encode -> device array).  Weights [rows, K] bf16 row-major, box = (64 columns) x (rows of one slice).
    CUtensorMap h_maps[OTB_MEGA_MAX_LAYERS * DG_LAYER_MAPS + DG_SHARED_MAPS];
    const char* err;
    for (int l = 0; l < m.n_layers; ++l) {
        const otb_mega_layer& ly = m.layers[l];
        CUtensorMap* lm = h_maps + l * DG_LAYER_MAPS;
        if ((err = encode_tmap_2d(&lm[MAP_WQKV], ly.wqkv, DG_D, 3 * DG_D, DG_D, 64, 48))) return err;
        if ((err = encode_tmap_2d(&lm[MAP_WO], ly.wo, DG_D, DG_D, DG_D, 64, 256))) return err;
        if ((err = encode_tmap_2d(&lm[MAP_WQ], ly.wq, DG_D, DG_D, DG_D, 64, 256))) return err;
        if ((err = encode_tmap_2d(&lm[MAP_WO2], ly.wo2, DG_D, DG_D, DG_D, 64, 256))) return err;
        if ((err = encode_tmap_2d(&lm[MAP_W1], ly.w1, DG_D, 2 * DG_DFF, DG_D, 64, 128))) return err;
        if ((err = encode_tmap_2d(&lm[MAP_W2], ly.w2, DG_DFF, DG_D, DG_DFF, 64, 256))) return err;
        DgLayer& d = p.layers[l];
        d.bqkv = ly.bqkv; d.bo = ly.bo; d.bq = ly.bq; d.bo2 = ly.bo2; d.b1 = ly.b1; d.b2 = ly.b2;
        d.g1 = ly.g1; d.be1 = ly.be1; d.g2 = ly.g2; d.be2 = ly.be2; d.g3 = ly.g3; d.be3 = ly.be3;
    }
    CUtensorMap* sm = h_maps + m.n_layers * DG_LAYER_MAPS;
    if ((err = encode_tmap_2d(&sm[MAP_WOUT], m.wout, DG_D, (uint64_t)V, DG_D, 64, 128))) return err;
    if ((err = encode_tmap_2d(&sm[MAP_KVX], kvx, 2 * DG_D, (uint64_t)m.n_layers * B * T, 2 * DG_D, 64, 256))) return err;
    if ((err = encode_tmap_2d(&sm[MAP_X], p.xbuf, DG_D, (uint64_t)N + 128, DG_D, 64, 128))) return err;
    if ((err = encode_tmap_2d(&sm[MAP_X2], p.x2buf, DG_D, (uint64_t)N + 128, DG_D, 64, 128))) return err;
    if ((err = encode_tmap_2d_f32(&sm[MAP_LG], p.logits, 512, (uint64_t)G * (p.ldv / 4), 512, (uint32_t)(beam | 1) * 4, 64))) return err;
    const size_t n_maps = (size_t)m.n_layers * DG_LAYER_MAPS + DG_SHARED_MAPS;
    cudaError_t e = cudaMemcpyAsync(p.maps, h_maps, n_maps * sizeof(CUtensorMap), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return cudaGetErrorString(e);
    if ((e = cudaMemsetAsync(p.bar, 0, (size_t)G * 128, st)) != cudaSuccess) return cudaGetErrorString(e);
    if ((e = cudaMemsetAsync(p.gstate, 0, (size_t)G * bs.Lmax * 4, st)) != cudaSuccess) return cudaGetErrorString(e);

    p.n_layers = m.n_layers; p.V = V; p.G = G; p.utts_per_group = 128 / beam;
    p.emb = reinterpret_cast<const bf16*>(m.emb); p.bout = m.bout; p.pe = m.pe;
    p.mem_len = mem_len; p.kc = kc; p.vc = vc;
    p.st = bs; p.B = B; p.T = T; p.max_steps = max_steps; p.eps = m.ln_eps;
    p.dbg_logp = dbg_logp; p.dbg_scores = dbg_scores;
    p.dbg_clk = g_dg_dbg; p.dbg_step = g_dg_dbg_step;

    // Preferred launch: one thread-block CLUSTER of 16 CTAs per row group (a GPC holds about 16-18 SMs, so at most one such
    // cluster per GPC is co-resident): the group barrier becomes barrier.cluster (hardware, ~0.3 us, and the CTAs of a group
    // are co-scheduled by construction).  Whether the device grants that shape is probed once.  Without it, or with
    // otb_set_decode_barrier(0), the group barrier is the software one on a counter in L2 (plain launch; needs G * 16 <=
    // #SMs co-resident CTAs).  The software barrier spins: it is only safe when every CTA of every batch in flight (all
    // streams together) is resident at once, e.g. 2 batches of 32 utterances (96 CTAs) on a 132-SM H100.
    static const bool cluster_ok = [] {
        // the question is about a DG_SMEM launch, so the kernel's shared-memory cap has to be raised before it is asked
        if (prepare<decode_group_kernel<false>>() || prepare<decode_group_kernel<true>>() ||
            cudaFuncSetAttribute(decode_group_kernel<false>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
            cudaFuncSetAttribute(decode_group_kernel<true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) {
            (void)cudaGetLastError();
            return false;
        }
        // one row group: a cluster of 16 CTAs (non-portable cluster size)
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = DG_P; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cudaLaunchConfig_t q;
        memset(&q, 0, sizeof(q));
        q.gridDim = dim3(DG_P); q.blockDim = dim3(DG_THREADS); q.dynamicSmemBytes = DG_SMEM;
        q.attrs = at; q.numAttrs = 1;
        int nclus = 0;
        if (cudaOccupancyMaxActiveClusters(&nclus, decode_group_kernel<false>, &q) != cudaSuccess || nclus < 1) {
            (void)cudaGetLastError();
            return false;
        }
        return true;
    }();
    // an explicit request for clusters is never served by the spinning software barrier: the caller may keep more CTAs in
    // flight than can be resident at once, which only gang-scheduled clusters tolerate
    if (g_dg_barrier == 1 && !cluster_ok) return "decode_persistent: thread-block clusters of 16 are not available on this device";
    p.cluster = (cluster_ok && g_dg_barrier != 0) ? 1 : 0;
    if (p.dbg_clk != nullptr)      // otb_debug_decode_timing: the stamped instantiation
        return p.cluster ? launch<decode_group_kernel<true>, DG_P>(G * DG_P, DG_THREADS, DG_SMEM, st, p)
                         : launch<decode_group_kernel<true>>(G * DG_P, DG_THREADS, DG_SMEM, st, p);
    return p.cluster ? launch<decode_group_kernel<false>, DG_P>(G * DG_P, DG_THREADS, DG_SMEM, st, p)
                     : launch<decode_group_kernel<false>>(G * DG_P, DG_THREADS, DG_SMEM, st, p);
}

}  // namespace otb
