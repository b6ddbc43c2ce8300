// extern "C" boundary of libotb200.so (declared in include/otb200.h).  Argument checking, error
// reporting (thread-local string, integer status, no aborts) and dispatch to the kernel launchers.
#include <stdio.h>
#include <string.h>

#include "../../include/otb200.h"
#include "dropout.cuh"
#include "otb_internal.h"

namespace otb {


static thread_local char g_err[512] = "";
void set_error(const char* msg) {
    strncpy(g_err, msg ? msg : "", sizeof(g_err) - 1);
    g_err[sizeof(g_err) - 1] = 0;
}
static int fail(const char* where, const char* msg) {
    char buf[512];
    snprintf(buf, sizeof(buf), "%s: %s", where, msg);
    set_error(buf);
    return 1;
}
static BeamState to_state(const otb_beam_state* s) {
    BeamState b;
    b.tok_hist = s->tok_hist; b.par_hist = s->par_hist; b.last_tok = (long long*)s->last_tok;
    b.scores = s->scores; b.flag = s->flag; b.anc = s->anc; b.ctrl = s->ctrl;
    b.N = s->N; b.beam = s->beam; b.Lmax = s->Lmax;
    return b;
}

// The front end's geometry (frontend/conv.py:10-11,27,78-83): per axis floor((n + 2 p - k) / s) + 1 with time unpadded
// and p = kf / 2 in frequency.  T1s / F1s: conv1 buffer rows / columns per conv2 stride phase, enough for every row conv1
// writes and every column conv2 reads (F1s >= F2 so the TMA box fits the view).
static const char* conv_geometry(int T, int F, int kt1, int kf1, int st1, int sf1, int kt2, int kf2, int st2, int sf2, ConvGeom* g) {
    const int k[4] = {kt1, kf1, kt2, kf2}, s[4] = {st1, sf1, st2, sf2};
    for (int i = 0; i < 4; ++i)
        if (k[i] < 1 || k[i] > 7 || s[i] < 1 || s[i] > 4) return "kernel sizes 1..7 and strides 1..4 only";
    if (F < 1) return "need F >= 1";
    if (T < kt1) return "input too short for one conv1 frame";
    g->kt1 = kt1; g->kf1 = kf1; g->st1 = st1; g->sf1 = sf1; g->kt2 = kt2; g->kf2 = kf2; g->st2 = st2; g->sf2 = sf2;
    g->T1 = (T - kt1) / st1 + 1;
    g->F1 = (F + 2 * (kf1 / 2) - kf1) / sf1 + 1;
    if (g->T1 < kt2) return "input too short for one conv2 frame";
    g->T2 = (g->T1 - kt2) / st2 + 1;
    g->F2 = (g->F1 + 2 * (kf2 / 2) - kf2) / sf2 + 1;
    g->T1s = (g->T1 + st2 - 1) / st2;
    g->F1s = max((g->F1 + sf2 - 1) / sf2, g->F2);
    return nullptr;
}

}  // namespace otb

using namespace otb;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define RET(where, expr)                      \
    do {                                      \
        const char* _e = (expr);              \
        if (_e) return fail(where, _e);       \
        return 0;                             \
    } while (0)
// the eight ints of the conv front end's geometry: kernel (kt, kf) and stride (st, sf) of conv1, then of conv2
#define CONV_GEOM int kt1, int kf1, int st1, int sf1, int kt2, int kf2, int st2, int sf2
#define CONV_ARGS kt1, kf1, st1, sf1, kt2, kf2, st2, sf2

extern "C" {

const char* otb_last_error(void) { return g_err; }
int otb_version(void) { return OTB_VERSION; }
int otb_num_sms(void) { return num_sms(); }

int otb_set_tile_policy(int policy) {
    if (policy != 0 && policy != 1) return fail("otb_set_tile_policy", "policy must be 0 (latency) or 1 (throughput)");
    g_tile_policy = policy;
    return 0;
}

int otb_debug_decode_timing(unsigned long long* buf, int step) {
    g_dg_dbg = buf;
    g_dg_dbg_step = step;
    return 0;
}

int otb_set_decode_barrier(int kind) {
    if (kind < -1 || kind > 1) return fail("otb_set_decode_barrier", "kind must be -1 (default), 0 (software) or 1 (cluster)");
    g_dg_barrier = kind;
    return 0;
}

int otb_conv_geometry(int T, int F, CONV_GEOM, int* out) {
    ConvGeom g;
    if (const char* e = conv_geometry(T, F, CONV_ARGS, &g)) return fail("otb_conv_geometry", e);
    if (out) {
        out[0] = g.T1; out[1] = g.F1; out[2] = g.T2; out[3] = g.F2;
        out[4] = g.st2 * g.T1s; out[5] = g.sf2 * g.F1s;
    }
    return 0;
}

int otb_conv1_relu(const float* x, const float* w, const float* bias, void* out, int B, int T, int F, int C1, CONV_GEOM,
                   void* stream) {
    ConvGeom g;
    if (const char* e = conv_geometry(T, F, CONV_ARGS, &g)) return fail("otb_conv1_relu", e);
    if (!x || !w || !bias || !out || B < 1) return fail("otb_conv1_relu", "null pointer or empty batch");
    RET("otb_conv1_relu", conv1_launch(ST(stream), x, w, bias, reinterpret_cast<bf16*>(out), B, T, F, g, C1));
}

int otb_conv2_relu(const void* in, const void* w, const float* bias, void* out, int B, int T, int F, int C1, int C2, CONV_GEOM,
                   void* stream) {
    ConvGeom g;
    if (const char* e = conv_geometry(T, F, CONV_ARGS, &g)) return fail("otb_conv2_relu", e);
    if (!in || !w || !bias || !out || B < 1) return fail("otb_conv2_relu", "null pointer or empty batch");
    if (C1 % 64) return fail("otb_conv2_relu", "C1 must be a multiple of 64 (one 128-byte tap per k-block)");
    if (C2 % 8) return fail("otb_conv2_relu", "C2 must be a multiple of 8");
    if (g.F2 > 128) return fail("otb_conv2_relu", "F2 > 128 not supported");
    int R = 128 / g.F2;
    if (R > g.T1s) R = g.T1s;
    if (R > 256) R = 256;
    CUtensorMap cmap;
    const char* e = encode_tmap_conv5d(&cmap, in, C1, g.sf2, g.F1s, g.st2, B * g.T1s, (uint32_t)g.F2, (uint32_t)R);
    if (e) return fail("otb_conv2_relu", e);
    const int K = kt2 * kf2 * C1;
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.M = B * g.T2 * g.F2;
    p.N = C2;
    p.K = K;
    p.bias = bias;
    p.out = out;
    p.ldc = C2;
    p.alpha = 1.f;
    p.conv = 1;
    p.conv_F2 = g.F2;
    p.conv_R = R;
    p.conv_T1h = g.T1s;
    p.conv_T2 = g.T2;
    p.conv_B = B;
    p.conv_cchunks = C1 / 64;
    for (int kh = 0; kh < kt2; ++kh)
        for (int kw = 0; kw < kf2; ++kw) {
            const int d = kw - kf2 / 2, par_f = ((d % sf2) + sf2) % sf2, f0 = (d - par_f) / sf2;
            p.conv_tap[kh * kf2 + kw] = (unsigned)par_f | (unsigned)(f0 + 8) << 8 | (unsigned)(kh % st2) << 16 | (unsigned)(kh / st2) << 24;
        }
    RET("otb_conv2_relu", gemm_launch(ST(stream), nullptr, 0, w, K, C2, EPI_RELU, p, &cmap));
}

int otb_linear(const void* a, int lda, const void* w, int ldw, const float* bias, void* out, int ldc, int M, int N,
               int K, int epilogue, int out_f32, const void* resid, int ldr, const float* gamma, const float* beta,
               float eps, float alpha, const float* table, int period, const int* row_len, int row_period,
               void* stream) {
    if (!a || !w || !out) return fail("otb_linear", "null operand");
    if (epilogue < 0 || epilogue > EPI_TANH) return fail("otb_linear", "unknown epilogue");
    if ((epilogue == EPI_RESID || epilogue == EPI_RESID_LN) && !resid) return fail("otb_linear", "residual epilogue without resid");
    if (epilogue == EPI_RESID_LN && (!gamma || !beta)) return fail("otb_linear", "LayerNorm epilogue without gamma/beta");
    if (epilogue == EPI_TABLE && (!table || period < 1)) return fail("otb_linear", "table epilogue without table/period");
    if (row_len && row_period < 1) return fail("otb_linear", "row_len without row_period");
    if (ldc < N) return fail("otb_linear", "ldc < N");
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.M = M; p.N = N; p.K = K;
    p.bias = bias;
    p.out = out; p.ldc = ldc; p.out_f32 = out_f32;
    p.resid = reinterpret_cast<const bf16*>(resid); p.ldr = ldr;
    p.gamma = gamma; p.beta = beta; p.eps = eps; p.alpha = alpha;
    p.table = table; p.period = period;
    p.row_len = row_len; p.row_period = row_period;
    const int w_rows = (epilogue == EPI_GLU) ? 2 * N : N;
    RET("otb_linear", gemm_launch(ST(stream), a, lda, w, ldw, w_rows, epilogue, p, nullptr));
}

int otb_gemm_config(int M, int N, int epilogue, int out_f32, int* bn) {
    if (epilogue < 0 || epilogue > EPI_TANH) return fail("otb_gemm_config", "unknown epilogue");
    if (M <= 0 || N <= 0) return fail("otb_gemm_config", "gemm: empty problem");
    int b = 0;
    const char* e = gemm_tile((M + 127) / 128, N, epilogue, out_f32 ? 1 : 0, &b);
    if (e) return fail("otb_gemm_config", e);
    if (bn) *bn = b;
    return 0;
}

int otb_linear_dropout_resid(const void* a, int lda, const void* w, int ldw, const float* bias, void* out, int ldc, int M, int N, int K,
                             const void* resid, int ldr, float alpha, float p_drop, const uint32_t* seed, uint32_t site, float p2,
                             uint32_t site2, void* stream) {
    if (!a || !w || !out || !resid || !seed) return fail("otb_linear_dropout_resid", "null operand");
    if (!(p_drop >= 0.f && p_drop < 1.f) || !(p2 >= 0.f && p2 < 1.f)) return fail("otb_linear_dropout_resid", "p must be in [0, 1)");
    if (ldc < N) return fail("otb_linear_dropout_resid", "ldc < N");
    // two masks only when both rates are non-zero; otherwise the one-mask instantiation with whichever rate is set
    const bool two = p_drop > 0.f && p2 > 0.f;
    if (p_drop == 0.f && p2 > 0.f) { p_drop = p2; site = site2; }
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.M = M; p.N = N; p.K = K;
    p.bias = bias;
    p.out = out; p.ldc = ldc; p.out_f32 = 0;
    p.resid = reinterpret_cast<const bf16*>(resid); p.ldr = ldr;
    p.alpha = alpha;
    p.drop_seed = seed; p.drop_site = site; p.drop_thresh = drop_threshold(p_drop); p.drop_scale = 1.0f / (1.0f - p_drop);
    if (two) { p.drop_site2 = site2; p.drop_thresh2 = drop_threshold(p2); p.drop_scale = drop_scale2(p_drop, p2); }
    RET("otb_linear_dropout_resid", gemm_launch(ST(stream), a, lda, w, ldw, N, two ? EPI_RESID_DROP2 : EPI_RESID, p, nullptr));
}

int otb_dropout_bwd(const void* dy, int lddy, void* out, int ldo, uint8_t* mask, int M, int N, float p, const uint32_t* seed,
                    uint32_t site, float p2, uint32_t site2, void* stream) {
    if ((!dy || !out) && !mask) return fail("otb_dropout_bwd", "nothing to do");
    RET("otb_dropout_bwd", dropout_bwd_launch(ST(stream), reinterpret_cast<const bf16*>(dy), lddy, reinterpret_cast<bf16*>(out), ldo, mask, M, N,
                                              p, seed, site, p2, site2));
}

int otb_attention(const void* q, int ldq, int q_rows, const void* k, int ldk, int k_rows, const void* v, int ldv,
                  void* out, int ldo, int B, int H, int Tq, int Tk, const int* kv_len, int causal, int q_col0,
                  int k_col0, int v_col0, const float* bd, int ldbd, const void* resid, int ldr, float* lse, int d_k,
                  void* stream) {
    if (!q || !k || !v || !out) return fail("otb_attention", "null operand");
    if (d_k != 64 && d_k != 96) return fail("otb_attention", "head width d_k must be 64 or 96");
    if (lse && d_k != 64) return fail("otb_attention", "lse is for the 64-wide backward: it needs d_k = 64");
    if (q_col0 % 8 || k_col0 % 8 || v_col0 % 8 || ldo % 8) return fail("otb_attention", "column offsets / ldo must be multiples of 8");
    if (bd) {   // the kernel reads band row i at columns Tq - 1 - i + j for every visible key j
        if (causal) return fail("otb_attention", "the rel-pos band is for non-causal attention");
        if (Tq != Tk) return fail("otb_attention", "the rel-pos band needs Tq == Tk");
        if (ldbd < 2 * Tq - 1) return fail("otb_attention", "band pitches must hold 2 Tq - 1 columns");
    }
    AttnParams p;
    p.B = B; p.H = H; p.Tq = Tq; p.Tk = Tk;
    p.kv_len = kv_len; p.causal = causal;
    p.scale_log2 = 1.4426950408889634f / sqrtf((float)d_k);   // log2(e) / sqrt(d_k); exactly 0.125 log2(e) at d_k 64
    p.out = reinterpret_cast<bf16*>(out); p.ldo = ldo;
    p.q_col0 = q_col0; p.k_col0 = k_col0; p.v_col0 = v_col0;
    p.bd = bd; p.ldbd = ldbd;
    p.resid = reinterpret_cast<const bf16*>(resid); p.ldr = ldr;
    p.lse = lse;
    if (resid && (ldr % 8)) return fail("otb_attention", "ldr must be a multiple of 8");
    RET("otb_attention", attn_launch(ST(stream), q, ldq, q_rows, k, ldk, k_rows, v, ldv, p, d_k));
}

int otb_attention_probs(const void* q, int ldq, int q_rows, const void* k, int ldk, int k_rows, float* out, int B, int H,
                        int Tq, int Tk, const int* kv_len, int causal, int q_col0, int k_col0, const float* bd, int ldbd,
                        int d_k, void* stream) {
    if (!q || !k || !out) return fail("otb_attention_probs", "null operand");
    if (d_k != 64 && d_k != 96) return fail("otb_attention_probs", "head width d_k must be 64 or 96");
    if (bd && (Tq != Tk || causal)) return fail("otb_attention_probs", "the rel-pos band needs Tq == Tk and no causal mask");
    if (q_col0 % 8 || k_col0 % 8 || ldq % 8 || ldk % 8)
        return fail("otb_attention_probs", "column offsets / leading dimensions must be multiples of 8");
    AttnProbsParams p;
    p.B = B; p.H = H; p.Tq = Tq; p.Tk = Tk;
    p.kv_len = kv_len; p.causal = causal;
    p.scale_log2 = 1.4426950408889634f / sqrtf((float)d_k);   // as otb_attention
    p.q_col0 = q_col0; p.k_col0 = k_col0;
    p.bd = bd; p.ldbd = ldbd;
    p.out = out;
    RET("otb_attention_probs", attn_probs_launch(ST(stream), q, ldq, q_rows, k, ldk, k_rows, p, d_k));
}

int otb_layernorm(const void* x, int ldx, void* out, int ldo, int out_f32, const float* g1, const float* b1,
                  const float* g2, const float* b2, float eps, int M, int N, void* stream) {
    if (!x || !out || !g1 || !b1) return fail("otb_layernorm", "null operand");
    if ((g2 == nullptr) != (b2 == nullptr)) return fail("otb_layernorm", "g2/b2 must both be given");
    RET("otb_layernorm", layernorm_launch(ST(stream), reinterpret_cast<const bf16*>(x), ldx, out, ldo, out_f32, g1, b1,
                                          g2, b2, eps, M, N));
}

int otb_scale_add_table(const void* x, int ldx, int x_f32, void* out, int ldo, float alpha, const float* table,
                        int period, int M, int N, const float* alpha_dev, void* stream) {
    if (!x || !out || M < 1 || N < 1) return fail("otb_scale_add_table", "bad arguments");
    if (table && period < 1) return fail("otb_scale_add_table", "table without period");
    RET("otb_scale_add_table", scale_add_table_launch(ST(stream), x, ldx, x_f32, reinterpret_cast<bf16*>(out), ldo, alpha,
                                                      table, period, M, N, alpha_dev));
}

int otb_dwconv_swish(const void* x, const float* w, const float* b, void* out, int B, int T, int d, int k,
                     void* stream) {
    if (!x || !w || !b || !out || B < 1 || T < 1) return fail("otb_dwconv_swish", "bad arguments");
    RET("otb_dwconv_swish", dwconv_swish_launch(ST(stream), reinterpret_cast<const bf16*>(x), w, b,
                                                reinterpret_cast<bf16*>(out), B, T, d, k));
}

int otb_sinusoid_table(float* out, int n_pos, int d, int first_pos, void* stream) {
    if (!out || n_pos < 1 || d < 2 || (d & 1)) return fail("otb_sinusoid_table", "bad arguments");
    RET("otb_sinusoid_table", sinusoid_table_launch(ST(stream), out, n_pos, d, first_pos));
}

int otb_embed_posenc(const int64_t* tok, int tok_stride, const void* emb, const float* table, void* out, int N,
                     int d, int period, const int* step_ptr, const int* row_pos, int vocab, void* stream) {
    if (!tok || !emb || !table || !out) return fail("otb_embed_posenc", "null operand");
    if (!row_pos && !step_ptr && period < 1) return fail("otb_embed_posenc", "need period, step_ptr or row_pos");
    RET("otb_embed_posenc",
        embed_posenc_launch(ST(stream), reinterpret_cast<const long long*>(tok), tok_stride,
                            reinterpret_cast<const bf16*>(emb), table, reinterpret_cast<bf16*>(out), N, d, period,
                            step_ptr, vocab, row_pos));
}

int otb_log_softmax(const float* x, int ldx, float* out, int ldo, int rows, int V, void* stream) {
    if (!x || !out || rows < 1 || V < 1) return fail("otb_log_softmax", "bad arguments");
    RET("otb_log_softmax", log_softmax_launch(ST(stream), x, ldx, out, ldo, rows, V));
}

int otb_decode_self_attn(const void* qkv, void* kc, void* vc, const int* anc, const int* step_ptr, const int* row_pos, void* out,
                         int N, int H, int Lmax, int d_k, void* stream) {
    if (!qkv || !kc || !vc || !anc || !out) return fail("otb_decode_self_attn", "null operand");
    if (!step_ptr == !row_pos) return fail("otb_decode_self_attn", "give exactly one of step_ptr and row_pos");
    if (d_k != 64 && d_k != 96) return fail("otb_decode_self_attn", "head width d_k must be 64 or 96");
    RET("otb_decode_self_attn",
        decode_self_attn_launch(ST(stream), reinterpret_cast<const bf16*>(qkv), reinterpret_cast<bf16*>(kc),
                                reinterpret_cast<bf16*>(vc), anc, step_ptr, reinterpret_cast<bf16*>(out), N, H, Lmax, d_k, row_pos));
}

int otb_ls_ce(const float* logits, int ldl, const int64_t* targets, int rows, int V, float smoothing, int pad_id,
              float* tok_loss, float* loss, int32_t* n_valid, void* dlogits, int ldd, int dlogits_bf16, void* stream) {
    if (!logits || !targets || !tok_loss || !loss || !n_valid) return fail("otb_ls_ce", "null operand");
    if (dlogits_bf16 && !dlogits) return fail("otb_ls_ce", "dlogits_bf16 without dlogits");
    if (dlogits_bf16 && (ldd < V || ldd % 8)) return fail("otb_ls_ce", "a bf16 dlogits needs ldd >= V and a multiple of 8");
    RET("otb_ls_ce", ls_ce_launch(ST(stream), logits, ldl, reinterpret_cast<const long long*>(targets), rows, V, smoothing,
                                  pad_id, tok_loss, loss, n_valid, dlogits_bf16 ? nullptr : static_cast<float*>(dlogits), ldd,
                                  dlogits_bf16 ? static_cast<bf16*>(dlogits) : nullptr));
}

int otb_beam_init(const otb_beam_state* st, void* stream) {
    if (!st) return fail("otb_beam_init", "null state");
    RET("otb_beam_init", beam_init_launch(ST(stream), to_state(st)));
}

int otb_beam_step(const float* logp, int ldl, int V, const float* lm_logp, int ld_lm, float lm_weight, const float* topk_val,
                  const int32_t* topk_idx, const otb_beam_state* st, int64_t* dbg_ktok, int32_t* dbg_offs, void* stream) {
    if (!st) return fail("otb_beam_step", "null state");
    if (logp ? (topk_val || topk_idx) : (!topk_val || !topk_idx))
        return fail("otb_beam_step", "give either logp or both topk_val and topk_idx");
    RET("otb_beam_step", beam_step_launch(ST(stream), logp, ldl, V, lm_logp, ld_lm, lm_weight, to_state(st),
                                          reinterpret_cast<long long*>(dbg_ktok), dbg_offs, topk_val, topk_idx));
}

int otb_logsoftmax_topk(const float* logits, int ldl, int V, const float* lm_logp, int ld_lm, float lm_weight, float lm_beta,
                        int lm_exempt, int k, int rows, float* out_val, int32_t* out_idx, float* out_logp, int ld_logp, void* stream) {
    if (!logits || !out_val || !out_idx || rows < 1) return fail("otb_logsoftmax_topk", "bad arguments");
    RET("otb_logsoftmax_topk", logsoftmax_topk_launch(ST(stream), logits, ldl, V, lm_logp, ld_lm, lm_weight, lm_beta, lm_exempt, k,
                                                      rows, out_val, out_idx, out_logp, ld_logp));
}

int otb_sample_step(const float* logits, int ldl, int V, const otb_beam_state* st, const int32_t* seed, void* stream) {
    if (!logits || !st || !seed) return fail("otb_sample_step", "null operand");
    RET("otb_sample_step", sample_step_launch(ST(stream), logits, ldl, V, to_state(st), seed));
}

int otb_beam_reconstruct(const otb_beam_state* st, int64_t* preds, int ld, int steps, void* stream) {
    if (!st || !preds) return fail("otb_beam_reconstruct", "null operand");
    RET("otb_beam_reconstruct", beam_reconstruct_launch(ST(stream), to_state(st), reinterpret_cast<long long*>(preds), ld, steps));
}

int otb_beam_finalize(const otb_beam_state* st, float penalty, float lamda, int nbest, int64_t* out_preds,
                      float* out_scores, void* stream) {
    if (!st || !out_preds || !out_scores) return fail("otb_beam_finalize", "null operand");
    RET("otb_beam_finalize", beam_finalize_launch(ST(stream), to_state(st), penalty, lamda, nbest,
                                                  reinterpret_cast<long long*>(out_preds), out_scores));
}

long long otb_decode_persistent_workspace(int N, int n_layers, int Lmax, int B, int beam, int vocab) {
    if (N < 1 || n_layers < 1 || Lmax < 1 || B < 1 || beam < 1 || beam > 16 || vocab < 1) return -1;
    return (long long)decode_group_workspace_bytes(N, n_layers, Lmax, B, beam, vocab);
}

int otb_decode_persistent(const otb_mega_model* model, const void* kvx, const int32_t* mem_len, void* kc, void* vc,
                          const otb_beam_state* st, int B, int T, int max_steps, void* workspace, long long workspace_bytes,
                          float* dbg_logp, float* dbg_scores, void* stream) {
    if (!model || !kvx || !mem_len || !kc || !vc || !st || !workspace) return fail("otb_decode_persistent", "null operand");
    if (model->n_layers < 1 || model->n_layers > OTB_MEGA_MAX_LAYERS) return fail("otb_decode_persistent", "1..8 decoder layers");
    if (!model->emb || !model->wout || !model->pe) return fail("otb_decode_persistent", "null model tensor");
    for (int l = 0; l < model->n_layers; ++l) {
        const otb_mega_layer& s = model->layers[l];
        const void* need[18] = {s.wqkv, s.wo, s.wq, s.wo2, s.w1, s.w2, s.bqkv, s.bo, s.bq, s.bo2, s.b1, s.b2,
                                s.g1, s.be1, s.g2, s.be2, s.g3, s.be3};
        for (int i = 0; i < 18; ++i)
            if (!need[i]) return fail("otb_decode_persistent", "null layer tensor (biases are required)");
    }
    RET("otb_decode_persistent", decode_group_launch(ST(stream), *model, reinterpret_cast<const bf16*>(kvx), mem_len,
                                                     reinterpret_cast<bf16*>(kc), reinterpret_cast<bf16*>(vc), to_state(st), B, T,
                                                     max_steps, dbg_logp, dbg_scores, workspace, (size_t)workspace_bytes));
}

int otb_attention_bwd(const void* q, int ldq, int q_rows, const void* k, int ldk, int k_rows, const void* v, int ldv,
                      const void* out, int ldo, const void* dout, int lddo, const float* lse, float* dsum, void* dq,
                      int lddq, int dq_col0, void* dk, int lddk, int dk_col0, void* dv, int lddv, int dv_col0, int B, int H,
                      int Tq, int Tk, const int* kv_len, int causal, int q_col0, int k_col0, int v_col0, const float* bd, int ldbd,
                      void* dbd, int lddbd, void* stream) {
    if (!q || !k || !v || !out || !dout || !lse || !dsum || !dq || !dk || !dv) return fail("otb_attention_bwd", "null operand");
    if ((q_col0 | k_col0 | v_col0 | dq_col0 | dk_col0 | dv_col0 | ldo | lddo | lddq | lddk | lddv) % 8)
        return fail("otb_attention_bwd", "column offsets / leading dimensions must be multiples of 8");
    if (!bd != !dbd) return fail("otb_attention_bwd", "bd and dbd must both be given or both be NULL");
    if (bd) {
        if (causal) return fail("otb_attention_bwd", "the rel-pos band is for non-causal attention");
        if (Tq != Tk) return fail("otb_attention_bwd", "the rel-pos band needs Tq == Tk");
        if (ldbd < 2 * Tq - 1 || lddbd < 2 * Tq - 1 || lddbd % 8)
            return fail("otb_attention_bwd", "band pitches must hold 2 Tq - 1 columns; the gradient's must be a multiple of 8");
    }
    AttnBwdParams p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.H = H; p.Tq = Tq; p.Tk = Tk; p.kv_len = kv_len; p.causal = causal;
    p.scale_log2 = 0.125f * 1.4426950408889634f;
    p.q_col0 = q_col0; p.k_col0 = k_col0; p.v_col0 = v_col0;
    p.o = reinterpret_cast<const bf16*>(out); p.ldo = ldo;
    p.dout = reinterpret_cast<const bf16*>(dout); p.lddo = lddo;
    p.lse = lse; p.dsum = dsum;
    p.dq = reinterpret_cast<bf16*>(dq); p.lddq = lddq; p.dq_col0 = dq_col0;
    p.dk = reinterpret_cast<bf16*>(dk); p.lddk = lddk; p.dk_col0 = dk_col0;
    p.dv = reinterpret_cast<bf16*>(dv); p.lddv = lddv; p.dv_col0 = dv_col0;
    p.bd = bd; p.ldbd = ldbd;
    p.dbd = reinterpret_cast<bf16*>(dbd); p.lddbd = lddbd;
    RET("otb_attention_bwd", attn_bwd_launch(ST(stream), q, ldq, q_rows, k, ldk, k_rows, v, ldv, p));
}

int otb_dropout_add(const void* x, int ldx, const void* resid, int ldr, void* out, int ldo, int M, int N, float alpha, float p,
                    const uint32_t* seed, uint32_t site, const int32_t* row_len, int row_period, void* stream) {
    if (!x || !out) return fail("otb_dropout_add", "null operand");
    RET("otb_dropout_add", dropout_add_launch(ST(stream), reinterpret_cast<const bf16*>(x), ldx, reinterpret_cast<const bf16*>(resid), ldr,
                                              reinterpret_cast<bf16*>(out), ldo, M, N, alpha, p, seed, site, row_len, row_period));
}

int otb_conformer_conv_train(const void* x, const int32_t* len, const float* w, const float* wb, const float* gamma, const float* beta,
                             float* running_mean, float* running_var, int64_t* num_batches, float momentum, float eps, float* c,
                             float* stats, void* out, int B, int T, int d, int k, void* stream) {
    if (!x || !len || !w || !gamma || !beta || !c || !stats || !out) return fail("otb_conformer_conv_train", "null operand");
    RET("otb_conformer_conv_train", conv_bn_train_launch(ST(stream), reinterpret_cast<const bf16*>(x), len, w, wb, gamma, beta,
                                                         running_mean, running_var, reinterpret_cast<long long*>(num_batches),
                                                         momentum, eps, c, stats, reinterpret_cast<bf16*>(out), B, T, d, k));
}

int otb_conformer_conv_bwd(const void* dy, const void* x, const int32_t* len, const float* w, const float* gamma, const float* beta,
                           const float* c, const float* stats, float* red, float* dc, void* dx, float* dw, float* dwb, float* dgamma,
                           float* dbeta, int accumulate, int B, int T, int d, int k, void* stream) {
    if (!dy || !x || !len || !w || !gamma || !beta || !c || !stats || !red || !dc || !dx || !dw || !dgamma || !dbeta)
        return fail("otb_conformer_conv_bwd", "null operand");
    RET("otb_conformer_conv_bwd", conv_bn_bwd_launch(ST(stream), reinterpret_cast<const bf16*>(dy), reinterpret_cast<const bf16*>(x), len,
                                                     w, gamma, beta, c, stats, red, dc, reinterpret_cast<bf16*>(dx), dw, dwb, dgamma,
                                                     dbeta, accumulate, B, T, d, k));
}

int otb_linear_wgrad(const void* dy, int lddy, const void* x, int ldx, float* dw, int lddw, int M, int N, int K, int accumulate,
                     void* stream) {
    if (!dy || !x || !dw) return fail("otb_linear_wgrad", "null operand");
    RET("otb_linear_wgrad", gemm_wgrad_launch(ST(stream), dy, lddy, x, ldx, dw, lddw, M, N, K, accumulate));
}

int otb_colsum(const void* x, int ldx, float* out, int M, int N, int accumulate, void* stream) {
    if (!x || !out || M < 1 || N < 1) return fail("otb_colsum", "bad arguments");
    RET("otb_colsum", colsum_launch(ST(stream), reinterpret_cast<const bf16*>(x), ldx, out, M, N, accumulate));
}

int otb_layernorm_bwd(const void* dy, int lddy, const void* z, int ldz, const float* gamma, void* dz, int lddz,
                      float* dgamma, float* dbeta, float eps, int M, int N, int accumulate, void* stream) {
    if (!dy || !z || !gamma || !dz || !dgamma || !dbeta) return fail("otb_layernorm_bwd", "null operand");
    RET("otb_layernorm_bwd", layernorm_bwd_launch(ST(stream), reinterpret_cast<const bf16*>(dy), lddy,
                                                  reinterpret_cast<const bf16*>(z), ldz, gamma, reinterpret_cast<bf16*>(dz),
                                                  lddz, dgamma, dbeta, eps, M, N, accumulate));
}

int otb_glu_fwd(const void* u, void* h, int M, int F, void* stream) {
    if (!u || !h || M < 1 || F < 8) return fail("otb_glu_fwd", "bad arguments");
    RET("otb_glu_fwd", glu_launch(ST(stream), reinterpret_cast<const bf16*>(u), nullptr, reinterpret_cast<bf16*>(h), M, F));
}

int otb_glu_bwd(const void* dh, const void* u, void* du, int M, int F, void* stream) {
    if (!dh || !u || !du || M < 1 || F < 8) return fail("otb_glu_bwd", "bad arguments");
    RET("otb_glu_bwd", glu_launch(ST(stream), reinterpret_cast<const bf16*>(u), reinterpret_cast<const bf16*>(dh),
                                  reinterpret_cast<bf16*>(du), M, F));
}

int otb_act_fwd(const void* u, void* h, int M, int N, int act, void* stream) {
    if (!u || !h || M < 1 || N < 1) return fail("otb_act_fwd", "bad arguments");
    RET("otb_act_fwd", act_launch(ST(stream), act, reinterpret_cast<const bf16*>(u), nullptr, reinterpret_cast<bf16*>(h),
                                  (size_t)M * (size_t)N));
}

int otb_act_bwd(const void* dh, const void* u, void* du, int M, int N, int act, void* stream) {
    if (!dh || !u || !du || M < 1 || N < 1) return fail("otb_act_bwd", "bad arguments");
    RET("otb_act_bwd", act_launch(ST(stream), act, reinterpret_cast<const bf16*>(u), reinterpret_cast<const bf16*>(dh),
                                  reinterpret_cast<bf16*>(du), (size_t)M * (size_t)N));
}

int otb_relu_bwd(const void* dy, const void* y, void* dx, long long n, void* stream) {
    if (!dy || !y || !dx || n < 8) return fail("otb_relu_bwd", "bad arguments");
    RET("otb_relu_bwd", relu_bwd_launch(ST(stream), reinterpret_cast<const bf16*>(dy), reinterpret_cast<const bf16*>(y),
                                        reinterpret_cast<bf16*>(dx), (size_t)n));
}

int otb_embed_bwd(const int64_t* tok, const void* dx, float* dE, int N, int d, int vocab, float scale, void* stream) {
    if (!tok || !dx || !dE || N < 1) return fail("otb_embed_bwd", "bad arguments");
    RET("otb_embed_bwd", embed_bwd_launch(ST(stream), reinterpret_cast<const long long*>(tok), reinterpret_cast<const bf16*>(dx),
                                          dE, N, d, vocab, scale));
}

int otb_sumsq(const float* g, long long n, float* out, int zero_first, void* stream) {
    if (!g || !out || n < 1) return fail("otb_sumsq", "bad arguments");
    RET("otb_sumsq", sumsq_launch(ST(stream), g, (size_t)n, out, zero_first));
}

int otb_adam_step_sched(float* p, const float* g, float* m, float* v, long long n, const float* sumsq, float max_norm,
                        float base_lr, float model_size, float warmup_steps, float factor, float beta1, float beta2, float eps,
                        float weight_decay, int32_t* counters, float* hyper, float noise_std, const int32_t* noise_seed,
                        const uint8_t* noise_mask, void* stream) {
    if (!p || !g || !m || !v || !sumsq || !counters || !hyper || n < 1) return fail("otb_adam_step_sched", "bad arguments");
    if (!(noise_std >= 0.f)) return fail("otb_adam_step_sched", "noise_std must be >= 0");
    if (noise_std > 0.f && (!noise_seed || !noise_mask)) return fail("otb_adam_step_sched", "noise without seed or mask");
    RET("otb_adam_step_sched", adam_sched_launch(ST(stream), p, g, m, v, (size_t)n, sumsq, max_norm, base_lr, model_size, warmup_steps,
                                                 factor, beta1, beta2, eps, weight_decay, counters, hyper, noise_std, noise_seed,
                                                 noise_mask));
}

int otb_mixspeech(const float* x, const uint8_t* mask, int B, int T, int F, const int32_t* seed, const int32_t* step, float scale,
                  float* lam_out, float* x_out, uint8_t* mask_out, void* stream) {
    if (!x || !mask || !seed || !step || !lam_out || !x_out || !mask_out) return fail("otb_mixspeech", "null operand");
    RET("otb_mixspeech", mixspeech_launch(ST(stream), x, mask, B, T, F, seed, step, scale, lam_out, x_out, mask_out));
}

int otb_frame_stack(const float* x, int B, int T, int F, int n, int s, int T2, void* out, int ldo, float alpha, const float* table,
                    void* stream) {
    if (!x || !out) return fail("otb_frame_stack", "null operand");
    RET("otb_frame_stack", frame_stack_launch(ST(stream), x, B, T, F, n, s, T2, reinterpret_cast<bf16*>(out), ldo, alpha, table));
}

int otb_fbank(const float* wave, int ld_wave, const int32_t* n_samples, const float* gain, int B, const float* window,
              const float* bank, const int32_t* bank_range, float* out, int Tmax, int F, int frame_len, int frame_shift, float preemph,
              void* stream) {
    if (!wave || !n_samples || !window || !bank || !bank_range || !out) return fail("otb_fbank", "null operand");
    RET("otb_fbank", fbank_launch(ST(stream), wave, ld_wave, n_samples, gain, B, window, bank, bank_range, out, Tmax, F, frame_len,
                                  frame_shift, preemph));
}

int otb_utt_cmvn(float* x, int B, int Tmax, int F, const int32_t* n_frames, const float* gmean, const float* gstd, const float* noise,
                 void* stream) {
    if (!x || !n_frames) return fail("otb_utt_cmvn", "null operand");
    RET("otb_utt_cmvn", utt_cmvn_launch(ST(stream), x, B, Tmax, F, n_frames, gmean, gstd, noise));
}

int otb_resample(const float* x, int ldx, const int32_t* n_in, const int32_t* orig, const int32_t* new_rate, float* y, int ldy,
                 int32_t* n_out, int B, int width, void* stream) {
    if (!x || !n_in || !orig || !new_rate || !y || !n_out) return fail("otb_resample", "null operand");
    if (B < 1 || width < 1) return fail("otb_resample", "need B >= 1 and width >= 1");
    if (ldx < 1 || ldy < width) return fail("otb_resample", "row pitch smaller than the row");
    RET("otb_resample", resample_launch(ST(stream), x, ldx, n_in, orig, new_rate, y, ldy, n_out, B, width));
}

int otb_ctc_loss(const float* logp, int ldl, int B, int T, int V, const int32_t* in_len, const int64_t* targets, int ldt,
                 const int32_t* tgt_len, int max_tgt, int blank, float* nll, float* loss, float* ws, void* dlogits_bf16, int ldd,
                 float grad_scale, const float* grad_scale_dev, void* stream) {
    if (!logp || !in_len || !targets || !tgt_len || !nll || !loss || !ws) return fail("otb_ctc_loss", "null operand");
    if (ldl < V || (dlogits_bf16 && ldd < V)) return fail("otb_ctc_loss", "row pitch < V");
    RET("otb_ctc_loss", ctc_launch(ST(stream), logp, ldl, B, T, V, in_len, reinterpret_cast<const long long*>(targets), ldt, tgt_len, max_tgt,
                                   blank, nll, loss, ws, reinterpret_cast<bf16*>(dlogits_bf16), ldd, grad_scale,
                                   grad_scale_dev));
}

int otb_ctc_frame_topk(const float* logits, int ld, int B, int T, int V, const int32_t* in_len, int K, float* top_lp,
                       int32_t* top_id, void* stream) {
    if (!logits || !in_len || !top_lp || !top_id) return fail("otb_ctc_frame_topk", "null operand");
    if (ld < V) return fail("otb_ctc_frame_topk", "row pitch < V");
    RET("otb_ctc_frame_topk", ctc_frame_topk_launch(ST(stream), logits, ld, B, T, V, in_len, K, top_lp, top_id));
}

int otb_ctc_greedy(const float* top_lp, const int32_t* top_id, int ldk, int B, int T, const int32_t* in_len, int blank,
                   int32_t* ids, int32_t* lengths, float* scores, void* stream) {
    if (!top_lp || !top_id || !in_len || !ids || !lengths || !scores) return fail("otb_ctc_greedy", "null operand");
    RET("otb_ctc_greedy", ctc_greedy_launch(ST(stream), top_lp, top_id, ldk, B, T, in_len, blank, ids, lengths, scores));
}

int otb_ctc_prefix_beam(const float* top_lp, const int32_t* top_id, int K, int B, int T, const int32_t* in_len, int blank, int beam,
                        int32_t* nodes, int32_t* ids, int32_t* lengths, float* scores, void* stream) {
    if (!top_lp || !top_id || !in_len || !nodes || !ids || !lengths || !scores) return fail("otb_ctc_prefix_beam", "null operand");
    RET("otb_ctc_prefix_beam", ctc_prefix_beam_launch(ST(stream), top_lp, top_id, K, B, T, in_len, blank, beam, nodes, ids,
                                                      lengths, scores));
}

int otb_ctc_prefix_beam_slots_bytes(int B) { return B < 1 ? -1 : ctc_prefix_beam_slots_bytes(B); }

int otb_ctc_prefix_beam_step(const float* top_lp, const int32_t* top_id, int K, int B, int T, const int32_t* in_len, int blank,
                             int beam, const float* lm, int ld_lm, float lm_weight, float beta, void* slots, int32_t* ctl,
                             int32_t* nodes, int32_t* src, int64_t* tok, int32_t* ext, int32_t* anc, int32_t* anc_tmp,
                             int32_t* pos, int Lpos, int32_t* ids, int32_t* lengths, float* scores, void* stream) {
    if (!top_lp || !top_id || !in_len || !lm || !slots || !ctl || !nodes || !src || !tok || !ext || !ids || !lengths || !scores)
        return fail("otb_ctc_prefix_beam_step", "null operand");
    CtcStepArgs a;
    a.top_lp = top_lp; a.top_id = top_id; a.K = K; a.T = T; a.in_len = in_len; a.blank = blank; a.beam = beam;
    a.lm = lm; a.ld_lm = ld_lm; a.lm_w = lm_weight; a.beta = beta; a.slots = slots; a.ctl = ctl; a.nodes = nodes;
    a.src = src; a.tok = reinterpret_cast<long long*>(tok); a.ext = ext; a.anc = anc; a.anc_tmp = anc_tmp; a.pos = pos;
    a.Lpos = Lpos; a.ids = ids; a.lengths = lengths; a.scores = scores;
    RET("otb_ctc_prefix_beam_step", ctc_prefix_beam_step_launch(ST(stream), a, B));
}

int otb_ctc_lm_carry(void* dst, int ldd, const void* a, int lda, const void* b, int ldb, const int32_t* idx, const int32_t* ext,
                     int rows, int width, void* stream) {
    if (!dst || !b) return fail("otb_ctc_lm_carry", "null operand");
    RET("otb_ctc_lm_carry", ctc_lm_carry_launch(ST(stream), dst, ldd, a, lda, b, ldb, idx, ext, rows, width));
}

int otb_ctc_align(const float* rows, int ld, int B, int T, int V, const float* lse, const int32_t* in_len, const int64_t* targets,
                  int ldt, const int32_t* tgt_len, int max_tgt, int blank, uint8_t* bp, int32_t* labels, float* frame_scores,
                  int32_t* spans, float* path_score, void* stream) {
    if (!rows || !in_len || !tgt_len || !bp || !labels || !frame_scores || !path_score || (max_tgt > 0 && (!targets || !spans)))
        return fail("otb_ctc_align", "null operand");
    if (ld < V) return fail("otb_ctc_align", "row pitch < V");
    if (max_tgt > 0 && ldt < max_tgt) return fail("otb_ctc_align", "target row pitch < max_tgt");
    RET("otb_ctc_align", ctc_align_launch(ST(stream), rows, ld, B, T, V, lse, in_len, reinterpret_cast<const long long*>(targets), ldt,
                                          tgt_len, max_tgt, blank, bp, labels, frame_scores, spans, path_score));
}

int otb_ctc_prefix_init(const float* lp, int ld, int B, int T, const int32_t* in_len, int blank, int beam, float* gamma,
                        float* psi, void* stream) {
    if (!lp || !in_len || !gamma || !psi) return fail("otb_ctc_prefix_init", "null operand");
    if (blank < 0 || blank >= ld) return fail("otb_ctc_prefix_init", "bad blank id");
    RET("otb_ctc_prefix_init", ctc_prefix_init_launch(ST(stream), lp, ld, B, T, in_len, blank, beam, gamma, psi));
}

int otb_ctc_prefix_score(const float* lp, int ld, int T, int V, const int32_t* in_len, int blank, const float* gamma,
                         const float* psi, const float* cand_val, const int32_t* cand_id, int P, const float* lm_logp, int ld_lm,
                         float lm_weight, float ctc_weight, const otb_beam_state* st, float* gamma_cand, float* psi_cand,
                         float* out_val, int32_t* out_idx, void* stream) {
    if (!lp || !in_len || !gamma || !psi || !cand_val || !cand_id || !st || !gamma_cand || !psi_cand || !out_val || !out_idx)
        return fail("otb_ctc_prefix_score", "null operand");
    RET("otb_ctc_prefix_score", ctc_prefix_score_launch(ST(stream), lp, ld, T, V, in_len, blank, gamma, psi, cand_val, cand_id, P,
                                                        lm_logp, ld_lm, lm_weight, ctc_weight, to_state(st), gamma_cand, psi_cand,
                                                        out_val, out_idx));
}

int otb_ctc_prefix_advance(const otb_beam_state* st, const int32_t* cand_id, int P, int T, const int32_t* in_len,
                           const float* gamma_cand, const float* psi_cand, float* gamma, float* psi, void* stream) {
    if (!st || !cand_id || !in_len || !gamma_cand || !psi_cand || !gamma || !psi) return fail("otb_ctc_prefix_advance", "null operand");
    RET("otb_ctc_prefix_advance", ctc_prefix_advance_launch(ST(stream), to_state(st), cand_id, P, T, in_len, gamma_cand, psi_cand,
                                                            gamma, psi));
}

int otb_ctc_nbest_score(const float* logp, int ld, int B, int T, int V, const int32_t* in_len, const int32_t* targets, int K,
                        int Lp, int blank, float* out, void* stream) {
    if (!logp || !in_len || !targets || !out) return fail("otb_ctc_nbest_score", "null operand");
    RET("otb_ctc_nbest_score", ctc_nbest_score_launch(ST(stream), logp, ld, B, T, V, in_len, targets, K, Lp, blank, out));
}

int otb_token_logprob(const float* logits, int ld, int rows, int V, const int32_t* target, float* out, void* stream) {
    if (rows > 0 && (!logits || !target || !out)) return fail("otb_token_logprob", "null operand");
    RET("otb_token_logprob", token_logprob_launch(ST(stream), logits, ld, rows, V, target, out));
}

static const char* rnnt_lattice_check(int B, int T, int U1, const void* t_len, const void* u_len, int64_t row0, int rows) {
    if (B < 1 || T < 1 || U1 < 1) return "empty lattice";
    if (!t_len || !u_len) return "null lengths";
    if (row0 < 0 || rows < 0 || row0 + rows > (int64_t)B * T * U1) return "rows outside the lattice";
    return nullptr;
}

// rows of the stored lattice: B T U1, or B T S when banded
static int64_t rnnt_rows(int B, int T, int U1, const void* s_begin, int S) { return (int64_t)B * T * (s_begin ? S : U1); }

int otb_rnnt_joint(const void* ep, const void* pp, int B, int T, int U1, int D, const int32_t* t_len, const int32_t* u_len, void* out,
                   const int32_t* s_begin, int S, void* stream) {
    if (!ep || !pp || !out) return fail("otb_rnnt_joint", "null operand");
    if ((t_len == nullptr) != (u_len == nullptr)) return fail("otb_rnnt_joint", "t_len and u_len are given together");
    RET("otb_rnnt_joint", rnnt_joint_launch(ST(stream), reinterpret_cast<const bf16*>(ep), reinterpret_cast<const bf16*>(pp), B, T, U1,
                                            D, t_len, u_len, s_begin, S, reinterpret_cast<bf16*>(out)));
}

int otb_rnnt_joint_bwd(const void* dh, const void* h, int B, int T, int U1, int D, const int32_t* t_len, const int32_t* u_len,
                       void* dep, void* dpp, const int32_t* s_begin, int S, void* stream) {
    if (!dh || !h || !dep || !dpp) return fail("otb_rnnt_joint_bwd", "null operand");
    if (const char* e = rnnt_lattice_check(B, T, U1, t_len, u_len, 0, 0)) return fail("otb_rnnt_joint_bwd", e);
    RET("otb_rnnt_joint_bwd", rnnt_joint_bwd_launch(ST(stream), reinterpret_cast<const bf16*>(dh), reinterpret_cast<const bf16*>(h), B,
                                                    T, U1, D, t_len, u_len, s_begin, S, reinterpret_cast<bf16*>(dep),
                                                    reinterpret_cast<bf16*>(dpp)));
}

int otb_rnnt_logprob(const float* logits, int ld, int rows, int64_t row0, int V, int B, int T, int U1, const int32_t* t_len,
                     const int32_t* u_len, const int32_t* labels, int ldy, float* lp, const int32_t* s_begin, int S, void* stream) {
    if ((rows > 0 && !logits) || !labels || !lp) return fail("otb_rnnt_logprob", "null operand");
    if (const char* e = rnnt_lattice_check(B, T, U1, t_len, u_len, 0, 0)) return fail("otb_rnnt_logprob", e);
    if (row0 < 0 || rows < 0 || row0 + rows > rnnt_rows(B, T, U1, s_begin, S)) return fail("otb_rnnt_logprob", "rows outside the lattice");
    RET("otb_rnnt_logprob", rnnt_logprob_launch(ST(stream), logits, ld, rows, (long long)row0, V, T, U1, t_len, u_len, labels, ldy,
                                                s_begin, S, lp));
}

int otb_rnnt_loss(const float* lp, int B, int T, int U1, const int32_t* t_len, const int32_t* u_len, double* alpha, float* nll,
                  float* loss, float* grad, float grad_scale, const float* grad_scale_dev, const int32_t* s_begin, int S, void* stream) {
    if (!lp || !alpha || !nll || !loss || !grad) return fail("otb_rnnt_loss", "null operand");
    if (const char* e = rnnt_lattice_check(B, T, U1, t_len, u_len, 0, 0)) return fail("otb_rnnt_loss", e);
    RET("otb_rnnt_loss", rnnt_loss_launch(ST(stream), lp, B, T, U1, t_len, u_len, s_begin, S, alpha, nll, loss, grad, grad_scale,
                                          grad_scale_dev));
}

int otb_rnnt_dlogits(const float* logits, int ld, int rows, int64_t row0, int V, int B, int T, int U1, const int32_t* t_len,
                     const int32_t* u_len, const int32_t* labels, int ldy, const float* lp, const float* grad, void* dz, int ldd,
                     const int32_t* s_begin, int S, void* stream) {
    if ((rows > 0 && !logits) || !labels || !lp || !grad || !dz) return fail("otb_rnnt_dlogits", "null operand");
    if (const char* e = rnnt_lattice_check(B, T, U1, t_len, u_len, 0, 0)) return fail("otb_rnnt_dlogits", e);
    if (row0 < 0 || rows < 0 || row0 + rows > rnnt_rows(B, T, U1, s_begin, S)) return fail("otb_rnnt_dlogits", "rows outside the lattice");
    RET("otb_rnnt_dlogits", rnnt_dlogits_launch(ST(stream), logits, ld, rows, (long long)row0, V, T, U1, t_len, u_len, labels, ldy, lp,
                                                grad, s_begin, S, reinterpret_cast<bf16*>(dz), ldd));
}

int otb_rnnt_simple_lse(const float* am, int lda, const float* lm, int ldl, int V, int B, int T, int U1, const int32_t* t_len,
                        const int32_t* u_len, const int32_t* labels, int ldy, float* lp, float* m_am, float* m_lm, void* stream) {
    if (!am || !lm || !labels || !lp || !m_am || !m_lm) return fail("otb_rnnt_simple_lse", "null operand");
    if (const char* e = rnnt_lattice_check(B, T, U1, t_len, u_len, 0, 0)) return fail("otb_rnnt_simple_lse", e);
    RET("otb_rnnt_simple_lse", rnnt_simple_lse_launch(ST(stream), am, lda, lm, ldl, V, B, T, U1, t_len, u_len, labels, ldy, lp, m_am,
                                                      m_lm));
}

int otb_rnnt_simple_bwd(const float* am, int lda, const float* lm, int ldl, int V, int B, int T, int U1, const int32_t* t_len,
                        const int32_t* u_len, const int32_t* labels, int ldy, const float* lp, const float* m_am, const float* m_lm,
                        const float* grad, float scale, const float* scale_dev, void* d_am, void* d_lm, int ldd, void* stream) {
    if (!am || !lm || !labels || !lp || !m_am || !m_lm || !grad || !d_am || !d_lm) return fail("otb_rnnt_simple_bwd", "null operand");
    if (const char* e = rnnt_lattice_check(B, T, U1, t_len, u_len, 0, 0)) return fail("otb_rnnt_simple_bwd", e);
    RET("otb_rnnt_simple_bwd", rnnt_simple_bwd_launch(ST(stream), am, lda, lm, ldl, V, B, T, U1, t_len, u_len, labels, ldy, lp, m_am,
                                                      m_lm, grad, scale, scale_dev, reinterpret_cast<bf16*>(d_am),
                                                      reinterpret_cast<bf16*>(d_lm), ldd));
}

int otb_rnnt_prune_ranges(const float* grad, int B, int T, int U1, const int32_t* t_len, const int32_t* u_len, int S, int32_t* s_begin,
                          void* stream) {
    if (!grad || !s_begin) return fail("otb_rnnt_prune_ranges", "null operand");
    if (const char* e = rnnt_lattice_check(B, T, U1, t_len, u_len, 0, 0)) return fail("otb_rnnt_prune_ranges", e);
    RET("otb_rnnt_prune_ranges", rnnt_prune_ranges_launch(ST(stream), grad, B, T, U1, t_len, u_len, S, s_begin));
}

int otb_rnnt_greedy_step(const int32_t* idx, const float* logp, int ldlp, const float* h_new, const float* c_new, const void* pp_new,
                         float* h, float* c, void* pp, int layers, int B, int H, int D, const void* ep, int T, void* ep_cur,
                         const int32_t* t_len, int32_t* frame, int32_t* n_sym, int32_t* n_out, int32_t* ids, int max_len,
                         int max_sym, float* score, int32_t* active, const float* val, int32_t* emit, int32_t* lm_pos,
                         void* stream) {
    if (!idx || !logp || !h_new || !c_new || !pp_new || !h || !c || !pp || !ep || !ep_cur || !t_len || !frame || !n_sym || !n_out ||
        !ids || !score || !active)
        return fail("otb_rnnt_greedy_step", "null operand");
    RET("otb_rnnt_greedy_step",
        rnnt_greedy_step_launch(ST(stream), idx, logp, ldlp, h_new, c_new, reinterpret_cast<const bf16*>(pp_new), h, c,
                                reinterpret_cast<bf16*>(pp), layers, B, H, D, reinterpret_cast<const bf16*>(ep), T,
                                reinterpret_cast<bf16*>(ep_cur), t_len, frame, n_sym, n_out, ids, max_len, max_sym, score, active, val,
                                emit, lm_pos));
}

int otb_rnnt_beam_step(const float* logp, int ldlp, const float* val, const int32_t* idx, int k1, int B, int K, int W, int V, int T,
                       int max_len, const int32_t* t_len, float* score, int32_t* slot_u, int32_t* frame, int32_t* node, int32_t* par,
                       int64_t* tok, int32_t* node_par, int32_t* node_tok, int n_cap, int32_t* n_nodes, float* f_score,
                       int32_t* f_node, int32_t* f_u, int32_t* f_n, int32_t* done, int32_t* active, int32_t* ids, int32_t* lengths,
                       float* out_score, float beta, int32_t* lm_src, int32_t* lm_ext, int32_t* anc, int32_t* anc_tmp, int32_t* lm_pos,
                       int Lpos, void* stream) {
    if (!logp || !val || !idx || !t_len || !score || !slot_u || !frame || !node || !par || !tok || !node_par || !node_tok ||
        !n_nodes || !f_score || !f_node || !f_u || !f_n || !done || !active || !ids || !lengths || !out_score)
        return fail("otb_rnnt_beam_step", "null operand");
    RET("otb_rnnt_beam_step",
        rnnt_beam_step_launch(ST(stream), logp, ldlp, val, idx, k1, B, K, W, V, T, max_len, t_len, score, slot_u, frame, node, par,
                              reinterpret_cast<long long*>(tok), node_par, node_tok, n_cap, n_nodes, f_score, f_node, f_u, f_n, done,
                              active, ids, lengths, out_score, beta, lm_src, lm_ext, anc, anc_tmp, lm_pos, Lpos));
}

int otb_rnnt_beam_gather(const int32_t* par, const int32_t* frame, int B, int K, int layers, int H, int D, int T, const float* h,
                         const float* c, const void* pp, const void* ep, float* hg, float* cg, void* ppg, void* ep_cur, void* stream) {
    if (!par || !frame || !h || !c || !pp || !ep || !hg || !cg || !ppg || !ep_cur) return fail("otb_rnnt_beam_gather", "null operand");
    RET("otb_rnnt_beam_gather",
        rnnt_beam_gather_launch(ST(stream), par, frame, B, K, layers, H, D, T, h, c, reinterpret_cast<const bf16*>(pp),
                                reinterpret_cast<const bf16*>(ep), hg, cg, reinterpret_cast<bf16*>(ppg), reinterpret_cast<bf16*>(ep_cur)));
}

int otb_rnnt_beam_commit(const int64_t* tok, int rows, int layers, int H, int D, const float* hg, const float* cg, const void* ppg,
                         const float* hn, const float* cn, const void* ppn, float* h, float* c, void* pp, void* stream) {
    if (!tok || !hg || !cg || !ppg || !hn || !cn || !ppn || !h || !c || !pp) return fail("otb_rnnt_beam_commit", "null operand");
    RET("otb_rnnt_beam_commit",
        rnnt_beam_commit_launch(ST(stream), reinterpret_cast<const long long*>(tok), rows, layers, H, D, hg, cg,
                                reinterpret_cast<const bf16*>(ppg), hn, cn, reinterpret_cast<const bf16*>(ppn), h, c,
                                reinterpret_cast<bf16*>(pp)));
}

int otb_nbest_rescore(const int32_t* tgt, int Lp, const int32_t* len, const float* s1, const float* tok_lp, int M, int B, int K,
                      float weight, int nbest, int Lout, int64_t pad_id, int64_t* ids, int32_t* out_len, float* out_score,
                      void* stream) {
    if (!tgt || !len || !s1 || (M > 0 && !tok_lp) || !ids || !out_len || !out_score) return fail("otb_nbest_rescore", "null operand");
    RET("otb_nbest_rescore", nbest_rescore_launch(ST(stream), tgt, Lp, len, s1, tok_lp, M, B, K, weight, nbest, Lout, (long long)pad_id,
                                                  reinterpret_cast<long long*>(ids), out_len, out_score));
}

int otb_edit_distance(const int32_t* hyp, int ldh, const int32_t* hyp_len, const int32_t* ref, int ldr, const int32_t* ref_len, int N,
                      int K, int max_hyp, int max_ref, int32_t* out, void* stream) {
    if (N > 0 && (!hyp || !hyp_len || !ref || !ref_len || !out)) return fail("otb_edit_distance", "null operand");
    RET("otb_edit_distance", edit_distance_launch(ST(stream), hyp, ldh, hyp_len, ref, ldr, ref_len, N, K, max_hyp, max_ref, out));
}

int otb_mwer_coeff(const int32_t* len, const int32_t* err, const float* tok_lp, int Lp, const int32_t* tgt, int B, int K, float scale,
                   const float* scale_dev, float* coeff, float* loss, void* stream) {
    if (!len || !err || !tok_lp || !tgt || !coeff || !loss) return fail("otb_mwer_coeff", "null operand");
    RET("otb_mwer_coeff", mwer_coeff_launch(ST(stream), len, err, tok_lp, Lp, tgt, B, K, scale, scale_dev, coeff, loss));
}

int otb_mwer_sample_coeff(const int32_t* err, int B, int K, float scale, const float* scale_dev, float* coeff, float* loss,
                          void* stream) {
    if (!err || !coeff || !loss) return fail("otb_mwer_sample_coeff", "null operand");
    RET("otb_mwer_sample_coeff", mwer_sample_coeff_launch(ST(stream), err, B, K, scale, scale_dev, coeff, loss));
}

int otb_mwer_grad(const float* logits, int ld, int rows, int V, const int32_t* target, const float* tok_lp, const float* coeff, int Lp,
                  void* dlogits, void* stream) {
    if (rows > 0 && (!logits || !target || !tok_lp || !coeff || !dlogits)) return fail("otb_mwer_grad", "null operand");
    RET("otb_mwer_grad", mwer_grad_launch(ST(stream), logits, ld, rows, V, target, tok_lp, coeff, Lp, reinterpret_cast<bf16*>(dlogits)));
}

int otb_conv_im2col(const void* h1, void* col, int B, int T, int F, int C1, CONV_GEOM, void* stream) {
    ConvGeom g;
    if (const char* e = conv_geometry(T, F, CONV_ARGS, &g)) return fail("otb_conv_im2col", e);
    if (!h1 || !col) return fail("otb_conv_im2col", "null operand");
    RET("otb_conv_im2col", im2col_launch(ST(stream), reinterpret_cast<const bf16*>(h1), reinterpret_cast<bf16*>(col), B, g, C1));
}

int otb_conv_col2im_relu(const void* dcol, const void* h1, void* dpre1, int B, int T, int F, int C1, CONV_GEOM, void* stream) {
    ConvGeom g;
    if (const char* e = conv_geometry(T, F, CONV_ARGS, &g)) return fail("otb_conv_col2im_relu", e);
    if (!dcol || !h1 || !dpre1) return fail("otb_conv_col2im_relu", "null operand");
    RET("otb_conv_col2im_relu", col2im_relu_launch(ST(stream), reinterpret_cast<const bf16*>(dcol), reinterpret_cast<const bf16*>(h1),
                                                   reinterpret_cast<bf16*>(dpre1), B, g, C1));
}

int otb_conv1_wgrad(const void* dpre1, const float* x, float* out, int B, int T, int F, int C1, CONV_GEOM, void* stream) {
    ConvGeom g;
    if (const char* e = conv_geometry(T, F, CONV_ARGS, &g)) return fail("otb_conv1_wgrad", e);
    if (!dpre1 || !x || !out) return fail("otb_conv1_wgrad", "null operand");
    RET("otb_conv1_wgrad", conv1_wgrad_launch(ST(stream), reinterpret_cast<const bf16*>(dpre1), x, out, B, T, F, g, C1));
}

int otb_spec_augment(float* x, const int32_t* bands, int B, int T, int F, int n_freq, int n_time, void* stream) {
    if (!x || !bands || B < 1 || T < 1 || F < 1 || n_freq < 0 || n_time < 0) return fail("otb_spec_augment", "bad arguments");
    RET("otb_spec_augment", spec_augment_launch(ST(stream), x, bands, B, T, F, n_freq, n_time));
}

int otb_lstm_config(int H, int sms, int smem_optin, int* units, int* smem_fwd, int* smem_bwd) {
    LstmPlan pl;
    if (const char* e = lstm_plan(H, sms, smem_optin, &pl)) return fail("otb_lstm_config", e);
    if (units) *units = pl.units;
    if (smem_fwd) *smem_fwd = (int)pl.smem_fwd;
    if (smem_bwd) *smem_bwd = (int)pl.smem_bwd;
    return 0;
}

int otb_lstm_fwd(const float* gx, const void* w_hh, const float* h0, const float* c0, void* y, float* h_n, float* c_n, float* gates,
                 float* c_all, uint32_t* barrier, int L, int B, int H, void* stream) {
    if (!gx || !w_hh || !y || !h_n || !c_n || !barrier) return fail("otb_lstm_fwd", "null operand");
    if ((gates == nullptr) != (c_all == nullptr)) return fail("otb_lstm_fwd", "gates and c_all are recorded together");
    RET("otb_lstm_fwd", lstm_fwd_launch(ST(stream), gx, reinterpret_cast<const bf16*>(w_hh), h0, c0, reinterpret_cast<bf16*>(y), h_n,
                                        c_n, gates, c_all, barrier, L, B, H));
}

int otb_lstm_bwd(const void* dy, const void* w_hh, const float* gates, const float* c_all, const float* c0, void* dg, float* dc,
                 uint32_t* barrier, int L, int B, int H, void* stream) {
    if (!dy || !w_hh || !gates || !c_all || !dg || !dc || !barrier) return fail("otb_lstm_bwd", "null operand");
    RET("otb_lstm_bwd", lstm_bwd_launch(ST(stream), reinterpret_cast<const bf16*>(dy), reinterpret_cast<const bf16*>(w_hh), gates, c_all,
                                        c0, reinterpret_cast<bf16*>(dg), dc, barrier, L, B, H));
}

int otb_embedding(const int64_t* tok, const void* emb, void* out, int N, int d, int vocab, void* stream) {
    if (!tok || !emb || !out || N < 1 || vocab < 1) return fail("otb_embedding", "bad arguments");
    RET("otb_embedding", embedding_launch(ST(stream), reinterpret_cast<const long long*>(tok), reinterpret_cast<const bf16*>(emb),
                                          reinterpret_cast<bf16*>(out), N, d, vocab));
}

}  // extern "C"
