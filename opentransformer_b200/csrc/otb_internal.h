// Internal declarations shared by the .cu translation units of libotb200.so.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/otb200.h"

namespace otb {

typedef __nv_bfloat16 bf16;

// ---- epilogues of the wgmma GEMM (C = A[M,K] * W[N,K]^T, fp32 accumulate in registers) ----
enum Epilogue : int {
    EPI_BIAS = 0,      // out = acc + bias
    EPI_RELU = 1,      // out = relu(acc + bias)
    EPI_GLU = 2,       // W has 2*Nh rows; out[:, j] = (acc_j + b_j) * sigmoid(acc_{Nh+j} + b_{Nh+j})
    EPI_TABLE = 3,     // out = (acc + bias) * alpha + table[(row % period) * N + col]     (x*sqrt(d)+PE)
    EPI_RESID = 4,     // out = resid + alpha * (acc + bias)
    EPI_RESID_LN = 5,  // out = LayerNorm(resid + acc + bias) * gamma + beta   (tile spans the whole row)
    EPI_SWISH = 6,     // out = v * sigmoid(v), v = acc + bias
    EPI_GELU = 7,      // out = gelu(v) (erf form, as F.gelu)
    EPI_TANH = 8,      // out = tanh(v)
    // internal (not an otb_linear epilogue): EPI_RESID with two independent dropout masks on (acc + bias), the
    // attention's output dropout under the residual dropout (otb_linear_dropout_resid with both rates non-zero)
    EPI_RESID_DROP2 = 9,
};

struct GemmParams {
    int M, N, K;  // N = number of output columns (for GLU: Nh); K multiple of 8
    const float* bias;
    void* out;
    int ldc;
    int out_f32;
    const bf16* resid;
    int ldr;
    const float* gamma;
    const float* beta;
    float eps;
    float alpha;
    const float* table;
    int period;
    const int* row_len;  // optional: rows with (m % row_period) >= row_len[m / row_period] produce 0 (before resid)
    int row_period;
    // implicit-GEMM convolution mode (A operand gathered by a 5-D TMA map, one k-block = one tap of 64 channels)
    int conv;
    int conv_F2;       // output frequency bins
    int conv_R;        // output time rows per M tile (R * F2 <= 128)
    int conv_T1h;      // input time rows per utterance / time stride (ConvGeom::T1s)
    int conv_T2;       // valid output time rows per utterance
    int conv_B;        // batch
    int conv_cchunks;  // C_in / 64
    // per tap (kh, kw) of conv2: bytes {f stride phase, f offset + 8, t stride phase, t offset}, computed on the host
    // (integer division by run-time strides in the TMA producer cost the shipped conv2 a third of its time on H100)
    unsigned conv_tap[49];
    int splitk;        // TN (weight-gradient) mode: number of contraction splits (fp32 atomics when > 1)
    int accum;         // TN mode: add into `out` instead of overwriting it
    // training-mode dropout of the projection BEFORE the residual add (EPI_RESID only): out = resid + alpha * keep * (.) / (1-p)
    const unsigned* drop_seed;    // device scalar, null = no dropout
    unsigned drop_site, drop_thresh;
    float drop_scale;             // EPI_RESID_DROP2: 1 / ((1 - p) (1 - p2))
    unsigned drop_site2, drop_thresh2;   // EPI_RESID_DROP2 only: the second mask
};

const char* gemm_launch(cudaStream_t st, const void* A, int lda, const void* W, int ldw, int w_rows, int epi,
                        GemmParams p, const CUtensorMap* conv_map);
// shape / epilogue checks of gemm_launch and the tile width it picks for m_tiles 128-row blocks (host only)
const char* gemm_tile(int m_tiles, int N, int epi, int out_f32, int* bn);

const char* gemm_wgrad_launch(cudaStream_t st, const void* dY, int lddy, const void* X, int ldx, float* out, int ldc,
                              int Mact, int Nw, int Kw, int accumulate);

// encode helpers (driver entry point fetched at runtime; libcuda is not a link-time dependency)
const char* encode_tmap_2d(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint64_t ld_elems,
                           uint32_t box_cols, uint32_t box_rows);
const char* encode_tmap_2d_f32(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint64_t ld_elems,
                               uint32_t box_cols, uint32_t box_rows);
const char* encode_tmap_conv5d(CUtensorMap* m, const void* base, int C, int sf, int F1s, int st, int T1s_total, uint32_t boxF,
                               uint32_t boxR);

// Two-layer Conv2d front end (frontend/conv.py:15-48,86-129): layer i has kernel (kt, kf), stride (st, sf) and padding
// (0, kf / 2).  conv1's output buffer is NHWC bf16 [B, st2 * T1s, sf2 * F1s, C1]: conv2 reads it through the 5-D view
// (c, f mod sf2, f / sf2, t mod st2, b * T1s + t / st2), and columns F1 .. sf2 * F1s - 1 are written as zero (the right
// frequency padding of conv2).
struct ConvGeom {
    int kt1, kf1, st1, sf1, kt2, kf2, st2, sf2;
    int T1, F1, T2, F2;
    int T1s, F1s;
};

struct AttnParams {
    int B, H, Tq, Tk;
    const int* kv_len;  // [B] or null
    int causal;
    float scale_log2;   // (1/sqrt(dk)) * log2(e)
    bf16* out;
    int ldo;
    int q_col0, k_col0, v_col0;
    const float* bd;    // optional relative-position scores, [H,B,Tq,ldbd]; bias(i,j) = bd[h,b,i, j - i + Tq - 1]
    int ldbd;
    const bf16* resid;  // optional: out = resid + softmax(..)V   (rel-pos attention has no output projection)
    int ldr;
    float* lse;         // optional [B,H,Tq]: row log-sum-exp of the scaled scores in log2 units (saved for the backward)
};

struct AttnBwdParams {
    int B, H, Tq, Tk;
    const int* kv_len;
    int causal;
    float scale_log2;
    int q_col0, k_col0, v_col0;
    const bf16* o;      // forward output [B*Tq, ldo]
    int ldo;
    const bf16* dout;   // gradient of the forward output [B*Tq, lddo]
    int lddo;
    const float* lse;   // [B,H,Tq] from the forward
    float* dsum;        // [B,H,Tq] scratch: D_i = dO_i . O_i (written by the dQ kernel, read by the dK/dV kernel)
    bf16* dq; int lddq, dq_col0;
    bf16* dk; int lddk, dk_col0;
    bf16* dv; int lddv, dv_col0;
    const float* bd;    // optional rel-pos band of the forward (AttnParams::bd, Tq == Tk), null for plain attention
    int ldbd;
    bf16* dbd;          // with bd: its gradient [H,B,Tq,lddbd], zeroed by the caller; dS(i,j) lands at column j - i + Tq - 1
    int lddbd;
};
const char* attn_bwd_launch(cudaStream_t st, const void* q, int ldq, int q_rows, const void* k, int ldk, int k_rows,
                            const void* v, int ldv, const AttnBwdParams& p);
const char* colsum_launch(cudaStream_t st, const bf16* x, int ldx, float* out, int M, int N, int accumulate);
const char* layernorm_bwd_launch(cudaStream_t st, const bf16* dy, int lddy, const bf16* z, int ldz, const float* gamma,
                                 bf16* dz, int lddz, float* dgamma, float* dbeta, float eps, int M, int N, int accumulate);
const char* glu_launch(cudaStream_t st, const bf16* u, const bf16* dh, bf16* out, int M, int F);
const char* relu_bwd_launch(cudaStream_t st, const bf16* dy, const bf16* y, bf16* dx, size_t n);
const char* dropout_bwd_launch(cudaStream_t st, const bf16* dy, int lddy, bf16* out, int ldo, unsigned char* mask, int M, int N, float p,
                               const unsigned* seed, unsigned site, float p2, unsigned site2);
const char* act_launch(cudaStream_t st, int act, const bf16* u, const bf16* dh, bf16* out, size_t n);
const char* embed_bwd_launch(cudaStream_t st, const long long* tok, const bf16* dx, float* dE, int N, int d, int vocab, float scale);
const char* im2col_launch(cudaStream_t st, const bf16* h1, bf16* col, int B, const ConvGeom& g, int C);
const char* col2im_relu_launch(cudaStream_t st, const bf16* dcol, const bf16* h1, bf16* dpre1, int B, const ConvGeom& g, int C);
const char* conv1_wgrad_launch(cudaStream_t st, const bf16* dpre1, const float* x, float* out, int B, int T, int F,
                               const ConvGeom& g, int C);
const char* spec_augment_launch(cudaStream_t st, float* x, const int* bands, int B, int T, int F, int nf, int nt);
const char* sumsq_launch(cudaStream_t st, const float* g, size_t n, float* out, int zero_first);
const char* adam_sched_launch(cudaStream_t st, float* p, const float* g, float* m, float* v, size_t n, const float* sumsq,
                              float max_norm, float base_lr, float model_size, float warmup, float factor, float b1, float b2,
                              float eps, float wd, int* counters, float* hyper, float noise, const int* noise_seed,
                              const uint8_t* noise_mask);
const char* mixspeech_launch(cudaStream_t st, const float* x, const uint8_t* mask, int B, int T, int F, const int* seed, const int* step,
                             float scale, float* lam_out, float* x_out, uint8_t* mask_out);
const char* frame_stack_launch(cudaStream_t st, const float* x, int B, int T, int F, int n, int s, int T2, bf16* out, int ldo,
                               float alpha, const float* table);

struct BeamState {
    int* tok_hist;
    int* par_hist;
    long long* last_tok;
    float* scores;
    unsigned char* flag;
    int* anc;
    int* ctrl;
    int N, beam, Lmax;
};

// ---- persistent decode kernel (decode_group.cu): row groups of <= 128 hypotheses x 16 CTAs, wgmma GEMMs.  The model is
// the public otb_mega_model; the launch checks that the kernel supports it.
extern unsigned long long* g_dg_dbg;
extern int g_dg_dbg_step;
extern int g_dg_barrier;
size_t decode_group_workspace_bytes(int N, int n_layers, int Lmax, int B, int beam, int V);
const char* decode_group_launch(cudaStream_t st, const otb_mega_model& m, const bf16* kvx, const int* mem_len, bf16* kc,
                                bf16* vc, const BeamState& bs, int B, int T, int max_steps, float* dbg_logp,
                                float* dbg_scores, void* workspace, size_t workspace_bytes);

// d_k: head width, 64 or 96 (head h starts at column col0 + d_k * h)
const char* attn_launch(cudaStream_t st, const void* q, int ldq, int q_rows, const void* k, int ldk, int k_rows,
                        const void* v, int ldv, const AttnParams& p, int d_k);
// attention weights (attn_probs.cu): the score operands of attn_launch, P written as f32 [B, H, Tq, Tk]
struct AttnProbsParams {
    int B, H, Tq, Tk;
    const int* kv_len;  // [B] or null
    int causal;
    float scale_log2;   // (1/sqrt(dk)) * log2(e)
    int q_col0, k_col0;
    const float* bd;    // optional rel-pos band as AttnParams::bd (Tq == Tk, not causal)
    int ldbd;
    float* out;         // [B, H, Tq, Tk], row pitch Tk
};
const char* attn_probs_launch(cudaStream_t st, const void* q, int ldq, int q_rows, const void* k, int ldk, int k_rows,
                              const AttnProbsParams& p, int d_k);
const char* conv1_launch(cudaStream_t st, const float* x, const float* w, const float* bias, bf16* out, int B, int T,
                         int F, const ConvGeom& g, int C1);
const char* layernorm_launch(cudaStream_t st, const bf16* x, int ldx, void* out, int ldo, int out_f32, const float* g1,
                             const float* b1, const float* g2, const float* b2, float eps, int M, int N);
const char* scale_add_table_launch(cudaStream_t st, const void* x, int ldx, int x_f32, bf16* out, int ldo, float alpha,
                                   const float* table, int period, int M, int N, const float* alpha_dev);
// Conformer convolution module in training mode (conformer_train.cu)
const char* conv_bn_train_launch(cudaStream_t st, const bf16* x, const int* len, const float* w, const float* wb, const float* gamma,
                                 const float* beta, float* run_mean, float* run_var, long long* n_batches, float momentum, float eps,
                                 float* c, float* stats, bf16* out, int B, int T, int d, int k);
const char* conv_bn_bwd_launch(cudaStream_t st, const bf16* dy, const bf16* x, const int* len, const float* w, const float* gamma,
                               const float* beta, const float* c, const float* stats, float* red, float* dc, bf16* dx, float* dw,
                               float* dwb, float* dgamma, float* dbeta, int accumulate, int B, int T, int d, int k);
const char* dropout_add_launch(cudaStream_t st, const bf16* x, int ldx, const bf16* resid, int ldr, bf16* out, int ldo, int M, int N,
                               float alpha, float p, const unsigned* seed, unsigned site, const int* row_len, int row_period);
const char* dwconv_swish_launch(cudaStream_t st, const bf16* x, const float* w, const float* b, bf16* out, int B, int T,
                                int d, int k);
const char* sinusoid_table_launch(cudaStream_t st, float* out, int n_pos, int d, int first_pos);
const char* embed_posenc_launch(cudaStream_t st, const long long* tok, int tok_stride, const bf16* emb,
                                const float* table, bf16* out, int N, int d, int period, const int* step_ptr,
                                int vocab, const int* row_pos = nullptr);
const char* log_softmax_launch(cudaStream_t st, const float* x, int ldx, float* out, int ldo, int rows, int V);
const char* decode_self_attn_launch(cudaStream_t st, const bf16* qkv, bf16* kc, bf16* vc, const int* anc,
                                    const int* step_ptr, bf16* out, int N, int H, int Lmax, int d_k, const int* row_pos = nullptr);
const char* beam_init_launch(cudaStream_t stream, BeamState st);
const char* beam_step_launch(cudaStream_t stream, const float* logp, int ldl, int V, const float* lm_logp, int ld_lm,
                             float lm_weight, BeamState st, long long* dbg_ktok, int* dbg_offs, const float* pre_val,
                             const int* pre_idx);
const char* logsoftmax_topk_launch(cudaStream_t stream, const float* logits, int ldl, int V, const float* lm_logp,
                                   int ld_lm, float lm_weight, float lm_beta, int lm_exempt, int k, int rows, float* out_val,
                                   int* out_idx, float* out_logp, int ld_logp);
const char* sample_step_launch(cudaStream_t stream, const float* logits, int ldl, int V, BeamState st, const int* seed);
const char* beam_reconstruct_launch(cudaStream_t stream, BeamState st, long long* preds, int ld, int steps);
const char* beam_finalize_launch(cudaStream_t stream, BeamState st, float penalty, float lamda, int nbest,
                                 long long* out_preds, float* out_scores);

const char* ls_ce_launch(cudaStream_t st, const float* logits, int ldl, const long long* tgt, int rows, int V, float eps,
                         int pad_id, float* tok_loss, float* loss, int* n_valid, float* dlogits, int ldd,
                         bf16* dlogits_bf16 = nullptr);

const char* ctc_launch(cudaStream_t st, const float* logp, int ldl, int B, int T, int V, const int* in_len, const long long* targets,
                       int ldt, const int* tgt_len, int max_tgt, int blank, float* nll, float* loss, float* ws, bf16* dlogits, int ldd,
                       float grad_scale, const float* scale_dev);
const char* ctc_frame_topk_launch(cudaStream_t st, const float* logits, int ld, int B, int T, int V, const int* in_len, int K,
                                  float* top_lp, int* top_id);
const char* ctc_greedy_launch(cudaStream_t st, const float* top_lp, const int* top_id, int ldk, int B, int T, const int* in_len,
                              int blank, int* ids, int* lengths, float* scores);
// One frame of the LM-fused CTC prefix beam search (ctc_prefix_beam_step_kernel, DESIGN.md 4.19).
static constexpr int CTC_LM_BOS = 1;          // <S/E>: the LM's first input, and the token of a row with an empty prefix
struct CtcStepArgs {
    const float* top_lp;
    const int* top_id;
    int K, T;
    const int* in_len;
    int blank, beam;
    const float* lm;          // f32 [B*beam, ld_lm]: row b*beam + i = log p_lm(. | BOS, prefix of slot i)
    int ld_lm;
    float lm_w, beta;
    void* slots;              // [2, B] slot states (ctc_prefix_beam_slots_bytes)
    int* ctl;                 // [2]: frame counter, arrival counter (both 0 before frame 0)
    int* nodes;               // i32 [B, 1 + T*beam, 2]
    int* src;                 // [B*beam] source row of each new slot
    long long* tok;           // [B*beam] the LM input of each row: its newest token (BOS for the empty prefix)
    int* ext;                 // [B*beam] 1 where the new slot extended its source
    int* anc;                 // Transformer LM or null: i32 [B*beam, Lpos] cache rows of each slot's prefix
    int* anc_tmp;             // i32 [B*beam, Lpos] scratch
    int* pos;                 // [B*beam] query position of each row, -1: nothing to compute
    int Lpos;
    int* ids;                 // written at the last frame: i32 [B, beam, T], lengths i32 [B, beam], scores f32 [B, beam]
    int* lengths;
    float* scores;
};
const char* ctc_prefix_beam_step_launch(cudaStream_t st, const CtcStepArgs& a, int B);
int ctc_prefix_beam_slots_bytes(int B);
const char* ctc_lm_carry_launch(cudaStream_t st, void* dst, int ldd, const void* a, int lda, const void* b, int ldb, const int* idx,
                                const int* ext, int rows, int width);
const char* ctc_prefix_beam_launch(cudaStream_t st, const float* top_lp, const int* top_id, int K, int B, int T, const int* in_len,
                                   int blank, int beam, int* nodes, int* ids, int* lengths, float* scores);
const char* ctc_align_launch(cudaStream_t st, const float* rows, int ld, int B, int T, int V, const float* lse, const int* in_len,
                             const long long* targets, int ldt, const int* tgt_len, int max_tgt, int blank, uint8_t* bp, int* labels,
                             float* frame_scores, int* spans, float* path_score);

const char* ctc_prefix_init_launch(cudaStream_t stream, const float* lp, int ld, int B, int T, const int* in_len, int blank,
                                   int beam, float* gamma, float* psi);
const char* ctc_prefix_score_launch(cudaStream_t stream, const float* lp, int ld, int T, int V, const int* in_len, int blank,
                                    const float* gamma, const float* psi, const float* cand_val, const int* cand_id, int P,
                                    const float* lm_logp, int ld_lm, float lm_weight, float ctc_weight, BeamState st,
                                    float* gamma_cand, float* psi_cand, float* out_val, int* out_idx);
const char* ctc_prefix_advance_launch(cudaStream_t stream, BeamState st, const int* cand_id, int P, int T, const int* in_len,
                                      const float* gamma_cand, const float* psi_cand, float* gamma, float* psi);

const char* ctc_nbest_score_launch(cudaStream_t st, const float* logp, int ld, int B, int T, int V, const int* in_len,
                                   const int* targets, int K, int Lp, int blank, float* out);

const char* token_logprob_launch(cudaStream_t stream, const float* logits, int ld, int rows, int V, const int* target, float* out);
const char* nbest_rescore_launch(cudaStream_t stream, const int* tgt, int Lp, const int* len, const float* s1, const float* tok_lp,
                                 int M, int B, int K, float weight, int nbest, int Lout, long long pad_id, long long* ids,
                                 int* out_len, float* out_score);

const char* edit_distance_launch(cudaStream_t stream, const int* hyp, int ldh, const int* hyp_len, const int* ref, int ldr,
                                 const int* ref_len, int N, int K, int max_h, int max_r, int* out);
const char* mwer_coeff_launch(cudaStream_t stream, const int* len, const int* err, const float* tok_lp, int Lp, const int* tgt, int B,
                              int K, float scale, const float* scale_dev, float* coeff, float* loss);
const char* mwer_sample_coeff_launch(cudaStream_t stream, const int* err, int B, int K, float scale, const float* scale_dev,
                                     float* coeff, float* loss);
const char* mwer_grad_launch(cudaStream_t stream, const float* logits, int ld, int rows, int V, const int* target, const float* tok_lp,
                             const float* coeff, int Lp, bf16* dlogits);

const char* fbank_launch(cudaStream_t st, const float* wave, int ld_wave, const int* n_samples, const float* gain, int B,
                         const float* window, const float* bank, const int* bank_range, float* out, int Tmax, int F, int frame_len,
                         int frame_shift, float preemph);
const char* utt_cmvn_launch(cudaStream_t st, float* x, int B, int Tmax, int F, const int* n_frames, const float* gmean, const float* gstd,
                            const float* noise);
const char* resample_launch(cudaStream_t st, const float* x, int ldx, const int* n_in, const int* orig, const int* new_rate, float* y,
                            int ldy, int* n_out, int B, int width);

const char* rnnt_joint_launch(cudaStream_t st, const bf16* ep, const bf16* pp, int B, int T, int U1, int D, const int* t_len,
                              const int* u_len, const int* s_begin, int S, bf16* out);
const char* rnnt_joint_bwd_launch(cudaStream_t st, const bf16* dh, const bf16* h, int B, int T, int U1, int D, const int* t_len,
                                  const int* u_len, const int* s_begin, int S, bf16* dep, bf16* dpp);
const char* rnnt_logprob_launch(cudaStream_t st, const float* logits, int ld, int rows, long long row0, int V, int T, int U1,
                                const int* t_len, const int* u_len, const int* labels, int ldy, const int* s_begin, int S, float* lp);
const char* rnnt_loss_launch(cudaStream_t st, const float* lp, int B, int T, int U1, const int* t_len, const int* u_len,
                             const int* s_begin, int S, double* alpha, float* nll, float* loss, float* grad, float grad_scale,
                             const float* scale_dev);
const char* rnnt_dlogits_launch(cudaStream_t st, const float* logits, int ld, int rows, long long row0, int V, int T, int U1,
                                const int* t_len, const int* u_len, const int* labels, int ldy, const float* lp, const float* grad,
                                const int* s_begin, int S, bf16* dz, int ldd);
const char* rnnt_simple_lse_launch(cudaStream_t st, const float* am, int lda, const float* lm, int ldl, int V, int B, int T, int U1,
                                   const int* t_len, const int* u_len, const int* labels, int ldy, float* lp, float* m_am,
                                   float* m_lm);
const char* rnnt_simple_bwd_launch(cudaStream_t st, const float* am, int lda, const float* lm, int ldl, int V, int B, int T, int U1,
                                   const int* t_len, const int* u_len, const int* labels, int ldy, const float* lp, const float* m_am,
                                   const float* m_lm, const float* grad, float scale, const float* scale_dev, bf16* d_am,
                                   bf16* d_lm, int ldd);
const char* rnnt_prune_ranges_launch(cudaStream_t st, const float* grad, int B, int T, int U1, const int* t_len, const int* u_len,
                                     int S, int* s_begin);
const char* rnnt_greedy_step_launch(cudaStream_t st, const int* idx, const float* logp, int ldlp, const float* h_new,
                                    const float* c_new, const bf16* pp_new, float* h, float* c, bf16* pp, int layers, int B, int H,
                                    int D, const bf16* ep, int T, bf16* ep_cur, const int* t_len, int* frame, int* n_sym, int* n_out,
                                    int* ids, int max_len, int max_sym, float* score, int* active, const float* val, int* emit,
                                    int* lm_pos);
const char* rnnt_beam_step_launch(cudaStream_t st, const float* logp, int ldlp, const float* val, const int* idx, int k1, int B, int K,
                                  int W, int V, int T, int max_len, const int* t_len, float* score, int* slot_u, int* frame, int* node,
                                  int* par, long long* tok, int* node_par, int* node_tok, int n_cap, int* n_nodes, float* f_score,
                                  int* f_node, int* f_u, int* f_n, int* done, int* active, int* ids, int* lengths, float* out_score,
                                  float beta, int* lm_src, int* lm_ext, int* anc, int* anc_tmp, int* lm_pos, int Lpos);
const char* rnnt_beam_gather_launch(cudaStream_t st, const int* par, const int* frame, int B, int K, int layers, int H, int D, int T,
                                    const float* h, const float* c, const bf16* pp, const bf16* ep, float* hg, float* cg, bf16* ppg,
                                    bf16* ep_cur);
const char* rnnt_beam_commit_launch(cudaStream_t st, const long long* tok, int rows, int layers, int H, int D, const float* hg,
                                    const float* cg, const bf16* ppg, const float* hn, const float* cn, const bf16* ppn, float* h,
                                    float* c, bf16* pp);

// LSTM recurrence (lstm.cu): units per CTA, grid and dynamic shared memory of the two persistent kernels for hidden size H
struct LstmPlan {
    int units, grid;
    size_t smem_fwd, smem_bwd;
};
const char* lstm_plan(int H, int sms, int smem_optin, LstmPlan* plan);
const char* lstm_fwd_launch(cudaStream_t st, const float* gx, const bf16* w, const float* h0, const float* c0, bf16* y, float* hn,
                            float* cn, float* gates, float* call, unsigned* bar, int L, int B, int H);
const char* lstm_bwd_launch(cudaStream_t st, const bf16* dy, const bf16* w, const float* gates, const float* call, const float* c0,
                            bf16* dg, float* dc, unsigned* bar, int L, int B, int H);
const char* embedding_launch(cudaStream_t st, const long long* tok, const bf16* emb, bf16* out, int N, int d, int vocab);

int num_sms();
extern int g_tile_policy;
void set_error(const char* msg);

}  // namespace otb
