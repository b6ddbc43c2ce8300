/*
 * libotb200 -- H100 (sm_90a) hot path for the OpenTransformer speech transformer, C ABI.
 *
 * The reference has no FFI / operator API: its boundary is the Python nn.Module surface
 * (SURVEY.md 8b).  Every entry point below therefore names the reference *module method* whose
 * per-call compute it replaces (file:line under the reference tree); the Python classes in
 * opentransformer_b200/ keep the reference's constructor kwargs / state_dict keys and call these
 * functions through ctypes (see INTEGRATION.md for the binding a maintainer would add).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless stated; "bf16" buffers are uint16 bfloat16, row-major
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream)
 *   - functions return 0 on success, non-zero on error; otb_last_error() gives the message
 *     (thread-local).  Nothing aborts; kernels are asynchronous on `stream`.
 *   - the library keeps no global mutable state besides the per-thread error string and lazily
 *     set function attributes, so one thread per GPU (nn.DataParallel, trainer.py:65) is safe.
 */
#ifndef OTB200_H_
#define OTB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OTB_VERSION 4

/* GEMM epilogues (otb_linear) */
enum {
    OTB_EPI_BIAS = 0,     /* y = x W^T + b                                   nn.Linear                          */
    OTB_EPI_RELU = 1,     /* relu(.)                                          ffn.py:16, conv.py:64              */
    OTB_EPI_GLU = 2,      /* W has 2N rows: (a + b_a) * sigmoid(g + b_g)      ffn.py:18 F.glu, conformer.py:45   */
    OTB_EPI_TABLE = 3,    /* (.) * alpha + table[row % period]                pos.py:56  x*sqrt(d)+PE            */
    OTB_EPI_RESID = 4,    /* resid + alpha * (.)                              encoder/conformer.py:53,72         */
    OTB_EPI_RESID_LN = 5, /* LayerNorm(resid + (.)) * gamma + beta            encoder/transformer.py:54-56,61-63 */
    OTB_EPI_SWISH = 6,    /* v * sigmoid(v)                                   ffn.py:20                          */
    OTB_EPI_GELU = 7,     /* F.gelu                                           ffn.py:17                          */
    OTB_EPI_TANH = 8      /* tanh                                             ffn.py:19                          */
};

const char* otb_last_error(void);
int otb_version(void);
int otb_num_sms(void);
/* Tiling policy of small GEMMs (M <= 512 rows, the decode step): 0 (default) = shortest launch -- the tiling with the
 * fewest MMA waves; 1 = least SM-time -- the widest tile on the fewest CTAs, for servers that keep several utterance
 * batches in flight on separate streams.  Process-wide; set it before CUDA graphs are captured. */
int otb_set_tile_policy(int policy);
/* Profiling aid: buf (device, u64 [>= 256]) receives clock64 stamps at every phase boundary of decode step `step`
 * of the next otb_decode_persistent launches (group 0, CTA 0); NULL disables. */
int otb_debug_decode_timing(unsigned long long* buf, int step);
/* Serving knob of otb_decode_persistent (no counterpart in the reference): how the 16 CTAs of a row group synchronise.
 * 1 = thread-block cluster of 16 + barrier.cluster (lowest latency; one cluster per GPC, i.e. at most 8 groups in flight),
 * 0 = plain CTAs + a release/acquire counter in L2 (every SM usable; every CTA of every batch in flight must be resident),
 * -1 = default: clusters when the device grants clusters of 16 (probed once), else the software barrier.  With 1, a launch
 * on a device that refuses clusters of 16 fails instead of falling back to the software barrier.  Process-wide. */
int otb_set_decode_barrier(int kind);

/* The two-layer conv front end (frontend/conv.py:10-11,15-48,50-76,131-153).  Every conv entry point takes its geometry as
 * eight ints kt1, kf1, st1, sf1, kt2, kf2, st2, sf2: layer i has kernel (kt_i, kf_i), stride (st_i, sf_i) and padding
 * (0, kf_i / 2), so per axis n' = (n + 2 p - k) / s + 1.  Kernel sizes 1..7 and strides 1..4; an input with fewer than one
 * output frame is refused.  The shipped front end is 3, 3, 2, 2, 3, 3, 2, 2 (two 3x3 convolutions at stride 2).
 *
 * Conv2dLayer output geometry, host only: out (may be NULL) receives {T1, F1, T2, F2, T1p, F1p}: the conv1 activation
 * buffer is NHWC bf16 [B, T1p, F1p, C1] (T1p a multiple of st2, F1p of sf2; conv2 reads it per stride phase). */
int otb_conv_geometry(int T, int F, int kt1, int kf1, int st1, int sf1, int kt2, int kf2, int st2, int sf2, int* out);

/* Conv2dLayer.forward #1 (C_in = 1): relu(conv2d(x, w) + b).
 * x f32 [B,T,F]; w f32 [C1,1,kt1,kf1]; bias f32 [C1]; out bf16 NHWC conv1 buffer (otb_conv_geometry), columns F1 ..
 * F1p-1 written as zero.  C1 % 8 == 0, at most 2048 (1024 for kernels wider than 3, 512 wider than 5). */
int otb_conv1_relu(const float* x, const float* w, const float* bias, void* out, int B, int T, int F, int C1, int kt1, int kf1,
                   int st1, int sf1, int kt2, int kf2, int st2, int sf2, void* stream);

/* Conv2dLayer.forward #2 + the transpose/reshape of ConvFrontEnd.forward (frontend/conv.py:63-64,145)
 * as a wgmma implicit GEMM.  in = conv1 buffer; w bf16 [C2, kt2*kf2*C1] with k = (kh*kf2+kw)*C1 + c;
 * out bf16 [B*T2, F2*C2] with feature index f*C2 + c (the caller permutes output_layer.weight columns
 * from the reference's c*F2 + f order once at load time).  C1 % 64 == 0, C2 % 8 == 0, F2 <= 128. */
int otb_conv2_relu(const void* in, const void* w, const float* bias, void* out, int B, int T, int F, int C1, int C2, int kt1,
                   int kf1, int st1, int sf1, int kt2, int kf2, int st2, int sf2, void* stream);

/* nn.Linear with a fused epilogue on wgmma tensor cores: out[M,N] = epi(a[M,K] w[N(,2N),K]^T + bias).
 * a, w bf16 (lda, ldw in elements, multiples of 8); out bf16 or f32 (out_f32; RESID and RESID_LN write bf16 only and
 * refuse out_f32); unused pointers NULL.  Only the [M, N] window of out (row pitch ldc) is written.
 * row_len/row_period: optional key-padding mask (conformer.py:46,55 masked_fill).  A masked row, one with
 * (m % row_period) >= row_len[m / row_period], has its GEMM result and bias replaced by 0 before the epilogue's
 * residual is added: it yields resid for RESID, LayerNorm(resid) * gamma + beta for RESID_LN, and 0 for every other
 * epilogue (TABLE included: a masked row gets 0, not its table row).
 * Replaces attention.py:68,128-129,44; ffn.py:39-41; frontend/conv.py:146; decoder/transformer.py:181. */
int otb_linear(const void* a, int lda, const void* w, int ldw, const float* bias, void* out, int ldc, int M, int N,
               int K, int epilogue, int out_f32, const void* resid, int ldr, const float* gamma, const float* beta,
               float eps, float alpha, const float* table, int period, const int* row_len, int row_period,
               void* stream);
/* Host only, launches nothing: the N tile width (64, 128 or 256) otb_linear would launch for an M x N output with this
 * epilogue and output type under the current tile policy (otb_set_tile_policy), in *bn.  Returns non-zero, with the
 * message otb_linear would give, for the combinations otb_linear refuses whatever its operands. */
int otb_gemm_config(int M, int N, int epilogue, int out_f32, int* bn);

/* Training-mode residual connection with nn.Dropout on the sub-layer output (encoder/transformer.py:32-33,54,61;
 * decoder/transformer.py:36-38 `residual_dropout`): out bf16 = resid + alpha * keep * (a w^T + bias) / (1 - p), where
 * keep(seed, site, row, col) is a counter-based Bernoulli(1-p) mask (csrc/dropout.cuh) -- a pure function of the per-step
 * seed (*seed is read on the DEVICE at run time, so a captured CUDA graph draws a fresh mask per replay), the dropout
 * site id and the element, so the backward replays it instead of storing it.
 * (p2, site2): a second, independent mask on the same tensor -- the attention's own dropout on its projected output
 * (attention.py:46, `slf_attn_dropout` / `src_attn_dropout`) under the residual dropout:
 *   out = resid + alpha * keep(site) * keep2(site2) * (a w^T + bias) / ((1 - p) (1 - p2)).
 * p2 = 0 is exactly the one-mask call; p = 0 < p2 draws site2's mask alone. */
int otb_linear_dropout_resid(const void* a, int lda, const void* w, int ldw, const float* bias, void* out, int ldc, int M, int N,
                             int K, const void* resid, int ldr, float alpha, float p, const uint32_t* seed, uint32_t site,
                             float p2, uint32_t site2, void* stream);
/* Backward of that dropout: out = dy * keep * keep2 / ((1 - p) (1 - p2)) (bf16 [M,N]); mask (optional, u8 [M,N]) receives
 * keep * keep2 -- with dy / out NULL this only exports the mask (parity tests replay it in the oracle). */
int otb_dropout_bwd(const void* dy, int lddy, void* out, int ldo, uint8_t* mask, int M, int N, float p, const uint32_t* seed,
                    uint32_t site, float p2, uint32_t site2, void* stream);

/* Fused masked multi-head attention (attention.py:80,34-41): for batch b, head h
 *   out[b*Tq+i, h*d_k:(h+1)*d_k] = softmax_j((q_i . k_j + bd) / sqrt(d_k), j < kv_len[b], causal: j <= i) V
 * q/k/v are row-major bf16 matrices; batch b owns rows [b*Tq, (b+1)*Tq) of q and [b*Tk, (b+1)*Tk) of k,v;
 * head h starts at column q_col0/k_col0/v_col0 + d_k*h.  d_k is 64 or 96 (96 is the width of the shipped Conformer
 * configuration, d_model 384 / 4 heads); any other value returns non-zero with otb_last_error().
 * bd (optional, f32 [H,B,Tq,ldbd]) holds relative-position scores, bias(i,j) = bd[h,b,i, j-i+Tq-1] (the gather of
 * attention.py:196-215 done by indexing); it needs Tq == Tk, no causal mask and ldbd >= 2 Tq - 1, as otb_attention_bwd
 * and otb_attention_probs do, and is refused otherwise.  resid (optional, bf16 [B*Tq, ldr]) is added to the output (the rel-pos
 * attention of the shipped Conformer has no output projection, SURVEY.md 8a quirks).  lse (optional, f32 [B,H,Tq])
 * receives the per-row log-sum-exp (log2 units) otb_attention_bwd needs; the backward is 64-wide, so lse requires
 * d_k = 64. */
int otb_attention(const void* q, int ldq, int q_rows, const void* k, int ldk, int k_rows, const void* v, int ldv,
                  void* out, int ldo, int B, int H, int Tq, int Tk, const int* kv_len, int causal, int q_col0,
                  int k_col0, int v_col0, const float* bd, int ldbd, const void* resid, int ldr, float* lse, int d_k,
                  void* stream);

/* Attention weights of otb_attention (module/attention.py:34-36): out f32 [B, H, Tq, Tk], contiguous and caller-allocated,
 * = softmax(Q K^T / sqrt(d_k) (+ bd) + mask) over the same q / k operands, column offsets, kv_len, causal flag and band
 * (Tq == Tk, not causal).  Masked entries are exactly 0; every entry of a batch entry with kv_len 0 is NaN.  q_col0,
 * k_col0, ldq and ldk must be multiples of 8; d_k 64 or 96.  No allocation and no host synchronisation. */
int otb_attention_probs(const void* q, int ldq, int q_rows, const void* k, int ldk, int k_rows, float* out, int B, int H,
                        int Tq, int Tk, const int* kv_len, int causal, int q_col0, int k_col0, const float* bd, int ldbd,
                        int d_k, void* stream);

/* ConformerConvolutionModule middle (module/conformer.py:48-52): depthwise Conv1d(k, pad (k-1)/2) over time +
 * eval-mode BatchNorm1d + swish.  x, out bf16 [B*T, d]; w f32 [k, d] and b f32 [d] carry the BatchNorm affine
 * folded in by the caller (w' = w * gamma/sqrt(var+eps), b' = (b - mean) * gamma/sqrt(var+eps) + beta). */
int otb_dwconv_swish(const void* x, const float* w, const float* b, void* out, int B, int T, int d, int k,
                     void* stream);

/* nn.LayerNorm (eps as given), optionally two in a row (encoder/conformer.py:87-89). g2/b2 may be NULL. */
int otb_layernorm(const void* x, int ldx, void* out, int ldo, int out_f32, const float* g1, const float* b1,
                  const float* g2, const float* b2, float eps, int M, int N, void* stream);

/* PositionalEncoding.forward stand-alone (module/pos.py:56): out bf16 = x * alpha + table[row % period];
 * x is f32 (x_f32 != 0) or bf16; table may be NULL (pure scale / dtype conversion).  alpha_dev (may be NULL): a device f32
 * scalar alpha is multiplied by, read on the device (a loss-gradient scale that exists only on the device). */
int otb_scale_add_table(const void* x, int ldx, int x_f32, void* out, int ldo, float alpha, const float* table,
                        int period, int M, int N, const float* alpha_dev, void* stream);

/* PositionalEncoding._embedding_from_positions (module/pos.py:30-42): out f32 [n_pos, d] for positions
 * first_pos .. first_pos + n_pos - 1 (negative allowed). */
int otb_sinusoid_table(float* out, int n_pos, int d, int first_pos, void* stream);

/* embedding + PositionalEncoding.forward (decoder/transformer.py:163,169; pos.py:56):
 * out[n] = emb[tok[n*tok_stride]] * sqrt(d) + table[pos], pos = row_pos ? max(row_pos[n], 0) : step_ptr ? *step_ptr :
 * n % period (row_pos: per-row positions, the LM-fused CTC search; NULL in every other caller). */
int otb_embed_posenc(const int64_t* tok, int tok_stride, const void* emb, const float* table, void* out, int N,
                     int d, int period, const int* step_ptr, const int* row_pos, int vocab, void* stream);

/* F.log_softmax over the last dim, fp32 (decoder/transformer.py:206). */
int otb_log_softmax(const float* x, int ldx, float* out, int ldo, int rows, int V, void* stream);

/* Decode-step self-attention over a per-hypothesis KV cache (the cache API the reference left as a
 * stub, decoder/transformer.py:92-126,188-203): qkv bf16 [N,3d] of the newest token; out bf16 [N,d]; head width d_k 64 or
 * 96 (d = H*d_k).  Give exactly one of step_ptr and row_pos; the other is NULL.  Two cache layouts:
 *   step_ptr (the beam search): *step_ptr = the 0-based position of every row; kc/vc bf16 [Lmax,N,d]; anc i32 [2,N,Lmax].
 *   row_pos (the LM-fused CTC prefix beam search, where slots hold prefixes of different lengths): row n's query is at
 *   position row_pos[n] (-1: the row computes nothing and gets zeros); kc/vc bf16 [cache rows, d]; anc i32 [N, Lmax]
 *   lists the cache row of each position 0..row_pos[n] of row n, and the newest K/V are written to cache row
 *   anc[n][row_pos[n]].
 * Lmax <= 1023; above 128 the prefix is read in chunks of 128 keys with an online softmax.  Shared memory per CTA:
 * min(H, 4) * (min(Lmax rounded up to 32, 128) * d_k * 2 + d_k * 4) bytes. */
int otb_decode_self_attn(const void* qkv, void* kc, void* vc, const int* anc, const int* step_ptr, const int* row_pos, void* out,
                         int N, int H, int Lmax, int d_k, void* stream);

/* LabelSmoothingLoss.forward (module/loss.py:21-48) fused: per-token KL(smoothed one-hot || softmax), PAD rows 0,
 * mean over in-range non-PAD tokens (a target outside [0, V) counts as PAD: loss 0, gradient 0, not in n_valid).
 * logits f32 [rows, ldl]; targets i64 [rows]; tok_loss f32 [rows]; loss f32 [1]; n_valid i32 [1]; dlogits (optional)
 * receives d(mean loss)/dlogits: f32 [rows, ldd] with dlogits_bf16 = 0, or bf16 [rows, ldd] with dlogits_bf16 != 0 for
 * the backward GEMMs (ldd >= V and a multiple of 8, columns [V, ldd) zeroed). */
int otb_ls_ce(const float* logits, int ldl, const int64_t* targets, int rows, int V, float smoothing, int pad_id,
              float* tok_loss, float* loss, int32_t* n_valid, void* dlogits, int ldd, int dlogits_bf16, void* stream);

/* Device-resident beam-search state, N = B*beam hypotheses (all device pointers). */
typedef struct {
    int32_t* tok_hist;  /* [Lmax, N] */
    int32_t* par_hist;  /* [Lmax, N] */
    int64_t* last_tok;  /* [N]       */
    float* scores;      /* [N]       */
    uint8_t* flag;      /* [N]       */
    int32_t* anc;       /* [2, N, Lmax] */
    int32_t* ctrl;      /* [4] = {step, done, ended_now, -} */
    int32_t N, beam, Lmax;
} otb_beam_state;

/* recognize() initial state (recognize/speech2text.py:54-58). */
int otb_beam_init(const otb_beam_state* st, void* stream);
/* SpeechToTextRecognizer.decode_step after the decoder call (recognize/speech2text.py:102-153,156-192).  Give either
 * logp f32 [N, ldl] log-probs, with lm_logp optional (shallow fusion, :102-105), or the per-hypothesis top-k already
 * computed by otb_logsoftmax_topk (k == beam): topk_val f32 / topk_idx i32 [N, beam], with logp NULL and ldl, V, lm_logp,
 * ld_lm, lm_weight unused.  dbg_ktok i64 [N,beam] and dbg_offs i32 [N] (optional) receive last_k_preds / offset_k_indices
 * for parity traces. */
int otb_beam_step(const float* logp, int ldl, int V, const float* lm_logp, int ld_lm, float lm_weight, const float* topk_val,
                  const int32_t* topk_idx, const otb_beam_state* st, int64_t* dbg_ktok, int32_t* dbg_offs, void* stream);
/* Fused log_softmax (+ lm_weight * lm_logp) + per-row top-k (decoder/transformer.py:206 + speech2text.py:102-112):
 * logits f32 [rows, ldl] -> out_val f32 [rows,k] (log-prob values, descending), out_idx i32 [rows,k];
 * out_logp (optional, f32 [rows, ld_logp]) additionally receives the full log-prob rows.  1 <= k <= min(16, V), V <= 49152;
 * ties go to the lower vocabulary id.  lm_exempt < 0 (lm_beta must be 0): as above.  lm_exempt in [0, V) (the transducer's
 * shallow fusion, DESIGN.md 4.22): column lm_exempt keeps its log-prob, every other column i gets
 * + (lm_weight * lm_logp[i] + lm_beta) (+ lm_beta when lm_logp is NULL), and out_logp receives the plain log-probs. */
int otb_logsoftmax_topk(const float* logits, int ldl, int V, const float* lm_logp, int ld_lm, float lm_weight, float lm_beta,
                        int lm_exempt, int k, int rows, float* out_val, int32_t* out_idx, float* out_logp, int ld_logp, void* stream);
/* One step of ancestral sampling from logits f32 [N, ldl] (DESIGN.md 4.11) on the beam state, rows never reordered: every
 * live row n draws token = argmax_{v < V} (logits[n, v] - log(-log u)), ties to the lower id, with
 * u = rng_u01(rng_key(rng_key(rng_key(seed, step), n), v)) (csrc/counter_rng.cuh), step = st->ctrl[0] and seed the int32
 * device scalar *seed; the token is distributed as softmax(logits[n, :V]).  The row adds logits[n, token] -
 * logsumexp(logits[n, :V]) to its score; <S/E> ends it, and an ended row emits <S/E> and keeps its score.  tok_hist,
 * par_hist (= n), anc, last_tok, flag and ctrl move as otb_beam_step moves them.  1 <= V <= 49152, N >= 1. */
int otb_sample_step(const float* logits, int ldl, int V, const otb_beam_state* st, const int32_t* seed, void* stream);
/* Materialise preds i64 [N, ld] (column 0 = BOS) after `steps` steps from the back-pointers. */
int otb_beam_reconstruct(const otb_beam_state* st, int64_t* preds, int ld, int steps, void* stream);
/* Tail of recognize() (recognize/speech2text.py:70-91). out_preds i64 [B,nbest,Lmax], out_scores f32 [B,nbest]. */
int otb_beam_finalize(const otb_beam_state* st, float penalty, float lamda, int nbest, int64_t* out_preds,
                      float* out_scores, void* stream);

/* ---- Persistent decode loop --------------------------------------------------------------------------------
 * The whole loop of SpeechToTextRecognizer.recognize (recognize/speech2text.py:60-68: decode_step :95-153 ->
 * TransformerDecoder.inference, decoder/transformer.py:185-208) for ALL steps in one launch (csrc/decode_group.cu):
 * the hypotheses of up to 128 / beam utterances form one 128-row wgmma tile owned by a group of 16 co-operating CTAs
 * (projections split by output column / contraction slice, weights streamed from L2 by TMA, accumulators in registers,
 * activations exchanged through L2 behind a group-local barrier), search state on the device, no kernel launch or host
 * round trip inside the loop.  Post-norm GLU decoder, d_model 256, 4 heads, d_ff 2048, beam <= 16, T <= 256 memory
 * frames, max_steps <= st->Lmax <= 128, ceil(B / (128 / beam)) * 16 <= number of SMs (other configurations: per-step
 * calls above).  All pointers are device pointers; weights bf16 [N,K] row-major exactly as nn.Linear stores them. */
#define OTB_MEGA_MAX_LAYERS 8
typedef struct {
    const void *wqkv, *wo, *wq, *wo2, *w1, *w2;                 /* slf_attn.qvk_proj, .output_proj, src_attn.q_proj, .output_proj, feed_forward.w_1, .w_2 */
    const float *bqkv, *bo, *bq, *bo2, *b1, *b2;
    const float *g1, *be1, *g2, *be2, *g3, *be3;                /* norm1/2/3 weight, bias */
} otb_mega_layer;
typedef struct {
    int32_t n_layers, d_model, n_heads, d_ff, vocab;
    const void* emb;       /* embedding.weight bf16 [V, d] */
    const void* wout;      /* output_layer.weight bf16 [V, d] (== emb when tied, decoder/transformer.py:156-158) */
    const float* bout;     /* output_layer.bias [V] or NULL */
    const float* pe;       /* sinusoid table f32 [>= max_steps, d] (otb_sinusoid_table) */
    otb_mega_layer layers[OTB_MEGA_MAX_LAYERS];
    float ln_eps;
} otb_mega_model;
/* Scratch the launch needs (activations, partial sums, barrier counters, TMA descriptors), in bytes; -1 on bad arguments. */
long long otb_decode_persistent_workspace(int N, int n_layers, int Lmax, int B, int beam, int vocab);
/* kvx bf16 [n_layers, B*T, 2d]: src_attn.vk_proj(memory) per layer (K | V, attention.py:134), projected once per
 * utterance by otb_linear; mem_len i32 [B]; kc/vc bf16 [n_layers, st->Lmax, N, d] self-attention cache (scratch);
 * st: search state, initialised by otb_beam_init (ctrl zeroed); workspace: 256-byte aligned device scratch of at least
 * otb_decode_persistent_workspace() bytes.  On return tok_hist / par_hist hold max_steps steps (a group of utterances
 * that ended early is padded with EOS / identity parents, exactly what the reference's finished-hypothesis masking
 * produces), scores / flag / last_tok the final state, ctrl[0] the reference's executed step count (first step at which
 * every hypothesis of every utterance has ended, else max_steps).
 * dbg_logp (optional, f32 [max_steps, N, vocab]) receives every step's log-probs, dbg_scores (optional, f32
 * [max_steps, N]) every step's hypothesis scores -- parity traces. */
int otb_decode_persistent(const otb_mega_model* model, const void* kvx, const int32_t* mem_len, void* kc, void* vc,
                          const otb_beam_state* st, int B, int T, int max_steps, void* workspace, long long workspace_bytes,
                          float* dbg_logp, float* dbg_scores, void* stream);

/* ---- Training step (SpeechToText.forward + loss.backward() + clip + Adam, model/speech2text.py:39-64,
 * train/trainer.py:206-234).  The reference differentiates through torch autograd; the entry points below are the
 * hand-written backward of each forward op above.  bf16 activations / gradients, fp32 parameter gradients. */

/* Backward of otb_attention (d_k = 64, no resid; lse as that forward stored it): dq, dk, dv written at column offsets
 * d*_col0 + 64*h of their matrices (e.g. the three thirds of one [M,3d] dqkv buffer).  out and dout are read at rows
 * [0, B*Tq) only, however many rows q has.  dsum f32 [B,H,Tq] receives D = rowsum(dout * out).
 * wgmma, scores recomputed.  bd and dbd are both NULL, or both set for rel-pos attention: the forward was otb_attention with
 * the band bd f32 [H, B*Tq, ldbd] (Tq == Tk, not causal).  The band is added to the recomputed scores, and its gradient dS
 * (the gradient of the raw score sum, which includes 1/sqrt(d_k)) is written to dbd bf16 [H, B*Tq, lddbd] at column
 * j - i + Tq - 1 (lddbd: 2 Tq - 1 rounded up to 8).  The caller zeroes dbd: entries without a visible key are not written. */
int otb_attention_bwd(const void* q, int ldq, int q_rows, const void* k, int ldk, int k_rows, const void* v, int ldv,
                      const void* out, int ldo, const void* dout, int lddo, const float* lse, float* dsum, void* dq,
                      int lddq, int dq_col0, void* dk, int lddk, int dk_col0, void* dv, int lddv, int dv_col0, int B, int H,
                      int Tq, int Tk, const int* kv_len, int causal, int q_col0, int k_col0, int v_col0, const float* bd, int ldbd,
                      void* dbd, int lddbd, void* stream);
/* Residual dropout without a GEMM in front: out = resid + alpha * keep(seed, site, row, col) / (1 - p) * x, with the mask of
 * otb_linear_dropout_resid / otb_dropout_bwd.  resid may be NULL (out = alpha * dropout_p(x): also the backward of such a
 * site).  row_len (optional, i32 [M / row_period]): rows with row % row_period >= row_len[row / row_period] read x as zero.
 * seed may be NULL when p = 0.  bf16 [M, N], N and the row pitches multiples of 8. */
int otb_dropout_add(const void* x, int ldx, const void* resid, int ldr, void* out, int ldo, int M, int N, float alpha, float p,
                    const uint32_t* seed, uint32_t site, const int32_t* row_len, int row_period, void* stream);
/* Conformer convolution module, middle part, in training mode (module/conformer.py:46-52): x bf16 [B*T, d] = GLU output, read as
 * zero on padded frames (t >= min(len[b], T): a length above T means every frame is valid, and no conv tap reads past the
 * utterance's T rows); c f32 [B*T, d] = depthwise_conv(x) + wb (w f32 [d, k] as nn.Conv1d stores it, k odd,
 * wb may be NULL); BatchNorm with batch statistics over all B*T rows -> stats f32 [2, d] = (mean, 1/sqrt(biased var + eps));
 * running_mean / running_var (optional) updated with `momentum` and the unbiased variance, *num_batches (optional) += 1;
 * out bf16 [B*T, d] = swish(BN(c)), zero on padded frames. */
int otb_conformer_conv_train(const void* x, const int32_t* len, const float* w, const float* wb, const float* gamma, const float* beta,
                             float* running_mean, float* running_var, int64_t* num_batches, float momentum, float eps, float* c,
                             float* stats, void* out, int B, int T, int d, int k, void* stream);
/* Its backward: dy bf16 [B*T, d] (gradient of out), x / c / stats as the forward left them; red f32 [2, d] and dc f32 [B*T, d]
 * are scratch; lengths are clamped to T as in the forward.  dx bf16 [B*T, d] (zero on padded frames); dw f32 [d, k], dwb
 * f32 [d] (NULL without conv bias), dgamma, dbeta f32 [d]: overwritten, or added to with accumulate != 0. */
int otb_conformer_conv_bwd(const void* dy, const void* x, const int32_t* len, const float* w, const float* gamma, const float* beta,
                           const float* c, const float* stats, float* red, float* dc, void* dx, float* dw, float* dwb, float* dgamma,
                           float* dbeta, int accumulate, int B, int T, int d, int k, void* stream);
/* nn.Linear weight gradient dW[N,K] (fp32) = dy[M,N]^T x[M,K] (bf16), wgmma with MN-major operands + split-K.
 * (The input gradient dx = dy W is otb_linear with the transposed weight.)  accumulate != 0: dW += ... (gradient
 * accumulation straight into the optimizer's flat gradient buffer, the way autograd accumulates into .grad). */
int otb_linear_wgrad(const void* dy, int lddy, const void* x, int ldx, float* dw, int lddw, int M, int N, int K, int accumulate,
                     void* stream);
/* nn.Linear bias gradient: out[n] (+)= sum_m x[m,n]. */
int otb_colsum(const void* x, int ldx, float* out, int M, int N, int accumulate, void* stream);
/* nn.LayerNorm backward (N <= 256): dz, dgamma (+)=, dbeta (+)= from dy and the pre-norm input z. */
int otb_layernorm_bwd(const void* dy, int lddy, const void* z, int ldz, const float* gamma, void* dz, int lddz,
                      float* dgamma, float* dbeta, float eps, int M, int N, int accumulate, void* stream);
/* F.glu (ffn.py:18) un-fused for training: u = [a | g] bf16 [M,2F] -> h [M,F]; and its backward. */
int otb_glu_fwd(const void* u, void* h, int M, int F, void* stream);
int otb_glu_bwd(const void* dh, const void* u, void* du, int M, int F, void* stream);
/* The other feed-forward activations (ffn.py:15-41) un-fused for training: h = act(u) and du = dh * act'(u), bf16 [M,N]
 * contiguous and 16-byte aligned (any M, N >= 1), fp32 math.  act: OTB_EPI_GELU (F.gelu, erf form: act' = Phi(u) +
 * u phi(u)), OTB_EPI_TANH or OTB_EPI_SWISH (u sigmoid(u)). */
int otb_act_fwd(const void* u, void* h, int M, int N, int act, void* stream);
int otb_act_bwd(const void* dh, const void* u, void* du, int M, int N, int act, void* stream);
/* ReLU backward through the output (frontend/conv.py:64). */
int otb_relu_bwd(const void* dy, const void* y, void* dx, long long n, void* stream);
/* nn.Embedding backward: dE[tok[n]] += scale * dx[n]  (fp32 atomics). */
int otb_embed_bwd(const int64_t* tok, const void* dx, float* dE, int N, int d, int vocab, float scale, void* stream);
/* out (+)= sum g^2 over a flat fp32 buffer (global gradient norm, trainer.py:221). */
int otb_sumsq(const float* g, long long n, float* out, int zero_first, void* stream);

/* clip_grad_norm_(max_norm) + torch.optim.Adam step on flat fp32 buffers (trainer.py:221-234); `sumsq` is the device scalar
 * written by otb_sumsq.  The step counters and the LR schedule live on the DEVICE (no host sync, CUDA-graph friendly):
 * counters i32 [3] = {optimizer steps, scheduler global_step, skipped steps}; when sqrt(*sumsq) is finite both counts
 * advance and lr = factor * model_size^-0.5 * min(s^-0.5, s * warmup^-1.5) (TransformerScheduler, train/scheduler.py:137-138;
 * warmup_steps <= 0: lr = base_lr), else only `skipped` advances and nothing is updated -- the reference skips
 * scheduler.step() and optimizer.step() together (trainer.py:229-233).  hyper f32 [4] receives {lr, 1-b1^t, 1-b2^t, applied}.
 * Gradient noise (trainer.py:223-227) when noise_std > 0: the clipped gradient of every element whose bit is set in
 * noise_mask (u8 [(n + 7) / 8], bit i & 7 of byte i >> 3) gets noise_std * z before the weight decay, z ~ N(0, 1) a
 * counter hash of (*noise_seed, the step t, i) through Box-Muller (DESIGN.md 4.5).  noise_std = 0: seed and mask unused. */
int otb_adam_step_sched(float* p, const float* g, float* m, float* v, long long n, const float* sumsq, float max_norm,
                        float base_lr, float model_size, float warmup_steps, float factor, float beta1, float beta2, float eps,
                        float weight_decay, int32_t* counters, float* hyper, float noise_std, const int32_t* noise_seed,
                        const uint8_t* noise_mask, void* stream);

/* MixSpeech input (trainer.py:155-201): x f32 [B, T, F] and mask u8 [B, T] (0 / 1) of B >= 2 utterances -> P = B / 2 pairs,
 * x_out f32 [P, T, F] = lambda * x[2p] + (1 - lambda) * x[2p + 1] (two separately rounded fp32 products, then their sum),
 * mask_out u8 [P, T] = mask[2p] | mask[2p + 1].  lambda ~ Beta(1/2, 1/2) = sin^2(pi u / 2), u a counter hash of (*seed,
 * *step) (both i32 device scalars); lam_out f32 [3] = {lambda, lambda * scale, (1 - lambda) * scale}. */
int otb_mixspeech(const float* x, const uint8_t* mask, int B, int T, int F, const int32_t* seed, const int32_t* step, float scale,
                  float* lam_out, float* x_out, uint8_t* mask_out, void* stream);

/* Low-frame-rate frame stacking (frontend/concat.py:11-56, the concat front ends): x f32 [B, T, F] -> out bf16 [B*T2, ldo],
 * row b*T2 + i = the n frames x[b, i*s .. i*s + n - 1] flattened frame-major (column j*F + f, nn.Unfold's order), frames at
 * or past T read as zero.  Columns [0, W) are written, W = n*F rounded up to 8; columns n*F .. W - 1 are zero and columns
 * from W to ldo are not touched (ldo >= W, a multiple of 8; out 16-byte aligned).  With table f32 [T2, n*F] each of the
 * n*F columns of row i becomes y * alpha + table[i] (two separately rounded fp32 operations), else y * alpha. */
int otb_frame_stack(const float* x, int B, int T, int F, int n, int s, int T2, void* out, int ldo, float alpha, const float* table,
                    void* stream);

/* ---- Recurrent language model (model/lm.py:31-90, rnnlm.yaml): nn.LSTM layers, gates ordered i, f, g, o.  Sequences are
 * time-major (row t*B + b, as nn.LSTM without batch_first).  The input projection gx f32 [L*B, 4H] = x W_ih^T + b_ih + b_hh
 * is otb_linear in front; these run the recurrence as persistent cooperative kernels (CTA j keeps the W_hh slice of its
 * hidden units in shared memory; one grid barrier per step).  H must be a multiple of 8 and the slice must fit shared
 * memory (otb_lstm_config); otherwise they return an error and launch nothing.  barrier u32 [2]: zeroed once, then reused
 * by launches that run one after another (one per stream).
 *
 * Host-only plan for hidden size H on a device with `sms` SMs and `smem_optin` bytes of opt-in shared memory per block:
 * hidden units per CTA, and the dynamic shared memory of the forward and backward kernels; an error where they refuse H. */
int otb_lstm_config(int H, int sms, int smem_optin, int* units, int* smem_fwd, int* smem_bwd);
/* Forward of one layer: w_hh bf16 [4H, H]; h0 / c0 f32 [B, H] or NULL (zero state); y bf16 [L*B, H] = h_t; h_n / c_n f32
 * [B, H] = the last step's h and c (fp32; outputs must not alias the inputs).  For training, gates (f32 [L*B, 4H],
 * post-activation, may alias gx) and c_all (f32 [L*B, H], c_t) record what otb_lstm_bwd reads; both NULL or both set. */
int otb_lstm_fwd(const float* gx, const void* w_hh, const float* h0, const float* c0, void* y, float* h_n, float* c_n, float* gates,
                 float* c_all, uint32_t* barrier, int L, int B, int H, void* stream);
/* Backward through time of one layer run with zero or given c0: dy bf16 [L*B, H] = gradient of y (h_n and c_n get none);
 * gates / c_all as otb_lstm_fwd recorded them -> dg bf16 [L*B, 4H] = gradient of the pre-activation gates, from which
 * dW_hh = dg[B:]^T y[:-B] and dW_ih = dg^T x (otb_linear_wgrad), db = colsum(dg) and dx = dg W_ih (otb_linear).
 * dc f32 [B, H] is scratch. */
int otb_lstm_bwd(const void* dy, const void* w_hh, const float* gates, const float* c_all, const float* c0, void* dg, float* dc,
                 uint32_t* barrier, int L, int B, int H, void* stream);
/* nn.Embedding lookup without scale: out bf16 [N, d] = emb[tok[n]] (d a multiple of 8; out-of-range ids read row 0). */
int otb_embedding(const int64_t* tok, const void* emb, void* out, int N, int d, int vocab, void* stream);

/* Log-mel filterbank features on the device (data/audio.py:117-120: ta.compliance.kaldi.fbank with Kaldi defaults, dither 0):
 * wave f32 [B, ld_wave] (zero padded), n_samples i32 [B]; gain f32 [B] or NULL scales each waveform where its samples are
 * loaded, before DC removal (volume_perturb, audio.py:112-114); window f32 [frame_len] (povey), 2 <= frame_len <= 2048; the
 * FFT has n_fft = round_to_power_of_two(frame_len) points; bank f32 [F, n_fft/2] triangular mel weights over the first
 * n_fft/2 bins of the spectrum and bank_range i32 [F, 2] their non-zero [lo, hi) ranges (built by
 * opentransformer_b200/features.py); out f32 [B, Tmax, F], frames >= 1 + (n - frame_len) / frame_shift are zero. */
int otb_fbank(const float* wave, int ld_wave, const int32_t* n_samples, const float* gain, int B, const float* window,
              const float* bank, const int32_t* bank_range, float* out, int Tmax, int F, int frame_len, int frame_shift, float preemph,
              void* stream);
/* `normalization` (data/audio.py:22-24): (x - mean) / std over all valid elements of each utterance (unbiased std), in place;
 * or, with gmean / gstd f32 [F], the global CMVN of audio.py:131-132.  x f32 [B, Tmax, F], n_frames i32 [B].  noise f32
 * [B, F] or NULL (gaussian_noise, audio.py:131-133) is added to every valid frame of utterance b in the same store; padded
 * frames stay zero.  gmean 0 / gstd 1 leave x as it is and only add the noise. */
int otb_utt_cmvn(float* x, int B, int Tmax, int F, const int32_t* n_frames, const float* gmean, const float* gstd, const float* noise,
                 void* stream);
/* Band-limited resampling, one rate pair per row (speed perturbation, data/audio.py:63-67,106-110, and audio at another
 * rate): row b of y equals torchaudio.functional.resample(x[b, :n_in[b]], orig[b], new_rate[b]) with its defaults
 * (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99).  x f32 [B, ldx] (only the first n_in[b] <= ldx samples of a row
 * are read), 1 <= B <= 65535; orig / new_rate i32 [B] on the device; y f32 [B, ldy], width <= ldy columns written; n_out i32 [B] = ceil(n *
 * n_in / o) with o / n the rates divided by their gcd, at most width (a row longer than width is cut there); columns from
 * n_out[b] to width are zero.  Rows with orig == new_rate are copied bit for bit; rows with a rate <= 0 are empty. */
int otb_resample(const float* x, int ldx, const int32_t* n_in, const int32_t* orig, const int32_t* new_rate, float* y, int ldy,
                 int32_t* n_out, int B, int width, void* stream);

/* Joint-CTC loss of SpeechToText.forward (model/speech2text.py:60-72 -> CTCAssistor.compute_loss, model/ctc.py:48-52):
 * nn.CTCLoss(blank, reduction 'mean', zero_infinity = True) and its gradient with respect to the LOGITS.
 * logp f32 [B*T, ldl] = log_softmax of the assistor's logits (otb_log_softmax); in_len i32 [B] valid frames; targets i64
 * [B, ldt] label rows (the first tgt_len[b] entries count); max_tgt >= every tgt_len, at most 1023 (one state per thread up
 * to 64, two per thread above); nll f32 [B] per-utterance
 * negative log-likelihood (+inf if infeasible); loss f32 [1]; ws f32 [B, T, 2 max_tgt + 1] scratch (alpha + beta; 262 MB
 * at B 32, T 1000, max_tgt 1023);
 * dlogits_bf16 (optional, bf16 [B*T, ldd]) = grad_scale * d loss / d logits (padded frames / infeasible utterances: 0).
 * grad_scale_dev (may be NULL): a device f32 scalar grad_scale is multiplied by, read on the device. */
int otb_ctc_loss(const float* logp, int ldl, int B, int T, int V, const int32_t* in_len, const int64_t* targets, int ldt,
                 const int32_t* tgt_len, int max_tgt, int blank, float* nll, float* loss, float* ws, void* dlogits_bf16, int ldd,
                 float grad_scale, const float* grad_scale_dev, void* stream);

/* CTC decoding (CTCRecognizer, recognize/ctc.py) on the CTC head's logits f32 [B*T, ld]; in_len i32 [B] valid frames.
 * otb_ctc_frame_topk: per frame, the K (1..min(64, V)) best tokens as log-probs (log-softmax over the first V columns), best
 *   first, ties to the lower index: top_lp f32 [B*T, K], top_id i32 [B*T, K]; frames at or past in_len, and ranks beyond
 *   the number of non-NaN logits of a row, get -inf / -1 (the greedy and beam kernels skip id -1).
 * otb_ctc_greedy: the greedy collapse on top_id[:, 0] (row pitch ldk): a frame's token is kept unless it is 0 (PAD), blank,
 *   or the previous frame's token.  ids i32 [B, T] (compacted, 0 after the end), lengths i32 [B], scores f32 [B] = sum of
 *   the best log-probs over the valid frames.
 * otb_ctc_prefix_beam: CTC prefix beam search (no LM) over each frame's top-K tokens, beam 1..16, one CTA per utterance.
 *   nodes i32 [B, 1 + T*beam, 2] workspace (back-pointer table); ids i32 [B, beam, T] best first (0 after the end),
 *   lengths i32 [B, beam], scores f32 [B, beam] = log(p_blank + p_nonblank) (-inf for unused slots). */
int otb_ctc_frame_topk(const float* logits, int ld, int B, int T, int V, const int32_t* in_len, int K, float* top_lp,
                       int32_t* top_id, void* stream);
int otb_ctc_greedy(const float* top_lp, const int32_t* top_id, int ldk, int B, int T, const int32_t* in_len, int blank,
                   int32_t* ids, int32_t* lengths, float* scores, void* stream);
int otb_ctc_prefix_beam(const float* top_lp, const int32_t* top_id, int K, int B, int T, const int32_t* in_len, int blank, int beam,
                        int32_t* nodes, int32_t* ids, int32_t* lengths, float* scores, void* stream);

/* The prefix beam search with a neural LM as ctcdecode's scorer (DESIGN.md 4.19), ONE frame per call, one CTA per
 * utterance; the frame index is ctl[0] (ctl i32 [2] zeroed before frame 0; the call moves ctl[0] on).  Extending slot i by
 * token c adds lm_weight * lm[b*beam + i][c] + beta (lm f32 [B*beam, ld_lm], the LM's next-token log-probs of each slot's
 * prefix after BOS).  slots: otb_ctc_prefix_beam_slots_bytes(B) bytes of slot state; nodes as otb_ctc_prefix_beam.  Per new
 * slot (row b*beam + s): src i32 its source row, tok i64 its newest token (BOS = 1 for the empty prefix), ext i32 1 where it
 * extended the source.  Transformer LM (anc non-null): anc i32 [B*beam, Lpos] cache rows (b*(1 + T*beam) + node) of each
 * slot's prefix from position 0 (BOS), rewritten for the new slots, anc_tmp the same size of scratch, pos i32 [B*beam] each
 * row's query position (-1: nothing to compute).  ids / lengths / scores as otb_ctc_prefix_beam, written at frame T - 1. */
int otb_ctc_prefix_beam_slots_bytes(int B);
int otb_ctc_prefix_beam_step(const float* top_lp, const int32_t* top_id, int K, int B, int T, const int32_t* in_len, int blank,
                             int beam, const float* lm, int ld_lm, float lm_weight, float beta, void* slots, int32_t* ctl,
                             int32_t* nodes, int32_t* src, int64_t* tok, int32_t* ext, int32_t* anc, int32_t* anc_tmp,
                             int32_t* pos, int Lpos, int32_t* ids, int32_t* lengths, float* scores, void* stream);
/* The fused search's LM rows and state follow its slots: row n of dst = row n of a where ext[n] != 0 (left as it is when a
 * is NULL), else row idx[n] of b (row n without idx).  Rows of `width` 4-byte words, pitches in words. */
int otb_ctc_lm_carry(void* dst, int ldd, const void* a, int lda, const void* b, int ldb, const int32_t* idx, const int32_t* ext,
                     int rows, int width, void* stream);

/* CTC forced alignment: the best path (Viterbi) through the CTC trellis of each utterance's target, one CTA per utterance.
 * rows f32 [B*T, ld]: log-probs when lse is NULL, else logits with lse f32 [B*T] each frame's log-sum-exp (lp = row - lse);
 * only the columns the targets name and the blank are read.  in_len i32 [B] valid frames; targets i64 [B, ldt], the first
 * tgt_len[b] entries count (0 <= tgt_len <= max_tgt <= 1023); bp u8 [B, T, 2 max_tgt + 1] workspace (back-pointers).
 * labels i32 [B, T] = the token aligned to each frame (blank included), -1 at or past in_len; frame_scores f32 [B, T] = its
 * log-prob (-inf where the label is -1); spans i32 [B, max_tgt, 2] = [start, end) of each target token in frames, -1 past
 * tgt_len; path_score f32 [B] = the path's log-prob.  Ties prefer the state itself, then one back, then two back; the end
 * state prefers the last token's blank.  An utterance without an alignment of finite log-prob (too few frames, a blank or
 * out-of-range token, tgt_len outside 0..max_tgt) gets path_score -inf and labels / spans -1. */
int otb_ctc_align(const float* rows, int ld, int B, int T, int V, const float* lse, const int32_t* in_len, const int64_t* targets,
                  int ldt, const int32_t* tgt_len, int max_tgt, int blank, uint8_t* bp, int32_t* labels, float* frame_scores,
                  int32_t* spans, float* path_score, void* stream);

/* CTC prefix scoring for joint CTC/attention decoding (Watanabe et al. 2017): the CTC term of the beam search's step score.
 * lp f32 [B*T, ld] log-probs of the joint-CTC head, in_len i32 [B] valid frames.  For a hypothesis g (its tokens after
 * <S/E>), gamma(g)[t] = {log-prob that frames 0..t emit exactly g ending in a non-blank, ... ending in a blank} and psi(g) =
 * the log-probability that the labels start with g; the closing <S/E> is a label like any other, so psi(g <S/E>) is the
 * log-probability of the whole label sequence g <S/E>.  gamma f32 [2, N, T, 2] and psi f32 [2, N] hold the state of the N
 * hypotheses of a search; the half in use is the parity of its step counter (st->ctrl[0]).
 * otb_ctc_prefix_init: gamma and psi of the empty prefix for every row, in half 0. */
int otb_ctc_prefix_init(const float* lp, int ld, int B, int T, const int32_t* in_len, int blank, int beam, float* gamma,
                        float* psi, void* stream);
/* One step's scores: for every unfinished hypothesis n and each of its P candidates (cand_val f32 / cand_id i32 [N, P] of
 * otb_logsoftmax_topk with k = P, beam <= P <= 16; cand_val = logp_att + lm_weight * lm_logp[cand_id] when lm_logp is given)
 * gamma_cand f32 [N, P, T, 2] and psi_cand f32 [N, P] of the hypothesis extended by the candidate, the joint score
 * (1 - ctc_weight) logp_att + ctc_weight (psi_cand - psi) + lm_weight lm_logp (-inf where psi_cand is -inf, never NaN), and
 * the `beam` best candidates by it into out_val f32 / out_idx i32 [N, beam] (descending, ties to the lower id), the top-k
 * layout otb_beam_step takes.  Does nothing once the search has ended. */
int otb_ctc_prefix_score(const float* lp, int ld, int T, int V, const int32_t* in_len, int blank, const float* gamma,
                         const float* psi, const float* cand_val, const int32_t* cand_id, int P, const float* lm_logp, int ld_lm,
                         float lm_weight, float ctc_weight, const otb_beam_state* st, float* gamma_cand, float* psi_cand,
                         float* out_val, int32_t* out_idx, void* stream);
/* After otb_beam_step on those top-k: every new row takes gamma_cand / psi_cand of its parent's candidate that names its
 * token into the other half of gamma / psi; a row whose token is <S/E> keeps its parent's state.  Does nothing once the
 * search has ended. */
int otb_ctc_prefix_advance(const otb_beam_state* st, const int32_t* cand_id, int P, int T, const int32_t* in_len,
                           const float* gamma_cand, const float* psi_cand, float* gamma, float* psi, void* stream);

/* CTC rescoring of an attention n-best (SpeechToTextRecognizer's apply_ctc_rescoring): out f32 [B*K] = log p_ctc(target_r |
 * x_b) of target row r of utterance b = r / K, by the blank-extended forward recursion (log domain, fp32), one CTA per row.
 * logp f32 [B*T, ld] the head's log-probs, of which the first in_len[b] (i32 [B], clamped to T) frames of utterance b count;
 * targets i32 [B*K, Lp], 1 <= Lp <= 1024: a row's labels are its entries before the first negative one.  -inf where no
 * alignment exists: a label equal to blank or outside [0, V), in_len <= 0, or too few frames for the labels and their
 * repeats.  Forward only: no workspace. */
int otb_ctc_nbest_score(const float* logp, int ld, int B, int T, int V, const int32_t* in_len, const int32_t* targets, int K,
                        int Lp, int blank, float* out, void* stream);

/* N-best rescoring (the recognizers' apply_rescoring / apply_lm_rescoring; no reference entry point computes it:
 * eval.py's -resc / -lm_resc / -rw are parsed and never used).
 * otb_token_logprob: out f32 [rows] = logits[r, target[r]] - logsumexp(logits[r, :V]) of logits f32 [rows, ld], 0 where
 * target[r] < 0 (the row is not read) and NaN where target[r] >= V.  ld % 4 == 0 and a 16-byte aligned base.  Each row is
 * read once; the reduction order is fixed, so repeated calls are bit-identical. */
int otb_token_logprob(const float* logits, int ld, int rows, int V, const int32_t* target, float* out, void* stream);
/* One warp per utterance over its K <= 32 first-pass hypotheses, hypothesis h = b * K + k: tgt i32 [B*K, Lp] its scored
 * tokens y <S/E> (-1 after), len i32 [B*K] the length n of y, s1 f32 [B*K] its first-pass score, tok_lp f32 [M, B*K, Lp]
 * the token log-probs of M second-pass models.  A hypothesis equal to one of a lower k of its utterance is dropped; the
 * others score s = s1 + weight * sum_m sum_{t <= n} tok_lp[m, h, t] (position order, then model order, fp32 without
 * contraction).  Ranked: kept before dropped, then descending s, then k.  The first nbest (<= K) go to ids i64
 * [B, nbest, Lout] (y, then pad_id), out_len i32 [B, nbest] (n; 0 when dropped) and out_score f32 [B, nbest] (-inf when
 * dropped). */
int otb_nbest_rescore(const int32_t* tgt, int Lp, const int32_t* len, const float* s1, const float* tok_lp, int M, int B, int K,
                      float weight, int nbest, int Lout, int64_t pad_id, int64_t* ids, int32_t* out_len, float* out_score,
                      void* stream);

/* Minimum word error rate training (Prabhavalkar et al. 2018; the reference has no counterpart).
 * otb_edit_distance: out i32 [N] = the Levenshtein distance (unit costs) between hypothesis i, the first hyp_len[i] tokens of
 * hyp i32 [N, ldh], and reference i / K, the first ref_len[i / K] tokens of ref i32 [ceil(N / K), ldr].  Lengths are clamped
 * to [0, max_hyp] and [0, max_ref]; max_hyp, max_ref <= 1023 (refused otherwise, before any launch).  Exact. */
int otb_edit_distance(const int32_t* hyp, int ldh, const int32_t* hyp_len, const int32_t* ref, int ldr, const int32_t* ref_len, int N,
                      int K, int max_hyp, int max_ref, int32_t* out, void* stream);
/* One warp per utterance over its K <= 32 hypotheses, h = b * K + k, laid out as otb_nbest_rescore's: tgt i32 [B*K, Lp] the
 * scored tokens y <S/E> (-1 after), len i32 [B*K] the length n of y (clamped to [0, Lp - 1]), err i32 [B*K] its edit distance W,
 * tok_lp f32 [B*K, Lp] its token log-probs.  A hypothesis equal to one of a lower k is dropped.  Over the kept ones: l = sum_{t <= n} tok_lp[h, t]
 * (position order, fp32 without contraction), P = softmax(l), loss f32 [B] = sum_k P_k (W_k - mean W) and coeff f32 [B*K] =
 * P_k (W_k - sum_j P_j W_j) * scale (* *scale_dev when scale_dev is not NULL); coeff is 0 for a dropped hypothesis. */
int otb_mwer_coeff(const int32_t* len, const int32_t* err, const float* tok_lp, int Lp, const int32_t* tgt, int B, int K, float scale,
                   const float* scale_dev, float* coeff, float* loss, void* stream);
/* The sampled estimator of the same gradient: one warp per utterance over its K <= 32 samples, drawn with replacement (no
 * duplicate rule, no softmax).  err i32 [B*K] the edit distances W; loss f32 [B] = W^_b = mean_k W_k and coeff f32 [B*K] =
 * (W_k - W^_b) / K * scale (* *scale_dev when scale_dev is not NULL), exactly 0 when all W of an utterance are equal. */
int otb_mwer_sample_coeff(const int32_t* err, int B, int K, float scale, const float* scale_dev, float* coeff, float* loss,
                          void* stream);
/* dlogits bf16 [rows, ld] = coeff[r / Lp] * (onehot(target[r]) - softmax(logits[r, :V])) of logits f32 [rows, ld], with
 * tok_lp f32 [rows] = otb_token_logprob of the same logits and targets (its log-sum-exp is reused); columns >= V, rows with
 * target < 0 or >= V and rows with coeff 0 are zero.  ld % 4 == 0 and 16-byte aligned logits. */
int otb_mwer_grad(const float* logits, int ld, int rows, int V, const int32_t* target, const float* tok_lp, const float* coeff, int Lp,
                  void* dlogits, void* stream);

/* Conv2d front end backward (frontend/conv.py:50-76 under autograd), at the geometry of the forward.  h1 = conv1
 * activation buffer (layout of otb_conv1_relu).  col bf16 [B*T2*F2, kt2*kf2*C1] = im2col of h1 for conv2
 * (k = (kh*kf2+kw)*C1 + c): conv2's weight gradient is otb_linear_wgrad(dpre2, col) and its input gradient
 * dcol = otb_linear(dpre2, W2^T).  otb_conv_col2im_relu folds dcol back onto the conv1 grid and applies ReLU' -> dpre1
 * (h1 layout).  otb_conv1_wgrad: out f32 [C1, kt1*kf1 + 1] = tap gradients + the bias gradient of conv1 (C_in = 1;
 * C1 <= 256). */
int otb_conv_im2col(const void* h1, void* col, int B, int T, int F, int C1, int kt1, int kf1, int st1, int sf1, int kt2,
                    int kf2, int st2, int sf2, void* stream);
int otb_conv_col2im_relu(const void* dcol, const void* h1, void* dpre1, int B, int T, int F, int C1, int kt1, int kf1,
                         int st1, int sf1, int kt2, int kf2, int st2, int sf2, void* stream);
int otb_conv1_wgrad(const void* dpre1, const float* x, float* out, int B, int T, int F, int C1, int kt1, int kf1, int st1,
                    int sf1, int kt2, int kf2, int st2, int sf2, void* stream);

/* ---- Transducer (RNN-T) model (DESIGN.md 4.22).  The lattice of utterance b: nodes (t, u), t < t_len[b] <= T frames and
 * u <= u_len[b] <= U1 - 1 labels, stored padded as [B, T, U1] with u fastest; node (b, t, u) is row (b T + t) U1 + u.  Every
 * call skips the nodes past t_len or u_len and writes zeros for them.  Blank is token 0; labels i32 [B, ldy] hold y_1 .. y_U
 * (u_len[b] of each row count; a label outside [1, V) has no arc).
 * otb_rnnt_joint: Hj bf16 [B T U1, D] = tanh(Ep[b T + t] + Pp[b U1 + u]) of Ep bf16 [B T, D] and Pp bf16 [B U1, D], D % 8 == 0.
 *   t_len / u_len may be NULL: every node is valid.
 * otb_rnnt_joint_bwd: dZ = dHj (1 - Hj^2) -> dEp bf16 [B T, D] (sum over u <= u_len) and dPp bf16 [B U1, D] (sum over
 *   t < t_len), each in ascending order in fp32: no atomics, repeated calls are bit-identical.  D even.
 * otb_rnnt_logprob: rows [row0, row0 + rows) of the lattice, logits f32 [rows, ld] (ld % 4 == 0, 16-byte aligned) ->
 *   lp f32 [B T U1, 3] rows row0.. = (logsumexp, log p(blank), log p(y_{u+1}); -inf at u = u_len).
 * otb_rnnt_loss: one CTA per utterance over lp, in fp64: alpha f64 [B T U1] scratch, nll f32 [B] the negative log-likelihood summed
 *   over all alignments (+inf when t_len <= 0), loss f32 [1] = mean_b nll, grad f32 [B T U1, 2] = grad_scale
 *   (* *grad_scale_dev when not NULL) / B * d nll_b / d (log p(blank), log p(y_{u+1})).  U1 <= 1024.
 * otb_rnnt_dlogits: dz bf16 [rows, ldd] = [k = 0] a + [k = y] c - softmax(logits)_k (a + c) of the same rows, with lp's
 *   logsumexp and (a, c) = grad of the node; columns >= V are zero.
 * otb_rnnt_greedy_step: one step of batched greedy search over B utterances, after otb_logsoftmax_topk (k = 1) of the joint's
 *   logits: idx i32 [B] the arg-max, logp f32 [B, ldlp] the log-probs.  A row whose frame[b] < t_len[b] takes idx, or blank
 *   when n_sym[b] >= max_sym or n_out[b] >= max_len, and adds its log-prob to score[b].  A label goes to ids i32 [B, max_len]
 *   at n_out[b], and the predictor state computed from it (h_new / c_new f32 [layers, B, H], pp_new bf16 [B, D]) replaces the
 *   row's (h, c, pp); blank moves frame[b] on and copies ep bf16 [B T, D] row b T + frame[b] into ep_cur bf16 [B, D], or,
 *   past the last frame, decrements *active.  Ended rows are left unchanged.  LM shallow fusion (all three optional, NULL:
 *   none): val f32 [B] the fused value of idx (otb_logsoftmax_topk with blank exempt), which a label adds to score in place
 *   of its log-prob; emit i32 [B] = 1 where the row emitted a label this step, else 0; lm_pos i32 [B] = the label's LM
 *   position (n_out after it, 1..max_len) where it emitted, else -1.
 * Pruned lattice (pruned RNN-T): joint, joint_bwd, logprob, loss and dlogits take (s_begin, S).  s_begin i32 [B, T] non-NULL
 *   keeps at frame t the S label positions u = s_begin[b T + t] + k, k < S (2 <= S <= 1024), stored [B, T, S] with k
 *   fastest: node (b, t, k) is row (b T + t) S + k, and every [B T U1, .] array above is [B T S, .].  A node outside its
 *   frame's band does not exist: the loss's alignments stay inside the bands, and an utterance without such an alignment
 *   gets nll +inf and zero gradients.  dPp row (b, u) sums over the frames whose band holds u.  NULL: the full lattice.
 * otb_rnnt_simple_lse: the simple joint's node log-probs for logits am[b T + t] + lm[b U1 + u] (am f32 [B T, lda], lm f32
 *   [B U1, ldl]) -> lp f32 [B T U1, 3] as otb_rnnt_logprob writes them, in fp32 through one [T, V] x [V, U1] product per
 *   utterance, and the row maxima m_am f32 [B T], m_lm f32 [B U1] the backward reads.
 * otb_rnnt_simple_bwd: from otb_rnnt_loss's grad over that lp, scaled by scale (* *scale_dev when not NULL): d am bf16
 *   [B T, ldd] and d lm bf16 [B U1, ldd], columns >= V zero; the one-hot terms summed in a fixed order, no atomics.
 * otb_rnnt_prune_ranges: s_begin i32 [B, T] from the simple loss's grad [B T U1, 2]: the S-wide window of largest occupancy
 *   at each frame, then the range rule of DESIGN.md 4.22 (s_0 = 0, non-decreasing, consecutive bands overlap, the last
 *   band holds U_b).  Frames past t_len get 0. */
int otb_rnnt_joint(const void* ep, const void* pp, int B, int T, int U1, int D, const int32_t* t_len, const int32_t* u_len, void* out,
                   const int32_t* s_begin, int S, void* stream);
int otb_rnnt_joint_bwd(const void* dh, const void* h, int B, int T, int U1, int D, const int32_t* t_len, const int32_t* u_len,
                       void* dep, void* dpp, const int32_t* s_begin, int S, void* stream);
int otb_rnnt_logprob(const float* logits, int ld, int rows, int64_t row0, int V, int B, int T, int U1, const int32_t* t_len,
                     const int32_t* u_len, const int32_t* labels, int ldy, float* lp, const int32_t* s_begin, int S, void* stream);
int otb_rnnt_loss(const float* lp, int B, int T, int U1, const int32_t* t_len, const int32_t* u_len, double* alpha, float* nll,
                  float* loss, float* grad, float grad_scale, const float* grad_scale_dev, const int32_t* s_begin, int S, void* stream);
int otb_rnnt_dlogits(const float* logits, int ld, int rows, int64_t row0, int V, int B, int T, int U1, const int32_t* t_len,
                     const int32_t* u_len, const int32_t* labels, int ldy, const float* lp, const float* grad, void* dz, int ldd,
                     const int32_t* s_begin, int S, void* stream);
int otb_rnnt_simple_lse(const float* am, int lda, const float* lm, int ldl, int V, int B, int T, int U1, const int32_t* t_len,
                        const int32_t* u_len, const int32_t* labels, int ldy, float* lp, float* m_am, float* m_lm, void* stream);
int otb_rnnt_simple_bwd(const float* am, int lda, const float* lm, int ldl, int V, int B, int T, int U1, const int32_t* t_len,
                        const int32_t* u_len, const int32_t* labels, int ldy, const float* lp, const float* m_am, const float* m_lm,
                        const float* grad, float scale, const float* scale_dev, void* d_am, void* d_lm, int ldd, void* stream);
int otb_rnnt_prune_ranges(const float* grad, int B, int T, int U1, const int32_t* t_len, const int32_t* u_len, int S, int32_t* s_begin,
                          void* stream);
int otb_rnnt_greedy_step(const int32_t* idx, const float* logp, int ldlp, const float* h_new, const float* c_new, const void* pp_new,
                         float* h, float* c, void* pp, int layers, int B, int H, int D, const void* ep, int T, void* ep_cur,
                         const int32_t* t_len, int32_t* frame, int32_t* n_sym, int32_t* n_out, int32_t* ids, int max_len,
                         int max_sym, float* score, int32_t* active, const float* val, int32_t* emit, int32_t* lm_pos,
                         void* stream);

/* ---- Transducer beam search: alignment-length synchronous decoding (ALSD), DESIGN.md 4.22.  Utterance b owns the K
 * hypothesis slots (1 <= K <= 15) of rows b K .. b K + K - 1 of every [B K, ...] array.  A slot holds score f32 (-inf:
 * empty), slot_u its label count u, frame its frame t (t < t_len[b] while live) and node its last label's node in the
 * utterance's node table (node_par / node_tok i32 [B, n_cap], n_cap >= K (T + max_len) + 1; node 0 is the empty sequence,
 * n_nodes i32 [B] the nodes in use).
 * otb_rnnt_beam_step: one search step for every utterance with done[b] == 0, after otb_logsoftmax_topk (k1 = min(K + 1, V))
 *   of the joint's logits at each slot: logp f32 [B K, ldlp] the log-probs (column 0 blank), val / idx [B K, k1] the top
 *   k1.  Each live slot forms a blank candidate (a final when t + 1 = t_len[b]) and, while u < max_len, one per each of its
 *   min(K, V - 1) best labels; a label candidate whose sequence equals a live blank candidate's is log-added into it; the K
 *   best (score descending, ties to the lower parent slot, blank before labels, labels in top-k order) become the new slots,
 *   with par i32 [B K] the parent slot (0..K-1) and tok i64 [B K] the label taken (0: blank or empty).  Finals go into the
 *   n-best f_score / f_node / f_u [B, W] (f_n i32 [B] entries; ties to the earlier step, then the lower slot).  The
 *   utterance ends when no slot is live, or f_n = W and logsumexp(live scores) <= f_score[W - 1]: done[b] = 1, *active -= 1,
 *   and ids i32 [B, W, max_len] (0-padded), lengths i32 [B, W] and out_score f32 [B, W] get the n-best, best first (unfilled
 *   entries: length 0, score -inf).  An ended utterance's slots get par = their own slot and tok = 0.
 *   LM shallow fusion: val holds the fused label values (otb_logsoftmax_topk with blank exempt) and no decision changes;
 *   beta > 0 makes the end bound logsumexp(live score + beta (max_len - u)).  lm_src / lm_ext (optional, i32 [B K]): each
 *   new slot's parent row b K + par and 1 where it took a label.  anc (optional, i32 [B K, Lpos], Lpos >= max_len + 1,
 *   with anc_tmp the same size of scratch and lm_pos i32 [B K]): each slot's LM cache rows b n_cap + node of its labels,
 *   position 0 the empty sequence's node 0, kept up to date; lm_pos = the new label's position u where the slot took one,
 *   else -1.  Ended utterances: lm_src = the row itself, lm_ext = 0, lm_pos = -1.
 * otb_rnnt_beam_gather: (h, c) f32 [layers, B K, H] and pp bf16 [B K, D] of row b K + par[r] -> (hg, cg, ppg) row r, and ep
 *   bf16 [B T, D] row b T + frame[r] -> ep_cur bf16 [B K, D] row r.
 * otb_rnnt_beam_commit: (h, c, pp) row r = (hn, cn, ppn) row r where tok[r] > 0, else (hg, cg, ppg) row r. */
int otb_rnnt_beam_step(const float* logp, int ldlp, const float* val, const int32_t* idx, int k1, int B, int K, int W, int V, int T,
                       int max_len, const int32_t* t_len, float* score, int32_t* slot_u, int32_t* frame, int32_t* node, int32_t* par,
                       int64_t* tok, int32_t* node_par, int32_t* node_tok, int n_cap, int32_t* n_nodes, float* f_score,
                       int32_t* f_node, int32_t* f_u, int32_t* f_n, int32_t* done, int32_t* active, int32_t* ids, int32_t* lengths,
                       float* out_score, float beta, int32_t* lm_src, int32_t* lm_ext, int32_t* anc, int32_t* anc_tmp, int32_t* lm_pos,
                       int Lpos, void* stream);
int otb_rnnt_beam_gather(const int32_t* par, const int32_t* frame, int B, int K, int layers, int H, int D, int T, const float* h,
                         const float* c, const void* pp, const void* ep, float* hg, float* cg, void* ppg, void* ep_cur, void* stream);
int otb_rnnt_beam_commit(const int64_t* tok, int rows, int layers, int H, int D, const float* hg, const float* cg, const void* ppg,
                         const float* hn, const float* cn, const void* ppn, float* h, float* c, void* pp, void* stream);

/* SpecAugment (data/augment.py:9-41) applied on the device: zero n_freq frequency bands and n_time time bands per
 * utterance.  x f32 [B,T,F] in place; bands i32 [B, 2*(n_freq+n_time)] = (f0, width)*n_freq, (t0, width)*n_time drawn
 * on the host with the reference's RNG call order. */
int otb_spec_augment(float* x, const int32_t* bands, int B, int T, int F, int n_freq, int n_time, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* OTB200_H_ */
