/*
 * avsr_b200.h -- C ABI of libavsr_b200.so: the H100 (sm_90a) Conformer-encoder forward path.
 *
 * The reference (mpc001/auto_avsr @ 182b628) has no FFI layer: its boundary for this path is the
 * Python nn.Module surface (SURVEY.md section 8b).  These entry points are what a binding for that
 * surface needs; auto_avsr_b200/_cabi.py binds them with ctypes and the modules in
 * auto_avsr_b200/espnet_dropin/ call them.  Each entry names the reference interface it replaces
 * (paths relative to /root/reference).
 *
 * Conventions
 *   - plain C types only: raw DEVICE pointers (unless a parameter says host), ints, sizes.
 *   - the caller owns every buffer (inputs, outputs, prepared weights, workspace); the library never
 *     allocates device memory and keeps no global device state.
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises.
 *   - return value: 0 = success, non-zero = AVSR_E_*; avsr_last_error() gives the message
 *     (thread-local, valid until the next call on that thread).
 *   - all float tensors are fp32, contiguous, row-major; "frames" are rows r = b*T + t.
 *   - there is NO CPU fallback: without a CUDA device every compute call fails with AVSR_E_CUDA.
 */
#ifndef AVSR_B200_H_
#define AVSR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AVSR_ABI_VERSION 12

enum {
  AVSR_OK = 0,
  AVSR_E_INVALID = 1,   /* bad argument / unsupported shape */
  AVSR_E_CUDA = 2,      /* CUDA runtime / driver error (message has the CUDA error string) */
  AVSR_E_WORKSPACE = 3  /* workspace or prepared-weight buffer too small */
};

/* Arithmetic of the GEMM / attention contractions. */
enum {
  AVSR_PREC_FP32 = 0,  /* CUDA-core fp32 FMA kernels: the on-device exact reference path (slow) */
  AVSR_PREC_TF32 = 1,  /* wgmma .tf32: operands kept as fp32 rounded to TF32, fp32 accumulate */
  AVSR_PREC_F16 = 2,   /* wgmma .f16: operands stored as IEEE half (same 10-bit mantissa as TF32, saturating
                          conversion), fp32 accumulate; residual stream, LayerNorm, softmax, conv stay fp32.
                          Half the operand bytes and twice the MMA rate of TF32: the product path. */
  AVSR_PREC_BF16 = 16  /* wgmma .bf16: operands stored as bfloat16 (7-bit mantissa, fp32's 8-bit exponent, round to
                          nearest even, no saturation), fp32 accumulate; the bytes and rate of AVSR_PREC_F16 with
                          fp32's range.  Every *_bytes entry returns its AVSR_PREC_F16 value. */
};

/* Hyper-parameters hard-wired in E2E.__init__ (espnet/nets/pytorch_backend/e2e_asr_conformer.py:33-39):
 * d_model 768, n_heads 12, linear_units 3072, num_blocks 12, cnn_kernel 31.  d_model/n_heads must be 64. */
typedef struct AvsrEncoderConfig {
  int32_t d_model;
  int32_t n_heads;
  int32_t linear_units;
  int32_t num_blocks;
  int32_t cnn_kernel;
} AvsrEncoderConfig;

/* One EncoderLayer's parameters in the reference's own layout and naming
 * (espnet/nets/pytorch_backend/encoder/conformer_encoder.py:61-94; the 40 state-dict keys of SURVEY.md 8a,
 * minus num_batches_tracked).  Linear weights are (out, in); conv weights keep their trailing 1-dims. */
typedef struct AvsrLayerParams {
  /* feed_forward_macaron.{w_1,w_2} + norm_ff_macaron   (positionwise_feed_forward.py:24-30) */
  const float *ffm_w1, *ffm_b1, *ffm_w2, *ffm_b2, *norm_ffm_w, *norm_ffm_b;
  /* self_attn.*  + norm_mha                            (transformer/attention.py:31-34,118-129) */
  const float *q_w, *q_b, *k_w, *k_b, *v_w, *v_b, *out_w, *out_b, *pos_w, *pos_bias_u, *pos_bias_v;
  const float *norm_mha_w, *norm_mha_b;
  /* conv_module.* + norm_conv                          (conformer_encoder.py:20-28) */
  const float *pw1_w, *pw1_b, *dw_w, *dw_b, *bn_w, *bn_b, *bn_mean, *bn_var, *pw2_w, *pw2_b;
  const float *norm_conv_w, *norm_conv_b;
  /* feed_forward.{w_1,w_2} + norm_ff */
  const float *ff_w1, *ff_b1, *ff_w2, *ff_b2, *norm_ff_w, *norm_ff_b;
  /* norm_final */
  const float *norm_final_w, *norm_final_b;
} AvsrLayerParams;

/* ---- library / error -------------------------------------------------------------------------- */
int avsr_abi_version(void);
const char *avsr_last_error(void);
/* number of kernels this library has launched in the calling process (bench.py's gpu_launches) */
uint64_t avsr_launch_count(void);

/* ---- weight preparation ------------------------------------------------------------------------
 * Replaces nothing in the reference (it uses nn.Parameters in place); it is the one-off layout step
 * of this implementation: QK weights concatenated, pointwise_cov1 rows interleaved so a GEMM tile
 * holds GLU value+gate pairs, depthwise taps transposed to (K, C), BatchNorm running statistics
 * (conformer_encoder.py:26, eval mode) folded into scale/shift, linear_pos of all layers stacked, and --
 * GEMM weights converted to the precision's operand storage (TF32-rounded fp32, or fp16).  `layers` is a HOST array of num_blocks structs holding DEVICE pointers.
 * Must be re-run after the parameters change. */
size_t avsr_prepared_bytes(const AvsrEncoderConfig *cfg);
int avsr_prepare_weights(const AvsrEncoderConfig *cfg, const AvsrLayerParams *layers,
                         const float *after_norm_w, const float *after_norm_b,
                         void *prepared, size_t prepared_bytes, int precision, void *stream);

/* ---- whole-encoder forward ---------------------------------------------------------------------
 * ConformerEncoder.forward(xs, masks) in eval mode (conformer_encoder.py:264-282): embed (x*sqrt(d),
 * rel-pos sinusoid table, transformer/embedding.py:171-184) -> num_blocks x EncoderLayer.forward
 * (conformer_encoder.py:96-170) -> after_norm.
 *   xs      (B, T, d_model) fp32      lengths (B) int32 DEVICE array or NULL
 *   out     (B, T, d_model) fp32
 * `lengths` is the prefix form of the reference's masks (B,1,T) = make_non_pad_mask(lengths)
 * (nets_utils.py:183); NULL == masks None == every frame valid.  As in the reference only attention
 * KEYS are masked: padded frames are computed as data everywhere else (SURVEY.md D6). */
size_t avsr_workspace_bytes(const AvsrEncoderConfig *cfg, int B, int T);
int avsr_encoder_forward(const AvsrEncoderConfig *cfg, const void *prepared, const float *xs,
                         const int32_t *lengths, int B, int T, float *out, void *workspace,
                         size_t workspace_bytes, int precision, void *stream);

/* Diagnostic variant of avsr_encoder_forward for AVSR_PREC_F16: fp16 operand stores saturate at +-65504
 * (cvt.rn.satfinite) where the fp32 reference would carry on.  The other precisions cannot saturate (AVSR_PREC_BF16
 * has fp32's range): for them this is the plain forward and *saturated stays 0.  This entry scans every operand tensor (LayerNorm
 * outputs, FFN hidden, q/k/v, rel-pos table, attention context, conv activations) right after its producer and
 * leaves in *saturated (DEVICE uint64, zeroed by the call) the number of elements that sit at the saturation value or
 * are NaN.  0 == the fp16 path stayed in range for these weights and inputs.  Direct launches, ~2x slower. */
int avsr_encoder_forward_checked(const AvsrEncoderConfig *cfg, const void *prepared, const float *xs,
                                 const int32_t *lengths, int B, int T, float *out, void *workspace,
                                 size_t workspace_bytes, int precision, uint64_t *saturated, void *stream);

/* Same computation replayed from a CUDA graph captured once per (B, T, buffers): removes the ~190
 * per-forward launches' host cost.  The plan is HOST state only (tensor maps + graph); it borrows
 * `prepared` and `workspace`, which must outlive it and must not be used by another plan concurrently. */
typedef struct AvsrPlan AvsrPlan;
int avsr_plan_create(const AvsrEncoderConfig *cfg, const void *prepared, int B, int T, void *workspace,
                     size_t workspace_bytes, int precision, void *stream, AvsrPlan **plan);
int avsr_plan_forward(AvsrPlan *plan, const float *xs, const int32_t *lengths, float *out, void *stream);
void avsr_plan_destroy(AvsrPlan *plan);

/* layer-0 residual-stage taps for parity debugging: after avsr_encoder_forward with taps enabled the
 * 5 stage outputs of layer 0 (conformer_encoder.py:110-162) are copied to `taps` (5, B*T, d_model). */
int avsr_encoder_forward_taps(const AvsrEncoderConfig *cfg, const void *prepared, const float *xs,
                              const int32_t *lengths, int B, int T, float *out, float *taps,
                              void *workspace, size_t workspace_bytes, int precision, void *stream);

/* ---- per-op entry points (unit parity) --------------------------------------------------------- */

/* LayerNorm(d, eps=1e-12) over the last dim (transformer/layer_norm.py:12-33).  rows x d. */
int avsr_layernorm(const float *x, const float *gamma, const float *beta, float *y, int rows, int d,
                   void *stream);

/* torch.nn.Linear: y = x W^T + b, optionally ReLU (positionwise_feed_forward.py:30) and/or
 * y = resid + alpha*y (conformer_encoder.py:115,140,150,158).  x (rows,k); w (n,k); bias (n) or NULL;
 * resid (rows,n) or NULL (may alias y).  All tensors fp32; for AVSR_PREC_F16 / BF16 x and w are first converted
 * to half / bfloat16 into `workspace` (>= avsr_linear_workspace_bytes), for AVSR_PREC_TF32 the tensor core truncates them. */
size_t avsr_linear_workspace_bytes(int rows, int n, int k, int precision);
int avsr_linear(const float *x, const float *w, const float *bias, const float *resid, float alpha,
                int relu, float *y, int rows, int n, int k, int precision, void *workspace,
                size_t workspace_bytes, void *stream);

/* A projection GEMM exactly as the encoder runs it: x and w ALREADY in `precision`'s operand storage (fp32 for
 * FP32/TF32, IEEE half for F16, bfloat16 for BF16); y = [resid + alpha *] act(x W^T + b), stored as an operand (y_is_operand != 0,
 * e.g. the FFN hidden) or as fp32 (the residual stream).  Used by bench.py / the tile sweep to time the dominant
 * kernel in isolation (roofline), not by the modules. */
int avsr_linear_operands(const void *x_op, const void *w_op, const float *bias, const float *resid, float alpha,
                         void *y, int rows, int n, int k, int relu, int y_is_operand, int precision, void *stream);
/* The same with the split workspace the encoder gives its residual-stream GEMMs, so that one GEMM takes the schedule
 * decision it takes inside the forward (stream-K or split-K when y is fp32, resid != NULL and relu == 0):
 * partial: 8 x rows x n fp32 scratch; counters: 4096 ints, zero on entry (the kernel leaves them zero again). */
int avsr_linear_operands_split(const void *x_op, const void *w_op, const float *bias, const float *resid,
                               float alpha, void *y, int rows, int n, int k, int relu, int y_is_operand,
                               int precision, float *partial, int *counters, void *stream);

/* RelPositionMultiHeadedAttention core (transformer/attention.py:174-189 + :59-82), d_k = 64:
 *   scores[b,h,i,j] = ((q_i+u_h).k_j + (q_i+v_h).p_h[rel=i-j]) / 8, key mask j >= lengths[b],
 *   softmax over j (fully masked row -> zeros), ctx = attn @ v.
 *   q,k,v (B,T,H*64) already projected (biases added); p (2T-1, H*64) = linear_pos(pos_emb), row m <-> rel=T-1-m;
 *   u,v_bias (H,64); ctx (B,T,H*64).  workspace >= avsr_attention_workspace_bytes(B,T,H). */
size_t avsr_attention_workspace_bytes(int B, int T, int H);
int avsr_relpos_attention(const float *q, const float *k, const float *v, const float *p,
                          const float *pos_bias_u, const float *pos_bias_v, const int32_t *lengths,
                          float *ctx, int B, int T, int H, void *workspace, size_t workspace_bytes,
                          int precision, void *stream);

/* Depthwise Conv1d(C, C, K, padding=(K-1)/2, groups=C) + BatchNorm1d(eval) + SiLU over (B,T,C)
 * (conformer_encoder.py:33 with :25-28); zero 'same' padding per utterance row, no length mask.
 *   w (C,1,K) reference layout; everything else (C).  workspace >= (K+2)*C floats (folded taps/scale/shift). */
int avsr_dwconv_bn_silu(const float *x, const float *w, const float *b, const float *bn_w,
                        const float *bn_b, const float *bn_mean, const float *bn_var, float *y, int B,
                        int T, int C, int K, void *workspace, size_t workspace_bytes, void *stream);

/* pointwise_cov1 + GLU (conformer_encoder.py:32): y = glu(x W^T + b) over channels, W (2C, C[,1]), b (2C),
 * x (rows, C) -> y (rows, C).  workspace >= avsr_pointwise_glu_workspace_bytes (interleaved W, b; converted x). */
size_t avsr_pointwise_glu_workspace_bytes(int rows, int C);
int avsr_pointwise_glu(const float *x, const float *w, const float *b, float *y, int rows, int C,
                       void *workspace, size_t workspace_bytes, int precision, void *stream);

/* pos_emb table of RelPositionalEncoding (transformer/embedding.py:139-184): (2T-1, d) fp32, row m = sinusoid(T-1-m). */
int avsr_rel_sinusoid_table(float *pe, int T, int d, void *stream);

/* ---- the step behind the encoder (SURVEY.md 8f #1) ------------------------------------------------------------
 * CTC.log_softmax / CTC.argmax (espnet/nets/pytorch_backend/ctc.py:77-93) over logits that avsr_linear produced
 * (ctc_lo: Linear(768 -> odim), ctc.py:21): y[r, 0..n) = x[r, 0..n) - logsumexp(x[r, 0..n)), argmax[r] = first index
 * of the row maximum.  x has row stride ldx >= n (the GEMM output may be padded), y row stride ldy >= n; y or argmax
 * may be NULL (not both). */
int avsr_log_softmax(const float *x, long ldx, float *y, long ldy, int32_t *argmax, int rows, int n, void *stream);

/* Prepared weights of the two projections: proj_encoder = torch.nn.Linear(idim, d_model)
 * (e2e_asr_conformer.py:31) and ctc.ctc_lo = torch.nn.Linear(d_model, odim) (ctc.py:21), converted ONCE to the
 * precision's operand storage: proj both plain and pre-multiplied by sqrt(d_model) (the encoder's embed scale,
 * transformer/embedding.py:178), ctc_lo with odim padded to a multiple of 512 zero rows.  idim % 8 == 0.
 * proj_w (d_model, idim), proj_b (d_model), ctc_w (odim, d_model), ctc_b (odim): fp32 device pointers; one of the two
 * pairs may be NULL (a module that owns only that projection prepares its half). */
size_t avsr_head_prepared_bytes(const AvsrEncoderConfig *cfg, int idim, int odim);
int avsr_prepare_head(const AvsrEncoderConfig *cfg, int idim, int odim, const float *proj_w, const float *proj_b,
                      const float *ctc_w, const float *ctc_b, void *prepared_head, size_t prepared_bytes,
                      int precision, void *stream);

/* E2E's inference path from front-end features to CTC log-probabilities in ONE call
 * (e2e_asr_conformer.py:70-71 + ctc.py:77-84; lightning.py:70-72 for B = 1, lengths NULL):
 *   x = proj_encoder(feats) * sqrt(d) -> written by the GEMM epilogue straight into the residual stream,
 *   12 x EncoderLayer, after_norm -> enc_out (B,T,d_model) fp32 (NULL: not needed) AND ctc_lo's fp16 operand,
 *   ctc_lo GEMM into fp32 logits, one row-wise log-softmax pass -> logp (B,T,odim) fp32,
 *   argmax (B*T) int32 greedy ids (either may be NULL, not both).
 * feats (B,T,idim) fp32.  workspace >= avsr_head_workspace_bytes. */
size_t avsr_head_workspace_bytes(const AvsrEncoderConfig *cfg, int B, int T, int idim, int odim);
int avsr_features_to_logprobs(const AvsrEncoderConfig *cfg, const void *prepared, const void *prepared_head,
                              const float *feats, const int32_t *lengths, int B, int T, int idim, int odim,
                              float *enc_out, float *logp, int32_t *argmax, void *workspace,
                              size_t workspace_bytes, int precision, void *stream);

/* avsr_features_to_logprobs replayed from a CUDA graph (fixed B, T).  The plan bakes in `workspace`
 * (>= avsr_head_plan_workspace_bytes) AND the output buffers given at creation: every avsr_head_plan_forward copies the
 * features into the plan's staging buffer, replays the graph and leaves its results in those same enc_out / logp /
 * argmax buffers (enc_out / argmax may be NULL).  Destroy with avsr_plan_destroy. */
size_t avsr_head_plan_workspace_bytes(const AvsrEncoderConfig *cfg, int B, int T, int idim, int odim);
int avsr_head_plan_create(const AvsrEncoderConfig *cfg, const void *prepared, const void *prepared_head, int B, int T,
                          int idim, int odim, float *enc_out, float *logp, int32_t *argmax, void *workspace,
                          size_t workspace_bytes, int precision, void *stream, AvsrPlan **plan);
int avsr_head_plan_forward(AvsrPlan *plan, const float *feats, const int32_t *lengths, void *stream);

/* The two projections on their own, on the prepared weights (what the ProjEncoder / CTC drop-in modules call when the
 * reference's E2E.forward drives them one by one): y = feats Wp^T + bp (rows, d_model) fp32, workspace >= rows*idim*4;
 * logp / argmax = log_softmax / arg max of hs Wc^T + bc over odim, hs (rows, d_model) fp32 = the encoder output,
 * workspace >= avsr_ctc_workspace_bytes. */
int avsr_proj_encoder(const AvsrEncoderConfig *cfg, const void *prepared_head, const float *feats, int rows, int idim,
                      int odim, float *y, void *workspace, size_t workspace_bytes, int precision, void *stream);
size_t avsr_ctc_workspace_bytes(const AvsrEncoderConfig *cfg, int rows, int odim);
int avsr_ctc_logprobs(const AvsrEncoderConfig *cfg, const void *prepared_head, const float *hs, int rows, int idim,
                      int odim, float *logp, int32_t *argmax, void *workspace, size_t workspace_bytes,
                      int precision, void *stream);

/* ---- training slice (SURVEY.md 8f #2, first slice) ------------------------------------------------------------
 * Backward of the HBM-bound kernels and what a Linear's backward needs around the tensor-core GEMMs (dgrad / wgrad are
 * avsr_linear_operands on transposed operands: avsr_linear_bwd).  What they replace is torch.autograd's backward of layer_norm.py:21,
 * positionwise_feed_forward.py:28-30 and conformer_encoder.py:30-35 under lightning.py:86-94.  All fp32; every
 * cross-row reduction is two-stage with a fixed order (deterministic).  workspace >= avsr_train_workspace_bytes. */
size_t avsr_train_workspace_bytes(int rows, int d, int K);
/* LayerNorm(d, eps 1e-12) backward: dx (rows,d), dgamma (d), dbeta (d) from x, gamma, dy (mean / rstd recomputed) */
int avsr_layernorm_bwd(const float *x, const float *gamma, const float *dy, float *dx, float *dgamma, float *dbeta,
                       int rows, int d, void *workspace, size_t workspace_bytes, void *stream);
/* out[c] = sum over rows of y[r][c] (bias gradients) */
int avsr_colsum(const float *y, float *out, int rows, int cols, void *workspace, size_t workspace_bytes, void *stream);
/* fp32 (rows, cols) -> a GEMM operand: AVSR_PREC_FP32 a plain fp32 copy, AVSR_PREC_BF16 converted to bf16; other
 * precisions are refused.  Transposed, dst (cols, ld_dst >= rows) with dst[c][r] = src[r][c]; else dst
 * (rows, ld_dst >= cols).  The padding columns are written as zeros.  The backward's dgrad / wgrad operands,
 * transposed, padded and converted in one pass for avsr_linear_operands. */
int avsr_pack_operand(const float *src, void *dst, int rows, int cols, long ld_dst, int transpose, int precision,
                      void *stream);
/* Both GEMMs of a Linear's backward in one call: dx (rows, k) = dy w and dw (n, k) = dy^T x, for dy (rows, n),
 * x (rows, k), w (n, k), all fp32; dx or dw may be NULL (not wanted).  precision: AVSR_PREC_FP32, AVSR_PREC_TF32 or
 * AVSR_PREC_BF16 (AVSR_PREC_F16 is refused: gradients overflow its range).  The operands are packed with
 * avsr_pack_operand into the workspace (>= avsr_linear_bwd_workspace_bytes), K zero-padded to 128 bytes (TF32 ones as
 * unrounded fp32), then avsr_linear_operands runs on them; an fp32 / TF32 dy whose n is a multiple of 32 is read in
 * place. */
size_t avsr_linear_bwd_workspace_bytes(int rows, int n, int k, int precision);
int avsr_linear_bwd(const float *dy, const float *x, const float *w, float *dx, float *dw, int rows, int n, int k,
                    int precision, void *workspace, size_t workspace_bytes, void *stream);
/* dx = dy * (y > 0) */
int avsr_relu_bwd(const float *y, const float *dy, float *dx, long n, void *stream);
/* F.glu over channels (conformer_encoder.py:32): in (rows, 2C) -> y (rows, C); and its backward din (rows, 2C) */
int avsr_glu_fwd(const float *in, float *y, long rows, int C, void *stream);
int avsr_glu_bwd(const float *in, const float *dy, float *din, long rows, int C, void *stream);
/* depthwise Conv1d(C,C,K,groups=C) of the conformer conv module (conformer_encoder.py:33), its training BatchNorm1d
 * being the avsr_bn_train_* entries below.
 *   avsr_dwconv_raw      y = conv(x) + b, raw fp32 (flip != 0: taps reversed, b may be NULL = the input gradient)
 *   avsr_dwconv_wgrad    dw (C,1,K), db (C) */
int avsr_dwconv_raw(const float *x, const float *w, const float *b, float *y, int B, int T, int C, int K, int flip,
                    void *workspace, size_t workspace_bytes, void *stream);
int avsr_dwconv_wgrad(const float *x, const float *dconv, float *dw, float *db, int B, int T, int C, int K,
                      void *workspace, size_t workspace_bytes, void *stream);

/* ---- BatchNorm with batch statistics (training), shared by the conformer conv module and the ResNet front-ends, in
 * the pieces a (Sync)BatchNorm needs: the statistics and the backward sums leave the library between the pieces, so
 * that the host can gather / all-reduce them over the ranks (train.py:31 sync_batchnorm=True).  z, y, dy, resid, dz,
 * dres are DEVICE fp32 (rows, C); the workspace is >= avsr_bn_train_workspace_bytes(rows, C).
 *   avsr_bn_train_stats     stats (3, C) fp64 = each channel's (count, mean, M2) over the rows: per-tile two-pass sums,
 *                           merged in a fixed order with Chan's formula.  avsr_frontend_train_conv_fwd computes the
 *                           same for its output.
 *   avsr_bn_train_finalize  stats (ranks, 3, C), merged in rank order -> mean, invstd = 1 / sqrt(biased var + eps) (C
 *                           fp32).  When running_mean / running_var are given they become (1 - factor) * old + factor *
 *                           (mean, unbiased var).
 *   avsr_bn_train_act_fwd   y = [SiLU]((z - mean) * invstd * gamma + beta [+ resid]); resid may be NULL
 *   avsr_bn_train_bwd_sums  sums (2, C) = [sum ds, sum ds * x_hat] with ds = dL/d(BatchNorm output) (dy through the
 *                           SiLU when act), summed in a fixed order
 *   avsr_bn_train_bwd_dx    dz = gamma * invstd * (ds - inv_count * (sums[0] + x_hat * sums[1])) and, when dres is
 *                           given, dres = ds (the residual's gradient); sums and inv_count over all ranks */
size_t avsr_bn_train_workspace_bytes(long rows, int C);
int avsr_bn_train_stats(const float *z, long rows, int C, double *stats, void *workspace, size_t workspace_bytes,
                        void *stream);
int avsr_bn_train_finalize(const double *stats, int ranks, int C, double eps, double factor, float *running_mean,
                           float *running_var, float *mean, float *invstd, void *stream);
int avsr_bn_train_act_fwd(const float *z, const float *mean, const float *invstd, const float *gamma, const float *beta,
                          const float *resid, int act, float *y, long rows, int C, void *stream);
int avsr_bn_train_bwd_sums(const float *z, const float *dy, const float *mean, const float *invstd, const float *gamma,
                           const float *beta, const float *resid, int act, float *sums, long rows, int C,
                           void *workspace, size_t workspace_bytes, void *stream);
int avsr_bn_train_bwd_dx(const float *z, const float *dy, const float *mean, const float *invstd, const float *gamma,
                         const float *beta, const float *resid, int act, const float *sums, float inv_count, float *dz,
                         float *dres, long rows, int C, void *stream);

/* Backward of the rel-pos attention core (avsr_relpos_attention; transformer/attention.py:174-189 + :59-82), fp32:
 * from q, k, v (B,T,H*64: the projected tensors, biases included), p (2T-1, H*64), pos_bias_u / v (H,64), lengths, the
 * forward's ctx and the incoming dctx (B,T,H*64) it returns dk, dv, dp and dq in two parts -- dq = dq_k + dq_p, whose
 * column sums over (b, t) are the gradients of pos_bias_u and pos_bias_v.  Scores are recomputed (nothing of size T^2
 * is stored); every output element is written by one warp (no atomics). */
size_t avsr_relpos_attention_bwd_workspace_bytes(int B, int T, int H);
int avsr_relpos_attention_bwd(const float *q, const float *k, const float *v, const float *p, const float *pos_bias_u,
                              const float *pos_bias_v, const int32_t *lengths, const float *ctx, const float *dctx,
                              float *dq_k, float *dq_p, float *dk, float *dv, float *dp, int B, int T, int H,
                              void *workspace, size_t workspace_bytes, void *stream);

/* The same backward on the tensor cores (wgmma), replacing the same reference lines
 * (transformer/attention.py:174-189 + :59-82): the arguments and outputs of avsr_relpos_attention_bwd, plus
 * `precision`, which must be AVSR_PREC_BF16 (bf16 operands, fp32 accumulation; any other value is an error naming it).
 * q+u, q+v, k, v, dctx and p are converted to bf16 head-major copies in the workspace; Delta is computed in fp32 from
 * ctx and dctx; the backward computes its own row log-sum-exp from the bf16 operands.  Scores are recomputed (nothing
 * of size T^2 is stored), no atomics, every sum in a fixed order: repeated calls are bit-identical.
 * avsr_relpos_attention_bwd_tc_workspace_bytes returns 0 for a precision other than AVSR_PREC_BF16. */
size_t avsr_relpos_attention_bwd_tc_workspace_bytes(int B, int T, int H, int precision);
int avsr_relpos_attention_bwd_tc(const float *q, const float *k, const float *v, const float *p, const float *pos_bias_u,
                                 const float *pos_bias_v, const int32_t *lengths, const float *ctx, const float *dctx,
                                 float *dq_k, float *dq_p, float *dk, float *dv, float *dp, int B, int T, int H,
                                 int precision, void *workspace, size_t workspace_bytes, void *stream);

/* CTC loss of the head (espnet/nets/pytorch_backend/ctc.py:32-65: CTC.forward -> loss_fn):
 * torch.nn.CTCLoss(reduction="none", zero_infinity=True), blank 0, on log_softmax of the logits, per utterance.
 *   logits  (B*Tmax, ld) fp32 = ctc_lo(hs_pad), rows r = b*Tmax + t; the first odim columns are the vocabulary
 *   hlens   (B) int32 frames per utterance;  ys_pad (B, Lmax) int64 padded label rows: every entry equal to ignore_id is
 *           dropped wherever it sits (ctc.py:52, y[y != ignore_id]); the rows are compacted on the device
 *   nll     (B) fp32 negative log-likelihoods (0 where it is +inf: zero_infinity)
 * The forward leaves in `state` (>= avsr_ctc_loss_state_bytes) what the backward needs: the compacted labels, the
 * per-frame log-sum-exp, the log-probs of blank and of the labels, alpha and -- want_grad != 0 only -- beta.  The
 * backward writes dlogits (B*Tmax, ldd >= odim) = dnll[b] * d nll_b / d logits: 0 on frames t >= hlens[b], on columns
 * [odim, ldd) and on utterances whose nll is +inf.  dnll (B) is a DEVICE array (nothing is read on the host).
 * A label outside [1, odim) or hlens[b] outside [0, Tmax] makes that utterance's nll NaN.  Lmax <= 1024.  Every sum has
 * a fixed order: repeated calls give identical bits. */
size_t avsr_ctc_loss_state_bytes(int B, int Tmax, int Lmax);
int avsr_ctc_loss_fwd(const float *logits, long ld, const int32_t *hlens, const int64_t *ys_pad, int B, int Tmax,
                      int Lmax, int odim, int ignore_id, int want_grad, float *nll, void *state, size_t state_bytes,
                      void *stream);
int avsr_ctc_loss_bwd(const float *logits, long ld, const int32_t *hlens, const int64_t *ys_pad, int B, int Tmax,
                      int Lmax, int odim, const float *dnll, const void *state, size_t state_bytes, float *dlogits,
                      long ldd, void *stream);

/* ---- teacher-forced training pass of the attention decoder (transformer_decoder.py:229-258) ------------------------
 * Masked multi-head attention core (transformer/attention.py:59-88), d_k = 64, fp32:
 *   q (B, Lq, H*64) row stride ldq, k / v (B, Lk, H*64) row strides ldk / ldv (multiples of 4, 16-byte aligned bases:
 *   the fused self q|k|v and source k|v GEMM outputs are read in place).  Query row i of utterance b sees keys
 *   j < min(key_lengths[b], Lk) (key_lengths NULL = all) and, when causal != 0, j <= i.  keep (B, H, Lq, Lk) uint8 or
 *   NULL: dropout on the probabilities, kept entries scaled by keep_scale = 1 / (1 - p).
 *   fwd: ctx (B, Lq, H*64) contiguous; probs (B, H, Lq, Lk) fp32 post-softmax, pre-dropout (0 on masked keys), or NULL
 *        when no backward follows.  A row that sees no key gives ctx 0.
 *   bwd: from probs, keep and dctx (B, Lq, H*64) contiguous -> dq (row stride lddq), dk and dv (row stride lddkv):
 *        dS = P o (dP - rowsum(dP o P)) / 8.  workspace >= avsr_mha_core_bwd_workspace_bytes.
 * Label smoothing (transformer/label_smoothing_loss.py:41-63, KLDivLoss against the smoothed target, per row):
 *   logits (rows, ld) fp32, the first odim columns the vocabulary; target (rows) int64, ignore_id rows give 0, a target
 *   outside [0, odim) that is not ignore_id gives NaN.  fwd -> row_loss (rows) and lse (rows, kept for the backward);
 *   bwd -> dlogits (rows, ldd) = *dscale * (softmax - smoothed target), 0 on ignored rows and on columns [odim, ldd).
 *   dscale is a DEVICE scalar.
 * Embedding + positional encoding (embedding.py:60-90): x (rows, D) = embed[tokens] * sqrt(D) + pe(row mod L); a token
 *   outside [0, odim) gives a NaN row.  bwd: dembed (odim, D) dense, positions grouped by token on the device and summed
 *   in position order (rows of unused tokens 0).
 * Every output element has one writer and a fixed summation order: repeated calls give identical bits. */
int avsr_mha_core_fwd(const float *q, long ldq, const float *k, long ldk, const float *v, long ldv, int B, int H, int Lq,
                      int Lk, int causal, const int32_t *key_lengths, const uint8_t *keep, float keep_scale, float *ctx,
                      float *probs, void *stream);
size_t avsr_mha_core_bwd_workspace_bytes(int B, int H, int Lq);
int avsr_mha_core_bwd(const float *q, long ldq, const float *k, long ldk, const float *v, long ldv, int B, int H, int Lq,
                      int Lk, int causal, const int32_t *key_lengths, const uint8_t *keep, float keep_scale,
                      const float *probs, const float *dctx, float *dq, long lddq, float *dk, float *dv, long lddkv,
                      void *workspace, size_t workspace_bytes, void *stream);
/* The same backward on the tensor cores (wgmma): the arguments and outputs of avsr_mha_core_bwd, plus ctx (B, Lq, H*64)
 * contiguous, the forward's output, and `precision`, which must be AVSR_PREC_BF16 (bf16 operands, fp32 accumulation;
 * any other value is an error naming it).  Delta = rowsum(dctx o ctx) is computed in fp32; the stored probabilities are
 * read tile by tile (nothing is recomputed).  Row strides, dq / dk / dv strides included, are multiples of 4 and
 * >= H*64; q / k / v / ctx / dctx / dq / dk / dv are 16-byte aligned.  Two launches, no atomics, every sum in a fixed
 * order: repeated calls are bit-identical.  Keys at or past the key length, and a zero-length utterance, get exact zeros.
 * avsr_mha_core_bwd_tc_workspace_bytes returns 0 for a precision other than AVSR_PREC_BF16. */
size_t avsr_mha_core_bwd_tc_workspace_bytes(int B, int H, int Lq, int Lk, int precision);
int avsr_mha_core_bwd_tc(const float *q, long ldq, const float *k, long ldk, const float *v, long ldv, int B, int H,
                         int Lq, int Lk, int causal, const int32_t *key_lengths, const uint8_t *keep, float keep_scale,
                         const float *probs, const float *ctx, const float *dctx, float *dq, long lddq, float *dk,
                         float *dv, long lddkv, int precision, void *workspace, size_t workspace_bytes, void *stream);
int avsr_label_smoothing_fwd(const float *logits, long ld, const int64_t *target, int rows, int odim, int ignore_id,
                             float smoothing, float *row_loss, float *lse, void *stream);
int avsr_label_smoothing_bwd(const float *logits, long ld, const int64_t *target, int rows, int odim, int ignore_id,
                             float smoothing, const float *lse, const float *dscale, float *dlogits, long ldd,
                             void *stream);
int avsr_embed_fwd(const int64_t *tokens, const float *embed, int rows, int L, int D, int odim, float *x, void *stream);
size_t avsr_embed_bwd_workspace_bytes(int rows, int odim);
int avsr_embed_bwd(const int64_t *tokens, const float *dx, int rows, int D, int odim, float *dembed, void *workspace,
                   size_t workspace_bytes, void *stream);

/* ---- on-device collate (SURVEY.md 8f #4) ------------------------------------------------------------------------
 * datamodule/data_module.py:10-41 (`pad` / `collate_pad`) on the GPU: the utterances of a max-frames bucket lie back to
 * back in `flat` (sum of lengths rows x d; offsets[B+1] int64 DEVICE prefix sums), the zero-padded (B, Tmax, d) batch and
 * its int32 lengths are formed on the device; avsr_unpack_padded is the inverse (valid rows only). */
int avsr_pack_padded(const float *flat, const int64_t *offsets, float *out, int32_t *lengths_out, int B, int Tmax, int d,
                     float pad_value, void *stream);
int avsr_unpack_padded(const float *padded, const int64_t *offsets, float *flat, int B, int Tmax, int d, void *stream);

/* ---- attention-decoder scoring path + CTC prefix scorer (SURVEY.md 8f #3) ----------------------------------------------
 * What the reference's BatchBeamSearch asks of its two scorers at every step (espnet/nets/batch_beam_search.py:208-285):
 *   TransformerDecoder.batch_score -> forward_one_step  (espnet/nets/pytorch_backend/decoder/transformer_decoder.py:260-334,
 *                                                        DecoderLayer.forward :63-140; 6 pre-norm layers, d 768, ff 3072)
 *   CTCPrefixScorer.batch_score_partial -> CTCPrefixScoreTH.__call__  (espnet/nets/scorers/ctc.py:99-130,
 *                                                        espnet/nets/ctc_prefix_score.py:72-200)
 * The reference keeps every layer's OUTPUT per hypothesis and re-projects K/V of the whole prefix and of the whole
 * encoder memory at every step; here K/V are projected once into a per-utterance SESSION buffer the caller owns:
 * source-attention K|V of all layers at avsr_decoder_begin, self-attention q|k|v of a position when it is decoded,
 * addressed (layer, position, beam slot).  A hypothesis is the list of slots of its prefix: re-ordering the beam copies
 * nothing. */
typedef struct AvsrDecoderConfig {
  int32_t d_model;       /* 768 (e2e_asr_conformer.py:41-47) */
  int32_t n_heads;       /* 12 */
  int32_t linear_units;  /* 3072 */
  int32_t num_blocks;    /* 6 (<= 16) */
  int32_t odim;          /* vocabulary, 5049 */
} AvsrDecoderConfig;

/* One DecoderLayer's parameters under the reference's names (transformer_decoder.py:36-61): Linear weights (out, in). */
typedef struct AvsrDecoderLayerParams {
  const float *self_q_w, *self_q_b, *self_k_w, *self_k_b, *self_v_w, *self_v_b, *self_out_w, *self_out_b;
  const float *src_q_w, *src_q_b, *src_k_w, *src_k_b, *src_v_w, *src_v_b, *src_out_w, *src_out_b;
  const float *ff_w1, *ff_b1, *ff_w2, *ff_b2;
  const float *norm1_w, *norm1_b, *norm2_w, *norm2_b, *norm3_w, *norm3_b;
} AvsrDecoderLayerParams;

/* One-off layout step (after every parameter update): self q|k|v and source k|v weights concatenated, GEMM weights in the
 * precision's operand storage, output_layer padded to a multiple of 64 rows.  `layers` is a HOST array of num_blocks
 * structs of DEVICE pointers; embed_w (odim, d) = embed.0.weight, out_w (odim, d) / out_b = output_layer. */
size_t avsr_decoder_prepared_bytes(const AvsrDecoderConfig *cfg);
int avsr_prepare_decoder(const AvsrDecoderConfig *cfg, const AvsrDecoderLayerParams *layers, const float *embed_w,
                         const float *after_norm_w, const float *after_norm_b, const float *out_w, const float *out_b,
                         void *prepared, size_t prepared_bytes, int precision, void *stream);

/* Utterance start (what batch_init_state + the first batch_score do in the reference): K|V of `memory` (T, d_model) fp32 =
 * the encoder output, for the source attention of every layer.  The session holds up to max_steps positions x max_hyps
 * beam slots. */
size_t avsr_decoder_session_bytes(const AvsrDecoderConfig *cfg, int T, int max_steps, int max_hyps);
int avsr_decoder_begin(const AvsrDecoderConfig *cfg, const void *prepared, const float *memory, int T, int max_steps,
                       int max_hyps, void *session, size_t session_bytes, int precision, void *stream);

/* One step of TransformerDecoder.batch_score for n <= max_hyps hypotheses of equal length step + 1:
 *   tokens (n) int32 DEVICE   the last token of each hypothesis (yseq[:, -1]); hypothesis i occupies beam slot i of
 *                             position `step`
 *   anc (step, n) int32 DEVICE  anc[s][i] = beam slot that holds position s < step of hypothesis i's prefix (NULL at step 0)
 *   logp (n, odim) fp32        log_softmax(output_layer(after_norm(x_last)))  -- transformer_decoder.py:283-289
 * workspace >= avsr_decoder_step_workspace_bytes. */
size_t avsr_decoder_step_workspace_bytes(const AvsrDecoderConfig *cfg, int T, int max_steps, int max_hyps);
int avsr_decoder_step(const AvsrDecoderConfig *cfg, const void *prepared, void *session, size_t session_bytes, int T,
                      int max_steps, int max_hyps, const int32_t *tokens, const int32_t *anc, int step, int n, float *logp,
                      void *workspace, size_t workspace_bytes, int precision, void *stream);

/* CTCPrefixScoreTH for ONE utterance (batch 1, no windowing).  logp (T, O) fp32 CTC log-posteriors (ctc.log_softmax);
 * forward variables use the reference's stacked layouts: r_prev (T, 2, n), r (T, 2, n, S), index 0 = prefix ends in a
 * non-blank, 1 = in blank; logzero = -1e10.
 *   avsr_ctc_prefix_init    r0 (T, 2): state of the empty prefix (ctc_prefix_score.py:87-98); its prefix score is 0
 *   avsr_ctc_prefix_score   one __call__: out_len = tokens after <sos>, last_ids (n) int32, s_prev (n), cand (n, S) int32
 *                           candidate ids (the pre-beam, unique per row) -> local (n, O) = log_psi - s_prev (logzero off the
 *                           candidates, <eos> = total prefix probability, blank = logzero), r, log_psi (n, O)
 *   avsr_ctc_prefix_select  CTCPrefixScorer.select_state for the m kept (parent, token) pairs: r_next (T, 2, m), s_next (m) */
int avsr_ctc_prefix_init(const float *logp, int T, int O, int blank, float *r0, void *stream);
int avsr_ctc_prefix_score(const float *logp, int T, int O, int blank, int eos, int out_len, const int32_t *last_ids,
                          const float *r_prev, const float *s_prev, const int32_t *cand, int n, int S, float *local,
                          float *r, float *log_psi, void *stream);
int avsr_ctc_prefix_select(const float *r, const float *log_psi, const int32_t *cand, const int32_t *parent,
                           const int32_t *token, int T, int O, int n, int S, int m, float *r_next, float *s_next,
                           void *stream);

/* ---- U utterances decoded in lock-step (one beam search over a batch) ----------------------------------------------
 * A batch session holds the source K|V of U utterances packed frame after frame, (L, sum T_u, 2d), with their frame
 * offsets and lengths, and the self-attention slots as above with max_hyps = U x beam slots.  Row i of a step belongs
 * to utterance row_utt[i]; rows may come in any order and take beam slot i of the position being decoded.  A row's
 * log-probabilities have the bits of the same hypothesis scored in a one-utterance session.
 *   lengths (U) int32 HOST      frames of each utterance, 1 <= T_u <= T_max; pass the same array to begin and every step
 *   memory (U, T_max, d) fp32   encoder output, utterance u's first T_u frames read
 *   row_utt (n) int32 DEVICE    utterance of each row, in 0..U-1 (not checked per call)
 * The workspace is the one-utterance step's at T = T_max. */
size_t avsr_decoder_batch_session_bytes(const AvsrDecoderConfig *cfg, int U, const int32_t *lengths, int max_steps,
                                        int max_hyps);
size_t avsr_decoder_batch_step_workspace_bytes(const AvsrDecoderConfig *cfg, int T_max, int max_steps, int max_hyps);
int avsr_decoder_batch_begin(const AvsrDecoderConfig *cfg, const void *prepared, const float *memory,
                             const int32_t *lengths, int U, int T_max, int max_steps, int max_hyps, void *session,
                             size_t session_bytes, int precision, void *stream);
int avsr_decoder_batch_step(const AvsrDecoderConfig *cfg, const void *prepared, void *session, size_t session_bytes,
                            const int32_t *lengths, int U, int T_max, int max_steps, int max_hyps, const int32_t *tokens,
                            const int32_t *anc, const int32_t *row_utt, int step, int n, float *logp, void *workspace,
                            size_t workspace_bytes, int precision, void *stream);

/* CTCPrefixScoreTH over U utterances with xlens (ctc_prefix_score.py:21-54): logp (U, T_max, O) fp32, row_utt (n) int32
 * DEVICE.  r0 (T_max, 2, U); r_prev (T_max, 2, n); r (T_max, 2, n, S).  A row's recursion stops at its utterance's T_u,
 * <eos> reads frame T_u - 1, and state entries at frames >= T_u are logzero.  avsr_ctc_prefix_select carries the states
 * over with T = T_max.
 *   avsr_ctc_prefix_batch_init   lengths (U) int32 HOST, checked (1..T_max); writes their device copy to lengths_dev (U)
 *   avsr_ctc_prefix_batch_score  lengths_dev = the device copy batch_init wrote for the same logp */
int avsr_ctc_prefix_batch_init(const float *logp, const int32_t *lengths, int U, int T_max, int O, int blank,
                               int32_t *lengths_dev, float *r0, void *stream);
int avsr_ctc_prefix_batch_score(const float *logp, const int32_t *lengths_dev, int U, int T_max, int O, int blank, int eos,
                                int out_len, const int32_t *last_ids, const float *r_prev, const float *s_prev,
                                const int32_t *cand, const int32_t *row_utt, int n, int S, float *local, float *r,
                                float *log_psi, void *stream);

/* ---- ResNet front-ends, inference (eval-mode BatchNorm): Conv3dResNet (frontend/resnet.py:176-233) and
 * Conv1dResNet (frontend/resnet1d.py:204-234) with relu_type "swish".  Activations are channels-last in the precision's
 * operand storage: (frames, H, W, C) for video, (utterances, L, C) for audio.  AVSR_PREC_TF32, F16 and BF16 run the
 * trunk convolutions and both stems as implicit GEMMs on wgmma; AVSR_PREC_FP32 runs a CUDA-core direct convolution
 * (the exact reference path). */
enum { AVSR_FRONTEND_VIDEO = 0, AVSR_FRONTEND_AUDIO = 1 };
#define AVSR_FRONTEND_CONVS 20

/* One convolution and the BatchNorm after it, as the module holds them (DEVICE fp32, contiguous): conv_w is
 * (C_out, C_in, [KT,] [KH,] KW); the BatchNorm's weight, bias, running_mean, running_var are (C_out); eps is the module's. */
typedef struct AvsrConvBnParams {
  const float *conv_w;
  const float *bn_w;
  const float *bn_b;
  const float *bn_mean;
  const float *bn_var;
  double eps;
} AvsrConvBnParams;

/* params: HOST array of AVSR_FRONTEND_CONVS entries in the reference's state-dict order (the stem, then per
 * BasicBlock conv1, conv2 and, in the first block of layer2..4, downsample).  Weights are reordered to
 * (C_out, taps * C_in) in operand storage; BatchNorm becomes an fp32 scale and shift.  Re-run whenever a parameter or
 * running statistic changes. */
size_t avsr_frontend_prepared_bytes(int modality, int precision);
int avsr_prepare_frontend(int modality, const AvsrConvBnParams *params, void *prepared, size_t prepared_bytes,
                          int precision, void *stream);
/* video x: (B, T_in, 1, H, W) fp32 -> out (B, T_in, 512) fp32.
 * audio x: (B, T_in, 1) fp32 samples (H, W ignored) -> out (B, T_in / 640, 512) fp32.
 * Padded frames are data: the front-end takes no lengths.  Temporal taps stay inside each utterance's row. */
size_t avsr_frontend_workspace_bytes(int modality, int B, int T_in, int H, int W, int precision);
int avsr_frontend_forward(int modality, const void *prepared, const float *x, int B, int T_in, int H, int W,
                          float *out, void *workspace, size_t workspace_bytes, int precision, void *stream);
/* Stage taps for parity tests: the same forward, and taps[i] != NULL (HOST array of AVSR_FRONTEND_TAPS device
 * pointers) receives stage i as fp32, channels-last (frames or utterances, H, W, C): 0 the stem after BN + SiLU (video:
 * before the max-pool), 1 the trunk input (video: after the max-pool; audio: the stem again), 2..9 the output of each
 * BasicBlock, layer1.0 .. layer4.1.  avsr_frontend_tap_shape writes a tap's 4 dims; audio taps are (B, 1, L, C). */
#define AVSR_FRONTEND_TAPS 10
int avsr_frontend_forward_taps(int modality, const void *prepared, const float *x, int B, int T_in, int H, int W,
                               float *out, float *const *taps, void *workspace, size_t workspace_bytes, int precision,
                               void *stream);
int avsr_frontend_tap_shape(int modality, int B, int T_in, int H, int W, int tap, int dims[4]);

/* One trunk convolution + BatchNorm (as scale, shift) [+ residual] [+ SiLU] on channels-last fp32 tensors, computed in
 * `precision` (inputs converted to operand storage in the workspace): x (N, H, W, C_in), w (C_out, C_in, KH, KW) in
 * torch layout, resid / y (N, Ho, Wo, C_out).  Padding is (KH - 1) / 2, (KW - 1) / 2; audio convs are KH = H = 1. */
size_t avsr_conv_bn_act_workspace_bytes(int N, int H, int W, int C_in, int C_out, int KH, int KW, int stride,
                                        int precision);
int avsr_conv_bn_act(const float *x, const float *w, const float *scale, const float *shift, const float *resid,
                     int act, float *y, int N, int H, int W, int C_in, int C_out, int KH, int KW, int stride,
                     void *workspace, size_t workspace_bytes, int precision, void *stream);

/* ---- ResNet front-ends, training (batch-statistics BatchNorm).  Building blocks that auto_avsr_b200/frontend_train.py
 * chains per conv unit (conv -> BatchNorm -> [+ residual] -> [SiLU]); every tensor is DEVICE fp32, channels-last.
 * `stem`: 0 a trunk conv, x (N, H, W, C_in), w (C_out, C_in, KH, KW), padding (K - 1) / 2, stride 1 or 2 (audio: H = KH =
 * 1); 1 the video stem, x (N = B * T frames, H, W) with T frames per utterance, w (64, 1, 5, 7, 7); 2 the audio stem,
 * x (N, W) samples with W a multiple of 640, w (64, 1, 80).  C_in, C_out and KH, KW, stride are ignored for the stems.
 *
 * avsr_frontend_train_conv_fwd: z (output pixels, C_out) = conv(x, w) in `precision` (TF32 / F16 / BF16 on wgmma, FP32 on
 * CUDA cores), and stats (3, C_out) fp64 = each channel's (count, mean, M2) over all output pixels, merged in a fixed order
 * with Chan's formula (the avsr_bn_train_stats of z).  BatchNorm then runs on the avsr_bn_train_* entries. */
size_t avsr_frontend_train_conv_workspace_bytes(int stem, int N, int T, int H, int W, int C_in, int C_out, int KH,
                                                int KW, int stride, int precision);
int avsr_frontend_train_conv_fwd(const float *x, const float *w, float *z, double *stats, int stem, int N, int T, int H,
                                 int W, int C_in, int C_out, int KH, int KW, int stride, void *workspace,
                                 size_t workspace_bytes, int precision, void *stream);
/* Input gradient of a trunk conv: dx (N, H, W, C_in) from dz (N, Ho, Wo, C_out), one stride-1 implicit GEMM per parity
 * class of the input (TF32 / F16 / BF16 on wgmma, FP32 on CUDA cores). */
size_t avsr_frontend_train_dgrad_workspace_bytes(int N, int H, int W, int C_in, int C_out, int KH, int KW, int stride,
                                                 int precision);
int avsr_frontend_train_conv_dgrad(const float *dz, const float *w, float *dx, int N, int H, int W, int C_in, int C_out,
                                   int KH, int KW, int stride, void *workspace, size_t workspace_bytes, int precision,
                                   void *stream);
/* Weight gradient dw (torch layout, like w) = sum over output pixels of dz x im2col(x): wgmma with TF32 operands
 * (AVSR_PREC_TF32 / F16 / BF16) or fp32 on CUDA cores (AVSR_PREC_FP32); the pixel axis is split across the SMs and
 * the partials are summed in a fixed order. */
size_t avsr_frontend_train_wgrad_workspace_bytes(int stem, int N, int T, int H, int W, int C_in, int C_out, int KH,
                                                 int KW, int stride);
int avsr_frontend_train_conv_wgrad(const float *x, const float *dz, float *dw, int stem, int N, int T, int H, int W,
                                   int C_in, int C_out, int KH, int KW, int stride, void *workspace,
                                   size_t workspace_bytes, int precision, void *stream);
/* MaxPool (1,3,3) / (1,2,2) / pad (0,1,1) on (N, Hi, Wi, C): idx (N, Ho, Wo, C) records the winner dy * 3 + dx, the first
 * maximum in window scan order (a NaN wins); the backward gathers dy into each pixel from the windows that chose it. */
int avsr_frontend_train_maxpool_fwd(const float *x, float *y, uint8_t *idx, int N, int Hi, int Wi, int C, void *stream);
int avsr_frontend_train_maxpool_bwd(const float *dy, const uint8_t *idx, float *dx, int N, int Hi, int Wi, int C,
                                    void *stream);
/* out (G, C) = mean of each group of P consecutive rows of x (G * P, C); the backward broadcasts dout / P */
int avsr_frontend_train_mean_rows(const float *x, float *out, long G, int P, int C, void *stream);
int avsr_frontend_train_mean_rows_bwd(const float *dout, float *dx, long G, int P, int C, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* AVSR_B200_H_ */
