// Teacher-forced training pass of the attention decoder (espnet/nets/pytorch_backend/decoder/transformer_decoder.py:
// 229-258 and the LabelSmoothingLoss of transformer/label_smoothing_loss.py:41-63): the per-element math, written as
// AVSR_HD code so that ONE source drives both the kernels of decoder_train.cu and the host replay the CPU tests build
// (tests/emu/decoder_train_emu.cu -- test infrastructure, never loaded by the package).
//
// Masked multi-head attention core (transformer/attention.py:59-88), d_k = 64, for query row i of utterance b:
//   keys j < n_i are visible, n_i = min(key_len[b], Lk) and, when causal, min(., i + 1)   (target_mask / memory_mask)
//   s_ij = q_i . k_j / 8 ;  A_ij = softmax_j(s_i) over the visible keys, 0 elsewhere (a row with n_i = 0 is all 0, as
//   the reference's masked_fill after the softmax leaves it) ;  A'_ij = A_ij * keep_ij / (1 - p) (dropout on the
//   probabilities, keep drawn by torch) ;  ctx_i = sum_j A'_ij v_j .
// Backward, with dA_ij = (dctx_i . v_j) * keep_ij / (1 - p) and Delta_i = sum_j A_ij dA_ij :
//   dS_ij = A_ij (dA_ij - Delta_i) / 8 ;  dq_i = sum_j dS_ij k_j ;  dk_j = sum_i dS_ij q_i ;  dv_j = sum_i A'_ij dctx_i .
//
// Label smoothing (smoothing s, V = odim classes), per row r with target y_r:
//   t_c = s / (V - 1) off the target, 1 - s on it ;  loss_r = sum_c t_c (log t_c - logp_c)   (0 log 0 = 0)
//       = c0 - off * sum_c x_c - (on - off) * x_y + lse        (sum_c t_c = 1;  c0 = sum_c t_c log t_c)
//   d loss_r / d x_c = softmax_c - t_c .  Rows whose target is ignore_id give 0; a target outside [0, V) that is not
//   ignore_id makes the row NaN.
#pragma once
#include <math.h>

#include "common.cuh"
#include "decoder_body.cuh"

namespace avsr {
namespace dtr {

constexpr float kAttnScale = 0.125f;   // 1 / sqrt(d_k), d_k = 64

// ------------------------------------------------------------------ attention masks and per-element steps
// number of keys query row i of utterance b sees: keys [0, n)
AVSR_HD int attn_row_keys(int i, int Lk, int causal, const int32_t* key_len, int b) {
  int n = Lk;
  if (key_len) {
    const int l = key_len[b];
    n = l < 0 ? 0 : (l < Lk ? l : Lk);
  }
  if (causal && i + 1 < n) n = i + 1;
  return n;
}
// first query row that sees key j (the key must also lie below the key length; see attn_row_keys)
AVSR_HD int attn_first_query(int j, int causal) { return causal ? j : 0; }
// dropout factor of probability element idx: keep / (1 - p), 1 without a keep-mask
AVSR_HD float keep_factor(const uint8_t* keep, long idx, float scale) { return keep ? (keep[idx] ? scale : 0.f) : 1.f; }
// d score of one visible (i, j) pair, the 1/8 of the scores included
AVSR_HD float attn_dscore(float a, float da, float delta) { return a * (da - delta) * kAttnScale; }

// ------------------------------------------------------------------ label smoothing
struct LsConst {
  float off, on, c0;   // t_c off / on the target, c0 = sum_c t_c log t_c
};
AVSR_HD LsConst ls_const(int V, float smoothing) {
  const double s = smoothing, off = V > 1 ? s / (double)(V - 1) : 0.0, on = 1.0 - s;
  double c0 = 0.0;
  if (off > 0.0) c0 += (double)(V - 1) * off * log(off);
  if (on > 0.0) c0 += on * log(on);
  return LsConst{(float)off, (float)on, (float)c0};
}
// 0 = ignored row, 1 = valid target, -1 = target outside [0, V)
AVSR_HD int ls_row_kind(int64_t tgt, int64_t ignore_id, int V) {
  return tgt == ignore_id ? 0 : ((tgt >= 0 && tgt < V) ? 1 : -1);
}
AVSR_HD float ls_row_loss(const LsConst& k, float lse, float sum_x, float x_tgt) {
  return k.c0 - k.off * sum_x - (k.on - k.off) * x_tgt + lse;
}
AVSR_HD float ls_grad(const LsConst& k, float x, float lse, float dscale, bool is_target) {
  return dscale * (expf(x - lse) - (is_target ? k.on : k.off));
}

// ------------------------------------------------------------------ embedding + positional encoding
// x[r, c] = embed[tokens[r], c] * sqrt(d) + pe(r mod L, c) over (B*L, D); a token outside [0, odim) gives a NaN row
// (nothing is indexed with it).  Unlike the scoring step (EmbedElem) the tokens are not clamped.
struct EmbedTrainElem {
  const int64_t* tokens; const float* emb; float* x;
  int D, L, odim;
  float xscale, kf;
  AVSR_HD void operator()(long idx) const {
    const long r = idx / D;
    const int c = (int)(idx - r * D), pos = (int)(r % L);
    const int64_t tok = tokens[r];
    x[idx] = (tok < 0 || tok >= odim) ? NAN : emb[tok * D + c] * xscale + dec::pe_value(pos, c, kf);
  }
};
AVSR_HD bool embed_token_ok(int64_t tok, int odim) { return tok >= 0 && tok < odim; }

}  // namespace dtr
}  // namespace avsr
