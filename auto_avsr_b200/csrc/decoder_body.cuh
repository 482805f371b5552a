// Attention-decoder scoring path (SURVEY.md 8f #3): buffer layouts, per-element functors and the launch schedule,
// written against a small backend interface so that ONE source drives both the device library (decoder.cu: wgmma /
// CUDA-core GEMMs, the LayerNorm / log-softmax kernels of the encoder path, functors as grid kernels) and the host
// replay the CPU tests build (tests/emu/decoder_emu.cu: the same schedule and the same functors as plain loops --
// test infrastructure, never loaded by the package).
//
// What it replaces in the reference (paths relative to the reference tree):
//   TransformerDecoder.forward_one_step / batch_score  espnet/nets/pytorch_backend/decoder/transformer_decoder.py:260-334
//   DecoderLayer.forward (pre-norm, cache)              transformer_decoder.py:63-140
//   CTCPrefixScoreTH.__call__                           espnet/nets/ctc_prefix_score.py:72-200
//   CTCPrefixScorer.select_state                        espnet/nets/scorers/ctc.py:37-60
//
// Design (GPU-first, not the reference's): the reference caches every layer's OUTPUT per hypothesis and re-projects
// K/V of the whole prefix -- and of the whole encoder memory -- at every step, then copies the caches around when
// the beam is re-ordered.  Here K/V are projected once: the source-attention K/V of all layers when an utterance
// starts, the self-attention K/V of a position when it is decoded, written straight into a slot (layer, position,
// beam slot) of the session buffer by the QKV GEMM.  Nothing is ever copied when the beam is re-ordered: a hypothesis
// is the list of slots of its prefix (`anc`, a (step, n) int32 table the host maintains), and the attention kernels
// follow it.
#pragma once
#include <math.h>

#include "common.cuh"

namespace avsr {
namespace dec {

constexpr int kMaxDecLayers = 16;
constexpr float kLogZero = -10000000000.0f;   // ctc_prefix_score.py:31

// ------------------------------------------------------------------ layouts (all slots 256-byte aligned, 4 B / element)

struct DecLayerPrep {
  float *self_qkv_w, *self_qkv_b, *self_out_w, *self_out_b;   // q|k|v rows concatenated: (3d, d)
  float *src_q_w, *src_q_b, *src_kv_w, *src_kv_b, *src_out_w, *src_out_b;   // k|v rows concatenated: (2d, d)
  float *ff_w1, *ff_b1, *ff_w2, *ff_b2;
  float *n1w, *n1b, *n2w, *n2b, *n3w, *n3b;
};
struct DecPrep {
  DecLayerPrep L[kMaxDecLayers];
  float *embed, *after_w, *after_b, *out_w, *out_b;   // out_w (npad, d) zero-padded rows, out_b (npad)
  int npad;
  size_t bytes;
};
static inline DecPrep layout_dec_prepared(const AvsrDecoderConfig& c, void* base) {
  DecPrep P{};
  Carver cv{reinterpret_cast<char*>(base)};
  const size_t D = c.d_model, F = c.linear_units;
  for (int l = 0; l < c.num_blocks && l < kMaxDecLayers; ++l) {
    DecLayerPrep& q = P.L[l];
    q.self_qkv_w = cv.take(3 * D * D); q.self_qkv_b = cv.take(3 * D);
    q.self_out_w = cv.take(D * D); q.self_out_b = cv.take(D);
    q.src_q_w = cv.take(D * D); q.src_q_b = cv.take(D);
    q.src_kv_w = cv.take(2 * D * D); q.src_kv_b = cv.take(2 * D);
    q.src_out_w = cv.take(D * D); q.src_out_b = cv.take(D);
    q.ff_w1 = cv.take(F * D); q.ff_b1 = cv.take(F);
    q.ff_w2 = cv.take(D * F); q.ff_b2 = cv.take(D);
    q.n1w = cv.take(D); q.n1b = cv.take(D); q.n2w = cv.take(D); q.n2b = cv.take(D); q.n3w = cv.take(D); q.n3b = cv.take(D);
  }
  P.npad = (int)align_up((size_t)c.odim, 64);
  P.embed = cv.take((size_t)c.odim * D);
  P.after_w = cv.take(D); P.after_b = cv.take(D);
  P.out_w = cv.take((size_t)P.npad * D); P.out_b = cv.take((size_t)P.npad);
  P.bytes = cv.off;
  return P;
}

// per-utterance state: source K/V of every layer and the self-attention q|k|v slots
struct DecSession {
  float* mem_kv;     // (L, T, 2d) fp32: k | v of the encoder memory
  float* self_qkv;   // (L, max_steps, max_hyps, 3d) fp32: q | k | v of (position, beam slot)
  float* mem_op;     // (T, d) operand copy of the memory (begin only)
  size_t bytes;
};
static inline DecSession layout_dec_session(const AvsrDecoderConfig& c, int T, int max_steps, int max_hyps, void* base) {
  DecSession S{};
  Carver cv{reinterpret_cast<char*>(base)};
  const size_t D = c.d_model, L = c.num_blocks;
  S.mem_kv = cv.take(L * (size_t)T * 2 * D);
  S.self_qkv = cv.take(L * (size_t)max_steps * max_hyps * 3 * D);
  S.mem_op = cv.take((size_t)T * D);
  S.bytes = cv.off;
  return S;
}

// U utterances decoded in lock-step: their source K/V packed frame after frame (no padding), the self-attention slots
// as in DecSession with max_hyps = U x beam slots (hypothesis row i of any utterance takes slot i of a position)
struct DecBatchSession {
  float* mem_kv;       // (L, sum_T, 2d) fp32: utterance u's frames are rows [utt_off[u], utt_off[u] + utt_len[u])
  float* self_qkv;     // (L, max_steps, max_hyps, 3d) fp32
  float* mem_op;       // (T_max, d) operand copy of one utterance's memory (begin only)
  int32_t* utt_off;    // (U) first packed frame of each utterance
  int32_t* utt_len;    // (U) frames of each utterance
  size_t bytes;
};
static inline DecBatchSession layout_dec_batch_session(const AvsrDecoderConfig& c, int U, long sum_T, int T_max,
                                                       int max_steps, int max_hyps, void* base) {
  DecBatchSession S{};
  Carver cv{reinterpret_cast<char*>(base)};
  const size_t D = c.d_model, L = c.num_blocks;
  S.mem_kv = cv.take(L * (size_t)sum_T * 2 * D);
  S.self_qkv = cv.take(L * (size_t)max_steps * max_hyps * 3 * D);
  S.mem_op = cv.take((size_t)T_max * D);
  S.utt_off = reinterpret_cast<int32_t*>(cv.take((size_t)U));
  S.utt_len = reinterpret_cast<int32_t*>(cv.take((size_t)U));
  S.bytes = cv.off;
  return S;
}

// lengths: HOST array of U utterance lengths, each in 1..T_max (T_max <= 0: no upper bound) -> total and longest
static inline int check_batch_lengths(const int32_t* lengths, int U, int T_max, long* sum_T, int* max_len) {
  AVSR_REQUIRE(U >= 1, "decoder batch: U=%d utterances", U);
  AVSR_REQUIRE(lengths != nullptr, "NULL lengths");
  long s = 0;
  int m = 0;
  for (int u = 0; u < U; ++u) {
    AVSR_REQUIRE(lengths[u] >= 1 && (T_max <= 0 || lengths[u] <= T_max),
                 "decoder batch: utterance %d has %d frames (must be 1..T_max = %d)", u, lengths[u], T_max);
    s += lengths[u];
    m = lengths[u] > m ? lengths[u] : m;
  }
  *sum_T = s;
  *max_len = m;
  return AVSR_OK;
}

struct DecWork {
  float *x, *xn, *q2, *scores, *ctx, *hid, *logits;
  size_t bytes;
};
static inline DecWork layout_dec_work(const AvsrDecoderConfig& c, int T, int max_steps, int max_hyps, void* base) {
  DecWork W{};
  Carver cv{reinterpret_cast<char*>(base)};
  const size_t D = c.d_model, n = max_hyps;
  const size_t smax = (size_t)(T > max_steps ? T : max_steps);
  W.x = cv.take(n * D); W.xn = cv.take(n * D); W.q2 = cv.take(n * D);
  W.scores = cv.take(n * c.n_heads * smax);
  W.ctx = cv.take(n * D);
  W.hid = cv.take(n * (size_t)c.linear_units);
  W.logits = cv.take(n * align_up((size_t)c.odim, 64));
  W.bytes = cv.off;
  return W;
}

// ------------------------------------------------------------------ per-element functors
AVSR_HD void store_operand(void* base, long idx, int kind, float v) {
#ifdef __CUDA_ARCH__
  if (kind == OP_F16) reinterpret_cast<__half*>(base)[idx] = to_half_sat(v);
  else reinterpret_cast<float*>(base)[idx] = kind == OP_TF32 ? round_tf32(v) : v;
#else
  if (kind == OP_F16) reinterpret_cast<__half*>(base)[idx] = __float2half_rn(v);
  else reinterpret_cast<float*>(base)[idx] = v;
#endif
}

AVSR_HD float logaddexp_f(float a, float b) {
  const float m = fmaxf(a, b);
  return m + log1pf(expf(-fabsf(a - b)));
}

// PositionalEncoding table entry (pos, c) (embedding.py:60-90), evaluated the way extend_pe does: fp32 exp of
// (2i * kf), kf = -(ln 1e4 / d), fp32 product with the position.  Shared by the scoring step (EmbedElem) and the
// teacher-forced training pass (decoder_train_body.cuh).
AVSR_HD float pe_value(int pos, int c, float kf) {
  const float ang = (float)pos * expf((float)(c & ~1) * kf);
  return (c & 1) ? cosf(ang) : sinf(ang);
}

// embed: Embedding row * sqrt(d) + PositionalEncoding row `pos` (transformer_decoder.py:163-167, embedding.py:60-90)
struct EmbedElem {
  const int32_t* tokens; const float* emb; float* x;
  int D, odim, pos;
  float xscale, kf;
  AVSR_HD void operator()(long idx) const {
    const int i = (int)(idx / D), c = (int)(idx - (long)i * D);
    int tok = tokens[i];
    tok = tok < 0 ? 0 : (tok >= odim ? odim - 1 : tok);
    x[idx] = emb[(long)tok * D + c] * xscale + pe_value(pos, c, kf);
  }
};

// where key / value row `s` of hypothesis i lives: the encoder frame s (source attention) or the slot of the
// hypothesis' prefix position s (self attention: its ancestors' slots for s < step, its own slot i at s == step)
struct KvIndex {
  const int32_t* anc;   // (step, n) slots, NULL for the source attention
  int n, step, max_hyps, self_mode;
  AVSR_HD long row(int s, int i) const {
    if (!self_mode) return s;
    const int slot = s < step ? anc[(long)s * n + i] : i;
    return (long)s * max_hyps + slot;
  }
};

// scores[i, h, s] = q_i,h . k_row(s,i),h / sqrt(d_k)   (attention.py:59-75 without mask: the prefix is causal by construction)
struct ScoresElem {
  const float* q; long ldq;
  const float* kv; long ld; int koff;
  KvIndex ix;
  int H, dk, S;
  float sqrt_dk;
  float* out;
  AVSR_HD void operator()(long idx) const {
    const int s = (int)(idx % S);
    const long ih = idx / S;
    const int h = (int)(ih % H), i = (int)(ih / H);
    const float* qp = q + (long)i * ldq + h * dk;
    const float* kp = kv + ix.row(s, i) * ld + koff + h * dk;
    float acc = 0.f;
    for (int e = 0; e < dk; ++e) acc = fmaf(qp[e], kp[e], acc);
    out[idx] = acc / sqrt_dk;
  }
};

// ctx[i, c] = sum_s softmax_s(scores[i, h(c), :]) * v_row(s,i)[c]   (attention.py:76-88), stored as a GEMM operand
struct PvElem {
  const float* scores;
  const float* kv; long ld; int voff;
  KvIndex ix;
  int H, dk, S, D, kind;
  void* ctx;
  AVSR_HD void operator()(long idx) const {
    const int i = (int)(idx / D), c = (int)(idx - (long)i * D);
    const int h = c / dk;
    const float* sc = scores + ((long)i * H + h) * S;
    float m = sc[0];
    for (int s = 1; s < S; ++s) m = fmaxf(m, sc[s]);
    float l = 0.f, acc = 0.f;
    for (int s = 0; s < S; ++s) {
      const float p = expf(sc[s] - m);
      l += p;
      acc = fmaf(p, kv[ix.row(s, i) * ld + voff + c], acc);
    }
    store_operand(ctx, idx, kind, acc / l);
  }
};

// Source attention of a batched step, row i over its own utterance's frames: the per-output operations and their order
// are ScoresElem's / PvElem's with S = utt_len[row_utt[i]] and the key rows offset by utt_off[row_utt[i]].  scores rows
// are strided by T_max; entries past the utterance's length are neither written nor read.  The host replay runs these;
// the device runs the grouped kernel of decoder.cu, which must give the same bits.
struct ScoresBatchElem {
  const float* q; const float* kv; const int32_t* row_utt; const int32_t* utt_off; const int32_t* utt_len;
  int H, dk, D, T_max;
  float sqrt_dk;
  float* out;
  AVSR_HD void operator()(long idx) const {
    const int s = (int)(idx % T_max);
    const long ih = idx / T_max;
    const int h = (int)(ih % H), i = (int)(ih / H);
    const int u = row_utt[i];
    if (s >= utt_len[u]) return;
    const float* qp = q + (long)i * D + h * dk;
    const float* kp = kv + (long)(utt_off[u] + s) * 2 * D + h * dk;
    float acc = 0.f;
    for (int e = 0; e < dk; ++e) acc = fmaf(qp[e], kp[e], acc);
    out[idx] = acc / sqrt_dk;
  }
};
struct PvBatchElem {
  const float* scores; const float* kv; const int32_t* row_utt; const int32_t* utt_off; const int32_t* utt_len;
  int H, dk, D, T_max, kind;
  void* ctx;
  AVSR_HD void operator()(long idx) const {
    const int i = (int)(idx / D), c = (int)(idx - (long)i * D);
    const int h = c / dk, u = row_utt[i], S = utt_len[u];
    const float* sc = scores + ((long)i * H + h) * T_max;
    const float* vp = kv + (long)utt_off[u] * 2 * D + D + c;
    float m = sc[0];
    for (int s = 1; s < S; ++s) m = fmaxf(m, sc[s]);
    float l = 0.f, acc = 0.f;
    for (int s = 0; s < S; ++s) {
      const float p = expf(sc[s] - m);
      l += p;
      acc = fmaf(p, vp[(long)s * 2 * D], acc);
    }
    store_operand(ctx, idx, kind, acc / l);
  }
};
// utt_off = exclusive prefix sum of utt_len (one thread: U is the number of utterances in a batch)
struct UttOffsetsElem {
  const int32_t* len; int32_t* off; int U;
  AVSR_HD void operator()(long) const {
    int32_t acc = 0;
    for (int u = 0; u < U; ++u) { off[u] = acc; acc += len[u]; }
  }
};

// generic copy with conversion into an operand storage kind (weights at preparation, the memory at begin)
struct ConvertElem {
  const float* src; void* dst; int kind;
  AVSR_HD void operator()(long idx) const { store_operand(dst, idx, kind, src[idx]); }
};
// rows [r0, r0 + rows) of a (rows_total, cols) destination <- a (rows, cols) source (concatenating q|k|v weights)
struct ConvertRowsElem {
  const float* src; void* dst; long dst_off; int kind;
  AVSR_HD void operator()(long idx) const { store_operand(dst, dst_off + idx, kind, src[idx]); }
};
struct FillElem {
  float* dst; float v;
  AVSR_HD void operator()(long idx) const { dst[idx] = v; }
};
struct CopyElem {
  const float* src; float* dst;
  AVSR_HD void operator()(long idx) const { dst[idx] = src[idx]; }
};

// ---- CTC prefix scorer (one utterance): r layouts follow the reference's stacked states,
//      r_prev (T, 2, n), r (T, 2, n, S); k = 0 non-blank ending, k = 1 blank ending ----------------------------------
struct CtcInitElem {        // state of the empty prefix: r^n = logzero, r^b_t = cumulative blank log-probability
  const float* logp; float* r0; int T, O, blank;
  AVSR_HD void operator()(long) const {
    float acc = 0.f;
    for (int t = 0; t < T; ++t) {
      acc += logp[(long)t * O + blank];
      r0[2 * t] = kLogZero;
      r0[2 * t + 1] = acc;
    }
  }
};
struct CtcFillElem {        // every token off the candidate list: logzero, except <eos> = total prefix probability
  const float* r_prev; const float* s_prev; float* local; float* log_psi;
  int T, O, n, blank, eos;
  AVSR_HD void operator()(long idx) const {
    const int i = (int)(idx / O), o = (int)(idx - (long)i * O);
    float v = kLogZero;
    if (o == eos) v = logaddexp_f(r_prev[((long)(T - 1) * 2 + 0) * n + i], r_prev[((long)(T - 1) * 2 + 1) * n + i]);
    if (o == blank) v = kLogZero;
    log_psi[idx] = v;
    local[idx] = v - s_prev[i];
  }
};
struct CtcCandElem {        // forward variables + prefix probability of (hypothesis i, candidate c)
  const float* logp; const float* r_prev; const float* s_prev; const int32_t* last_ids; const int32_t* cand;
  float* r; float* local; float* log_psi;
  int T, O, n, S, blank, eos, out_len;
  AVSR_HD void operator()(long idx) const {
    const int i = (int)(idx / S), c = (int)(idx - (long)i * S);
    const int tok = cand[idx];
    const bool same = tok == last_ids[i];
    const int start = out_len > 1 ? out_len : 1;
    const long plane = (long)n * S;                   // elements per (t, k)
    float* rp = r + (long)i * S + c;
    for (int t = 0; t < start && t < T; ++t) { rp[(long)(2 * t) * plane] = kLogZero; rp[(long)(2 * t + 1) * plane] = kLogZero; }
    float rn = kLogZero, rb = kLogZero;
    if (out_len == 0) { rn = logp[tok]; rp[0] = rn; }             // r[0, 0] = x[0, tok]
    float psi = rn;                                               // the r^n_{start-1} term
    for (int t = start; t < T; ++t) {
      const float pn = r_prev[((long)(t - 1) * 2 + 0) * n + i], pb = r_prev[((long)(t - 1) * 2 + 1) * n + i];
      const float phi = same ? pb : logaddexp_f(pn, pb);
      const float xt = logp[(long)t * O + tok], xb = logp[(long)t * O + blank];
      const float rn_new = logaddexp_f(rn, phi) + xt;
      const float rb_new = logaddexp_f(rn, rb) + xb;
      psi = logaddexp_f(psi, phi + xt);
      rp[(long)(2 * t) * plane] = rn_new;
      rp[(long)(2 * t + 1) * plane] = rb_new;
      rn = rn_new; rb = rb_new;
    }
    if (tok != eos && tok != blank) {                  // those two were set by CtcFillElem
      log_psi[(long)i * O + tok] = psi;
      local[(long)i * O + tok] = psi - s_prev[i];
    }
  }
};
struct CtcSelectElem {      // states of the kept hypotheses: r_next (T, 2, m) <- r[:, :, parent, position of token in cand[parent]]
  const float* r; const int32_t* cand; const int32_t* parent; const int32_t* token; float* r_next;
  int n, S, m;
  AVSR_HD void operator()(long idx) const {
    const int j = (int)(idx % m);
    const long tk = idx / m;
    const int p = parent[j], tok = token[j];
    int pos = -1;
    for (int c = 0; c < S; ++c) if (cand[(long)p * S + c] == tok) { pos = c; break; }
    r_next[idx] = pos >= 0 ? r[(tk * n + p) * S + pos] : kLogZero;
  }
};
struct CtcSelectScoreElem {
  const float* log_psi; const int32_t* parent; const int32_t* token; float* s_next; int O;
  AVSR_HD void operator()(long j) const { s_next[j] = log_psi[(long)parent[j] * O + token[j]]; }
};

// ---- CTC prefix scorer over U utterances of lengths len[u] <= T_max (CTCPrefixScoreTH with xlens,
//      ctc_prefix_score.py:21-54, :180-181): logp (U, T_max, O); row i belongs to utterance row_utt[i].  Per row, the
//      operations and their order are those of the one-utterance functors above with T = len[row_utt[i]]; state entries
//      at frames t >= T are logzero (CtcSelectElem copies all T_max frames) ---------------------------------------------
struct CtcInitBatchElem {   // r0 (T_max, 2, U)
  const float* logp; const int32_t* len; float* r0; int U, T_max, O, blank;
  AVSR_HD void operator()(long u) const {
    const int T = len[u];
    const float* lp = logp + u * (long)T_max * O;
    float acc = 0.f;
    for (int t = 0; t < T_max; ++t) {
      if (t < T) acc += lp[(long)t * O + blank];
      r0[(long)(2 * t) * U + u] = kLogZero;
      r0[(long)(2 * t + 1) * U + u] = t < T ? acc : kLogZero;
    }
  }
};
struct CtcFillBatchElem {
  const float* r_prev; const float* s_prev; const int32_t* row_utt; const int32_t* len; float* local; float* log_psi;
  int O, n, blank, eos;
  AVSR_HD void operator()(long idx) const {
    const int i = (int)(idx / O), o = (int)(idx - (long)i * O);
    const int T = len[row_utt[i]];
    float v = kLogZero;
    if (o == eos) v = logaddexp_f(r_prev[((long)(T - 1) * 2 + 0) * n + i], r_prev[((long)(T - 1) * 2 + 1) * n + i]);
    if (o == blank) v = kLogZero;
    log_psi[idx] = v;
    local[idx] = v - s_prev[i];
  }
};
struct CtcCandBatchElem {
  const float* logp; const float* r_prev; const float* s_prev; const int32_t* last_ids; const int32_t* cand;
  const int32_t* row_utt; const int32_t* len;
  float* r; float* local; float* log_psi;
  int T_max, O, n, S, blank, eos, out_len;
  AVSR_HD void operator()(long idx) const {
    const int i = (int)(idx / S), c = (int)(idx - (long)i * S);
    const int u = row_utt[i], T = len[u];
    const float* lp = logp + (long)u * T_max * O;
    const int tok = cand[idx];
    const bool same = tok == last_ids[i];
    const int start = out_len > 1 ? out_len : 1;
    const long plane = (long)n * S;
    float* rp = r + (long)i * S + c;
    for (int t = 0; t < start && t < T; ++t) { rp[(long)(2 * t) * plane] = kLogZero; rp[(long)(2 * t + 1) * plane] = kLogZero; }
    float rn = kLogZero, rb = kLogZero;
    if (out_len == 0) { rn = lp[tok]; rp[0] = rn; }
    float psi = rn;
    for (int t = start; t < T; ++t) {
      const float pn = r_prev[((long)(t - 1) * 2 + 0) * n + i], pb = r_prev[((long)(t - 1) * 2 + 1) * n + i];
      const float phi = same ? pb : logaddexp_f(pn, pb);
      const float xt = lp[(long)t * O + tok], xb = lp[(long)t * O + blank];
      const float rn_new = logaddexp_f(rn, phi) + xt;
      const float rb_new = logaddexp_f(rn, rb) + xb;
      psi = logaddexp_f(psi, phi + xt);
      rp[(long)(2 * t) * plane] = rn_new;
      rp[(long)(2 * t + 1) * plane] = rb_new;
      rn = rn_new; rb = rb_new;
    }
    for (int t = T; t < T_max; ++t) { rp[(long)(2 * t) * plane] = kLogZero; rp[(long)(2 * t + 1) * plane] = kLogZero; }
    if (tok != eos && tok != blank) {
      log_psi[(long)i * O + tok] = psi;
      local[(long)i * O + tok] = psi - s_prev[i];
    }
  }
};

// ------------------------------------------------------------------ schedules
// Backend BK provides: gemm(prec, A_op, W_op, M, N, K, bias, out, resid, alpha, relu, out_is_operand),
//   layernorm(x, g, b, y, rows, d, out_kind), log_softmax(x, ldx, y, ldy, rows, n), for_each(count, functor).
template <class BK>
int prepare_body(BK& bk, const AvsrDecoderConfig& c, const AvsrDecoderLayerParams* layers, const float* embed_w,
                 const float* after_w, const float* after_b, const float* out_w, const float* out_b, const DecPrep& P,
                 int prec) {
  const long D = c.d_model, F = c.linear_units;
  const int kind = operand_kind(prec);
  for (int l = 0; l < c.num_blocks; ++l) {
    const AvsrDecoderLayerParams& s = layers[l];
    const DecLayerPrep& q = P.L[l];
    const float* qkv_w[3] = {s.self_q_w, s.self_k_w, s.self_v_w};
    const float* qkv_b[3] = {s.self_q_b, s.self_k_b, s.self_v_b};
    for (int j = 0; j < 3; ++j) {
      AVSR_TRY(bk.for_each(D * D, ConvertRowsElem{qkv_w[j], q.self_qkv_w, j * D * D, kind}));
      AVSR_TRY(bk.for_each(D, CopyElem{qkv_b[j], q.self_qkv_b + j * D}));
    }
    const float* kv_w[2] = {s.src_k_w, s.src_v_w};
    const float* kv_b[2] = {s.src_k_b, s.src_v_b};
    for (int j = 0; j < 2; ++j) {
      AVSR_TRY(bk.for_each(D * D, ConvertRowsElem{kv_w[j], q.src_kv_w, j * D * D, kind}));
      AVSR_TRY(bk.for_each(D, CopyElem{kv_b[j], q.src_kv_b + j * D}));
    }
    AVSR_TRY(bk.for_each(D * D, ConvertElem{s.self_out_w, q.self_out_w, kind}));
    AVSR_TRY(bk.for_each(D * D, ConvertElem{s.src_q_w, q.src_q_w, kind}));
    AVSR_TRY(bk.for_each(D * D, ConvertElem{s.src_out_w, q.src_out_w, kind}));
    AVSR_TRY(bk.for_each(F * D, ConvertElem{s.ff_w1, q.ff_w1, kind}));
    AVSR_TRY(bk.for_each(D * F, ConvertElem{s.ff_w2, q.ff_w2, kind}));
    AVSR_TRY(bk.for_each(D, CopyElem{s.self_out_b, q.self_out_b}));
    AVSR_TRY(bk.for_each(D, CopyElem{s.src_q_b, q.src_q_b}));
    AVSR_TRY(bk.for_each(D, CopyElem{s.src_out_b, q.src_out_b}));
    AVSR_TRY(bk.for_each(F, CopyElem{s.ff_b1, q.ff_b1}));
    AVSR_TRY(bk.for_each(D, CopyElem{s.ff_b2, q.ff_b2}));
    AVSR_TRY(bk.for_each(D, CopyElem{s.norm1_w, q.n1w})); AVSR_TRY(bk.for_each(D, CopyElem{s.norm1_b, q.n1b}));
    AVSR_TRY(bk.for_each(D, CopyElem{s.norm2_w, q.n2w})); AVSR_TRY(bk.for_each(D, CopyElem{s.norm2_b, q.n2b}));
    AVSR_TRY(bk.for_each(D, CopyElem{s.norm3_w, q.n3w})); AVSR_TRY(bk.for_each(D, CopyElem{s.norm3_b, q.n3b}));
  }
  AVSR_TRY(bk.for_each((long)c.odim * D, CopyElem{embed_w, P.embed}));
  AVSR_TRY(bk.for_each(D, CopyElem{after_w, P.after_w}));
  AVSR_TRY(bk.for_each(D, CopyElem{after_b, P.after_b}));
  // output_layer padded to npad rows: zero weights, zero bias (the log-softmax only reads the first odim columns)
  AVSR_TRY(bk.for_each((long)P.npad * D, FillElem{P.out_w, 0.f}));     // 0.0f is all-zero bits in every operand kind
  AVSR_TRY(bk.for_each((long)P.npad, FillElem{P.out_b, 0.f}));
  AVSR_TRY(bk.for_each((long)c.odim * D, ConvertElem{out_w, P.out_w, kind}));
  AVSR_TRY(bk.for_each((long)c.odim, CopyElem{out_b, P.out_b}));
  return AVSR_OK;
}

// utterance start: source-attention K | V of every layer, once (the reference recomputes them at every step inside
// src_attn, transformer_decoder.py:119-127)
// source K|V of one utterance's T frames into rows [row0, row0 + T) of every layer's (rows_per_layer, 2d) block
template <class BK>
int project_memory_kv(BK& bk, const AvsrDecoderConfig& c, const DecPrep& P, const float* memory, int T, void* mem_op,
                      float* mem_kv, long rows_per_layer, long row0, int prec) {
  const int D = c.d_model;
  const void* a = memory;
  if (prec != AVSR_PREC_FP32) {
    AVSR_TRY(bk.for_each((long)T * D, ConvertElem{memory, mem_op, operand_kind(prec)}));
    a = mem_op;
  }
  // Row chunks of <= 192 frames: every launch stays in the M < 256 regime of the persistent one-CTA GEMM -- the same
  // kernel variant (fp32 output + bias) every step GEMM of this path uses; once per utterance, so the extra launches
  // do not matter.
  const size_t esz = prec == AVSR_PREC_F16 ? 2 : 4;
  constexpr int kChunk = 192;
  for (int l = 0; l < c.num_blocks; ++l)
    for (int r0 = 0; r0 < T; r0 += kChunk) {
      const int rows = T - r0 < kChunk ? T - r0 : kChunk;
      const void* a_rows = reinterpret_cast<const char*>(a) + (size_t)r0 * D * esz;
      AVSR_TRY(bk.gemm(prec, a_rows, P.L[l].src_kv_w, rows, 2 * D, D, P.L[l].src_kv_b,
                       mem_kv + ((size_t)l * rows_per_layer + row0 + r0) * 2 * D, nullptr, 0.f, 0, 0));
    }
  return AVSR_OK;
}

template <class BK>
int begin_body(BK& bk, const AvsrDecoderConfig& c, const DecPrep& P, const DecSession& S, const float* memory, int T,
               int prec) {
  return project_memory_kv(bk, c, P, memory, T, S.mem_op, S.mem_kv, T, 0, prec);
}

// U utterances: memory (U, T_max, d) fp32, lengths a HOST array.  Each utterance's K|V is projected with the chunks of
// begin_body, so it has the bits a one-utterance session would hold.
template <class BK>
int begin_batch_body(BK& bk, const AvsrDecoderConfig& c, const DecPrep& P, const DecBatchSession& S,
                     const float* memory, const int32_t* lengths, int U, int T_max, long sum_T, int prec) {
  AVSR_TRY(bk.upload_i32(S.utt_len, lengths, U));
  AVSR_TRY(bk.for_each(1, UttOffsetsElem{S.utt_len, S.utt_off, U}));
  long off = 0;
  for (int u = 0; u < U; ++u) {
    AVSR_TRY(project_memory_kv(bk, c, P, memory + (size_t)u * T_max * c.d_model, lengths[u], S.mem_op, S.mem_kv, sum_T,
                               off, prec));
    off += lengths[u];
  }
  return AVSR_OK;
}

// one decoding step for n hypotheses of equal length `step + 1` (their last tokens in `tokens`, their earlier
// positions' slots in `anc` (step, n)): next-token log-probabilities (n, odim).  `src_attn(l)` computes the source
// attention of layer l from W.q2 into W.ctx.
template <class BK, class SrcAttn>
int step_layers(BK& bk, const AvsrDecoderConfig& c, const DecPrep& P, float* self_qkv, const DecWork& W,
                const int32_t* tokens, const int32_t* anc, int step, int n, int max_steps, int max_hyps, float* logp,
                int prec, const SrcAttn& src_attn) {
  const int D = c.d_model, H = c.n_heads, F = c.linear_units, dk = D / H;
  const int kind = operand_kind(prec);
  const float sqrt_dk = (float)sqrt((double)dk);
  AVSR_TRY(bk.for_each((long)n * D, EmbedElem{tokens, P.embed, W.x, D, c.odim, step, (float)sqrt((double)D),
                                               (float)(-(log(10000.0) / D))}));
  const KvIndex self_ix{anc, n, step, max_hyps, 1};
  for (int l = 0; l < c.num_blocks; ++l) {
    const DecLayerPrep& q = P.L[l];
    float* qkv_l = self_qkv + (size_t)l * max_steps * max_hyps * 3 * D;          // row (position, slot)
    float* qkv_t = qkv_l + (size_t)step * max_hyps * 3 * D;                      // this step's rows: slot = hypothesis index
    // (1) x += self_attn(norm1(x)) over the prefix
    AVSR_TRY(bk.layernorm(W.x, q.n1w, q.n1b, W.xn, n, D, kind));
    AVSR_TRY(bk.gemm(prec, W.xn, q.self_qkv_w, n, 3 * D, D, q.self_qkv_b, qkv_t, nullptr, 0.f, 0, 0));
    AVSR_TRY(bk.for_each((long)n * H * (step + 1),
                         ScoresElem{qkv_t, 3L * D, qkv_l, 3L * D, D, self_ix, H, dk, step + 1, sqrt_dk, W.scores}));
    AVSR_TRY(bk.for_each((long)n * D, PvElem{W.scores, qkv_l, 3L * D, 2 * D, self_ix, H, dk, step + 1, D, kind, W.ctx}));
    AVSR_TRY(bk.gemm(prec, W.ctx, q.self_out_w, n, D, D, q.self_out_b, W.x, W.x, 1.f, 0, 0));
    // (2) x += src_attn(norm2(x), memory)
    AVSR_TRY(bk.layernorm(W.x, q.n2w, q.n2b, W.xn, n, D, kind));
    AVSR_TRY(bk.gemm(prec, W.xn, q.src_q_w, n, D, D, q.src_q_b, W.q2, nullptr, 0.f, 0, 0));
    AVSR_TRY(src_attn(l));
    AVSR_TRY(bk.gemm(prec, W.ctx, q.src_out_w, n, D, D, q.src_out_b, W.x, W.x, 1.f, 0, 0));
    // (3) x += w_2(relu(w_1(norm3(x))))
    AVSR_TRY(bk.layernorm(W.x, q.n3w, q.n3b, W.xn, n, D, kind));
    AVSR_TRY(bk.gemm(prec, W.xn, q.ff_w1, n, F, D, q.ff_b1, W.hid, nullptr, 0.f, 1, 1));
    AVSR_TRY(bk.gemm(prec, W.hid, q.ff_w2, n, D, F, q.ff_b2, W.x, W.x, 1.f, 0, 0));
  }
  // after_norm -> output_layer -> log_softmax (transformer_decoder.py:283-289)
  AVSR_TRY(bk.layernorm(W.x, P.after_w, P.after_b, W.xn, n, D, kind));
  AVSR_TRY(bk.gemm(prec, W.xn, P.out_w, n, P.npad, D, P.out_b, W.logits, nullptr, 0.f, 0, 0));
  return bk.log_softmax(W.logits, P.npad, logp, c.odim, n, c.odim);
}

template <class BK>
int step_body(BK& bk, const AvsrDecoderConfig& c, const DecPrep& P, const DecSession& S, const DecWork& W,
              const int32_t* tokens, const int32_t* anc, int step, int n, int T, int max_steps, int max_hyps, float* logp,
              int prec) {
  const int D = c.d_model, H = c.n_heads, dk = D / H;
  const int kind = operand_kind(prec);
  const float sqrt_dk = (float)sqrt((double)dk);
  const KvIndex src_ix{nullptr, n, 0, 0, 0};
  auto src_attn = [&](int l) {
    const float* mkv = S.mem_kv + (size_t)l * T * 2 * D;
    AVSR_TRY(bk.for_each((long)n * H * T, ScoresElem{W.q2, (long)D, mkv, 2L * D, 0, src_ix, H, dk, T, sqrt_dk, W.scores}));
    return bk.for_each((long)n * D, PvElem{W.scores, mkv, 2L * D, D, src_ix, H, dk, T, D, kind, W.ctx});
  };
  return step_layers(bk, c, P, S.self_qkv, W, tokens, anc, step, n, max_steps, max_hyps, logp, prec, src_attn);
}

// one step of U utterances in lock-step: rows in any order, row i of utterance row_utt[i] (DEVICE int32, not checked);
// everything but the source attention is step_body's code at M = n.  BK::src_attention_batch runs the source attention
// of every row over its own utterance's frames (the batched functors on the host, the grouped kernel on the device).
template <class BK>
int step_batch_body(BK& bk, const AvsrDecoderConfig& c, const DecPrep& P, const DecBatchSession& S, const DecWork& W,
                    const int32_t* tokens, const int32_t* anc, const int32_t* row_utt, int step, int n, int U, int T_max,
                    long sum_T, int max_steps, int max_hyps, float* logp, int prec) {
  const int D = c.d_model, H = c.n_heads, dk = D / H;
  const int kind = operand_kind(prec);
  const float sqrt_dk = (float)sqrt((double)dk);
  auto src_attn = [&](int l) {
    const float* mkv = S.mem_kv + (size_t)l * sum_T * 2 * D;
    return bk.src_attention_batch(W.q2, mkv, row_utt, S.utt_off, S.utt_len, U, sum_T, n, H, dk, T_max, sqrt_dk, W.scores,
                                  kind, W.ctx);
  };
  return step_layers(bk, c, P, S.self_qkv, W, tokens, anc, step, n, max_steps, max_hyps, logp, prec, src_attn);
}

template <class BK>
int ctc_prefix_body(BK& bk, const float* logp, int T, int O, int blank, int eos, int out_len, const int32_t* last_ids,
                    const float* r_prev, const float* s_prev, const int32_t* cand, int n, int S, float* local, float* r,
                    float* log_psi) {
  AVSR_TRY(bk.for_each((long)n * O, CtcFillElem{r_prev, s_prev, local, log_psi, T, O, n, blank, eos}));
  return bk.for_each((long)n * S, CtcCandElem{logp, r_prev, s_prev, last_ids, cand, r, local, log_psi, T, O, n, S, blank,
                                              eos, out_len});
}

template <class BK>
int ctc_prefix_batch_body(BK& bk, const float* logp, const int32_t* len, int T_max, int O, int blank, int eos,
                          int out_len, const int32_t* last_ids, const float* r_prev, const float* s_prev,
                          const int32_t* cand, const int32_t* row_utt, int n, int S, float* local, float* r,
                          float* log_psi) {
  AVSR_TRY(bk.for_each((long)n * O, CtcFillBatchElem{r_prev, s_prev, row_utt, len, local, log_psi, O, n, blank, eos}));
  return bk.for_each((long)n * S, CtcCandBatchElem{logp, r_prev, s_prev, last_ids, cand, row_utt, len, r, local, log_psi,
                                                   T_max, O, n, S, blank, eos, out_len});
}

template <class BK>
int ctc_select_body(BK& bk, const float* r, const float* log_psi, const int32_t* cand, const int32_t* parent,
                    const int32_t* token, int T, int O, int n, int S, int m, float* r_next, float* s_next) {
  AVSR_TRY(bk.for_each((long)T * 2 * m, CtcSelectElem{r, cand, parent, token, r_next, n, S, m}));
  return bk.for_each((long)m, CtcSelectScoreElem{log_psi, parent, token, s_next, O});
}

// ------------------------------------------------------------------ C-ABI entry bodies (include/avsr_b200.h)
// The argument contract of every decoder / CTC-prefix entry, written once: decoder.cu forwards the extern "C" names to
// these with its DeviceBackend, the host replay with its host backend.  What only one backend refuses stays in it.
static inline int check_dec_cfg(const AvsrDecoderConfig* c) {
  AVSR_REQUIRE(c != nullptr, "NULL decoder config");
  AVSR_REQUIRE(c->d_model > 0 && c->n_heads > 0 && c->d_model % c->n_heads == 0 && c->d_model % 64 == 0,
               "decoder: d_model=%d must be a multiple of 64 and of n_heads=%d", c->d_model, c->n_heads);
  AVSR_REQUIRE(c->linear_units > 0 && c->linear_units % 64 == 0, "decoder: linear_units=%d must be a multiple of 64",
               c->linear_units);
  AVSR_REQUIRE(c->num_blocks > 0 && c->num_blocks <= kMaxDecLayers, "decoder: num_blocks=%d outside 1..%d", c->num_blocks,
               kMaxDecLayers);
  AVSR_REQUIRE(c->odim > 1, "decoder: odim=%d", c->odim);
  return AVSR_OK;
}

static inline size_t decoder_prepared_bytes_entry(const AvsrDecoderConfig* cfg) {
  if (check_dec_cfg(cfg) != AVSR_OK) return 0;
  return layout_dec_prepared(*cfg, nullptr).bytes;
}

template <class BK>
int prepare_decoder_entry(BK bk, const AvsrDecoderConfig* cfg, const AvsrDecoderLayerParams* layers,
                          const float* embed_w, const float* after_norm_w, const float* after_norm_b, const float* out_w,
                          const float* out_b, void* prepared, size_t prepared_bytes, int precision) {
  AVSR_TRY(check_dec_cfg(cfg));
  AVSR_REQUIRE(layers && embed_w && after_norm_w && after_norm_b && out_w && out_b && prepared, "NULL argument");
  AVSR_REQUIRE(valid_precision(precision), "bad precision %d", precision);
  for (int l = 0; l < cfg->num_blocks; ++l) {
    const void* const* p = reinterpret_cast<const void* const*>(&layers[l]);
    for (size_t k = 0; k < sizeof(AvsrDecoderLayerParams) / sizeof(void*); ++k)
      AVSR_REQUIRE(p[k] != nullptr, "decoder layer %d: parameter %zu is NULL", l, k);
  }
  const DecPrep P = layout_dec_prepared(*cfg, prepared);
  AVSR_REQUIRE_BYTES(P.bytes, prepared_bytes, "decoder prepared buffer");
  return prepare_body(bk, *cfg, layers, embed_w, after_norm_w, after_norm_b, out_w, out_b, P, precision);
}

static inline size_t decoder_session_bytes_entry(const AvsrDecoderConfig* cfg, int T, int max_steps, int max_hyps) {
  if (check_dec_cfg(cfg) != AVSR_OK || T <= 0 || max_steps <= 0 || max_hyps <= 0) return 0;
  return layout_dec_session(*cfg, T, max_steps, max_hyps, nullptr).bytes;
}

template <class BK>
int decoder_begin_entry(BK bk, const AvsrDecoderConfig* cfg, const void* prepared, const float* memory, int T,
                        int max_steps, int max_hyps, void* session, size_t session_bytes, int precision) {
  AVSR_TRY(check_dec_cfg(cfg));
  AVSR_REQUIRE(prepared && memory && session, "NULL argument");
  AVSR_REQUIRE(T > 0 && max_steps > 0 && max_hyps > 0, "decoder_begin: bad T=%d max_steps=%d max_hyps=%d", T, max_steps, max_hyps);
  AVSR_REQUIRE(valid_precision(precision), "bad precision %d", precision);
  const DecSession S = layout_dec_session(*cfg, T, max_steps, max_hyps, session);
  AVSR_REQUIRE_BYTES(S.bytes, session_bytes, "decoder session");
  const DecPrep P = layout_dec_prepared(*cfg, const_cast<void*>(prepared));
  return begin_body(bk, *cfg, P, S, memory, T, precision);
}

static inline size_t decoder_step_workspace_bytes_entry(const AvsrDecoderConfig* cfg, int T, int max_steps,
                                                        int max_hyps) {
  if (check_dec_cfg(cfg) != AVSR_OK || T <= 0 || max_steps <= 0 || max_hyps <= 0) return 0;
  return layout_dec_work(*cfg, T, max_steps, max_hyps, nullptr).bytes;
}

template <class BK>
int decoder_step_entry(BK bk, const AvsrDecoderConfig* cfg, const void* prepared, void* session, size_t session_bytes,
                       int T, int max_steps, int max_hyps, const int32_t* tokens, const int32_t* anc, int step, int n,
                       float* logp, void* workspace, size_t workspace_bytes, int precision) {
  AVSR_TRY(check_dec_cfg(cfg));
  AVSR_REQUIRE(prepared && session && tokens && logp && workspace, "NULL argument");
  AVSR_REQUIRE(T > 0 && max_steps > 0 && max_hyps > 0, "decoder_step: bad T=%d max_steps=%d max_hyps=%d", T, max_steps, max_hyps);
  AVSR_REQUIRE(step >= 0 && step < max_steps, "decoder_step: step %d outside the session's %d positions", step, max_steps);
  AVSR_REQUIRE(n >= 0 && n <= max_hyps, "decoder_step: n=%d hypotheses exceed the session's %d beam slots", n, max_hyps);
  AVSR_REQUIRE(step == 0 || anc != nullptr, "decoder_step: step %d needs the ancestor table", step);
  AVSR_REQUIRE(valid_precision(precision), "bad precision %d", precision);
  if (n == 0) return AVSR_OK;
  const DecSession S = layout_dec_session(*cfg, T, max_steps, max_hyps, session);
  const DecWork W = layout_dec_work(*cfg, T, max_steps, max_hyps, workspace);
  AVSR_REQUIRE_BYTES(S.bytes, session_bytes, "decoder session");
  AVSR_REQUIRE_BYTES(W.bytes, workspace_bytes, "decoder step workspace");
  const DecPrep P = layout_dec_prepared(*cfg, const_cast<void*>(prepared));
  return step_body(bk, *cfg, P, S, W, tokens, anc, step, n, T, max_steps, max_hyps, logp, precision);
}

template <class BK>
int ctc_prefix_init_entry(BK bk, const float* logp, int T, int O, int blank, float* r0) {
  AVSR_REQUIRE(logp && r0, "NULL argument");
  AVSR_REQUIRE(T > 0 && O > 1 && blank >= 0 && blank < O, "ctc_prefix_init: bad T=%d O=%d blank=%d", T, O, blank);
  return bk.for_each(1, CtcInitElem{logp, r0, T, O, blank});
}

template <class BK>
int ctc_prefix_score_entry(BK bk, const float* logp, int T, int O, int blank, int eos, int out_len,
                           const int32_t* last_ids, const float* r_prev, const float* s_prev, const int32_t* cand, int n,
                           int S, float* local, float* r, float* log_psi) {
  AVSR_REQUIRE(logp && last_ids && r_prev && s_prev && cand && local && r && log_psi, "NULL argument");
  AVSR_REQUIRE(T > 0 && O > 1 && blank >= 0 && blank < O && eos >= 0 && eos < O && blank != eos,
               "ctc_prefix_score: bad T=%d O=%d blank=%d eos=%d", T, O, blank, eos);
  AVSR_REQUIRE(out_len >= 0 && n >= 0 && S > 0 && S <= O, "ctc_prefix_score: bad out_len=%d n=%d S=%d", out_len, n, S);
  if (n == 0) return AVSR_OK;
  return ctc_prefix_body(bk, logp, T, O, blank, eos, out_len, last_ids, r_prev, s_prev, cand, n, S, local, r, log_psi);
}

template <class BK>
int ctc_prefix_select_entry(BK bk, const float* r, const float* log_psi, const int32_t* cand, const int32_t* parent,
                            const int32_t* token, int T, int O, int n, int S, int m, float* r_next, float* s_next) {
  AVSR_REQUIRE(r && log_psi && cand && parent && token && r_next && s_next, "NULL argument");
  AVSR_REQUIRE(T > 0 && O > 1 && n > 0 && S > 0 && m >= 0, "ctc_prefix_select: bad T=%d O=%d n=%d S=%d m=%d", T, O, n, S, m);
  if (m == 0) return AVSR_OK;
  return ctc_select_body(bk, r, log_psi, cand, parent, token, T, O, n, S, m, r_next, s_next);
}

static inline size_t decoder_batch_session_bytes_entry(const AvsrDecoderConfig* cfg, int U, const int32_t* lengths,
                                                       int max_steps, int max_hyps) {
  long sum_T;
  int max_len;
  if (check_dec_cfg(cfg) != AVSR_OK || check_batch_lengths(lengths, U, 0, &sum_T, &max_len) != AVSR_OK ||
      max_steps <= 0 || max_hyps <= 0)
    return 0;
  return layout_dec_batch_session(*cfg, U, sum_T, max_len, max_steps, max_hyps, nullptr).bytes;
}

template <class BK>
int decoder_batch_begin_entry(BK bk, const AvsrDecoderConfig* cfg, const void* prepared, const float* memory,
                              const int32_t* lengths, int U, int T_max, int max_steps, int max_hyps, void* session,
                              size_t session_bytes, int precision) {
  AVSR_TRY(check_dec_cfg(cfg));
  AVSR_REQUIRE(prepared && memory && session, "NULL argument");
  AVSR_REQUIRE(T_max > 0 && max_steps > 0 && max_hyps > 0, "decoder_batch_begin: bad T_max=%d max_steps=%d max_hyps=%d",
               T_max, max_steps, max_hyps);
  AVSR_REQUIRE(valid_precision(precision), "bad precision %d", precision);
  long sum_T;
  int max_len;
  AVSR_TRY(check_batch_lengths(lengths, U, T_max, &sum_T, &max_len));
  const DecBatchSession S = layout_dec_batch_session(*cfg, U, sum_T, max_len, max_steps, max_hyps, session);
  AVSR_REQUIRE_BYTES(S.bytes, session_bytes, "decoder batch session");
  const DecPrep P = layout_dec_prepared(*cfg, const_cast<void*>(prepared));
  return begin_batch_body(bk, *cfg, P, S, memory, lengths, U, T_max, sum_T, precision);
}

template <class BK>
int decoder_batch_step_entry(BK bk, const AvsrDecoderConfig* cfg, const void* prepared, void* session,
                             size_t session_bytes, const int32_t* lengths, int U, int T_max, int max_steps, int max_hyps,
                             const int32_t* tokens, const int32_t* anc, const int32_t* row_utt, int step, int n,
                             float* logp, void* workspace, size_t workspace_bytes, int precision) {
  AVSR_TRY(check_dec_cfg(cfg));
  AVSR_REQUIRE(prepared && session && tokens && row_utt && logp && workspace, "NULL argument");
  AVSR_REQUIRE(T_max > 0 && max_steps > 0 && max_hyps > 0, "decoder_batch_step: bad T_max=%d max_steps=%d max_hyps=%d",
               T_max, max_steps, max_hyps);
  AVSR_REQUIRE(step >= 0 && step < max_steps, "decoder_batch_step: step %d outside the session's %d positions", step,
               max_steps);
  AVSR_REQUIRE(n >= 0 && n <= max_hyps, "decoder_batch_step: n=%d hypotheses exceed the session's %d beam slots", n,
               max_hyps);
  AVSR_REQUIRE(step == 0 || anc != nullptr, "decoder_batch_step: step %d needs the ancestor table", step);
  AVSR_REQUIRE(valid_precision(precision), "bad precision %d", precision);
  long sum_T;
  int max_len;
  AVSR_TRY(check_batch_lengths(lengths, U, T_max, &sum_T, &max_len));
  if (n == 0) return AVSR_OK;
  const DecBatchSession S = layout_dec_batch_session(*cfg, U, sum_T, max_len, max_steps, max_hyps, session);
  const DecWork W = layout_dec_work(*cfg, T_max, max_steps, max_hyps, workspace);
  AVSR_REQUIRE_BYTES(S.bytes, session_bytes, "decoder batch session");
  AVSR_REQUIRE_BYTES(W.bytes, workspace_bytes, "decoder batch step workspace");
  const DecPrep P = layout_dec_prepared(*cfg, const_cast<void*>(prepared));
  return step_batch_body(bk, *cfg, P, S, W, tokens, anc, row_utt, step, n, U, T_max, sum_T, max_steps, max_hyps, logp,
                         precision);
}

template <class BK>
int ctc_prefix_batch_init_entry(BK bk, const float* logp, const int32_t* lengths, int U, int T_max, int O, int blank,
                                int32_t* lengths_dev, float* r0) {
  AVSR_REQUIRE(logp && lengths_dev && r0, "NULL argument");
  AVSR_REQUIRE(T_max > 0 && O > 1 && blank >= 0 && blank < O, "ctc_prefix_batch_init: bad T_max=%d O=%d blank=%d", T_max,
               O, blank);
  long sum_T;
  int max_len;
  AVSR_TRY(check_batch_lengths(lengths, U, T_max, &sum_T, &max_len));
  AVSR_TRY(bk.upload_i32(lengths_dev, lengths, U));
  return bk.for_each(U, CtcInitBatchElem{logp, lengths_dev, r0, U, T_max, O, blank});
}

template <class BK>
int ctc_prefix_batch_score_entry(BK bk, const float* logp, const int32_t* lengths, int U, int T_max, int O, int blank,
                                 int eos, int out_len, const int32_t* last_ids, const float* r_prev, const float* s_prev,
                                 const int32_t* cand, const int32_t* row_utt, int n, int S, float* local, float* r,
                                 float* log_psi) {
  AVSR_REQUIRE(logp && lengths && last_ids && r_prev && s_prev && cand && row_utt && local && r && log_psi,
               "NULL argument");
  AVSR_REQUIRE(U >= 1 && T_max > 0 && O > 1 && blank >= 0 && blank < O && eos >= 0 && eos < O && blank != eos,
               "ctc_prefix_batch_score: bad U=%d T_max=%d O=%d blank=%d eos=%d", U, T_max, O, blank, eos);
  AVSR_REQUIRE(out_len >= 0 && n >= 0 && S > 0 && S <= O, "ctc_prefix_batch_score: bad out_len=%d n=%d S=%d", out_len, n,
               S);
  if (n == 0) return AVSR_OK;
  return ctc_prefix_batch_body(bk, logp, lengths, T_max, O, blank, eos, out_len, last_ids, r_prev, s_prev, cand, row_utt,
                               n, S, local, r, log_psi);
}

}  // namespace dec
}  // namespace avsr
