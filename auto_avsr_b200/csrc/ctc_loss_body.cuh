// CTC loss and its gradient (the training loss of the CTC head, espnet/nets/pytorch_backend/ctc.py:32-65): the state
// layout and every per-element step, written as AVSR_HD code so that ONE source drives both the kernels of
// ctc_loss.cu and the host replay the CPU tests build (tests/emu/ctc_loss_emu.cu -- test infrastructure, never loaded
// by the package).
//
// What it computes is torch.nn.CTCLoss(reduction="none", zero_infinity=True) with blank 0 on log_softmax(logits), per
// utterance b of a padded batch:
//   labels  l = ys_pad[b][ys_pad[b] != ignore_id] (in order), L = |l|; extended sequence l' = (0, l_1, 0, ..., l_L, 0),
//           S = 2L + 1 states; state s emits column lp_col(s) of the gathered table lp[b][t][0..L] (0 = blank, j = l_j)
//   alpha_t(s) = lp(t, l'_s) + logsumexp(alpha_{t-1}(s), alpha_{t-1}(s-1), alpha_{t-1}(s-2) if can_skip(s))
//   beta_t(s)  = lp(t, l'_s) + logsumexp(beta_{t+1}(s), beta_{t+1}(s+1), beta_{t+1}(s+2) if can_skip(s+2))
//   nll = -logsumexp(alpha_{T-1}(S-1), alpha_{T-1}(S-2)),  T = hlens[b]
//   d nll / d logits[t][c] = exp(x - lse_t) - sum_{s: l'_s = c} exp(alpha_t(s) + beta_t(s) - lp(t, c) + nll)
// (torch's convention: alpha and beta both include the emission at t).  alpha, beta and nll are fp64: over hundreds of
// frames they reach thousands in magnitude, and fp32 rounding there would leave ~1e-3 in the exponent of the gradient's
// state posteriors.  T = 0 gives nll 0 for L = 0 and +inf otherwise,
// as torch does.  An utterance whose nll is +inf contributes loss 0 and gradient 0 (zero_infinity).  A kept label
// outside [1, odim) or hlens[b] outside [0, Tmax] marks the utterance invalid: its loss is NaN and no table is indexed
// with the bad value.
#pragma once
#include <math.h>

#include "common.cuh"

namespace avsr {
namespace ctc {

constexpr int kMaxLabels = 1024;   // Lmax bound: the recursion keeps two state rows + an emission chunk in shared memory

// ------------------------------------------------------------------ state (caller-owned, 256-byte aligned slots)
struct CtcState {
  int32_t* labels;   // (B, max(Lmax, 1)) compacted label rows
  int32_t* nlab;     // (B) label count L, -1 = invalid utterance
  double* nll;       // (B) raw negative log-likelihood (+inf kept: the backward zeroes those utterances)
  float* lse;        // (B * Tmax) log-sum-exp of each valid logits row
  float* lp;         // (B, Tmax, Lmax + 1) log-probs of blank and of each label
  double* alpha;     // (B, Tmax, 2 Lmax + 1)
  double* beta;      // (B, Tmax, 2 Lmax + 1)
  size_t bytes;
};

static inline CtcState layout_ctc_state(int B, int Tmax, int Lmax, void* base) {
  CtcState s{};
  char* p = reinterpret_cast<char*>(base);
  size_t off = 0;
  auto take = [&](size_t n, size_t esz = 4) {
    char* r = p + off;
    off += align_up(n * esz, 256);
    return p ? r : nullptr;
  };
  const size_t BT = (size_t)B * Tmax, Smax = 2 * (size_t)Lmax + 1;
  s.labels = reinterpret_cast<int32_t*>(take((size_t)B * (Lmax > 0 ? Lmax : 1)));
  s.nlab = reinterpret_cast<int32_t*>(take((size_t)B));
  s.nll = reinterpret_cast<double*>(take((size_t)B, 8));
  s.lse = reinterpret_cast<float*>(take(BT));
  s.lp = reinterpret_cast<float*>(take(BT * (Lmax + 1)));
  s.alpha = reinterpret_cast<double*>(take(BT * Smax, 8));
  s.beta = reinterpret_cast<double*>(take(BT * Smax, 8));
  s.bytes = off;
  return s;
}

// ------------------------------------------------------------------ labels
// y[y != ignore_id] of one padded row into `out`; -> L, or -1 when a kept id lies outside [1, odim) (stored as 1 so
// that nothing downstream indexes with it)
AVSR_HD int compact_labels(const int64_t* row, int Lmax, int64_t ignore_id, int odim, int32_t* out) {
  int n = 0;
  bool bad = false;
  for (int j = 0; j < Lmax; ++j) {
    const int64_t y = row[j];
    if (y == ignore_id) continue;
    const bool ok = y >= 1 && y < odim;
    bad = bad || !ok;
    out[n++] = ok ? (int32_t)y : 1;
  }
  return bad ? -1 : n;
}

// L, or -1 when the utterance cannot be evaluated (bad label, hlen outside [0, Tmax])
AVSR_HD int utterance_labels(int compacted, int hlen, int Tmax) { return (hlen < 0 || hlen > Tmax) ? -1 : compacted; }

// ------------------------------------------------------------------ extended label sequence
AVSR_HD int lp_col(int s) { return (s & 1) ? (s >> 1) + 1 : 0; }
// may state s be entered from s - 2 (two different labels with no blank between them)
AVSR_HD bool can_skip(const int32_t* lab, int s) { return (s & 1) && s >= 3 && lab[s >> 1] != lab[(s >> 1) - 1]; }

// log(exp(a) + exp(b)) where either may be -inf (an unreachable state)
AVSR_HD double lae(double a, double b) {
  const double m = fmax(a, b);
  return m == -INFINITY ? m : m + log1p(exp(-fabs(a - b)));
}

// ------------------------------------------------------------------ recursion (one state per call; `em` = its emission)
AVSR_HD double alpha_first(int s, float em) { return s < 2 ? (double)em : -INFINITY; }
AVSR_HD double alpha_next(const double* prev, const int32_t* lab, int s, float em) {
  double a = prev[s];
  if (s >= 1) a = lae(a, prev[s - 1]);
  if (can_skip(lab, s)) a = lae(a, prev[s - 2]);
  return a + em;
}
AVSR_HD double beta_last(int s, int S, float em) { return s >= S - 2 ? (double)em : -INFINITY; }
AVSR_HD double beta_prev(const double* next, const int32_t* lab, int s, int S, float em) {
  double b = next[s];
  if (s + 1 < S) b = lae(b, next[s + 1]);
  if (s + 2 < S && can_skip(lab, s + 2)) b = lae(b, next[s + 2]);
  return b + em;
}
// nll from the state row at t = T - 1
AVSR_HD double nll_from_alpha(const double* last, int S) {
  const double a = S >= 2 ? lae(last[S - 1], last[S - 2]) : last[S - 1];
  return -a;
}
// nll of an utterance that has no frame (T = 0): torch gives 0 for the empty target, +inf otherwise
AVSR_HD double nll_no_frames(int L) { return L == 0 ? 0.0 : INFINITY; }
// what the loss reports: zero_infinity=True
AVSR_HD float reported_nll(double raw) { return raw == INFINITY ? 0.f : (float)raw; }

// ------------------------------------------------------------------ gradient
// Does compacted label j carry a token that no earlier label has?  Its thread then owns that token's logit.
AVSR_HD bool first_occurrence(const int32_t* lab, int j) {
  for (int i = 0; i < j; ++i)
    if (lab[i] == lab[j]) return false;
  return true;
}
// posterior of state s at frame t: exp(alpha + beta - lp + nll) (both alpha and beta contain the emission lp)
AVSR_HD float state_posterior(double a, double b, float lpv, double nll) { return (float)exp(a + b - (double)lpv + nll); }
// sum of the state posteriors `post` of the states emitting column `col` (0 = blank: all even states; j >= 1: every label
// position with the token of label j - 1, which must be its first occurrence), in state order
AVSR_HD float token_occupancy(const float* post, const int32_t* lab, int L, int col) {
  float acc = 0.f;
  if (col == 0) {
    for (int s = 0; s <= 2 * L; s += 2) acc += post[s];
  } else {
    const int32_t tok = lab[col - 1];
    for (int j = col - 1; j < L; ++j)
      if (lab[j] == tok) acc += post[2 * j + 1];
  }
  return acc;
}
// d logits = dnll * (softmax - occupancy)
AVSR_HD float logit_grad(float x, float lse, float dnll, float occupancy) { return dnll * (expf(x - lse) - occupancy); }

}  // namespace ctc
}  // namespace avsr
