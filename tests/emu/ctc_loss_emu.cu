// HOST replay of the CTC loss (csrc/ctc_loss.cu) -- TEST INFRASTRUCTURE ONLY (tests/emu/build.py builds it into
// tests/emu/_build/libavsr_ctc_loss_emu.so; nothing under auto_avsr_b200/ knows it exists).
//
// The CPU suite checks the label compaction, the extended-label mapping, the alpha / beta recursion and the gradient
// combination of csrc/ctc_loss_body.cuh by compiling that same header into plain loops that follow the kernels'
// schedule: per utterance the labels pass, per frame the row pass (log-sum-exp in fp32, then the gather), the two
// recursions frame by frame over two state rows, and the backward row pass.  Same extern "C" names and signatures as
// include/avsr_b200.h, HOST pointers.
#include <stdarg.h>

#include <algorithm>
#include <vector>

#include "../../auto_avsr_b200/csrc/ctc_loss_body.cuh"

namespace avsr {
static thread_local std::string g_emu_err;
void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_emu_err = buf;
}
}  // namespace avsr

using namespace avsr;
using namespace avsr::ctc;

static void recursion(const CtcState& st, int b, int T, int L, int Tmax, int Lmax, bool bwd, double* out) {
  const int S = 2 * L + 1, Smax = 2 * Lmax + 1, W = Lmax + 1;
  const int32_t* lab = st.labels + (long)b * (Lmax > 0 ? Lmax : 1);
  const float* lp = st.lp + (long)b * Tmax * W;
  std::vector<double> rows(2 * (size_t)Smax);
  for (int k = 0; k < T; ++k) {
    const int t = bwd ? T - 1 - k : k;
    double* cur = rows.data() + (k & 1) * Smax;
    const double* prev = rows.data() + ((k + 1) & 1) * Smax;
    for (int s = 0; s < S; ++s) {
      const float e = lp[(long)t * W + lp_col(s)];
      const double v = bwd ? (k == 0 ? beta_last(s, S, e) : beta_prev(prev, lab, s, S, e))
                          : (k == 0 ? alpha_first(s, e) : alpha_next(prev, lab, s, e));
      cur[s] = v;
      if (out) out[((long)b * Tmax + t) * Smax + s] = v;
    }
  }
  if (!bwd) {
    st.nll[b] = nll_from_alpha(rows.data() + ((T - 1) & 1) * Smax, S);
  }
}

extern "C" {
const char* avsr_last_error(void) { return g_emu_err.c_str(); }

size_t avsr_ctc_loss_state_bytes(int B, int Tmax, int Lmax) {
  if (B < 0 || Tmax < 0 || Lmax < 0) return 0;
  return layout_ctc_state(B, Tmax, Lmax, nullptr).bytes;
}

int avsr_ctc_loss_fwd(const float* logits, long ld, const int32_t* hlens, const int64_t* ys_pad, int B, int Tmax,
                      int Lmax, int odim, int ignore_id, int want_grad, float* nll, void* state, size_t state_bytes,
                      void*) {
  AVSR_REQUIRE(B >= 0 && Tmax >= 0 && Lmax >= 0 && Lmax <= kMaxLabels && odim >= 1 && ld >= odim, "emu: bad shape");
  const CtcState st = layout_ctc_state(B, Tmax, Lmax, state);
  if (st.bytes > state_bytes) return AVSR_E_WORKSPACE;
  const int Lstride = Lmax > 0 ? Lmax : 1, W = Lmax + 1;
  for (int b = 0; b < B; ++b)
    st.nlab[b] = utterance_labels(compact_labels(ys_pad + (long)b * Lmax, Lmax, ignore_id, odim, st.labels + (long)b * Lstride),
                                  hlens[b], Tmax);
  for (int b = 0; b < B; ++b) {
    const int L = st.nlab[b];
    if (L < 0) continue;
    for (int t = 0; t < hlens[b]; ++t) {
      const long row = (long)b * Tmax + t;
      const float* xr = logits + row * ld;
      float m = -INFINITY;
      for (int c = 0; c < odim; ++c) m = fmaxf(m, xr[c]);
      float s = 0.f;
      for (int c = 0; c < odim; ++c) s += xr[c] == -INFINITY ? 0.f : expf(xr[c] - m);
      const float lse = m + logf(s);
      st.lse[row] = lse;
      const int32_t* lab = st.labels + (long)b * Lstride;
      for (int j = 0; j <= L; ++j) st.lp[row * W + j] = xr[j == 0 ? 0 : lab[j - 1]] - lse;
    }
  }
  for (int b = 0; b < B; ++b) {
    const int L = st.nlab[b];
    const int T = L < 0 ? 0 : hlens[b];
    if (L < 0 || T == 0) {
      st.nll[b] = L < 0 ? NAN : nll_no_frames(L);
    } else {
      recursion(st, b, T, L, Tmax, Lmax, false, want_grad ? st.alpha : nullptr);
      if (want_grad) recursion(st, b, T, L, Tmax, Lmax, true, st.beta);
    }
    nll[b] = reported_nll(st.nll[b]);
  }
  return AVSR_OK;
}

int avsr_ctc_loss_bwd(const float* logits, long ld, const int32_t* hlens, const int64_t*, int B, int Tmax, int Lmax,
                      int odim, const float* dnll, const void* state, size_t state_bytes, float* dlogits, long ldd, void*) {
  AVSR_REQUIRE(ldd >= odim && ld >= odim, "emu: bad strides");
  const CtcState st = layout_ctc_state(B, Tmax, Lmax, const_cast<void*>(state));
  if (st.bytes > state_bytes) return AVSR_E_WORKSPACE;
  const int Lstride = Lmax > 0 ? Lmax : 1, W = Lmax + 1;
  const long Smax = 2 * Lmax + 1;
  for (int b = 0; b < B; ++b) {
    const int L = st.nlab[b];
    const double nll = st.nll[b];
    std::vector<float> post(Smax);
    for (int t = 0; t < Tmax; ++t) {
      const long row = (long)b * Tmax + t;
      float* dr = dlogits + row * ldd;
      const float* xr = logits + row * ld;
      if (L < 0) {
        const float v = t < std::min(std::max(hlens[b], 0), Tmax) ? NAN : 0.f;
        for (long c = 0; c < ldd; ++c) dr[c] = c < odim ? v : 0.f;
        continue;
      }
      if (t >= hlens[b] || nll == INFINITY) {
        for (long c = 0; c < ldd; ++c) dr[c] = 0.f;
        continue;
      }
      const float lse = st.lse[row], g = dnll[b];
      for (long c = 0; c < ldd; ++c) dr[c] = c < odim ? logit_grad(xr[c], lse, g, 0.f) : 0.f;
      const int32_t* lab = st.labels + (long)b * Lstride;
      for (int s = 0; s < 2 * L + 1; ++s)
        post[s] = state_posterior(st.alpha[row * Smax + s], st.beta[row * Smax + s], st.lp[row * W + lp_col(s)], nll);
      for (int j = 0; j <= L; ++j) {
        if (j > 0 && !first_occurrence(lab, j - 1)) continue;
        const int c = j == 0 ? 0 : lab[j - 1];
        dr[c] = logit_grad(xr[c], lse, g, token_occupancy(post.data(), lab, L, j));
      }
    }
  }
  return AVSR_OK;
}
}  // extern "C"
