// CTC loss forward / backward on the device (espnet/nets/pytorch_backend/ctc.py:32-65: torch.nn.CTCLoss(zero_infinity)
// on log_softmax(ctc_lo(hs))).  The math lives in ctc_loss_body.cuh; this file is the launch schedule:
//
//   ctc_labels_kernel      one thread per utterance: y[y != ignore_id] compacted on the device (no host copy)
//   ctc_rows_fwd_kernel    one 256-thread CTA per valid frame: ONE read of the logits row -> log-sum-exp (MaxSum),
//                          then the log-probs of blank and of the utterance's labels into lp (B, Tmax, Lmax+1)
//   ctc_recursion_kernel   one CTA per (utterance, direction): alpha (y = 0) and, for a gradient, beta (y = 1) over the
//                          S = 2L+1 extended states, states across threads, one barrier per frame; the emissions are
//                          staged a chunk of frames at a time in shared memory; y = 0 also writes nll
//   ctc_rows_bwd_kernel    one 256-thread CTA per frame: the frame's state posteriors staged in shared memory, then
//                          d logits = dnll * (softmax - occupancy), the occupancy of each distinct token summed by one
//                          thread in state order; padded frames / columns get 0
// The recursion runs in fp64 (see ctc_loss_body.cuh); it is latency-bound (one barrier per frame), not arithmetic-bound.
//
// Every sum has a fixed order (no atomics): two identical calls give identical bits.  HBM traffic: the forward reads the
// valid logits once, the backward reads them again and writes dlogits; everything else is (B, Tmax, O(L)).
#include "ctc_loss_body.cuh"
#include "maxsum.cuh"

namespace avsr {
namespace ctc {

constexpr int kSmemBudget = 48 * 1024;   // the recursion's shared memory (no opt-in needed)

__global__ void ctc_labels_kernel(const int64_t* __restrict__ ys, const int32_t* __restrict__ hlens, int B, int Tmax,
                                  int Lmax, int odim, long long ignore_id, CtcState st) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int n = compact_labels(ys + (long)b * Lmax, Lmax, (int64_t)ignore_id, odim, st.labels + (long)b * (Lmax > 0 ? Lmax : 1));
  st.nlab[b] = utterance_labels(n, hlens[b], Tmax);
}

__global__ void __launch_bounds__(256) ctc_rows_fwd_kernel(const float* __restrict__ x, long ld,
                                                           const int32_t* __restrict__ hlens, int Tmax, int Lmax,
                                                           int odim, CtcState st) {
  pdl_launch_dependents();
  const int row = blockIdx.x, b = row / Tmax, t = row - b * Tmax;
  pdl_wait();
  const int L = st.nlab[b];
  if (L < 0 || t >= hlens[b]) return;                    // CTA-uniform
  const float* xr = x + (long)row * ld;
  MaxSum acc{-INFINITY, 0.f, 0x7fffffff};
  for (int c = threadIdx.x; c < odim; c += 256) ms_push(acc, xr[c], c);
  const MaxSum tot = ms_block_reduce_256(acc);
  const float lse = tot.m + logf(tot.s);
  if (threadIdx.x == 0) st.lse[row] = lse;
  const int32_t* lab = st.labels + (long)b * (Lmax > 0 ? Lmax : 1);
  float* lpr = st.lp + (long)row * (Lmax + 1);
  for (int j = threadIdx.x; j <= L; j += 256) lpr[j] = xr[j == 0 ? 0 : lab[j - 1]] - lse;
}

// shared memory: [2][Smax] fp64 state rows | [F][Lmax+1] emission chunk | [Lmax] labels
__global__ void __launch_bounds__(1024) ctc_recursion_kernel(const int32_t* __restrict__ hlens, int Tmax, int Lmax,
                                                             int F, int store_alpha, float* __restrict__ nll_out,
                                                             CtcState st) {
  extern __shared__ double ctc_smem[];
  pdl_launch_dependents();
  const int b = blockIdx.x;
  const bool bwd = blockIdx.y == 1;
  pdl_wait();
  const int L = st.nlab[b];
  const int T = L < 0 ? 0 : hlens[b];
  if (L < 0 || T == 0) {
    if (!bwd && threadIdx.x == 0) {
      const double raw = L < 0 ? (double)NAN : nll_no_frames(L);
      st.nll[b] = raw;
      nll_out[b] = reported_nll(raw);
    }
    return;
  }
  const int S = 2 * L + 1, Smax = 2 * Lmax + 1, W = Lmax + 1;
  double* rows = ctc_smem;                                // [2][Smax]
  float* em = reinterpret_cast<float*>(ctc_smem + 2 * Smax);   // [F][W]
  int32_t* lab = reinterpret_cast<int32_t*>(em + (long)F * W);
  const int32_t* glab = st.labels + (long)b * (Lmax > 0 ? Lmax : 1);
  for (int j = threadIdx.x; j < L; j += blockDim.x) lab[j] = glab[j];
  const float* lp = st.lp + (long)b * Tmax * W;
  double* out = bwd ? st.beta : (store_alpha ? st.alpha : nullptr);
  if (out) out += (long)b * Tmax * Smax;
  for (int k = 0; k < T; ++k) {
    const int t = bwd ? T - 1 - k : k;
    const int kc = k % F;
    if (kc == 0) {                                        // stage the next chunk of frames (the previous one is consumed)
      const int n = min(F, T - k);
      for (int e = threadIdx.x; e < n * (L + 1); e += blockDim.x) {
        const int i = e / (L + 1), j = e - i * (L + 1);
        em[i * W + j] = lp[(long)(bwd ? t - i : t + i) * W + j];
      }
      __syncthreads();
    }
    const float* er = em + kc * W;
    double* cur = rows + (k & 1) * Smax;
    const double* prev = rows + ((k + 1) & 1) * Smax;
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
      const float e = er[lp_col(s)];
      const double v = bwd ? (k == 0 ? beta_last(s, S, e) : beta_prev(prev, lab, s, S, e))
                          : (k == 0 ? alpha_first(s, e) : alpha_next(prev, lab, s, e));
      cur[s] = v;
      if (out) out[(long)t * Smax + s] = v;
    }
    __syncthreads();
  }
  if (!bwd && threadIdx.x == 0) {
    const double raw = nll_from_alpha(rows + ((T - 1) & 1) * Smax, S);
    st.nll[b] = raw;
    nll_out[b] = reported_nll(raw);
  }
}

// shared memory: [Smax] state posteriors of the frame | [Lmax] labels
__global__ void __launch_bounds__(256) ctc_rows_bwd_kernel(const float* __restrict__ x, long ld,
                                                           const int32_t* __restrict__ hlens, int Tmax, int Lmax,
                                                           int odim, const float* __restrict__ dnll, CtcState st,
                                                           float* __restrict__ dx, long ldd) {
  extern __shared__ float ctc_post[];
  pdl_launch_dependents();
  const int row = blockIdx.x, b = row / Tmax, t = row - b * Tmax;
  float* dr = dx + (long)row * ldd;
  pdl_wait();
  const int L = st.nlab[b];
  const double nll = st.nll[b];
  if (L < 0) {                                           // invalid utterance: NaN loss, NaN gradient on its frames
    const int h = hlens[b];
    const float v = t < min(max(h, 0), Tmax) ? NAN : 0.f;
    for (int c = threadIdx.x; c < ldd; c += 256) dr[c] = c < odim ? v : 0.f;
    return;
  }
  if (t >= hlens[b] || nll == INFINITY) {                // padding frame, or zero_infinity
    for (int c = threadIdx.x; c < ldd; c += 256) dr[c] = 0.f;
    return;
  }
  const int S = 2 * L + 1, Smax = 2 * Lmax + 1;
  int32_t* lab = reinterpret_cast<int32_t*>(ctc_post + Smax);
  const int32_t* glab = st.labels + (long)b * (Lmax > 0 ? Lmax : 1);
  const double* a = st.alpha + (long)row * Smax;
  const double* be = st.beta + (long)row * Smax;
  const float* lpr = st.lp + (long)row * (Lmax + 1);
  for (int s = threadIdx.x; s < S; s += 256) ctc_post[s] = state_posterior(a[s], be[s], lpr[lp_col(s)], nll);
  for (int j = threadIdx.x; j < L; j += 256) lab[j] = glab[j];
  const float* xr = x + (long)row * ld;
  const float lse = st.lse[row], g = dnll[b];
  for (int c = threadIdx.x; c < ldd; c += 256) dr[c] = c < odim ? logit_grad(xr[c], lse, g, 0.f) : 0.f;
  __syncthreads();                                       // posteriors staged; token columns are rewritten below
  for (int j = threadIdx.x; j <= L; j += 256) {          // j = 0: blank, j >= 1: label j - 1
    if (j > 0 && !first_occurrence(lab, j - 1)) continue;
    const int c = j == 0 ? 0 : lab[j - 1];
    dr[c] = logit_grad(xr[c], lse, g, token_occupancy(ctc_post, lab, L, j));
  }
}

static int recursion_config(int Lmax, int* threads, int* frames, size_t* smem) {
  const int Smax = 2 * Lmax + 1, W = Lmax + 1;
  const size_t fixed = (size_t)2 * Smax * 8 + (size_t)(Lmax > 0 ? Lmax : 1) * 4;
  const long F = ((long)kSmemBudget - (long)fixed) / ((long)W * 4);
  if (F < 1) return AVSR_E_INVALID;
  *frames = (int)(F > 64 ? 64 : F);
  *threads = Smax >= 1024 ? 1024 : (Smax + 31) / 32 * 32;
  *smem = fixed + (size_t)(*frames) * W * 4;
  return AVSR_OK;
}

}  // namespace ctc
}  // namespace avsr

using namespace avsr;
using namespace avsr::ctc;

extern "C" {

size_t avsr_ctc_loss_state_bytes(int B, int Tmax, int Lmax) {
  if (B < 0 || Tmax < 0 || Lmax < 0) return 0;
  return layout_ctc_state(B, Tmax, Lmax, nullptr).bytes;
}

static int ctc_check(const float* logits, long ld, const int32_t* hlens, const int64_t* ys_pad, int B, int Tmax,
                     int Lmax, int odim, const void* state, size_t state_bytes) {
  AVSR_REQUIRE(B >= 0 && Tmax >= 0 && Lmax >= 0 && Lmax <= kMaxLabels && odim >= 1 && ld >= odim,
               "ctc_loss: bad B=%d Tmax=%d Lmax=%d (<= %d) odim=%d ld=%ld", B, Tmax, Lmax, kMaxLabels, odim, ld);
  AVSR_REQUIRE(B == 0 || (hlens && state && (Lmax == 0 || ys_pad) && (Tmax == 0 || logits)), "NULL argument");
  if (layout_ctc_state(B, Tmax, Lmax, nullptr).bytes > state_bytes) {
    set_error("ctc_loss: state too small: need %zu bytes, got %zu", layout_ctc_state(B, Tmax, Lmax, nullptr).bytes,
              state_bytes);
    return AVSR_E_WORKSPACE;
  }
  return AVSR_OK;
}

int avsr_ctc_loss_fwd(const float* logits, long ld, const int32_t* hlens, const int64_t* ys_pad, int B, int Tmax,
                      int Lmax, int odim, int ignore_id, int want_grad, float* nll, void* state, size_t state_bytes,
                      void* stream) {
  AVSR_TRY(ctc_check(logits, ld, hlens, ys_pad, B, Tmax, Lmax, odim, state, state_bytes));
  AVSR_REQUIRE(B == 0 || nll, "NULL argument");
  if (B == 0) return AVSR_OK;
  int threads = 0, frames = 0;
  size_t smem = 0;
  AVSR_TRY(recursion_config(Lmax, &threads, &frames, &smem));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const CtcState S = layout_ctc_state(B, Tmax, Lmax, state);
  AVSR_LAUNCH(ctc_labels_kernel, cdiv(B, 128), 128, 0, st, ys_pad, hlens, B, Tmax, Lmax, odim, (long long)ignore_id, S);
  if ((long)B * Tmax > 0)
    AVSR_LAUNCH(ctc_rows_fwd_kernel, B * Tmax, 256, 0, st, logits, ld, hlens, Tmax, Lmax, odim, S);
  AVSR_LAUNCH(ctc_recursion_kernel, dim3(B, want_grad ? 2 : 1), threads, smem, st, hlens, Tmax, Lmax, frames,
              want_grad ? 1 : 0, nll, S);
  return AVSR_OK;
}

int avsr_ctc_loss_bwd(const float* logits, long ld, const int32_t* hlens, const int64_t* ys_pad, int B, int Tmax,
                      int Lmax, int odim, const float* dnll, const void* state, size_t state_bytes, float* dlogits,
                      long ldd, void* stream) {
  AVSR_TRY(ctc_check(logits, ld, hlens, ys_pad, B, Tmax, Lmax, odim, state, state_bytes));
  AVSR_REQUIRE(ldd >= odim, "ctc_loss_bwd: ldd=%ld < odim=%d", ldd, odim);
  if ((long)B * Tmax == 0) return AVSR_OK;
  AVSR_REQUIRE(dnll && dlogits, "NULL argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const CtcState S = layout_ctc_state(B, Tmax, Lmax, const_cast<void*>(state));
  const size_t smem = (size_t)(2 * Lmax + 1) * 4 + (size_t)(Lmax > 0 ? Lmax : 1) * 4;   // <= 12 KB
  AVSR_LAUNCH(ctc_rows_bwd_kernel, B * Tmax, 256, smem, st, logits, ld, hlens, Tmax, Lmax, odim, dnll, S, dlogits, ldd);
  return AVSR_OK;
}

}  // extern "C"
