// Device side of the attention-decoder scoring path and the CTC prefix scorer (SURVEY.md 8f #3): the backend that
// runs decoder_body.cuh's schedule on the GPU, and the C ABI of include/avsr_b200.h for it.
//
// The projections are the library's GEMMs (wgmma gemm_tc for AVSR_PREC_F16 / TF32 -- at n <= 40 hypotheses they are
// weight-streaming launches of the persistent one-CTA kernel, the S1 regime of the encoder --, CUDA-core gemm_simt for
// AVSR_PREC_FP32), LayerNorm and log-softmax are the encoder path's kernels; the attention over the slot-addressed K/V
// cache, the embedding and the CTC forward recursion are per-element functors launched as plain grids (one thread per
// output element, no cross-thread communication: at 40 hypotheses x 12 heads these are microsecond kernels whose cost
// is the launch).  Plain launches (no PDL attribute): each waits for the full completion of its predecessor, and the
// PDL kernels that follow wait in griddepcontrol.wait for these.
#include "decoder_body.cuh"

namespace avsr {
namespace dec {

template <class F>
__global__ void __launch_bounds__(256) for_each_kernel(long count, F f) {
  const long idx = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (idx < count) f(idx);
}

struct DeviceBackend {
  cudaStream_t st;

  template <class F>
  int for_each(long count, const F& f) {
    if (count <= 0) return AVSR_OK;
    const long blocks = (count + 255) / 256;
    AVSR_REQUIRE(blocks <= 0x7fffffffL, "decoder: %ld elements exceed one grid", count);
    for_each_kernel<F><<<(unsigned)blocks, 256, 0, st>>>(count, f);
    AVSR_CHECK_LAUNCH();
    return AVSR_OK;
  }
  int gemm(int prec, const void* A, const void* W, int M, int N, int K, const float* bias, void* out, const float* resid,
           float alpha, int relu, int out_is_operand) {
    EpiParams e{};
    e.M = M; e.N = N; e.bias = bias; e.out = out; e.ldo = N; e.resid = resid; e.alpha = alpha; e.relu = relu;
    e.round_out = (out_is_operand && prec != AVSR_PREC_FP32) ? 1 : 0;
    if (prec == AVSR_PREC_FP32)
      return gemm_simt(EPI_LINEAR, reinterpret_cast<const float*>(A), reinterpret_cast<const float*>(W), M, N, K, e, st);
    return gemm_tc(EPI_LINEAR, dec_operand_kind(prec), A, W, M, N, K, e, st);
  }
  int layernorm(const float* x, const float* g, const float* b, void* y, int rows, int d, int out_kind) {
    return launch_layernorm(x, g, b, y, rows, d, out_kind, st);
  }
  int log_softmax(const float* x, long ldx, float* y, long ldy, int rows, int n) {
    return launch_log_softmax_rows(x, ldx, y, ldy, nullptr, rows, n, st);
  }
};

static int check_dec_cfg(const AvsrDecoderConfig* c) {
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
static inline bool dec_valid_precision(int p) { return p == AVSR_PREC_FP32 || p == AVSR_PREC_TF32 || p == AVSR_PREC_F16; }

}  // namespace dec
}  // namespace avsr

using namespace avsr;
using namespace avsr::dec;

extern "C" {

size_t avsr_decoder_prepared_bytes(const AvsrDecoderConfig* cfg) {
  if (check_dec_cfg(cfg) != AVSR_OK) return 0;
  return layout_dec_prepared(*cfg, nullptr).bytes;
}

int avsr_prepare_decoder(const AvsrDecoderConfig* cfg, const AvsrDecoderLayerParams* layers, const float* embed_w,
                         const float* after_norm_w, const float* after_norm_b, const float* out_w, const float* out_b,
                         void* prepared, size_t prepared_bytes, int precision, void* stream) {
  AVSR_TRY(check_dec_cfg(cfg));
  AVSR_REQUIRE(layers && embed_w && after_norm_w && after_norm_b && out_w && out_b && prepared, "NULL argument");
  AVSR_REQUIRE(dec_valid_precision(precision), "bad precision %d", precision);
  for (int l = 0; l < cfg->num_blocks; ++l) {
    const void* const* p = reinterpret_cast<const void* const*>(&layers[l]);
    for (size_t k = 0; k < sizeof(AvsrDecoderLayerParams) / sizeof(void*); ++k)
      AVSR_REQUIRE(p[k] != nullptr, "decoder layer %d: parameter %zu is NULL", l, k);
  }
  const DecPrep P = layout_dec_prepared(*cfg, prepared);
  if (P.bytes > prepared_bytes) {
    set_error("decoder prepared buffer too small: need %zu bytes, got %zu", P.bytes, prepared_bytes);
    return AVSR_E_WORKSPACE;
  }
  DeviceBackend bk{reinterpret_cast<cudaStream_t>(stream)};
  return prepare_body(bk, *cfg, layers, embed_w, after_norm_w, after_norm_b, out_w, out_b, P, precision);
}

size_t avsr_decoder_session_bytes(const AvsrDecoderConfig* cfg, int T, int max_steps, int max_hyps) {
  if (check_dec_cfg(cfg) != AVSR_OK || T <= 0 || max_steps <= 0 || max_hyps <= 0) return 0;
  return layout_dec_session(*cfg, T, max_steps, max_hyps, nullptr).bytes;
}

int avsr_decoder_begin(const AvsrDecoderConfig* cfg, const void* prepared, const float* memory, int T, int max_steps,
                       int max_hyps, void* session, size_t session_bytes, int precision, void* stream) {
  AVSR_TRY(check_dec_cfg(cfg));
  AVSR_REQUIRE(prepared && memory && session, "NULL argument");
  AVSR_REQUIRE(T > 0 && max_steps > 0 && max_hyps > 0, "decoder_begin: bad T=%d max_steps=%d max_hyps=%d", T, max_steps, max_hyps);
  AVSR_REQUIRE(dec_valid_precision(precision), "bad precision %d", precision);
  const DecSession S = layout_dec_session(*cfg, T, max_steps, max_hyps, session);
  if (S.bytes > session_bytes) {
    set_error("decoder session too small: need %zu bytes, got %zu", S.bytes, session_bytes);
    return AVSR_E_WORKSPACE;
  }
  const DecPrep P = layout_dec_prepared(*cfg, const_cast<void*>(prepared));
  DeviceBackend bk{reinterpret_cast<cudaStream_t>(stream)};
  return begin_body(bk, *cfg, P, S, memory, T, precision);
}

size_t avsr_decoder_step_workspace_bytes(const AvsrDecoderConfig* cfg, int T, int max_steps, int max_hyps) {
  if (check_dec_cfg(cfg) != AVSR_OK || T <= 0 || max_steps <= 0 || max_hyps <= 0) return 0;
  return layout_dec_work(*cfg, T, max_steps, max_hyps, nullptr).bytes;
}

int avsr_decoder_step(const AvsrDecoderConfig* cfg, const void* prepared, void* session, size_t session_bytes, int T,
                      int max_steps, int max_hyps, const int32_t* tokens, const int32_t* anc, int step, int n, float* logp,
                      void* workspace, size_t workspace_bytes, int precision, void* stream) {
  AVSR_TRY(check_dec_cfg(cfg));
  AVSR_REQUIRE(prepared && session && tokens && logp && workspace, "NULL argument");
  AVSR_REQUIRE(T > 0 && max_steps > 0 && max_hyps > 0, "decoder_step: bad T=%d max_steps=%d max_hyps=%d", T, max_steps, max_hyps);
  AVSR_REQUIRE(step >= 0 && step < max_steps, "decoder_step: step %d outside the session's %d positions", step, max_steps);
  AVSR_REQUIRE(n >= 0 && n <= max_hyps, "decoder_step: n=%d hypotheses exceed the session's %d beam slots", n, max_hyps);
  AVSR_REQUIRE(step == 0 || anc != nullptr, "decoder_step: step %d needs the ancestor table", step);
  AVSR_REQUIRE(dec_valid_precision(precision), "bad precision %d", precision);
  if (n == 0) return AVSR_OK;
  const DecSession S = layout_dec_session(*cfg, T, max_steps, max_hyps, session);
  const DecWork W = layout_dec_work(*cfg, T, max_steps, max_hyps, workspace);
  if (S.bytes > session_bytes) {
    set_error("decoder session too small: need %zu bytes, got %zu", S.bytes, session_bytes);
    return AVSR_E_WORKSPACE;
  }
  if (W.bytes > workspace_bytes) {
    set_error("decoder step workspace too small: need %zu bytes, got %zu", W.bytes, workspace_bytes);
    return AVSR_E_WORKSPACE;
  }
  const DecPrep P = layout_dec_prepared(*cfg, const_cast<void*>(prepared));
  DeviceBackend bk{reinterpret_cast<cudaStream_t>(stream)};
  return step_body(bk, *cfg, P, S, W, tokens, anc, step, n, T, max_steps, max_hyps, logp, precision);
}

int avsr_ctc_prefix_init(const float* logp, int T, int O, int blank, float* r0, void* stream) {
  AVSR_REQUIRE(logp && r0, "NULL argument");
  AVSR_REQUIRE(T > 0 && O > 1 && blank >= 0 && blank < O, "ctc_prefix_init: bad T=%d O=%d blank=%d", T, O, blank);
  DeviceBackend bk{reinterpret_cast<cudaStream_t>(stream)};
  return bk.for_each(1, CtcInitElem{logp, r0, T, O, blank});
}

int avsr_ctc_prefix_score(const float* logp, int T, int O, int blank, int eos, int out_len, const int32_t* last_ids,
                          const float* r_prev, const float* s_prev, const int32_t* cand, int n, int S, float* local,
                          float* r, float* log_psi, void* stream) {
  AVSR_REQUIRE(logp && last_ids && r_prev && s_prev && cand && local && r && log_psi, "NULL argument");
  AVSR_REQUIRE(T > 0 && O > 1 && blank >= 0 && blank < O && eos >= 0 && eos < O && blank != eos,
               "ctc_prefix_score: bad T=%d O=%d blank=%d eos=%d", T, O, blank, eos);
  AVSR_REQUIRE(out_len >= 0 && n >= 0 && S > 0 && S <= O, "ctc_prefix_score: bad out_len=%d n=%d S=%d", out_len, n, S);
  if (n == 0) return AVSR_OK;
  DeviceBackend bk{reinterpret_cast<cudaStream_t>(stream)};
  return ctc_prefix_body(bk, logp, T, O, blank, eos, out_len, last_ids, r_prev, s_prev, cand, n, S, local, r, log_psi);
}

int avsr_ctc_prefix_select(const float* r, const float* log_psi, const int32_t* cand, const int32_t* parent,
                           const int32_t* token, int T, int O, int n, int S, int m, float* r_next, float* s_next,
                           void* stream) {
  AVSR_REQUIRE(r && log_psi && cand && parent && token && r_next && s_next, "NULL argument");
  AVSR_REQUIRE(T > 0 && O > 1 && n > 0 && S > 0 && m >= 0, "ctc_prefix_select: bad T=%d O=%d n=%d S=%d m=%d", T, O, n, S, m);
  if (m == 0) return AVSR_OK;
  DeviceBackend bk{reinterpret_cast<cudaStream_t>(stream)};
  return ctc_select_body(bk, r, log_psi, cand, parent, token, T, O, n, S, m, r_next, s_next);
}

}  // extern "C"
