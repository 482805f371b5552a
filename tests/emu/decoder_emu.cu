// HOST replay of the decoder / CTC-prefix schedule -- TEST INFRASTRUCTURE ONLY (tests/emu/build.py builds it into
// tests/emu/_build/libavsr_decoder_emu.so; nothing under auto_avsr_b200/ knows it exists).
//
// There is no GPU in the build container, so the CPU suite checks the part of csrc/decoder.cu that is NOT one of the
// already GPU-verified kernels -- the launch schedule, the buffer layouts, the slot / ancestor addressing and every
// per-element functor of decoder_body.cuh -- by compiling that same header against this backend: functors run as plain
// loops, the GEMM / LayerNorm / log-softmax launchers (verified on the GPU by the encoder tests) are replaced by
// naive fp32 loops.  Same extern "C" names and signatures as include/avsr_b200.h, forwarded to the same entry bodies
// (argument checks, layouts, size checks) as csrc/decoder.cu; HOST pointers, AVSR_PREC_FP32 only.
#include <stdarg.h>

#include <vector>

#include "../../auto_avsr_b200/csrc/decoder_body.cuh"

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
std::atomic<uint64_t> g_launches{0};

namespace dec {
struct HostBackend {
  template <class F>
  int for_each(long count, const F& f) {
    for (long i = 0; i < count; ++i) f(i);
    g_launches.fetch_add(1);
    return AVSR_OK;
  }
  int gemm(int prec, const void* A, const void* W, int M, int N, int K, const float* bias, void* out, const float* resid,
           float alpha, int relu, int /*out_is_operand*/) {
    AVSR_REQUIRE(prec == AVSR_PREC_FP32, "emu: fp32 only");
    AVSR_REQUIRE(N % 8 == 0 && K % 64 == 0, "emu gemm: N=%d %% 8, K=%d %% 64 (the device GEMMs' contract)", N, K);
    const float* a = reinterpret_cast<const float*>(A);
    const float* w = reinterpret_cast<const float*>(W);
    float* o = reinterpret_cast<float*>(out);
    for (int m = 0; m < M; ++m)
      for (int n = 0; n < N; ++n) {
        double acc = 0.0;
        for (int k = 0; k < K; ++k) acc += (double)a[(long)m * K + k] * w[(long)n * K + k];
        float v = (float)acc + (bias ? bias[n] : 0.f);
        if (relu) v = v > 0.f ? v : 0.f;
        if (resid) v = resid[(long)m * N + n] + alpha * v;
        o[(long)m * N + n] = v;
      }
    g_launches.fetch_add(1);
    return AVSR_OK;
  }
  int layernorm(const float* x, const float* g, const float* b, void* y, int rows, int d, int out_kind) {
    AVSR_REQUIRE(out_kind == OP_F32, "emu: fp32 only");
    float* o = reinterpret_cast<float*>(y);
    for (int r = 0; r < rows; ++r) {
      double mu = 0, var = 0;
      for (int c = 0; c < d; ++c) mu += x[(long)r * d + c];
      mu /= d;
      for (int c = 0; c < d; ++c) { const double t = x[(long)r * d + c] - mu; var += t * t; }
      var /= d;
      const double rs = 1.0 / sqrt(var + 1e-12);
      for (int c = 0; c < d; ++c) o[(long)r * d + c] = (float)((x[(long)r * d + c] - mu) * rs * g[c] + b[c]);
    }
    g_launches.fetch_add(1);
    return AVSR_OK;
  }
  int log_softmax(const float* x, long ldx, float* y, long ldy, int rows, int n) {
    for (int r = 0; r < rows; ++r) {
      double m = x[r * ldx];
      for (int c = 1; c < n; ++c) m = x[r * ldx + c] > m ? x[r * ldx + c] : m;
      double s = 0;
      for (int c = 0; c < n; ++c) s += exp(x[r * ldx + c] - m);
      const double lse = m + log(s);
      for (int c = 0; c < n; ++c) y[r * ldy + c] = (float)(x[r * ldx + c] - lse);
    }
    g_launches.fetch_add(1);
    return AVSR_OK;
  }
};
}  // namespace dec
}  // namespace avsr

using namespace avsr;
using namespace avsr::dec;

extern "C" {
const char* avsr_last_error(void) { return g_emu_err.c_str(); }
uint64_t avsr_launch_count(void) { return g_launches.load(); }

size_t avsr_decoder_prepared_bytes(const AvsrDecoderConfig* cfg) { return decoder_prepared_bytes_entry(cfg); }
int avsr_prepare_decoder(const AvsrDecoderConfig* cfg, const AvsrDecoderLayerParams* layers, const float* embed_w,
                         const float* after_norm_w, const float* after_norm_b, const float* out_w, const float* out_b,
                         void* prepared, size_t prepared_bytes, int precision, void*) {
  return prepare_decoder_entry(HostBackend{}, cfg, layers, embed_w, after_norm_w, after_norm_b, out_w, out_b, prepared,
                               prepared_bytes, precision);
}
size_t avsr_decoder_session_bytes(const AvsrDecoderConfig* cfg, int T, int max_steps, int max_hyps) {
  return decoder_session_bytes_entry(cfg, T, max_steps, max_hyps);
}
int avsr_decoder_begin(const AvsrDecoderConfig* cfg, const void* prepared, const float* memory, int T, int max_steps,
                       int max_hyps, void* session, size_t session_bytes, int precision, void*) {
  return decoder_begin_entry(HostBackend{}, cfg, prepared, memory, T, max_steps, max_hyps, session, session_bytes,
                             precision);
}
size_t avsr_decoder_step_workspace_bytes(const AvsrDecoderConfig* cfg, int T, int max_steps, int max_hyps) {
  return decoder_step_workspace_bytes_entry(cfg, T, max_steps, max_hyps);
}
int avsr_decoder_step(const AvsrDecoderConfig* cfg, const void* prepared, void* session, size_t session_bytes, int T,
                      int max_steps, int max_hyps, const int32_t* tokens, const int32_t* anc, int step, int n, float* logp,
                      void* workspace, size_t workspace_bytes, int precision, void*) {
  return decoder_step_entry(HostBackend{}, cfg, prepared, session, session_bytes, T, max_steps, max_hyps, tokens, anc,
                            step, n, logp, workspace, workspace_bytes, precision);
}
int avsr_ctc_prefix_init(const float* logp, int T, int O, int blank, float* r0, void*) {
  return ctc_prefix_init_entry(HostBackend{}, logp, T, O, blank, r0);
}
int avsr_ctc_prefix_score(const float* logp, int T, int O, int blank, int eos, int out_len, const int32_t* last_ids,
                          const float* r_prev, const float* s_prev, const int32_t* cand, int n, int S, float* local,
                          float* r, float* log_psi, void*) {
  return ctc_prefix_score_entry(HostBackend{}, logp, T, O, blank, eos, out_len, last_ids, r_prev, s_prev, cand, n, S,
                                local, r, log_psi);
}
int avsr_ctc_prefix_select(const float* r, const float* log_psi, const int32_t* cand, const int32_t* parent,
                           const int32_t* token, int T, int O, int n, int S, int m, float* r_next, float* s_next, void*) {
  return ctc_prefix_select_entry(HostBackend{}, r, log_psi, cand, parent, token, T, O, n, S, m, r_next, s_next);
}
}  // extern "C"
