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

// ---- grouped source attention of a batched step: one CTA per (utterance, head) ------------------------------------
// ScoresBatchElem / PvBatchElem launch a thread per (row, head, frame) and per output element, and each thread gathers
// its own 256-byte key / value slice: every row re-reads its utterance's K/V.  Here a CTA stages the utterance's K head
// slice, then its V head slice, through shared memory in 64-frame tiles, ascending, and serves every query row of the
// utterance (64 at a time) from each staged tile, so K/V are read once per (utterance, head, 64 rows).
// Each output is computed with the functors' per-output operations in their order -- an fmaf chain over e ascending and
// a division by sqrt_dk per score; the row max (exact, so any order); p = expf(s - m) once per (row, key); l and the
// P.V sum accumulated over s ascending with += and fmaf -- so the context has the functors' bits.  Keys are never split
// across CTAs: that would change the summation order.  Scores go through the `scores` workspace between the passes.
constexpr int kGaRows = 64, kGaTile = 64, kGaLd = 65, kGaThreads = 256;
constexpr size_t kGaFixedSmem = (3 * kGaRows * kGaLd + kGaRows + 8) * sizeof(float);

__global__ void __launch_bounds__(kGaThreads) grouped_src_attention_kernel(
    const float* __restrict__ q, const float* __restrict__ kv, const int32_t* __restrict__ row_utt,
    const int32_t* __restrict__ utt_off, const int32_t* __restrict__ utt_len, int U, long sum_T, int n, int H, int dk,
    int D, int T_max, float sqrt_dk, float* __restrict__ scores, int kind, void* __restrict__ ctx) {
  extern __shared__ float sm[];
  float* q_s = sm;                                  // (64 rows, dk) of this chunk, row stride 65
  float* t_s = q_s + kGaRows * kGaLd;               // (64 frames, dk): the K tile, then the V tile
  float* p_s = t_s + kGaTile * kGaLd;               // (64 rows, 64 frames): expf(s - m) of the V tile
  float* m_s = p_s + kGaRows * kGaLd;               // (64) row max
  int* warp_cnt = reinterpret_cast<int*>(m_s + kGaRows);
  int* rows_s = warp_cnt + 8;                       // (n) rows of this utterance, ascending
  const int u = blockIdx.x / H, h = blockIdx.x - u * H;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tr = tid >> 4, tc = tid & 15;           // rows tr*4 .. +3; frames / columns tc + 16 j
  // The host lays the session out from the lengths it passes at every step; they must be the ones begin stored.  If
  // they are not (other total, or an utterance longer than T_max), the rows get a NaN context (0 / 0) instead of
  // another utterance's K/V.
  const bool stale = (long)utt_off[U - 1] + utt_len[U - 1] != sum_T || utt_len[u] > T_max;
  const int T = stale ? 0 : utt_len[u];
  const long f0 = utt_off[u];
  const long ld = 2L * D;

  int R = 0;
  for (int base = 0; base < n; base += kGaThreads) {
    const int i = base + tid;
    const bool mine = i < n && row_utt[i] == u;
    const unsigned ballot = __ballot_sync(0xffffffffu, mine);
    if (lane == 0) warp_cnt[warp] = __popc(ballot);
    __syncthreads();
    int before = R, total = 0;
    for (int w = 0; w < kGaThreads / 32; ++w) {
      before += w < warp ? warp_cnt[w] : 0;
      total += warp_cnt[w];
    }
    if (mine) rows_s[before + __popc(ballot & ((1u << lane) - 1u))] = i;
    __syncthreads();
    R += total;
  }

  for (int r0 = 0; r0 < R; r0 += kGaRows) {
    const int nr = min(kGaRows, R - r0);
    for (int idx = tid; idx < kGaRows * dk; idx += kGaThreads) {
      const int r = idx / dk, e = idx - r * dk;
      q_s[r * kGaLd + e] = r < nr ? q[(long)rows_s[r0 + r] * D + h * dk + e] : 0.f;
    }
    // pass 1: scores, running row max
    float mx[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    for (int t0 = 0; t0 < T; t0 += kGaTile) {
      const int nt = min(kGaTile, T - t0);
      __syncthreads();
      for (int idx = tid; idx < kGaTile * dk; idx += kGaThreads) {
        const int s = idx / dk, e = idx - s * dk;
        t_s[s * kGaLd + e] = s < nt ? kv[(f0 + t0 + s) * ld + h * dk + e] : 0.f;
      }
      __syncthreads();
      float acc[4][4] = {};
      for (int e = 0; e < dk; ++e) {
        float qv[4], kk[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) qv[a] = q_s[(tr * 4 + a) * kGaLd + e];
#pragma unroll
        for (int b = 0; b < 4; ++b) kk[b] = t_s[(tc + 16 * b) * kGaLd + e];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) acc[a][b] = fmaf(qv[a], kk[b], acc[a][b]);
      }
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const int r = tr * 4 + a;
        if (r >= nr) continue;
        float* out = scores + ((long)rows_s[r0 + r] * H + h) * T_max + t0;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const int s = tc + 16 * b;
          if (s < nt) {
            const float v = acc[a][b] / sqrt_dk;
            out[s] = v;
            mx[a] = fmaxf(mx[a], v);
          }
        }
      }
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      for (int o = 8; o > 0; o >>= 1) mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
      if (tc == 0) m_s[tr * 4 + a] = mx[a];
    }
    // pass 2: p = expf(s - m) once per (row, key); l and P.V over s ascending
    float o[4][4] = {}, l[4] = {};
    for (int t0 = 0; t0 < T; t0 += kGaTile) {
      const int nt = min(kGaTile, T - t0);
      __syncthreads();
      for (int idx = tid; idx < kGaTile * dk; idx += kGaThreads) {
        const int s = idx / dk, c = idx - s * dk;
        t_s[s * kGaLd + c] = s < nt ? kv[(f0 + t0 + s) * ld + D + h * dk + c] : 0.f;
      }
      for (int idx = tid; idx < kGaRows * kGaTile; idx += kGaThreads) {
        const int r = idx / kGaTile, s = idx - r * kGaTile;
        p_s[r * kGaLd + s] =
            (r < nr && s < nt) ? expf(scores[((long)rows_s[r0 + r] * H + h) * T_max + t0 + s] - m_s[r]) : 0.f;
      }
      __syncthreads();
      for (int s = 0; s < nt; ++s) {
        float pv[4], vv[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) pv[a] = p_s[(tr * 4 + a) * kGaLd + s];
#pragma unroll
        for (int b = 0; b < 4; ++b) vv[b] = t_s[s * kGaLd + tc + 16 * b];
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          l[a] += pv[a];
#pragma unroll
          for (int b = 0; b < 4; ++b) o[a][b] = fmaf(pv[a], vv[b], o[a][b]);
        }
      }
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int r = tr * 4 + a;
      if (r >= nr) continue;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int c = tc + 16 * b;
        if (c < dk) store_operand(ctx, (long)rows_s[r0 + r] * D + h * dk + c, kind, o[a][b] / l[a]);
      }
    }
    __syncthreads();
  }
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
    return gemm_tc(EPI_LINEAR, operand_kind(prec), A, W, M, N, K, e, st);
  }
  int layernorm(const float* x, const float* g, const float* b, void* y, int rows, int d, int out_kind) {
    return launch_layernorm(x, g, b, y, rows, d, out_kind, st);
  }
  int log_softmax(const float* x, long ldx, float* y, long ldy, int rows, int n) {
    return launch_log_softmax_rows(x, ldx, y, ldy, nullptr, rows, n, st);
  }
  // a small HOST array into device memory (pageable source: staged before the call returns)
  int upload_i32(int32_t* dst, const int32_t* src, int count) {
    AVSR_CUDA_TRY(cudaMemcpyAsync(dst, src, (size_t)count * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    return AVSR_OK;
  }
  int src_attention_batch(const float* q, const float* kv, const int32_t* row_utt, const int32_t* utt_off,
                          const int32_t* utt_len, int U, long sum_T, int n, int H, int dk, int T_max, float sqrt_dk,
                          float* scores, int kind, void* ctx) {
    AVSR_REQUIRE(dk <= kGaTile, "decoder batch step: head size %d > %d", dk, kGaTile);
    const size_t smem = kGaFixedSmem + (size_t)n * sizeof(int32_t);
    AVSR_REQUIRE(smem <= 227 * 1024, "decoder batch step: %d hypotheses exceed the grouped attention's row list", n);
    // raise the kernel's dynamic shared-memory limit only when a launch needs more than the device was given so far
    constexpr int kMaxDevices = 64;
    static std::atomic<size_t> smem_set[kMaxDevices];
    int devc = 0;
    AVSR_CUDA_TRY(cudaGetDevice(&devc));
    if (devc >= kMaxDevices || smem > smem_set[devc].load()) {
      AVSR_CUDA_TRY(cudaFuncSetAttribute(grouped_src_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
      if (devc < kMaxDevices) smem_set[devc].store(smem);
    }
    grouped_src_attention_kernel<<<(unsigned)(U * H), kGaThreads, smem, st>>>(q, kv, row_utt, utt_off, utt_len, U, sum_T,
                                                                              n, H, dk, H * dk, T_max, sqrt_dk, scores,
                                                                              kind, ctx);
    AVSR_CHECK_LAUNCH();
    return AVSR_OK;
  }
};

}  // namespace dec
}  // namespace avsr

using namespace avsr;
using namespace avsr::dec;

static DeviceBackend device(void* stream) { return DeviceBackend{reinterpret_cast<cudaStream_t>(stream)}; }

extern "C" {

size_t avsr_decoder_prepared_bytes(const AvsrDecoderConfig* cfg) { return decoder_prepared_bytes_entry(cfg); }

int avsr_prepare_decoder(const AvsrDecoderConfig* cfg, const AvsrDecoderLayerParams* layers, const float* embed_w,
                         const float* after_norm_w, const float* after_norm_b, const float* out_w, const float* out_b,
                         void* prepared, size_t prepared_bytes, int precision, void* stream) {
  return prepare_decoder_entry(device(stream), cfg, layers, embed_w, after_norm_w, after_norm_b, out_w, out_b, prepared,
                               prepared_bytes, precision);
}

size_t avsr_decoder_session_bytes(const AvsrDecoderConfig* cfg, int T, int max_steps, int max_hyps) {
  return decoder_session_bytes_entry(cfg, T, max_steps, max_hyps);
}

int avsr_decoder_begin(const AvsrDecoderConfig* cfg, const void* prepared, const float* memory, int T, int max_steps,
                       int max_hyps, void* session, size_t session_bytes, int precision, void* stream) {
  return decoder_begin_entry(device(stream), cfg, prepared, memory, T, max_steps, max_hyps, session, session_bytes,
                             precision);
}

size_t avsr_decoder_step_workspace_bytes(const AvsrDecoderConfig* cfg, int T, int max_steps, int max_hyps) {
  return decoder_step_workspace_bytes_entry(cfg, T, max_steps, max_hyps);
}

int avsr_decoder_step(const AvsrDecoderConfig* cfg, const void* prepared, void* session, size_t session_bytes, int T,
                      int max_steps, int max_hyps, const int32_t* tokens, const int32_t* anc, int step, int n, float* logp,
                      void* workspace, size_t workspace_bytes, int precision, void* stream) {
  return decoder_step_entry(device(stream), cfg, prepared, session, session_bytes, T, max_steps, max_hyps, tokens, anc,
                            step, n, logp, workspace, workspace_bytes, precision);
}

int avsr_ctc_prefix_init(const float* logp, int T, int O, int blank, float* r0, void* stream) {
  return ctc_prefix_init_entry(device(stream), logp, T, O, blank, r0);
}

int avsr_ctc_prefix_score(const float* logp, int T, int O, int blank, int eos, int out_len, const int32_t* last_ids,
                          const float* r_prev, const float* s_prev, const int32_t* cand, int n, int S, float* local,
                          float* r, float* log_psi, void* stream) {
  return ctc_prefix_score_entry(device(stream), logp, T, O, blank, eos, out_len, last_ids, r_prev, s_prev, cand, n, S,
                                local, r, log_psi);
}

size_t avsr_decoder_batch_session_bytes(const AvsrDecoderConfig* cfg, int U, const int32_t* lengths, int max_steps,
                                        int max_hyps) {
  return decoder_batch_session_bytes_entry(cfg, U, lengths, max_steps, max_hyps);
}

size_t avsr_decoder_batch_step_workspace_bytes(const AvsrDecoderConfig* cfg, int T_max, int max_steps, int max_hyps) {
  return decoder_step_workspace_bytes_entry(cfg, T_max, max_steps, max_hyps);
}

int avsr_decoder_batch_begin(const AvsrDecoderConfig* cfg, const void* prepared, const float* memory,
                             const int32_t* lengths, int U, int T_max, int max_steps, int max_hyps, void* session,
                             size_t session_bytes, int precision, void* stream) {
  return decoder_batch_begin_entry(device(stream), cfg, prepared, memory, lengths, U, T_max, max_steps, max_hyps, session,
                                   session_bytes, precision);
}

int avsr_decoder_batch_step(const AvsrDecoderConfig* cfg, const void* prepared, void* session, size_t session_bytes,
                            const int32_t* lengths, int U, int T_max, int max_steps, int max_hyps, const int32_t* tokens,
                            const int32_t* anc, const int32_t* row_utt, int step, int n, float* logp, void* workspace,
                            size_t workspace_bytes, int precision, void* stream) {
  return decoder_batch_step_entry(device(stream), cfg, prepared, session, session_bytes, lengths, U, T_max, max_steps,
                                  max_hyps, tokens, anc, row_utt, step, n, logp, workspace, workspace_bytes, precision);
}

int avsr_ctc_prefix_batch_init(const float* logp, const int32_t* lengths, int U, int T_max, int O, int blank,
                               int32_t* lengths_dev, float* r0, void* stream) {
  return ctc_prefix_batch_init_entry(device(stream), logp, lengths, U, T_max, O, blank, lengths_dev, r0);
}

int avsr_ctc_prefix_batch_score(const float* logp, const int32_t* lengths, int U, int T_max, int O, int blank, int eos,
                                int out_len, const int32_t* last_ids, const float* r_prev, const float* s_prev,
                                const int32_t* cand, const int32_t* row_utt, int n, int S, float* local, float* r,
                                float* log_psi, void* stream) {
  return ctc_prefix_batch_score_entry(device(stream), logp, lengths, U, T_max, O, blank, eos, out_len, last_ids, r_prev,
                                      s_prev, cand, row_utt, n, S, local, r, log_psi);
}

int avsr_ctc_prefix_select(const float* r, const float* log_psi, const int32_t* cand, const int32_t* parent,
                           const int32_t* token, int T, int O, int n, int S, int m, float* r_next, float* s_next,
                           void* stream) {
  return ctc_prefix_select_entry(device(stream), r, log_psi, cand, parent, token, T, O, n, S, m, r_next, s_next);
}

}  // extern "C"
