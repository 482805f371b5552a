// HOST replay of the batched decoder / CTC-prefix schedule (several utterances in one session) -- TEST INFRASTRUCTURE
// ONLY (tests/emu/build_decoder_batch.py builds it into tests/emu/_build/libavsr_decoder_batch_emu.so).
//
// It is the one-utterance replay of decoder_emu.cu plus the batched entries, so one library serves both sides of the
// "a batched row equals the same hypothesis decoded alone" checks.  The source attention of a batched step, which the
// device runs as the grouped kernel of csrc/decoder.cu, is replayed here with the batched functors of decoder_body.cuh
// (ScoresBatchElem / PvBatchElem); the GPU tests hold the kernel to those functors' bits.  HOST pointers, fp32 only.
#include <string.h>

#include "decoder_emu.cu"

namespace avsr {
namespace dec {
struct BatchHostBackend : HostBackend {
  int upload_i32(int32_t* dst, const int32_t* src, int count) {
    memcpy(dst, src, (size_t)count * sizeof(int32_t));
    return AVSR_OK;
  }
  int src_attention_batch(const float* q, const float* kv, const int32_t* row_utt, const int32_t* utt_off,
                          const int32_t* utt_len, int U, long sum_T, int n, int H, int dk, int T_max, float sqrt_dk,
                          float* scores, int kind, void* ctx) {
    // the device kernel answers stale lengths with a NaN context; the replay can read the session, so it refuses them
    AVSR_REQUIRE((long)utt_off[U - 1] + utt_len[U - 1] == sum_T, "emu: step lengths differ from the session's");
    const int D = H * dk;
    AVSR_TRY(for_each((long)n * H * T_max, ScoresBatchElem{q, kv, row_utt, utt_off, utt_len, H, dk, D, T_max, sqrt_dk,
                                                           scores}));
    return for_each((long)n * D, PvBatchElem{scores, kv, row_utt, utt_off, utt_len, H, dk, D, T_max, kind, ctx});
  }
};

}  // namespace dec
}  // namespace avsr

extern "C" {
size_t avsr_decoder_batch_session_bytes(const AvsrDecoderConfig* cfg, int U, const int32_t* lengths, int max_steps,
                                        int max_hyps) {
  long sum_T;
  int max_len;
  if (check_batch_lengths(lengths, U, 0, &sum_T, &max_len) != AVSR_OK || max_steps <= 0 || max_hyps <= 0) return 0;
  return layout_dec_batch_session(*cfg, U, sum_T, max_len, max_steps, max_hyps, nullptr).bytes;
}
size_t avsr_decoder_batch_step_workspace_bytes(const AvsrDecoderConfig* cfg, int T_max, int max_steps, int max_hyps) {
  return layout_dec_work(*cfg, T_max, max_steps, max_hyps, nullptr).bytes;
}
int avsr_decoder_batch_begin(const AvsrDecoderConfig* cfg, const void* prepared, const float* memory,
                             const int32_t* lengths, int U, int T_max, int max_steps, int max_hyps, void* session,
                             size_t session_bytes, int precision, void*) {
  AVSR_REQUIRE(T_max > 0 && max_steps > 0 && max_hyps > 0, "emu: bad T_max / max_steps / max_hyps");
  long sum_T;
  int max_len;
  AVSR_TRY(check_batch_lengths(lengths, U, T_max, &sum_T, &max_len));
  const DecBatchSession S = layout_dec_batch_session(*cfg, U, sum_T, max_len, max_steps, max_hyps, session);
  if (S.bytes > session_bytes) return AVSR_E_WORKSPACE;
  const DecPrep P = layout_dec_prepared(*cfg, const_cast<void*>(prepared));
  BatchHostBackend bk;
  return begin_batch_body(bk, *cfg, P, S, memory, lengths, U, T_max, sum_T, precision);
}
int avsr_decoder_batch_step(const AvsrDecoderConfig* cfg, const void* prepared, void* session, size_t session_bytes,
                            const int32_t* lengths, int U, int T_max, int max_steps, int max_hyps, const int32_t* tokens,
                            const int32_t* anc, const int32_t* row_utt, int step, int n, float* logp, void* workspace,
                            size_t workspace_bytes, int precision, void*) {
  AVSR_REQUIRE(T_max > 0 && max_steps > 0 && max_hyps > 0, "emu: bad T_max / max_steps / max_hyps");
  AVSR_REQUIRE(step >= 0 && step < max_steps, "decoder_batch_step: step %d outside %d positions", step, max_steps);
  AVSR_REQUIRE(n >= 0 && n <= max_hyps, "decoder_batch_step: n=%d hypotheses exceed %d beam slots", n, max_hyps);
  AVSR_REQUIRE((step == 0 || anc) && row_utt, "emu: NULL anc / row_utt");
  long sum_T;
  int max_len;
  AVSR_TRY(check_batch_lengths(lengths, U, T_max, &sum_T, &max_len));
  if (n == 0) return AVSR_OK;
  const DecBatchSession S = layout_dec_batch_session(*cfg, U, sum_T, max_len, max_steps, max_hyps, session);
  const DecWork W = layout_dec_work(*cfg, T_max, max_steps, max_hyps, workspace);
  if (S.bytes > session_bytes || W.bytes > workspace_bytes) return AVSR_E_WORKSPACE;
  const DecPrep P = layout_dec_prepared(*cfg, const_cast<void*>(prepared));
  BatchHostBackend bk;
  return step_batch_body(bk, *cfg, P, S, W, tokens, anc, row_utt, step, n, U, T_max, sum_T, max_steps, max_hyps, logp,
                         precision);
}
int avsr_ctc_prefix_batch_init(const float* logp, const int32_t* lengths, int U, int T_max, int O, int blank,
                               int32_t* lengths_dev, float* r0, void*) {
  AVSR_REQUIRE(T_max > 0, "emu: bad T_max");
  long sum_T;
  int max_len;
  AVSR_TRY(check_batch_lengths(lengths, U, T_max, &sum_T, &max_len));
  BatchHostBackend bk;
  AVSR_TRY(bk.upload_i32(lengths_dev, lengths, U));
  return bk.for_each(U, CtcInitBatchElem{logp, lengths_dev, r0, U, T_max, O, blank});
}
int avsr_ctc_prefix_batch_score(const float* logp, const int32_t* lengths, int U, int T_max, int O, int blank, int eos,
                                int out_len, const int32_t* last_ids, const float* r_prev, const float* s_prev,
                                const int32_t* cand, const int32_t* row_utt, int n, int S, float* local, float* r,
                                float* log_psi, void*) {
  AVSR_REQUIRE(U >= 1 && T_max > 0, "emu: bad U / T_max");
  if (n == 0) return AVSR_OK;
  BatchHostBackend bk;
  return ctc_prefix_batch_body(bk, logp, lengths, T_max, O, blank, eos, out_len, last_ids, r_prev, s_prev, cand, row_utt,
                               n, S, local, r, log_psi);
}
}  // extern "C"
