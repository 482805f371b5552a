// HOST replay of the batched decoder / CTC-prefix schedule (several utterances in one session) -- TEST INFRASTRUCTURE
// ONLY (tests/emu/build.py builds it into tests/emu/_build/libavsr_decoder_batch_emu.so).
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
  return decoder_batch_session_bytes_entry(cfg, U, lengths, max_steps, max_hyps);
}
size_t avsr_decoder_batch_step_workspace_bytes(const AvsrDecoderConfig* cfg, int T_max, int max_steps, int max_hyps) {
  return decoder_step_workspace_bytes_entry(cfg, T_max, max_steps, max_hyps);
}
int avsr_decoder_batch_begin(const AvsrDecoderConfig* cfg, const void* prepared, const float* memory,
                             const int32_t* lengths, int U, int T_max, int max_steps, int max_hyps, void* session,
                             size_t session_bytes, int precision, void*) {
  return decoder_batch_begin_entry(BatchHostBackend{}, cfg, prepared, memory, lengths, U, T_max, max_steps, max_hyps,
                                   session, session_bytes, precision);
}
int avsr_decoder_batch_step(const AvsrDecoderConfig* cfg, const void* prepared, void* session, size_t session_bytes,
                            const int32_t* lengths, int U, int T_max, int max_steps, int max_hyps, const int32_t* tokens,
                            const int32_t* anc, const int32_t* row_utt, int step, int n, float* logp, void* workspace,
                            size_t workspace_bytes, int precision, void*) {
  return decoder_batch_step_entry(BatchHostBackend{}, cfg, prepared, session, session_bytes, lengths, U, T_max,
                                  max_steps, max_hyps, tokens, anc, row_utt, step, n, logp, workspace, workspace_bytes,
                                  precision);
}
int avsr_ctc_prefix_batch_init(const float* logp, const int32_t* lengths, int U, int T_max, int O, int blank,
                               int32_t* lengths_dev, float* r0, void*) {
  return ctc_prefix_batch_init_entry(BatchHostBackend{}, logp, lengths, U, T_max, O, blank, lengths_dev, r0);
}
int avsr_ctc_prefix_batch_score(const float* logp, const int32_t* lengths, int U, int T_max, int O, int blank, int eos,
                                int out_len, const int32_t* last_ids, const float* r_prev, const float* s_prev,
                                const int32_t* cand, const int32_t* row_utt, int n, int S, float* local, float* r,
                                float* log_psi, void*) {
  return ctc_prefix_batch_score_entry(BatchHostBackend{}, logp, lengths, U, T_max, O, blank, eos, out_len, last_ids,
                                      r_prev, s_prev, cand, row_utt, n, S, local, r, log_psi);
}
}  // extern "C"
