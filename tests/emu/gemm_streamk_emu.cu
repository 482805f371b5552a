// Host build of the tensor-core GEMM's piece lists (csrc/gemm_schedule.cuh) for tests/test_gemm_streamk_cpu.py.
// TEST INFRASTRUCTURE ONLY.
#include "../../auto_avsr_b200/csrc/gemm_schedule.cuh"

extern "C" int tc_emu_max_splits() { return avsr::kMaxSplits; }

extern "C" int tc_emu_sk_ctas(int sms, int tiles, int nkb) { return avsr::tc_streamk_ctas(sms, tiles, nkb); }

// every piece of the stream-K list over `ctas` CTAs, in walk order per CTA: rows of
// {cta, j, tm, tn, kb0, kb1, piece, npieces}; returns the row count (at most `cap`)
extern "C" int tc_emu_sk_walk(int ctas, int tiles_m, int tiles_n, int nkb, int* out, int cap) {
  int n = 0;
  for (int c = 0; c < ctas; ++c) {
    const int np = avsr::tc_streamk_pieces(c, ctas, tiles_m * tiles_n, nkb);
    for (int j = 0; j < np && n < cap; ++j, ++n) {
      const avsr::TcPiece p = avsr::tc_streamk_piece(j, c, ctas, tiles_n, tiles_m * tiles_n, nkb);
      int* r = out + 8 * n;
      r[0] = c; r[1] = j; r[2] = p.tm; r[3] = p.tn; r[4] = p.kb0; r[5] = p.kb1; r[6] = p.piece; r[7] = p.npieces;
    }
  }
  return n;
}

// the same rows for the equal-slice split-K list of 1 x 1 clusters on `ctas` CTAs
extern "C" int tc_emu_slice_walk(int ctas, int tiles_m, int tiles_n, int nkb, int splits, int* out, int cap) {
  int n = 0;
  for (int c = 0; c < ctas; ++c) {
    const int np = avsr::tc_slice_pieces(c, ctas, tiles_m, tiles_n, splits, 1, 1);
    for (int j = 0; j < np && n < cap; ++j, ++n) {
      const avsr::TcPiece p = avsr::tc_slice_piece(j, c, ctas, 0, tiles_m, tiles_n, nkb, splits, 1, 1);
      int* r = out + 8 * n;
      r[0] = c; r[1] = j; r[2] = p.tm; r[3] = p.tn; r[4] = p.kb0; r[5] = p.kb1; r[6] = p.piece; r[7] = p.npieces;
    }
  }
  return n;
}
