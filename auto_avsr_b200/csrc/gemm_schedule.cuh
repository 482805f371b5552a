// Work list of the persistent tensor-core GEMM (gemm_tc.cu), shared with the host test that checks it (tests/emu).
//
// The output is cut into 128 x BN tiles, tiles_m x tiles_n of them.  CTAs run in clusters of CM x CN; a cluster owns
// a "cluster tile" of CM x CN neighbouring tiles (CTA rank r of the cluster -> cm = r % CM along M, cn = r / CM along
// N).  Clusters walk the cluster tiles c, c + clusters, ... (n fastest), each CTA taking its own tile of every
// cluster tile, so all CTAs of a cluster see the same number of items in the same order: every multicast load one
// CTA waits for is issued by its peers.  A tile past the matrix edge (M = 1600 has 13 m-tiles) is still walked: its
// CTA takes part in the shared loads and skips the stores.  Split-K (1 x 1 clusters only) repeats the tile list once
// per K-slice, slice-major.
//
// The kernel walks a CTA's work as pieces (TcPiece): k-blocks [kb0, kb1) of one tile.  Two lists produce them:
//   - the cluster / equal-slice list above: item j of a cluster is a piece, its K-slice is its piece rank;
//   - stream-K (1 x 1 clusters only): the tiles * nkb (tile, k-block) steps, tile-major with n fastest, are cut into
//     `ctas` contiguous shares [c * U / ctas, (c + 1) * U / ctas), and CTA c's share is split at tile boundaries.
//     Every CTA gets within one k-block of the same number of steps, whatever the tile count.
// A tile shared by npieces > 1 CTAs is finished by the last of them to arrive (a counter per tile), which sums the
// fp32 partials in piece order: the result depends on the list (M, N, K, CTA count), never on arrival order.
#pragma once
#include "common.cuh"

namespace avsr {

struct TcWork {
  int tm, tn, split;   // tile coordinates (may lie past the edge: valid == false) and K-slice
  bool valid;
};

struct TcPiece {
  int tm, tn;          // tile (may lie past the edge in a cluster list: valid == false)
  int kb0, kb1;        // k-blocks of the tile this piece computes
  int piece, npieces;  // rank of the piece in k order among the tile's pieces (selects the partial plane), and count
  bool valid;
};

AVSR_HD int tc_cluster_items(int tiles_m, int tiles_n, int splits, int CM, int CN) {
  return ((tiles_m + CM - 1) / CM) * ((tiles_n + CN - 1) / CN) * splits;
}

AVSR_HD TcWork tc_work_item(int item, int crank, int tiles_m, int tiles_n, int CM, int CN) {
  const int ctn = (tiles_n + CN - 1) / CN;
  const int ctiles = ((tiles_m + CM - 1) / CM) * ctn;
  const int ct = item % ctiles;
  TcWork w;
  w.split = item / ctiles;
  w.tm = (ct / ctn) * CM + crank % CM;
  w.tn = (ct % ctn) * CN + crank / CM;
  w.valid = w.tm < tiles_m && w.tn < tiles_n;
  return w;
}

// ---- cluster / equal-slice list: cluster `cluster` of `clusters` takes items cluster, cluster + clusters, ...
AVSR_HD int tc_slice_pieces(int cluster, int clusters, int tiles_m, int tiles_n, int splits, int CM, int CN) {
  const int total = tc_cluster_items(tiles_m, tiles_n, splits, CM, CN);
  return cluster < total ? (total - cluster + clusters - 1) / clusters : 0;
}

AVSR_HD TcPiece tc_slice_piece(int j, int cluster, int clusters, int crank, int tiles_m, int tiles_n, int nkb,
                               int splits, int CM, int CN) {
  const TcWork w = tc_work_item(cluster + j * clusters, crank, tiles_m, tiles_n, CM, CN);
  return TcPiece{w.tm, w.tn, w.split * nkb / splits, (w.split + 1) * nkb / splits, w.split, splits, w.valid};
}

// ---- stream-K list over `ctas` CTAs
AVSR_HD long long tc_sk_begin(int cta, int ctas, long long steps) { return steps * cta / ctas; }

// the CTA whose share holds global step g
AVSR_HD int tc_sk_owner(long long g, int ctas, long long steps) { return (int)(((g + 1) * ctas - 1) / steps); }

AVSR_HD int tc_streamk_pieces(int cta, int ctas, int tiles, int nkb) {
  const long long U = (long long)tiles * nkb, b = tc_sk_begin(cta, ctas, U), e = tc_sk_begin(cta + 1, ctas, U);
  return e > b ? (int)((e - 1) / nkb - b / nkb + 1) : 0;
}

AVSR_HD TcPiece tc_streamk_piece(int j, int cta, int ctas, int tiles_n, int tiles, int nkb) {
  const long long U = (long long)tiles * nkb, b = tc_sk_begin(cta, ctas, U), e = tc_sk_begin(cta + 1, ctas, U);
  const long long t = b / nkb + j, t0 = t * nkb, t1 = t0 + nkb;
  const int first = tc_sk_owner(t0, ctas, U);
  TcPiece p;
  p.tm = (int)(t / tiles_n);
  p.tn = (int)(t % tiles_n);
  p.kb0 = (int)((b > t0 ? b : t0) - t0);
  p.kb1 = (int)((e < t1 ? e : t1) - t0);
  p.piece = cta - first;
  p.npieces = tc_sk_owner(t1 - 1, ctas, U) - first + 1;
  p.valid = true;
  return p;
}

// Stream-K CTA count for `sms` SMs.  The piece selects one of kMaxSplits partial planes, so no tile may be split into
// more pieces: a tile touched by n CTAs holds n - 2 whole shares of at least floor(U / ctas) steps plus a step of
// each end CTA, so shares of at least (nkb - 2) / (kMaxSplits - 1) + 1 steps keep n <= kMaxSplits.  Small GEMMs get
// fewer CTAs rather than more pieces.
AVSR_HD int tc_streamk_ctas(int sms, int tiles, int nkb) {
  const long long U = (long long)tiles * nkb;
  const long long share = nkb > 2 ? (nkb - 2) / (kMaxSplits - 1) + 1 : 1;
  const long long ctas = U / share;
  return (int)(ctas < sms ? (ctas > 0 ? ctas : 1) : sms);
}

}  // namespace avsr
