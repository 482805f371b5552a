// Work list of the persistent tensor-core GEMM (gemm_tc.cu), shared with the host test that checks it (tests/emu).
//
// The output is cut into 128 x BN tiles, tiles_m x tiles_n of them.  CTAs run in clusters of CM x CN; a cluster owns
// a "cluster tile" of CM x CN neighbouring tiles (CTA rank r of the cluster -> cm = r % CM along M, cn = r / CM along
// N).  Clusters walk the cluster tiles c, c + clusters, ... (n fastest), each CTA taking its own tile of every
// cluster tile, so all CTAs of a cluster see the same number of items in the same order: every multicast load one
// CTA waits for is issued by its peers.  A tile past the matrix edge (M = 1600 has 13 m-tiles) is still walked: its
// CTA takes part in the shared loads and skips the stores.  Split-K (1 x 1 clusters only) repeats the tile list once
// per K-slice, slice-major.
#pragma once
#include "common.cuh"

namespace avsr {

struct TcWork {
  int tm, tn, split;   // tile coordinates (may lie past the edge: valid == false) and K-slice
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

}  // namespace avsr
