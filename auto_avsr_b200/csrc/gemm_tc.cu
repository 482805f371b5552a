// Tensor-core GEMM for the Conformer layer's projections (FFN x2, QK, V^T, out, pw1+GLU, pw2) and the stacked
// linear_pos:   acc[m][n] = sum_k A[m][k] * Bw[n][k]   (both K-major = torch.nn.Linear layout).
//
// Hopper pipeline (sm_90a).  One persistent CTA owns a 128 x BN output tile at a time:
//   warp 0        : TMA producer -- cp.async.bulk.tensor 2-D boxes (rows x 128 bytes, SWIZZLE_128B) of A and Bw into
//                   a STAGES-deep shared-memory ring, completion on `full` mbarriers
//   warpgroups 1-2: ping-pong consumers.  Warpgroup 1 owns the CTA's even work items, warpgroup 2 the odd ones; each
//                   runs the whole 128 x BN tile: wgmma.mma_async (two M = 64 chains, rows 0-63 and 64-127, N = BN,
//                   K = 32 bytes) x4 per stage straight from shared memory into register accumulators; a stage goes
//                   back to the producer (`empty` mbarrier) once the wgmma group that read it has retired.  Then the
//                   same 4 warps run the fused epilogue: accumulators -> fp32 tile in shared memory -> lane-per-row
//                   reads, bias / ReLU / residual / GLU / head-major scatter / conversion to the next operand's
//                   storage, coalesced global stores (epilogue.cuh).  Two ordering mbarriers alternate the
//                   warpgroups, one for main loops and one for epilogues, so one warpgroup's epilogue runs while the
//                   other's main loop issues wgmma, and only one epilogue at a time uses the shared fp32 tile
// Operand storage (template TOp): float = TF32 (8 elements per MMA-K), __half or __nv_bfloat16 (16 per MMA-K; half the
// bytes, twice the rate).  Out-of-bounds rows of edge tiles are zero-filled by TMA and masked in the
// epilogue.  The tile width is chosen per problem by a small cost model (bytes through L2 vs tensor-pipe time).
#include <cstring>

#include "common.cuh"
#include "epilogue.cuh"
#include "gemm_schedule.cuh"
#include "sm90.cuh"

namespace avsr {

using namespace sm90;

// ---------------------------------------------------------------- host: tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

static CUtensorMapDataType tmap_dtype(int kind) {
  return kind == OP_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                        : (kind == OP_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32);
}

int make_tmap_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                 int kind) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)"); return AVSR_E_CUDA; }
  const int esz = (int)operand_bytes(kind);
  AVSR_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0 && (ld * esz) % 16 == 0 && box_rows <= 256,
               "tensor map: base/stride must be 16-byte aligned (ld=%llu, esz=%d)", (unsigned long long)ld, esz);
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstr[1] = {ld * (uint64_t)esz};
  cuuint32_t box[2] = {(cuuint32_t)(128 / esz), box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, tmap_dtype(kind), 2,
                   const_cast<void*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(2d) failed: CUresult %d", (int)r); return AVSR_E_CUDA; }
  return AVSR_OK;
}

int make_tmap_3d(CUtensorMap* map, const void* base, uint64_t planes, uint64_t rows, uint64_t cols, uint64_t ld_row,
                 uint64_t ld_plane, uint32_t box_rows, int kind) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)"); return AVSR_E_CUDA; }
  const int esz = (int)operand_bytes(kind);
  AVSR_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0 && (ld_row * esz) % 16 == 0 &&
                   (ld_plane * esz) % 16 == 0 && box_rows <= 256,
               "tensor map 3d: base/strides must be 16-byte aligned");
  cuuint64_t gdim[3] = {cols, rows, planes};
  cuuint64_t gstr[2] = {ld_row * (uint64_t)esz, ld_plane * (uint64_t)esz};
  cuuint32_t box[3] = {(cuuint32_t)(128 / esz), box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, tmap_dtype(kind), 3,
                   const_cast<void*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(3d) failed: CUresult %d", (int)r); return AVSR_E_CUDA; }
  return AVSR_OK;
}

// ---------------------------------------------------------------- the kernel
constexpr int TC_BM = 128;          // rows per CTA tile / per A box (two wgmma chains of 64 rows)
constexpr int TC_THREADS = 384;     // warpgroup 0: TMA producer (warp 0); warpgroups 1-2: wgmma + epilogue
constexpr int TC_SMEM_BUDGET = 227 * 1024;   // one persistent CTA per SM

template <int BN>
struct TcCfg {
  static constexpr int kABytes = TC_BM * 128;
  static constexpr int kBBytes = BN * 128;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kAccLd = BN + 4;                 // fp32 accumulator tile row stride (conflict-free float4 rows)
  static constexpr int kAccBytes = TC_BM * kAccLd * 4;
  static constexpr int kVecBytes = 3 * BN * 4;          // bias / pos_bias_u / pos_bias_v of the tile's columns
  static constexpr int kFixedBytes = 1024 /*align slack*/ + 256 /*barriers*/ + kAccBytes + kVecBytes;
  static constexpr int kStagesFit = (TC_SMEM_BUDGET - kFixedBytes) / kStageBytes;
  static constexpr int kStages = kStagesFit > 8 ? 8 : kStagesFit;
  static constexpr int kSmem = kStages * kStageBytes + kFixedBytes;
  static_assert(kStages >= 2, "tile too large for shared memory");
};

template <typename TOp> struct OpTraits;
template <> struct OpTraits<float> {
  static constexpr int kElemsPerBlock = 32;  // 128 bytes of fp32
  template <int BN>
  __device__ static void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    if constexpr (BN == 64) wgmma_tf32_n64(d, a, b, acc); else wgmma_tf32_n128(d, a, b, acc);
  }
};
template <> struct OpTraits<__half> {
  static constexpr int kElemsPerBlock = 64;  // 128 bytes of fp16
  template <int BN>
  __device__ static void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    if constexpr (BN == 64) wgmma_f16_n64(d, a, b, acc); else wgmma_f16_n128(d, a, b, acc);
  }
};
template <> struct OpTraits<__nv_bfloat16> {
  static constexpr int kElemsPerBlock = 64;  // 128 bytes of bf16
  template <int BN>
  __device__ static void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    if constexpr (BN == 64) wgmma_bf16_n64(d, a, b, acc); else wgmma_bf16_n128(d, a, b, acc);
  }
};

template <int MODE, int BN, typename TOp, int CM, int CN>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int K, int tiles_m,
               int tiles_n, int splits, int streamk, EpiParams ep) {
  // PERSISTENT: cluster c processes cluster tiles c, c + clusters, ... (n fastest, so concurrently running CTAs share
  // A rows in L2; gemm_schedule.cuh).  The TMA ring never drains between tiles: the producer fills it in item order,
  // and the consumer warpgroups take turns on the items (even / odd), so stage ownership follows the item index.
  // The main-loop order barrier also keeps a warpgroup from waiting on a `full` phase that is two phases ahead.
  // Clusters of CM x CN CTAs (tensor maps with boxes of BN / CM rows of Bw and 128 / CN rows of A): the CM CTAs of a
  // cluster column share their Bw tile and each loads 1/CM of it, multicast to all of them; likewise the CN CTAs of a
  // cluster row share A.  Every warp of the consumer warpgroup that owns a stage's item releases the stage to the
  // producer of every CTA of the cluster (peers walk the same items, so their warpgroups of the same parity own it),
  // so a stage is refilled (by any peer) only after all CTAs it lands in are done with it.
  using Cfg = TcCfg<BN>;
  using Op = OpTraits<TOp>;
  constexpr int CS = CM * CN;
  static_assert(CS == 1 || (CM <= 2 && CN <= 2), "cluster shapes: 1x1, 2x1, 1x2, 2x2");
  constexpr int S = Cfg::kStages;
  constexpr int KE = Op::kElemsPerBlock;
  constexpr int LD = Cfg::kAccLd;
  extern __shared__ uint8_t tc_smem_raw[];
  const uint32_t raw = smem_u32(tc_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;       // SWIZZLE_128B tiles need 1024-byte alignment
  uint8_t* gen = tc_smem_raw + (base - raw);
  const uint32_t bars = base + S * Cfg::kStageBytes;  // full[S], empty[S], order[2][2]
  int* s_flag = reinterpret_cast<int*>(gen + S * Cfg::kStageBytes + (2 * S + 4) * 8);   // split-K: "arrived last"
  float* s_acc = reinterpret_cast<float*>(gen + S * Cfg::kStageBytes + 256);      // [TC_BM][LD]
  float* s_vec = s_acc + TC_BM * LD;                                               // [3][BN]
  auto full_bar = [&](int s) { return bars + 8u * s; };
  auto empty_bar = [&](int s) { return bars + 8u * (S + s); };
  // consumer warpgroup g waits on order_bar(phase, g) for its turn at the main loop (phase 0) or at the epilogue
  // (phase 1); the other warpgroup's 4 warps arrive on it when they finish theirs
  auto order_bar = [&](int phase, int g) { return bars + 8u * (2 * S + 2 * phase + g); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nkb = K / KE;
  // this CTA's pieces (gemm_schedule.cuh): the cluster / equal-slice list, or with `streamk` (LINEAR into the residual
  // stream only, 1 x 1 clusters) an equal share of the (tile, k-block) steps of all gridDim.x CTAs
  const bool sk = CS == 1 && streamk != 0;
  const int crank = CS > 1 ? (int)cluster_ctarank() : 0;
  const int cluster_id = blockIdx.x / CS, clusters = gridDim.x / CS;
  const int npieces = sk ? tc_streamk_pieces(blockIdx.x, gridDim.x, tiles_m * tiles_n, nkb)
                         : tc_slice_pieces(cluster_id, clusters, tiles_m, tiles_n, splits, CM, CN);
  auto piece_at = [&](int j) {
    return sk ? tc_streamk_piece(j, blockIdx.x, gridDim.x, tiles_n, tiles_m * tiles_n, nkb)
              : tc_slice_piece(j, cluster_id, clusters, crank, tiles_m, tiles_n, nkb, splits, CM, CN);
  };

  pdl_launch_dependents();
  // trace record: kernel 400 + MODE, aux = N | K << 16 (the GEMM's shape names its kind in the encoder's schedule)
  AVSR_TSPAN_OPEN(400 + MODE, (unsigned)ep.N | ((unsigned)K << 16));
#ifdef AVSR_TRACE
  __shared__ unsigned long long* s_trec;   // the record, for marks by threads other than thread 0
  if (threadIdx.x == 0) s_trec = _tsp;
#define TC_STAMP(slot) ::avsr::trace_stamp(s_trec, slot)
#else
#define TC_STAMP(slot) do { } while (0)
#endif
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    // empty: the 4 warps of the consumer warpgroup that owns the stage's item, in each CTA the stage's loads land in
    for (int s = 0; s < S; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 4 * CS); }
    for (int i = 0; i < 4; ++i) mbar_init(order_bar(i >> 1, i & 1), 4);
    fence_barrier_init();
  }
  __syncthreads();
  if constexpr (CS > 1) cluster_sync();   // peers' barriers are initialised before any multicast or remote arrive
  // Static-operand prologue (ep.b_static): Bw is a prepared weight that no kernel of this PDL chain writes, so it may be
  // read before griddepcontrol.wait.  Why that holds: with PDL, kernel k + 2 can run this section before kernel k has
  // finished, so only buffers that nothing in the chain writes may be read here.  The encoder forward is the only
  // caller that sets the flag; its weights are written by avsr_prepare_weights / the training refresh, which end
  // before the chain starts (the forward's first operation is a memset, the plan's body a graph launch, and the head's
  // proj GEMM follows a kernel launched without PDL, each a full dependency on the stream's earlier work).
  //   warp 0: arms `full` of the first min(S, k-blocks of its pieces) stages with the whole stage's bytes and issues
  //           their Bw boxes; their A boxes follow the wait (the barrier protocol is unchanged);
  //   warp 1: prefetches this CTA's share of the whole weight into L2, k-block-major (the order the CTAs consume it),
  //           so the k-blocks past the ring's first fill do not wait on HBM either.
  const bool pre = CS == 1 && MODE != EPI_VT && ep.b_static != 0;
  // Everything before each warp's pdl_wait() overlaps the previous kernel's tail; after it the warp touches that
  // kernel's outputs.  Warps 1-3 never touch them.
  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0) {
      int pre_its = 0;                              // ring iterations whose Bw box the prologue issued
      if (pre) {
        for (int j = 0; j < npieces && pre_its < S; ++j) {
          const TcPiece w = piece_at(j);
          for (int kb = w.kb0; kb < w.kb1 && pre_its < S; ++kb, ++pre_its) {
            if (elect_one_sync()) {
              mbar_expect_tx(full_bar(pre_its), Cfg::kStageBytes);
              tma_load_2d(base + pre_its * Cfg::kStageBytes + Cfg::kABytes, &tmB, kb * KE, w.tn * BN, full_bar(pre_its));
            }
          }
        }
        if (lane == 0) TC_STAMP(0);                 // the prologue's loads are issued
      }
      pdl_wait();
      AVSR_TSPAN_DEP();
      // TMA producer: warp-uniform loop, only the instruction issue is guarded by elect.sync
      const int cm = crank % CM, cn = crank / CM;
      uint16_t a_mask = 0, b_mask = 0;              // peers sharing this CTA's A rows / Bw rows
      for (int j = 0; j < CN; ++j) a_mask |= (uint16_t)(1u << (cm + CM * j));
      for (int i = 0; i < CM; ++i) b_mask |= (uint16_t)(1u << (i + CM * cn));
      int it = 0;                                   // running k-block counter across tiles
      for (int j = 0; j < npieces; ++j) {
        const TcPiece w = piece_at(j);
        const int m0 = w.tm * TC_BM, n0 = w.tn * BN;
        for (int kb = w.kb0; kb < w.kb1; ++kb, ++it) {
          const int s = it % S;
          const uint32_t ph = (it / S) & 1;
          const bool b_done = it < pre_its;           // armed and Bw issued by the prologue (a fresh stage)
          if (!b_done) mbar_wait(empty_bar(s), ph ^ 1);
          if (elect_one_sync()) {
            if (!b_done) mbar_expect_tx(full_bar(s), Cfg::kStageBytes);   // own slices + the peers' multicast slices
            const uint32_t a_dst = base + s * Cfg::kStageBytes;
            if constexpr (CN == 1) tma_load_2d(a_dst, &tmA, kb * KE, m0, full_bar(s));
            else tma_load_2d_mc(a_dst + cn * (TC_BM / CN) * 128, &tmA, kb * KE, m0 + cn * (TC_BM / CN), full_bar(s), a_mask);
            if (!b_done) {
              if constexpr (CM == 1) tma_load_2d(a_dst + Cfg::kABytes, &tmB, kb * KE, n0, full_bar(s));
              else tma_load_2d_mc(a_dst + Cfg::kABytes + cm * (BN / CM) * 128, &tmB, kb * KE, n0 + cm * (BN / CM),
                                  full_bar(s), b_mask);
            }
          }
        }
      }
      if (lane == 0) TC_STAMP(2);                   // every load of the CTA is issued
    } else if (warp == 1 && pre && lane == 0) {
      for (int i = blockIdx.x; i < tiles_n * nkb; i += gridDim.x)
        tma_prefetch_l2_2d(&tmB, (i / tiles_n) * KE, (i % tiles_n) * BN);
    }
  } else {
    setmaxnreg_inc<232>();
    pdl_wait();
    const int wg = (warp - 4) >> 2;              // consumer warpgroup: the CTA's items with index parity wg
    const int q = warp & 3;                      // 32-row slab of the tile this warp drains (all BN columns)
    constexpr int RB = LD * 4;                               // accumulator row stride in bytes
    // transpose buffer of a chunk: the warp's own accumulator rows, from the chunk's first column (epilogue.cuh)
    auto stg_at = [&](int c) { return reinterpret_cast<uint8_t*>(s_acc + (q * 32) * LD + c); };
    auto wg_sync = [&] { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); };   // this warpgroup only
    const int pr = lane >> 3;                                // row (of 4) this lane emits per read iteration
    const int pc = lane & 7;                                 // 16-byte piece of the 128-byte row segment
    constexpr int OC = StageOp<TOp>::kCols;                  // operand columns per row segment (32 tf32 / 64 f16)
    constexpr int ONE = 16 / (int)sizeof(TOp);               // operand elements per 16-byte piece
    const float* arow = s_acc + (q * 32 + lane) * LD;        // this lane's accumulator row
    auto acc_ld32 = [&](int c, float* v) {
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const float4 t = *reinterpret_cast<const float4*>(arow + c + j);
        v[j] = t.x; v[j + 1] = t.y; v[j + 2] = t.z; v[j + 3] = t.w;
      }
    };
    float acc[BN];                               // rows 0-63 of the tile in acc[0, BN/2), rows 64-127 in acc[BN/2, BN)
    // a stage is released to the producer of every CTA of the cluster (lane r -> CTA r)
    auto release = [&](int s) {
      if constexpr (CS == 1) { if (lane == 0) mbar_arrive(empty_bar(s)); }
      else { if (lane < CS) mbar_arrive_cluster(empty_bar(s), (uint32_t)lane); }
    };
    // this warp is done with its main loop / epilogue: the other warpgroup may start its own
    auto pass_turn = [&](int phase) { __syncwarp(); if (lane == 0) mbar_arrive(order_bar(phase, wg ^ 1)); };
    int it = 0, turn = 0;
#pragma unroll 1
    for (int idx = 0; idx < npieces; ++idx) {
    const TcPiece w = piece_at(idx);
    const int tile = w.tm * tiles_n + w.tn;
    const int m0 = w.tm * TC_BM, n0 = w.tn * BN;
    const int kb0 = w.kb0, kb1 = w.kb1;
    if ((idx & 1) != wg) { it += kb1 - kb0; continue; }   // the other warpgroup's piece: skip its stages
    // warpgroup 0 goes first: its first wait is on the parity of the phase before phase 0, which passes at once
    const uint32_t par = (uint32_t)(turn++ & 1) ^ (wg == 0 ? 1u : 0u);
    // the first wgmma of the item overwrites the accumulator; zeroing it here only tells the compiler that the previous
    // item's values are dead, so they need no registers during the epilogue
#pragma unroll
    for (int i = 0; i < BN; ++i) acc[i] = 0.f;
    // ---- main loop: one wgmma group in flight; a stage is released once the group that read it has retired
    mbar_wait(order_bar(0, wg), par);
    for (int kb = kb0; kb < kb1; ++kb, ++it) {
      const int s = it % S;
      mbar_wait(full_bar(s), (it / S) & 1);
      if (idx == 0 && kb == kb0 && q == 0 && lane == 0) TC_STAMP(1);   // the CTA's first stage landed
      const uint32_t a_addr = base + s * Cfg::kStageBytes;
      const uint64_t a_desc0 = wgmma_desc_sw128(a_addr);
      const uint64_t a_desc1 = wgmma_desc_sw128(a_addr + 64 * 128);
      const uint64_t b_desc = wgmma_desc_sw128(a_addr + Cfg::kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {  // one MMA-K = 32 bytes = +2 in the descriptor's 16-byte address field
        Op::template mma<BN>(acc, a_desc0 + 2 * k, b_desc + 2 * k, (kb != kb0) || (k != 0));
        Op::template mma<BN>(acc + BN / 2, a_desc1 + 2 * k, b_desc + 2 * k, (kb != kb0) || (k != 0));
      }
      wgmma_commit();
      wgmma_wait<1>();
      wgmma_fence_regs<BN>(acc);
      if (kb != kb0) release((it - 1) % S);
    }
    pass_turn(0);                                  // every k-block is issued: the other main loop may start
    wgmma_wait<0>();
    wgmma_fence_regs<BN>(acc);
    if (idx == npieces - 1 && q == 0 && lane == 0) TC_STAMP(3);       // the CTA's last main loop retired
    release((it - 1) % S);
    mbar_wait(order_bar(1, wg), par);              // the other warpgroup's epilogue is done with s_acc / s_vec
    if (!w.valid) { pass_turn(1); continue; }      // past the matrix edge: took part in the loads, stores nothing
    // ---- accumulator -> shared memory (fp32 rows), the tile's per-column vectors next to it
    // fp32 LINEAR into a residual, whole tile: the warp's residual slab is loaded 64 columns at a time, the first 64
    // once the accumulator registers are free, the next while the previous ones are stored (lane: rows it8 * 4 + pr of
    // the slab, columns 32 * cc + 4 * pc of the tile; every load of an element precedes its store by the same thread,
    // so resid may be out).  One round trip per 64 columns instead of one per 32.
    constexpr int RC = BN / 32 < 2 ? BN / 32 : 2;             // 32-column chunks of residual in registers
    float4 res[RC][8];
    const bool res_tile = MODE == EPI_LINEAR && !ep.round_out && w.npieces == 1 && ep.resid != nullptr;
    auto load_res = [&](int cc, float4* dst) {
      const int n = n0 + 32 * cc + pc * 4;
#pragma unroll
      for (int it8 = 0; it8 < 8; ++it8) {
        const int m = m0 + q * 32 + it8 * 4 + pr;
        dst[it8] = (m < ep.M && n < ep.N) ? *reinterpret_cast<const float4*>(ep.resid + (long)m * ep.ldo + n)
                                          : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    };
    {
      const int r = (warp & 3) * 16 + (lane >> 2);
      const int c = 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float* ah = acc + h * (BN / 2);
        float* sh = s_acc + (h * 64 + r) * LD + c;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          *reinterpret_cast<float2*>(sh + 8 * j) = make_float2(ah[4 * j], ah[4 * j + 1]);
          *reinterpret_cast<float2*>(sh + 8 * LD + 8 * j) = make_float2(ah[4 * j + 2], ah[4 * j + 3]);
        }
      }
      if constexpr (MODE == EPI_LINEAR) {
        if (res_tile) {
#pragma unroll
          for (int cc = 0; cc < RC; ++cc) load_res(cc, res[cc]);
        }
      }
      float* s_bias = s_vec;
      float* s_u = s_vec + BN;
      float* s_v = s_vec + 2 * BN;
      const int D = ep.H * kHeadDim;
      for (int cc = threadIdx.x & 127; cc < BN; cc += 128) {
        const int n = n0 + cc;
        float bv = 0.f, uv = 0.f, vv = 0.f;
        if constexpr (MODE != EPI_VT && MODE != EPI_POS) {
          if (ep.bias && n < ep.N) bv = ep.bias[n];
        }
        if constexpr (MODE == EPI_QK) {
          if (n < D) { uv = ep.pos_u[n]; vv = ep.pos_v[n]; }
        }
        s_bias[cc] = bv; s_u[cc] = uv; s_v[cc] = vv;
      }
    }
    wg_sync();
    {
      const int mw = m0 + q * 32;                            // first row of this warp's 32-row slab
      if constexpr (MODE == EPI_GLU) {
        static_assert(MODE != EPI_GLU || BN % 128 == 0, "GLU pairs live 64 columns apart inside a 128-wide group");
#pragma unroll 1
        for (int c = 0; c < BN; c += (c & 32) ? 96 : 32) {   // value columns [g, g + 64) of each 128-wide group g
          uint8_t* stg = stg_at(c);
          float val[32], gate[32];
          acc_ld32(c, val);
          acc_ld32(c + 64, gate);
          const float* sb = s_vec + c;
#pragma unroll
          for (int j = 0; j < 32; ++j) val[j] = (val[j] + sb[j]) * sigmoidf_fast(gate[j] + sb[64 + j]);
          stage_write_f32(stg, RB, lane, val, false);
          __syncwarp();
#pragma unroll
          for (int it8 = 0; it8 < 8; ++it8) emit_glu(ep, mw + it8 * 4 + pr, n0 + c + pc * 4, stage_read(stg, RB, it8, lane));
          __syncwarp();
        }
      } else if constexpr (MODE == EPI_LINEAR) {
        if (!ep.round_out && w.npieces == 1) {              // fp32 destination (+ residual), whole tile
          // the lane reads its output pieces straight from the accumulator rows (the layout emit reads)
#pragma unroll
          for (int cc = 0; cc < BN / 32; ++cc) {
            const int c = 32 * cc, n = n0 + c + pc * 4;
            const float4 bv = *reinterpret_cast<const float4*>(s_vec + c + pc * 4);
#pragma unroll
            for (int it8 = 0; it8 < 8; ++it8) {
              const int m = mw + it8 * 4 + pr;
              float4 o = *reinterpret_cast<const float4*>(s_acc + (q * 32 + it8 * 4 + pr) * LD + c + pc * 4);
              o.x += bv.x; o.y += bv.y; o.z += bv.z; o.w += bv.w;
              if (ep.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
              if (res_tile) {
                const float4 r = res[cc % RC][it8];
                o.x = r.x + ep.alpha * o.x; o.y = r.y + ep.alpha * o.y;
                o.z = r.z + ep.alpha * o.z; o.w = r.w + ep.alpha * o.w;
              }
              if (m < ep.M && n < ep.N)
                *reinterpret_cast<float4*>(reinterpret_cast<float*>(ep.out) + (long)m * ep.ldo + n) = o;
            }
            if (res_tile && cc + RC < BN / 32) load_res(cc + RC, res[cc % RC]);
          }
        } else if (!ep.round_out) {                          // fp32 partial of a piece of a shared tile
          // its raw partial tile goes to plane `piece` of the fp32 workspace (coalesced 16-byte stores); the last CTA
          // to arrive for this tile sums the pieces in fixed order (below) -> deterministic
          float* part = ep.partial + (long)w.piece * ep.M * ep.ldo;
#pragma unroll 1
          for (int c = 0; c < BN; c += 32) {
            const int n = n0 + c + pc * 4;
#pragma unroll
            for (int it8 = 0; it8 < 8; ++it8) {
              const int m = mw + it8 * 4 + pr;
              const float4 pay = *reinterpret_cast<const float4*>(s_acc + (q * 32 + it8 * 4 + pr) * LD + c + pc * 4);
              if (m < ep.M && n < ep.N) *reinterpret_cast<float4*>(part + (long)m * ep.ldo + n) = pay;
            }
          }
        } else {                                             // operand-typed destination (FFN hidden)
#pragma unroll 1
          for (int c = 0; c < BN; c += OC) {
            uint8_t* stg = stg_at(c);
            float v[OC];
#pragma unroll
            for (int k = 0; k < OC; k += 32) acc_ld32(c + k, v + k);
            const float* sb = s_vec + c;
#pragma unroll
            for (int j = 0; j < OC; ++j) { v[j] += sb[j]; if (ep.relu) v[j] = fmaxf(v[j], 0.f); }
            StageOp<TOp>::write(stg, RB, lane, v);
            __syncwarp();
#pragma unroll
            for (int it8 = 0; it8 < 8; ++it8)
              emit_linear_op<TOp>(ep, mw + it8 * 4 + pr, n0 + c + pc * ONE, stage_read(stg, RB, it8, lane));
            __syncwarp();
          }
        }
      } else {
        float row_bias = 0.f;                                // V^T: the bias is per output ROW (feature)
        if constexpr (MODE == EPI_VT) { const int m = mw + lane; row_bias = (m < ep.M) ? ep.bias[m] : 0.f; }
        const int D = ep.H * kHeadDim;
#pragma unroll 1
        for (int c = 0; c < BN; c += OC) {
          uint8_t* stg = stg_at(c);
          float v[OC];
#pragma unroll
          for (int k = 0; k < OC; k += 32) acc_ld32(c + k, v + k);
          const int n = n0 + c;
          if constexpr (MODE == EPI_QK) {
            const float* sb = s_vec + c;
#pragma unroll
            for (int j = 0; j < OC; ++j) v[j] += sb[j];
            // decode once per chunk / per lane: column -> (segment, head, offset); rows -> (utterance, frame)
            const int np = n + pc * ONE;
            const int seg = np / D, nn = np - seg * D;
            const int hh = nn >> 6, d0 = nn & 63;
            int rb[8], rt[8];
            bool rok[8];
            {
              const int mrow = mw + pr;                    // this lane's first row; the others follow 4 rows apart
              int bb = mrow / ep.T, tt = mrow - bb * ep.T;
#pragma unroll
              for (int it8 = 0; it8 < 8; ++it8) {
                rb[it8] = bb; rt[it8] = tt; rok[it8] = (mrow + it8 * 4 < ep.M) && (np < ep.N);
                tt += 4;
                while (tt >= ep.T) { tt -= ep.T; ++bb; }
              }
            }
            if (n < D) {                                     // q: two outputs, q + pos_bias_u and q + pos_bias_v
              // the first output's transpose overwrites the chunk's first 128 bytes: keep those accumulators
              float keep[32];
              acc_ld32(c, keep);
              const float* su = s_vec + BN + c;
#pragma unroll
              for (int j = 0; j < OC; ++j) v[j] += su[j];
              StageOp<TOp>::write(stg, RB, lane, v);
              __syncwarp();
#pragma unroll
              for (int it8 = 0; it8 < 8; ++it8)
                emit_heads<TOp>(ep, ep.qu, rok[it8], rb[it8], rt[it8], hh, d0, stage_read(stg, RB, it8, lane));
              __syncwarp();
              // second output: the accumulator chunk again (kept registers + the part still in shared memory)
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] = keep[j];
#pragma unroll
              for (int k = 32; k < OC; k += 32) acc_ld32(c + k, v + k);
              const float* sv = s_vec + 2 * BN + c;
#pragma unroll
              for (int j = 0; j < OC; ++j) v[j] += sb[j] + sv[j];
              StageOp<TOp>::write(stg, RB, lane, v);
              __syncwarp();
#pragma unroll
              for (int it8 = 0; it8 < 8; ++it8)
                emit_heads<TOp>(ep, ep.qv, rok[it8], rb[it8], rt[it8], hh, d0, stage_read(stg, RB, it8, lane));
              __syncwarp();
            } else {
              StageOp<TOp>::write(stg, RB, lane, v);
              __syncwarp();
              void* dst = n < 2 * D ? ep.kk : ep.vt;
#pragma unroll
              for (int it8 = 0; it8 < 8; ++it8)
                emit_heads<TOp>(ep, dst, rok[it8], rb[it8], rt[it8], hh, d0, stage_read(stg, RB, it8, lane));
              __syncwarp();
            }
          } else {
            if constexpr (MODE == EPI_VT) {
#pragma unroll
              for (int j = 0; j < OC; ++j) v[j] += row_bias;
            }
            StageOp<TOp>::write(stg, RB, lane, v);
            __syncwarp();
#pragma unroll
            for (int it8 = 0; it8 < 8; ++it8) {
              const uint4 pay = stage_read(stg, RB, it8, lane);
              if constexpr (MODE == EPI_VT) emit_vt<TOp>(ep, mw + it8 * 4 + pr, n + pc * ONE, pay);
              else emit_pos<TOp>(ep, mw + it8 * 4 + pr, n + pc * ONE, pay);
            }
            __syncwarp();
          }
        }
      }
    }
    if constexpr (MODE == EPI_LINEAR) {
      if (w.npieces > 1) {
        // ---- deterministic fix-up ("last block reduces"): publish the partial, count arrivals per tile.  No CTA
        // waits for another: the one that arrives last finishes the tile, the others are done.
        __threadfence();
        wg_sync();
        if ((threadIdx.x & 127) == 0) {
          const int old = atomicAdd(ep.counters + tile, 1);
          const int last = (old == w.npieces - 1);
          if (last) ep.counters[tile] = 0;                 // every piece has arrived: re-arm for the next launch
          *s_flag = last;
        }
        wg_sync();
        if (*s_flag) {
          __threadfence();                                 // acquire: the other pieces' partial tiles are visible
          const int mw = m0 + q * 32;
          const float* own = s_acc + (q * 32 + pr) * LD + pc * 4;   // this piece's partial, still in shared memory
#pragma unroll 1
          for (int c = 0; c < BN; c += 32) {
            const int n = n0 + c + pc * 4;
            const float4 bv = *reinterpret_cast<const float4*>(s_vec + c + pc * 4);
            // loads first (8 independent 16-byte loads in flight per slice, no store in between), stores last
            float4 a[8], t4[8];
            bool ok[8];
#pragma unroll
            for (int it8 = 0; it8 < 8; ++it8) { a[it8] = bv; ok[it8] = (mw + it8 * 4 + pr < ep.M) && (n < ep.N); }
            for (int sp = 0; sp < w.npieces; ++sp) {     // fixed order: piece 0, 1, ... regardless of arrival order
              const float* part = ep.partial + (long)sp * ep.M * ep.ldo;
              if (sp == w.piece) {
#pragma unroll
                for (int it8 = 0; it8 < 8; ++it8) t4[it8] = *reinterpret_cast<const float4*>(own + it8 * 4 * LD + c);
              } else {
#pragma unroll
                for (int it8 = 0; it8 < 8; ++it8)
                  t4[it8] = ok[it8] ? __ldcg(reinterpret_cast<const float4*>(part + (long)(mw + it8 * 4 + pr) * ep.ldo + n))
                                    : make_float4(0.f, 0.f, 0.f, 0.f);
              }
#pragma unroll
              for (int it8 = 0; it8 < 8; ++it8) { a[it8].x += t4[it8].x; a[it8].y += t4[it8].y; a[it8].z += t4[it8].z; a[it8].w += t4[it8].w; }
            }
#pragma unroll
            for (int it8 = 0; it8 < 8; ++it8)
              t4[it8] = ok[it8] ? *reinterpret_cast<const float4*>(ep.resid + (long)(mw + it8 * 4 + pr) * ep.ldo + n)
                                : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int it8 = 0; it8 < 8; ++it8) {
              if (ok[it8]) {
                float4 o;
                o.x = t4[it8].x + ep.alpha * a[it8].x; o.y = t4[it8].y + ep.alpha * a[it8].y;
                o.z = t4[it8].z + ep.alpha * a[it8].z; o.w = t4[it8].w + ep.alpha * a[it8].w;
                *reinterpret_cast<float4*>(reinterpret_cast<float*>(ep.out) + (long)(mw + it8 * 4 + pr) * ep.ldo + n) = o;
              }
            }
          }
        }
      }
    }
    pass_turn(1);                                  // this warp is done with s_acc / s_vec / s_flag
    }  // tile loop
  }
  __syncthreads();
  if constexpr (CS > 1) cluster_sync();   // no CTA leaves while a peer may still arrive on or load into its memory
  AVSR_TSPAN_CLOSE();
#undef TC_STAMP
}

AVSR_TRACE_DEFINE_BIND(trace_bind_gemm_tc)

static int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
  }
  return n;
}

// Most clusters of this kernel that can be resident at once (GPCs need not hold a multiple of the cluster size).
template <typename Kernel>
static int max_active_clusters(Kernel kernel, int cs, int smem) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(cs); cfg.blockDim = dim3(TC_THREADS); cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = cs; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
  cfg.attrs = &attr; cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess) return 0;
  return n;
}

template <int MODE, int BN, typename TOp, int CM, int CN>
static int launch_tc(const void* A, const void* Bw, int M, int N, int K, int splits, bool streamk,
                     const EpiParams& ep, cudaStream_t st) {
  using Cfg = TcCfg<BN>;
  constexpr int CS = CM * CN;
  auto kernel = gemm_tc_kernel<MODE, BN, TOp, CM, CN>;
  CUtensorMap tmA, tmB;
  AVSR_TRY(make_tmap_2d(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)K, TC_BM / CN, op_kind_of<TOp>()));
  AVSR_TRY(make_tmap_2d(&tmB, Bw, (uint64_t)N, (uint64_t)K, (uint64_t)K, BN / CM, op_kind_of<TOp>()));
  AVSR_SET_MAX_SMEM(kernel, Cfg::kSmem);
  const int tiles_m = cdiv(M, TC_BM), tiles_n = cdiv(N, BN);
  if (CS > 1 || splits > kMaxSplits || tiles_m * tiles_n > kSplitCounters) {   // caller's workspace contract
    splits = 1;
    streamk = false;
  }
  if (streamk) {
    const int grid = tc_streamk_ctas(num_sms(), tiles_m * tiles_n, K / OpTraits<TOp>::kElemsPerBlock);
    AVSR_LAUNCH_CLUSTER(kernel, grid, TC_THREADS, Cfg::kSmem, st, 1, tmA, tmB, K, tiles_m, tiles_n, 1, 1, ep);
    return AVSR_OK;
  }
  const int total = tc_cluster_items(tiles_m, tiles_n, splits, CM, CN);
  int slots = num_sms();
  if constexpr (CS > 1) {
    static int dev_done = -1, active = 0;
    int dev = 0;
    AVSR_CUDA_TRY(cudaGetDevice(&dev));
    if (dev_done != dev) { active = max_active_clusters(kernel, CS, Cfg::kSmem); dev_done = dev; }
    AVSR_REQUIRE(active > 0, "gemm_tc: no %dx%d cluster of this kernel fits on the device", CM, CN);
    slots = active;
  }
  const int grid = (total < slots ? total : slots) * CS;
  AVSR_LAUNCH_CLUSTER(kernel, grid, TC_THREADS, Cfg::kSmem, st, CS, tmA, tmB, K, tiles_m, tiles_n, splits, 0, ep);
  return AVSR_OK;
}

// ---------------------------------------------------------------- tile / split selection
// Cost model (SM cycles) of one GEMM on persistent CTAs, one per SM: the busier of the tensor pipe (dense wgmma rate
// per SM) and operand ingest (bytes the busiest SM pulls through L2, at an assumed ~64 B/cycle), plus one epilogue:
// the consumer warpgroups alternate items, so every epilogue but the SM's last runs under the other warpgroup's main
// loop.  Split-K and stream-K (only for GEMMs that accumulate into the fp32 residual stream) spread a long K over more
// SMs; stream-K is charged what it measured (below).
// It picks 1 x 1 clusters only.  Multicast clusters cut the modelled L2 -> SM bytes by 25 % (2x1, 1x2) or 50 % (2x2)
// but measured about 1.8x slower at the S2 shapes on an H100 80GB HBM3 at 400 W (FFN w_1 1600x3072x768: 22.7 us at
// 1x1, 42.6 us at 2x1): the main loop waits on load latency, not L2 bandwidth (DESIGN.md section 4); clusters stay
// reachable through AVSR_B200_TILE for sweeps.
struct TileChoice { int bn, splits, cm, cn; bool streamk; };
static const int kTileWidths[] = {64, 128};
// Stream-K as measured on an H100 80GB HBM3 at 700 W (1980 MHz), against the data-parallel schedule at the encoder's
// residual shapes (DESIGN.md section 4): the data-parallel w_2 main loop already pulls ~9 TB/s from L2 on its 78
// SMs, so on 132 SMs a k-block costs about 3x the modelled per-SM time (FFN w_2 1600x768x3072 f16: 28.4 k-blocks per
// SM in 41.7 us), and a launch carries ~20 us of partial-tile traffic and fix-up on its critical path (out
// 1600x768x768: 7.1 k-blocks per SM in 24.5 us).  So it stays a candidate for long-K GEMMs with few tiles, and the
// encoder's GEMMs keep the data-parallel schedule.
constexpr double kStreamKStepFactor = 3.0;
constexpr double kStreamKFixed = 40000.0;

static TileChoice choose_tile(int mode, int M, int N, int K, int esz, bool operand_dest, bool can_split,
                              bool can_streamk) {
  const double mac_per_cycle = esz == 2 ? 2048.0 : 1024.0;   // per SM, dense f16 / tf32
  const double ingest = 64.0;                                // operand bytes per cycle per SM
  const int nkb = K / (128 / esz);
  const int sms = num_sms();
  double best = 1e30;
  TileChoice pick{128, 1, 1, 1, false};
  for (const int bn : kTileWidths) {
    if (mode == EPI_GLU && bn % 128 != 0) continue;
    if (bn == 64 && esz == 2 && (mode != EPI_LINEAR || operand_dest)) continue;   // needs 64-column row segments
    if (bn > 64 && N <= bn / 2) continue;                                          // mostly empty tile
    const long tiles = (long)cdiv(M, 128) * cdiv(N, bn);
    const double t_epi = 128.0 * bn * 10.0 / 128.0 * 4.0;                          // the SM's last epilogue
    // the busiest SM's main loop over `steps` k-blocks
    auto t_main = [&](long steps) {
      const double t_mma = steps * 128.0 * bn * (128 / esz) / mac_per_cycle;
      const double t_in = steps * (128.0 + bn) * 128.0 / ingest;
      return t_mma > t_in ? t_mma : t_in;
    };
    for (int splits = 1; splits <= (can_split ? kMaxSplits : 1); ++splits) {
      if (splits > nkb) break;
      const long per_sm = (tiles * splits + sms - 1) / sms;
      // fix-up: the last arriver re-reads `splits` fp32 partial tiles through the same port
      const double t_red = splits > 1 ? (double)splits * 128.0 * bn * 4.0 / ingest : 0.0;
      const double est = t_main(per_sm * ((nkb + splits - 1) / splits)) + t_epi + t_red + 4000.0;
      if (est < best) { best = est; pick = TileChoice{bn, splits, 1, 1, false}; }
    }
    if (can_streamk && tiles <= kSplitCounters) {
      // stream-K: equal shares of the tiles * nkb steps at the measured rate
      const long ctas = tc_streamk_ctas(sms, (int)tiles, nkb);
      const double est = kStreamKStepFactor * t_main((tiles * nkb + ctas - 1) / ctas) + t_epi + kStreamKFixed;
      if (est < best) { best = est; pick = TileChoice{bn, 1, 1, 1, true}; }
    }
  }
  return pick;
}

template <int MODE, int BN, typename TOp>
static int dispatch_cluster(TileChoice t, const void* A, const void* Bw, int M, int N, int K, const EpiParams& ep,
                            cudaStream_t st) {
  if (t.cm == 1 && t.cn == 1) return launch_tc<MODE, BN, TOp, 1, 1>(A, Bw, M, N, K, t.splits, t.streamk, ep, st);
  if (t.cm == 2 && t.cn == 1) return launch_tc<MODE, BN, TOp, 2, 1>(A, Bw, M, N, K, 1, false, ep, st);
  if (t.cm == 1 && t.cn == 2) return launch_tc<MODE, BN, TOp, 1, 2>(A, Bw, M, N, K, 1, false, ep, st);
  if (t.cm == 2 && t.cn == 2) return launch_tc<MODE, BN, TOp, 2, 2>(A, Bw, M, N, K, 1, false, ep, st);
  set_error("gemm_tc: no kernel for cluster %dx%d", t.cm, t.cn);
  return AVSR_E_INVALID;
}

template <int MODE, typename TOp>
static int dispatch_tile(TileChoice t, const void* A, const void* Bw, int M, int N, int K, const EpiParams& ep,
                         cudaStream_t st) {
  if (t.bn == 64) {
    if constexpr (MODE != EPI_GLU) return dispatch_cluster<MODE, 64, TOp>(t, A, Bw, M, N, K, ep, st);
  }
  if (t.bn == 128) return dispatch_cluster<MODE, 128, TOp>(t, A, Bw, M, N, K, ep, st);
  set_error("gemm_tc: no kernel for tile 128x%d", t.bn);
  return AVSR_E_INVALID;
}

template <typename TOp>
static int dispatch_mode(int mode, const void* A, const void* Bw, int M, int N, int K, const EpiParams& ep,
                         cudaStream_t st) {
  const bool operand_dest = mode != EPI_GLU && (mode != EPI_LINEAR || ep.round_out != 0);
  // split-K and stream-K add partial sums into the destination: only when the destination IS the residual it
  // accumulates into.  Both need the caller's fp32 workspace + zeroed tile counters (EpiParams::partial / counters);
  // the pieces of a tile are summed in fixed order by the last-arriving CTA, so the result does not depend on
  // scheduling.  Stream-K is a candidate of the cost model whenever the workspace is there; equal-slice split-K is
  // opt-in (AVSR_B200_SPLITK=1).
  const bool can_streamk = mode == EPI_LINEAR && !ep.round_out && !ep.relu && ep.resid != nullptr &&
                           ep.partial != nullptr && ep.counters != nullptr;
  static const bool allow_split = [] { const char* e = getenv("AVSR_B200_SPLITK"); return e && e[0] == '1'; }();
  const bool can_split = allow_split && can_streamk;
  TileChoice t = choose_tile(mode, M, N, K, (int)sizeof(TOp), operand_dest, can_split, can_streamk);
  // "BN[,SPLITS[,CMxCN]]" runs exactly that tile, split and cluster shape; "BN,sk" runs stream-K at that tile width
  // where the GEMM can take it (tuning / profiling aid)
  if (const char* force = getenv("AVSR_B200_TILE")) {
    int bn = 0, sp = 1, cm = 1, cn = 1;
    const int got = sscanf(force, "%d,%d,%dx%d", &bn, &sp, &cm, &cn);
    if (got >= 1 && (bn == 64 || bn == 128) && (mode != EPI_GLU || bn % 128 == 0) &&
        !(bn == 64 && sizeof(TOp) == 2 && operand_dest)) {
      if (got < 4 || cm < 1 || cm > 2 || cn < 1 || cn > 2) cm = cn = 1;
      if (got < 2 || !can_split || sp < 1 || cm * cn > 1) sp = 1;
      const int nkb = K / (128 / (int)sizeof(TOp));
      const char* comma = strchr(force, ',');
      const bool sk = got == 1 && comma && strcmp(comma + 1, "sk") == 0 && can_streamk;
      t = TileChoice{bn, sp > nkb ? nkb : sp, cm, cn, sk};
    }
  }
  AVSR_REQUIRE(mode == EPI_VT || N % 8 == 0, "gemm_tc: N=%d must be a multiple of 8", N);
  if (mode == EPI_LINEAR) {
    AVSR_REQUIRE((ep.ldo % 8) == 0 && (reinterpret_cast<uintptr_t>(ep.out) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(ep.resid) & 15) == 0,
                 "gemm_tc: output / residual must be 16-byte aligned with a row stride that is a multiple of 8");
  }
  switch (mode) {
    case EPI_LINEAR: return dispatch_tile<EPI_LINEAR, TOp>(t, A, Bw, M, N, K, ep, st);
    case EPI_QK:
      AVSR_REQUIRE(N % 128 == 0, "gemm_tc: QK needs N %% 128 == 0 (N=%d)", N);
      return dispatch_tile<EPI_QK, TOp>(t, A, Bw, M, N, K, ep, st);
    case EPI_VT:
      AVSR_REQUIRE(M % 64 == 0, "gemm_tc: V^T needs M %% 64 == 0 (M=%d)", M);
      return dispatch_tile<EPI_VT, TOp>(t, A, Bw, M, N, K, ep, st);
    case EPI_GLU:
      AVSR_REQUIRE(N % 128 == 0, "gemm_tc: GLU needs N %% 128 == 0 (N=%d)", N);
      return dispatch_tile<EPI_GLU, TOp>(t, A, Bw, M, N, K, ep, st);
    case EPI_POS:
      AVSR_REQUIRE(N % 64 == 0, "gemm_tc: POS needs N %% 64 == 0 (N=%d)", N);
      return dispatch_tile<EPI_POS, TOp>(t, A, Bw, M, N, K, ep, st);
    default:
      AVSR_REQUIRE(false, "gemm_tc: bad epilogue mode %d", mode);
  }
  return AVSR_OK;
}

int gemm_tc(int mode, int opk, const void* A, const void* Bw, int M, int N, int K, const EpiParams& ep,
            cudaStream_t st) {
  AVSR_REQUIRE(opk == OP_TF32 || op16(opk), "gemm_tc: operand kind %d", opk);
  const int ke = op16(opk) ? 64 : 32;
  AVSR_REQUIRE(K >= ke && K % ke == 0, "gemm_tc: K=%d must be a multiple of %d", K, ke);
  if (M <= 0 || N <= 0) return AVSR_OK;
  // AVSR_B200_PROLOGUE=0 turns the static-operand prologue off (read per call, so one process can A/B both paths)
  EpiParams e = ep;
  if (const char* pro = getenv("AVSR_B200_PROLOGUE")) { if (pro[0] == '0') e.b_static = 0; }
  if (opk == OP_F16) return dispatch_mode<__half>(mode, A, Bw, M, N, K, e, st);
  if (opk == OP_BF16) return dispatch_mode<__nv_bfloat16>(mode, A, Bw, M, N, K, e, st);
  return dispatch_mode<float>(mode, A, Bw, M, N, K, e, st);
}

}  // namespace avsr
