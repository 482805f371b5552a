// Tensor-core GEMM for the Conformer layer's projections (FFN x2, QK, V^T, out, pw1+GLU, pw2) and the stacked
// linear_pos:   acc[m][n] = sum_k A[m][k] * Bw[n][k]   (both K-major = torch.nn.Linear layout).
//
// Hopper pipeline (sm_90a).  One persistent CTA owns a 128 x BN output tile at a time:
//   warp 0        : TMA producer -- cp.async.bulk.tensor 2-D boxes (rows x 128 bytes, SWIZZLE_128B) of A and Bw into
//                   a STAGES-deep shared-memory ring, completion on `full` mbarriers
//   warpgroups 1-2: wgmma.mma_async (M = 64 rows each, N = BN, K = 32 bytes) x4 per stage straight from shared memory
//                   into register accumulators; a stage goes back to the producer (`empty` mbarrier) once the wgmma
//                   group that read it has retired.  Then the same 8 warps run the fused epilogue: accumulators ->
//                   fp32 tile in shared memory -> lane-per-row reads, bias / ReLU / residual / GLU / head-major
//                   scatter / conversion to the next operand's storage, coalesced global stores (epilogue.cuh)
// Operand storage (template TOp): float = TF32 (8 elements per MMA-K) or __half (16 per MMA-K; same 10-bit mantissa,
// half the bytes, twice the rate).  Out-of-bounds rows of edge tiles are zero-filled by TMA and masked in the
// epilogue.  The tile width is chosen per problem by a small cost model (bytes through L2 vs tensor-pipe time).
#include "common.cuh"
#include "epilogue.cuh"
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

int make_tmap_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                 int esz) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)"); return AVSR_E_CUDA; }
  AVSR_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0 && (ld * esz) % 16 == 0 && box_rows <= 256 &&
                   (esz == 4 || esz == 2),
               "tensor map: base/stride must be 16-byte aligned (ld=%llu, esz=%d)", (unsigned long long)ld, esz);
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstr[1] = {ld * (uint64_t)esz};
  cuuint32_t box[2] = {(cuuint32_t)(128 / esz), box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, esz == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                   const_cast<void*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(2d) failed: CUresult %d", (int)r); return AVSR_E_CUDA; }
  return AVSR_OK;
}

int make_tmap_3d(CUtensorMap* map, const void* base, uint64_t planes, uint64_t rows, uint64_t cols, uint64_t ld_row,
                 uint64_t ld_plane, uint32_t box_rows, int esz) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)"); return AVSR_E_CUDA; }
  AVSR_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0 && (ld_row * esz) % 16 == 0 &&
                   (ld_plane * esz) % 16 == 0 && box_rows <= 256 && (esz == 4 || esz == 2),
               "tensor map 3d: base/strides must be 16-byte aligned");
  cuuint64_t gdim[3] = {cols, rows, planes};
  cuuint64_t gstr[2] = {ld_row * (uint64_t)esz, ld_plane * (uint64_t)esz};
  cuuint32_t box[3] = {(cuuint32_t)(128 / esz), box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, esz == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3,
                   const_cast<void*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(3d) failed: CUresult %d", (int)r); return AVSR_E_CUDA; }
  return AVSR_OK;
}

// ---------------------------------------------------------------- the kernel
constexpr int TC_BM = 128;          // rows per CTA tile / per A box (two warpgroups of 64 rows)
constexpr int TC_THREADS = 384;     // warpgroup 0: TMA producer (warp 0); warpgroups 1-2: wgmma + epilogue
constexpr int TC_EPI_THREADS = 256; // the two consumer warpgroups
constexpr int TC_SMEM_BUDGET = 227 * 1024;   // one persistent CTA per SM

template <int BN>
struct TcCfg {
  static constexpr int kABytes = TC_BM * 128;
  static constexpr int kBBytes = BN * 128;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kAccLd = BN + 4;                 // fp32 accumulator tile row stride (conflict-free float4 rows)
  static constexpr int kAccBytes = TC_BM * kAccLd * 4;
  static constexpr int kVecBytes = 3 * BN * 4;          // bias / pos_bias_u / pos_bias_v of the tile's columns
  static constexpr int kStagingBytes = 8 * STG_WARP;    // epilogue transpose buffers
  static constexpr int kFixedBytes = 1024 /*align slack*/ + 256 /*barriers*/ + kAccBytes + kVecBytes + kStagingBytes;
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

template <int MODE, int BN, typename TOp>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int K, int tiles_m,
               int tiles_n, int splits, EpiParams ep) {
  // PERSISTENT: CTA c processes tiles c, c + gridDim.x, ... (n fastest, so concurrently running CTAs share A rows in
  // L2).  The TMA ring never drains between tiles: the producer fetches the next tile's k-blocks while the consumer
  // warpgroups run the epilogue of the current one.
  using Cfg = TcCfg<BN>;
  using Op = OpTraits<TOp>;
  constexpr int S = Cfg::kStages;
  constexpr int KE = Op::kElemsPerBlock;
  constexpr int LD = Cfg::kAccLd;
  extern __shared__ uint8_t tc_smem_raw[];
  const uint32_t raw = smem_u32(tc_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;       // SWIZZLE_128B tiles need 1024-byte alignment
  uint8_t* gen = tc_smem_raw + (base - raw);
  const uint32_t bars = base + S * Cfg::kStageBytes;  // full[S], empty[S]
  int* s_flag = reinterpret_cast<int*>(gen + S * Cfg::kStageBytes + 2 * S * 8);   // split-K: "this CTA arrived last"
  float* s_acc = reinterpret_cast<float*>(gen + S * Cfg::kStageBytes + 256);      // [TC_BM][LD]
  float* s_vec = s_acc + TC_BM * LD;                                               // [3][BN]
  uint8_t* stg_base = reinterpret_cast<uint8_t*>(s_vec + 3 * BN);
  auto full_bar = [&](int s) { return bars + 8u * s; };
  auto empty_bar = [&](int s) { return bars + 8u * (S + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nkb = K / KE;
  const int total_tiles = tiles_m * tiles_n;
  // split-K (LINEAR into the residual stream only): work item = (tile, K-slice); slice-major order so that CTAs
  // running at the same time reduce into different tiles.
  const int total_items = total_tiles * splits;

  pdl_launch_dependents();
  AVSR_TSPAN_OPEN(400 + MODE, (unsigned)BN);
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < S; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 8); }   // 8 consumer warps
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();   // everything above overlapped the previous kernel's tail; from here on we touch its outputs
  AVSR_TSPAN_DEP();

  if (warp == 0) {
    // TMA producer: warp-uniform loop, only the instruction issue is guarded by elect.sync
    int it = 0;                                         // running k-block counter across tiles
    for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
      const int tile = item % total_tiles, split = item / total_tiles;
      const int m0 = (tile / tiles_n) * TC_BM, n0 = (tile % tiles_n) * BN;
      const int kb0 = split * nkb / splits, kb1 = (split + 1) * nkb / splits;
      for (int kb = kb0; kb < kb1; ++kb, ++it) {
        const int s = it % S;
        const uint32_t ph = (it / S) & 1;
        mbar_wait(empty_bar(s), ph ^ 1);
        if (elect_one_sync()) {
          mbar_expect_tx(full_bar(s), Cfg::kStageBytes);
          const uint32_t a_dst = base + s * Cfg::kStageBytes;
          tma_load_2d(a_dst, &tmA, kb * KE, m0, full_bar(s));
          tma_load_2d(a_dst + Cfg::kABytes, &tmB, kb * KE, n0, full_bar(s));
        }
      }
    }
  } else if (warp >= 4) {
    const int wg = (warp - 4) >> 2;              // consumer warpgroup: accumulator rows [64 wg, 64 wg + 64)
    const int e = warp - 4;                      // epilogue warp 0..7
    const int q = e & 3;                         // 32-row slab of the tile this warp drains
    const int chalf = e >> 2;                    // which half of the tile's columns this warp drains
    uint8_t* stg = stg_base + e * STG_WARP;
    const int cb = chalf * (BN / 2), ce = cb + BN / 2;      // this warp's columns of the tile
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
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int it = 0;
#pragma unroll 1
    for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
    const int tile = item % total_tiles, split = item / total_tiles;
    const int m0 = (tile / tiles_n) * TC_BM, n0 = (tile % tiles_n) * BN;
    const int kb0 = split * nkb / splits, kb1 = (split + 1) * nkb / splits;
    // ---- main loop: one wgmma group in flight; a stage is released once the group that read it has retired
    for (int kb = kb0; kb < kb1; ++kb, ++it) {
      const int s = it % S;
      mbar_wait(full_bar(s), (it / S) & 1);
      const uint32_t a_addr = base + s * Cfg::kStageBytes;
      const uint64_t a_desc = wgmma_desc_sw128(a_addr + wg * (64 * 128));
      const uint64_t b_desc = wgmma_desc_sw128(a_addr + Cfg::kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)  // one MMA-K = 32 bytes = +2 in the descriptor's 16-byte address field
        Op::template mma<BN>(acc, a_desc + 2 * k, b_desc + 2 * k, (kb != kb0) || (k != 0));
      wgmma_commit();
      wgmma_wait<1>();
      wgmma_fence_regs<BN / 2>(acc);
      if (kb != kb0 && lane == 0) mbar_arrive(empty_bar((it - 1) % S));
    }
    wgmma_wait<0>();
    wgmma_fence_regs<BN / 2>(acc);
    if (lane == 0) mbar_arrive(empty_bar((it - 1) % S));
    // ---- accumulator -> shared memory (fp32 rows), the tile's per-column vectors next to it
    asm volatile("bar.sync 1, 256;" ::: "memory");   // previous tile's readers of s_acc / s_vec are done
    {
      const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
      const int c = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        *reinterpret_cast<float2*>(s_acc + r * LD + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(s_acc + (r + 8) * LD + 8 * j + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
      float* s_bias = s_vec;
      float* s_u = s_vec + BN;
      float* s_v = s_vec + 2 * BN;
      const int D = ep.H * kHeadDim;
      for (int cc = threadIdx.x - 128; cc < BN; cc += TC_EPI_THREADS) {
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
    asm volatile("bar.sync 1, 256;" ::: "memory");
    {
      const int mw = m0 + q * 32;                            // first row of this warp's 32-row slab
      if constexpr (MODE == EPI_GLU) {
        static_assert(MODE != EPI_GLU || BN % 128 == 0, "GLU pairs live 64 columns apart inside a 128-wide group");
#pragma unroll 1
        for (int g = 0; g < BN; g += 128) {
          const int c = g + chalf * 32;
          float val[32], gate[32];
          acc_ld32(c, val);
          acc_ld32(c + 64, gate);
          const float* sb = s_vec + c;
#pragma unroll
          for (int j = 0; j < 32; ++j) val[j] = (val[j] + sb[j]) * sigmoidf_fast(gate[j] + sb[64 + j]);
          stage_write_f32(stg, lane, val, false);
          __syncwarp();
#pragma unroll
          for (int it8 = 0; it8 < 8; ++it8) emit_glu(ep, mw + it8 * 4 + pr, n0 + c + pc * 4, stage_read(stg, it8, lane));
          __syncwarp();
        }
      } else if constexpr (MODE == EPI_LINEAR) {
        if (!ep.round_out) {                                 // fp32 destination (+ residual)
#pragma unroll 1
          for (int c = cb; c < ce; c += 32) {
            float v[32];
            acc_ld32(c, v);
            const float* sb = s_vec + c;
            if (splits == 1) {
#pragma unroll
              for (int j = 0; j < 32; ++j) { v[j] += sb[j]; if (ep.relu) v[j] = fmaxf(v[j], 0.f); }
            }
            stage_write_f32(stg, lane, v, false);
            __syncwarp();
            const int n = n0 + c + pc * 4;
            if (splits > 1) {
              // split-K: this K-slice's raw partial tile goes to the fp32 workspace (coalesced 16-byte stores); the
              // last CTA to arrive for this tile sums the slices in fixed order (below) -> deterministic
              float* part = ep.partial + (long)split * ep.M * ep.ldo;
#pragma unroll
              for (int it8 = 0; it8 < 8; ++it8) {
                const int m = mw + it8 * 4 + pr;
                const uint4 pay = stage_read(stg, it8, lane);
                if (m < ep.M && n < ep.N) *reinterpret_cast<uint4*>(part + (long)m * ep.ldo + n) = pay;
              }
            } else {
            // residual pieces first (8 independent coalesced loads in flight), then combine + store: a load may not
            // be hoisted above a store by the compiler (possible aliasing), so the order is made explicit here
            float4 r[8];
            if (ep.resid) {
#pragma unroll
              for (int it8 = 0; it8 < 8; ++it8) {
                const int m = mw + it8 * 4 + pr;
                r[it8] = (m < ep.M && n < ep.N) ? *reinterpret_cast<const float4*>(ep.resid + (long)m * ep.ldo + n)
                                                : make_float4(0.f, 0.f, 0.f, 0.f);
              }
            }
#pragma unroll
            for (int it8 = 0; it8 < 8; ++it8) {
              const int m = mw + it8 * 4 + pr;
              const uint4 pay = stage_read(stg, it8, lane);
              float4 o = *reinterpret_cast<const float4*>(&pay);
              if (ep.resid) {
                o.x = r[it8].x + ep.alpha * o.x; o.y = r[it8].y + ep.alpha * o.y;
                o.z = r[it8].z + ep.alpha * o.z; o.w = r[it8].w + ep.alpha * o.w;
              }
              if (m < ep.M && n < ep.N)
                *reinterpret_cast<float4*>(reinterpret_cast<float*>(ep.out) + (long)m * ep.ldo + n) = o;
            }
            }
            __syncwarp();
          }
        } else {                                             // operand-typed destination (FFN hidden)
#pragma unroll 1
          for (int c = cb; c < ce; c += OC) {
            float v[OC];
#pragma unroll
            for (int k = 0; k < OC; k += 32) acc_ld32(c + k, v + k);
            const float* sb = s_vec + c;
#pragma unroll
            for (int j = 0; j < OC; ++j) { v[j] += sb[j]; if (ep.relu) v[j] = fmaxf(v[j], 0.f); }
            StageOp<TOp>::write(stg, lane, v);
            __syncwarp();
#pragma unroll
            for (int it8 = 0; it8 < 8; ++it8)
              emit_linear_op<TOp>(ep, mw + it8 * 4 + pr, n0 + c + pc * ONE, stage_read(stg, it8, lane));
            __syncwarp();
          }
        }
      } else {
        float row_bias = 0.f;                                // V^T: the bias is per output ROW (feature)
        if constexpr (MODE == EPI_VT) { const int m = mw + lane; row_bias = (m < ep.M) ? ep.bias[m] : 0.f; }
        const int D = ep.H * kHeadDim;
#pragma unroll 1
        for (int c = cb; c < ce; c += OC) {
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
              const float* su = s_vec + BN + c;
#pragma unroll
              for (int j = 0; j < OC; ++j) v[j] += su[j];
              StageOp<TOp>::write(stg, lane, v);
              __syncwarp();
#pragma unroll
              for (int it8 = 0; it8 < 8; ++it8)
                emit_heads<TOp>(ep, ep.qu, rok[it8], rb[it8], rt[it8], hh, d0, stage_read(stg, it8, lane));
              __syncwarp();
              // second output: re-read the accumulator chunk (cheaper than keeping two register copies)
#pragma unroll
              for (int k = 0; k < OC; k += 32) acc_ld32(c + k, v + k);
              const float* sv = s_vec + 2 * BN + c;
#pragma unroll
              for (int j = 0; j < OC; ++j) v[j] += sb[j] + sv[j];
              StageOp<TOp>::write(stg, lane, v);
              __syncwarp();
#pragma unroll
              for (int it8 = 0; it8 < 8; ++it8)
                emit_heads<TOp>(ep, ep.qv, rok[it8], rb[it8], rt[it8], hh, d0, stage_read(stg, it8, lane));
              __syncwarp();
            } else {
              StageOp<TOp>::write(stg, lane, v);
              __syncwarp();
              void* dst = n < 2 * D ? ep.kk : ep.vt;
#pragma unroll
              for (int it8 = 0; it8 < 8; ++it8)
                emit_heads<TOp>(ep, dst, rok[it8], rb[it8], rt[it8], hh, d0, stage_read(stg, it8, lane));
              __syncwarp();
            }
          } else {
            if constexpr (MODE == EPI_VT) {
#pragma unroll
              for (int j = 0; j < OC; ++j) v[j] += row_bias;
            }
            StageOp<TOp>::write(stg, lane, v);
            __syncwarp();
#pragma unroll
            for (int it8 = 0; it8 < 8; ++it8) {
              const uint4 pay = stage_read(stg, it8, lane);
              if constexpr (MODE == EPI_VT) emit_vt<TOp>(ep, mw + it8 * 4 + pr, n + pc * ONE, pay);
              else emit_pos<TOp>(ep, mw + it8 * 4 + pr, n + pc * ONE, pay);
            }
            __syncwarp();
          }
        }
      }
    }
    if constexpr (MODE == EPI_LINEAR) {
      if (splits > 1) {
        // ---- deterministic split-K fix-up ("last block reduces"): publish the partial, count arrivals per tile ----
        __threadfence();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (threadIdx.x == 128) {
          const int old = atomicAdd(ep.counters + tile, 1);
          const int last = (old == splits - 1);
          if (last) ep.counters[tile] = 0;                 // every slice has arrived: re-arm for the next launch
          *s_flag = last;
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (*s_flag) {
          __threadfence();                                 // acquire: the other slices' partial tiles are visible
          const int mw = m0 + q * 32;
#pragma unroll 1
          for (int c = cb; c < ce; c += 32) {
            const int n = n0 + c + pc * 4;
            const float4 bv = *reinterpret_cast<const float4*>(s_vec + c + pc * 4);
            // loads first (8 independent 16-byte loads in flight per slice, no store in between), stores last
            float4 a[8], t4[8];
            bool ok[8];
#pragma unroll
            for (int it8 = 0; it8 < 8; ++it8) { a[it8] = bv; ok[it8] = (mw + it8 * 4 + pr < ep.M) && (n < ep.N); }
            for (int sp = 0; sp < splits; ++sp) {        // fixed order: slice 0, 1, ... regardless of arrival order
              const float* part = ep.partial + (long)sp * ep.M * ep.ldo;
#pragma unroll
              for (int it8 = 0; it8 < 8; ++it8)
                t4[it8] = ok[it8] ? __ldcg(reinterpret_cast<const float4*>(part + (long)(mw + it8 * 4 + pr) * ep.ldo + n))
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
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
    }  // tile loop
  }
  __syncthreads();
  AVSR_TSPAN_CLOSE();
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

template <int MODE, int BN, typename TOp>
static int launch_tc(const void* A, const void* Bw, int M, int N, int K, int splits, const EpiParams& ep,
                     cudaStream_t st) {
  using Cfg = TcCfg<BN>;
  CUtensorMap tmA, tmB;
  AVSR_TRY(make_tmap_2d(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)K, TC_BM, (int)sizeof(TOp)));
  AVSR_TRY(make_tmap_2d(&tmB, Bw, (uint64_t)N, (uint64_t)K, (uint64_t)K, BN, (int)sizeof(TOp)));
  AVSR_SET_MAX_SMEM((gemm_tc_kernel<MODE, BN, TOp>), Cfg::kSmem);
  const int tiles_m = cdiv(M, TC_BM), tiles_n = cdiv(N, BN);
  if (splits > kMaxSplits || tiles_m * tiles_n > kSplitCounters) splits = 1;   // caller's workspace contract
  const int total = tiles_m * tiles_n * splits;
  const int grid = total < num_sms() ? total : num_sms();
  AVSR_LAUNCH((gemm_tc_kernel<MODE, BN, TOp>), grid, TC_THREADS, Cfg::kSmem, st, tmA, tmB, K, tiles_m, tiles_n, splits, ep);
  return AVSR_OK;
}

// ---------------------------------------------------------------- tile / split selection
// Cost model (SM cycles) of one GEMM on persistent CTAs, one per SM: the busier of the tensor pipe (dense wgmma rate
// per SM) and operand ingest (bytes the busiest SM pulls through L2, at an assumed ~64 B/cycle), plus the epilogue of
// the last item (it does not overlap the main loop of a following item: the accumulator lives in the registers of the
// warpgroups that also run the epilogue).  Split-K (only for GEMMs that accumulate into the fp32 residual stream)
// spreads a long K over more SMs.
struct TileChoice { int bn, splits; };
static const int kTileWidths[] = {64, 128};

static TileChoice choose_tile(int mode, int M, int N, int K, int esz, bool operand_dest, bool can_split) {
  const double mac_per_cycle = esz == 2 ? 2048.0 : 1024.0;   // per SM, dense f16 / tf32
  const double ingest = 64.0;                                // operand bytes per cycle per SM
  const int nkb = K / (128 / esz);
  const int sms = num_sms();
  double best = 1e30;
  TileChoice pick{128, 1};
  for (const int bn : kTileWidths) {
    if (mode == EPI_GLU && bn % 128 != 0) continue;
    if (bn == 64 && esz == 2 && (mode != EPI_LINEAR || operand_dest)) continue;   // needs 64-column row segments
    if (bn > 64 && N <= bn / 2) continue;                                          // mostly empty tile
    const long tiles = (long)cdiv(M, 128) * cdiv(N, bn);
    for (int splits = 1; splits <= (can_split ? kMaxSplits : 1); ++splits) {
      if (splits > nkb) break;
      const long items = tiles * splits;
      const long per_sm = (items + sms - 1) / sms;
      const double kfrac = (double)((nkb + splits - 1) / splits) * (128 / esz);    // K elements of the longest slice
      const double t_mma = per_sm * 128.0 * bn * kfrac / mac_per_cycle;
      const double t_in = per_sm * (128.0 + bn) * kfrac * esz / ingest;
      const double t_epi = per_sm * 128.0 * bn * 10.0 / 256.0 * 4.0;               // one item's epilogue, per item
      // fix-up: the last arriver re-reads `splits` fp32 partial tiles through the same port
      const double t_red = splits > 1 ? (double)splits * 128.0 * bn * 4.0 / ingest : 0.0;
      const double est = (t_mma > t_in ? t_mma : t_in) + t_epi + t_red + 4000.0;
      if (est < best) { best = est; pick = TileChoice{bn, splits}; }
    }
  }
  return pick;
}

template <int MODE, typename TOp>
static int dispatch_tile(TileChoice t, const void* A, const void* Bw, int M, int N, int K, const EpiParams& ep,
                         cudaStream_t st) {
  if (t.bn == 64) {
    if constexpr (MODE != EPI_GLU) return launch_tc<MODE, 64, TOp>(A, Bw, M, N, K, t.splits, ep, st);
  }
  if (t.bn == 128) return launch_tc<MODE, 128, TOp>(A, Bw, M, N, K, t.splits, ep, st);
  set_error("gemm_tc: no kernel for tile 128x%d", t.bn);
  return AVSR_E_INVALID;
}

template <typename TOp>
static int dispatch_mode(int mode, const void* A, const void* Bw, int M, int N, int K, const EpiParams& ep,
                         cudaStream_t st) {
  const bool operand_dest = mode != EPI_GLU && (mode != EPI_LINEAR || ep.round_out != 0);
  // split-K adds partial sums into the destination: only when the destination IS the residual it accumulates into.
  // Split-K needs the caller's fp32 workspace + zeroed tile counters (EpiParams::partial / counters); the slices
  // are summed in fixed order by the last-arriving CTA, so the result does not depend on scheduling.  Opt-in
  // (AVSR_B200_SPLITK=1): the fix-up re-reads `splits` fp32 tiles as a serial tail.
  static const bool allow_split = [] { const char* e = getenv("AVSR_B200_SPLITK"); return e && e[0] == '1'; }();
  const bool can_split = allow_split && mode == EPI_LINEAR && !ep.round_out && !ep.relu && ep.resid != nullptr &&
                         ep.partial != nullptr && ep.counters != nullptr;
  TileChoice t = choose_tile(mode, M, N, K, (int)sizeof(TOp), operand_dest, can_split);
  if (const char* force = getenv("AVSR_B200_TILE")) {        // "BN[,SPLITS]" -- tuning / profiling aid
    int bn = 0, sp = 1;
    const int got = sscanf(force, "%d,%d", &bn, &sp);
    if (got >= 1 && (bn == 64 || bn == 128) && (mode != EPI_GLU || bn % 128 == 0) &&
        !(bn == 64 && sizeof(TOp) == 2 && operand_dest)) {
      if (got < 2 || !can_split || sp < 1) sp = 1;
      const int nkb = K / (128 / (int)sizeof(TOp));
      t = TileChoice{bn, sp > nkb ? nkb : sp};
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
  AVSR_REQUIRE(opk == OP_TF32 || opk == OP_F16, "gemm_tc: operand kind %d", opk);
  const int ke = opk == OP_F16 ? 64 : 32;
  AVSR_REQUIRE(K >= ke && K % ke == 0, "gemm_tc: K=%d must be a multiple of %d", K, ke);
  if (M <= 0 || N <= 0) return AVSR_OK;
  if (opk == OP_F16) return dispatch_mode<__half>(mode, A, Bw, M, N, K, ep, st);
  return dispatch_mode<float>(mode, A, Bw, M, N, K, ep, st);
}

}  // namespace avsr
