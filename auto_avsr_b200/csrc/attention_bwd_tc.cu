// Backward of the rel-pos attention core on the Hopper tensor cores (wgmma): bf16 operands, fp32 accumulation.  The
// same five outputs as attention_bwd.cu (its header has the notation):
//   g_ij = A_ij (dctx_i . v_j - Delta_i) / 8 ,  Delta_i = dctx_i . ctx_i ,  table row m_ij = j - i + T - 1 ;
//   dq_k_i = sum_j g_ij k_j ,  dq_p_i = sum_j g_ij p[m_ij] ,  dk_j = sum_i g_ij (q_i + u) ,  dv_j = sum_i A_ij dctx_i ,
//   dp[m] = sum_{b, i} g_{i, j = m + i - (T-1)} (q_i + v) .
// Operands are the bf16 head-major copies (B,H,T,64) of q+u, q+v, k, v, dctx and the table (H, 2T-1, 64) that
// launch_split_heads writes (the step avsr_relpos_attention runs before its forward kernel).  Delta is fp32, from the
// fp32 ctx and dctx.  Like the fp32 kernels, the scores are recomputed tile by tile and nothing of size T^2 leaves the SM:
//   dq kernel   (h, b, 64 queries)   pass 1: S = Qu.K^T and the pre-skewed G = Qv.Pband^T (the forward's band trick:
//                                    the 127 table rows a 64 x 64 tile pair touches, one TMA box) -> the row
//                                    log-sum-exp, which goes to the workspace.  The backward computes its own from the
//                                    bf16 operands it builds A from, so A is normalised consistently whatever precision
//                                    the forward ran in.
//                                    pass 2: A, dP = dO.V^T, g -> dq_k += g.K, dq_p += g_band.Pband (K = 128), where
//                                    g_band is g skewed into the 64 x 128 band layout
//   dk/dv kernel (h, b, 64 keys)     over the query tiles: dv += A^T.dO, dk += g^T.Qu; wgmma reads both shared operands
//                                    MN-major, so A and g are stored once as [query][key] and need no transpose
//   dp kernel   (h, tile diagonal d = J - I, chunk of utterances)   over its b and I: dp_band (128 x 64) += g_band^T.Qv
//                                    as two m64 wgmmas.  Every tile pair of one diagonal has the same band (rows
//                                    64d + T - 64 ...), so the band stays in registers.  Short buckets have few
//                                    diagonals, so the utterances are split into chunks until the grid fills the SMs
//                                    (bw_dp_chunks).  Neighbouring diagonals' bands overlap by 63 rows; a fix-up kernel
//                                    sums each table row's partials in ascending (d, chunk).
// Keys j >= len[b] get A = 0; a zero-length utterance gives zero gradients; padded query rows (len <= i < T) are computed
// like any other row, rows i >= T of a tile (the next head's data) get A = 0 through an infinite log-sum-exp.  No atomics
// and every sum in a fixed order: repeated calls are bit-identical.
#include "bwd_tc_tiles.cuh"

namespace avsr {

using namespace sm90;

constexpr int BW_BAND = 128;                // table rows per tile pair (>= 2 * 64 - 1)
constexpr int BW_GLD = 64 + 4;              // fp32 row stride of the pre-skewed G tile
constexpr uint32_t BW_BB = BW_BAND * 128;   // the band: [128 rows][64 bf16]
constexpr uint32_t BW_GSK = 64 * BW_GLD * 4;
constexpr float BW_SCALE = 0.125f * 1.4426950408889634f;   // 1/sqrt(64) * log2(e): scores in log2 units

// shared-memory layouts (offsets from a 1024-aligned base; every operand tile 1024-aligned for the 128B swizzle)
struct BwDq {   // Qu, Qv, dO | K, V, Pband | g, g_band | Gsk | barriers
  static constexpr uint32_t kQu = 0, kQv = kQu + BW_TB, kO = kQv + BW_TB, kK = kO + BW_TB, kV = kK + BW_TB,
                            kPb = kV + BW_TB, kG = kPb + BW_BB, kGb = kG + BW_TB, kGsk = kGb + 2 * BW_TB,
                            kBars = kGsk + BW_GSK, kSmem = kBars + 64 + 1024;
};
struct BwKv {   // K, V | Qu, Qv, dO, Pband | A, g (or g_band for the dp kernel) | Gsk | lse, Delta of the query tile
  static constexpr uint32_t kK = 0, kV = kK + BW_TB, kQu = kV + BW_TB, kQv = kQu + BW_TB, kO = kQv + BW_TB,
                            kPb = kO + BW_TB, kA = kPb + BW_BB, kG = kA + BW_TB, kGsk = kG + BW_TB,
                            kRows = kGsk + BW_GSK, kBars = kRows + 2 * 64 * 4, kSmem = kBars + 64 + 1024;
};

// utterance chunks of the dp kernel: enough (h, diagonal, chunk) CTAs for 2 per SM on 132 SMs, each chunk non-empty;
// a function of the shape only, so the summation order is fixed
static inline void bw_dp_chunks(int B, int T, int H, int* chunks, int* per_chunk) {
  const int nd = 2 * cdiv(T, 64) - 1;
  int want = (2 * 132) / (H * nd);
  want = want < 1 ? 1 : (want > B ? B : want);
  *per_chunk = cdiv(B, want);
  *chunks = cdiv(B, *per_chunk);
}
__device__ __forceinline__ int bw_len(const int32_t* lengths, int b, int T) {
  int L = T;
  if (lengths) { L = lengths[b]; L = L < 0 ? 0 : (L > T ? T : L); }
  return L;
}

// S[64 x 64] = (Qu.K^T + shift(Qv.Pband^T)) in log2 units, in the accumulator layout: sc[4j + 2rr + e] is (row
// r0 + 8rr, key 8j + cq + e).  G column cb of row r is score column cb - 63 + r (attention_tc.cu); the skew goes through
// `gsk`, whose rows are private to a warp.
__device__ __forceinline__ void bw_scores(uint32_t qu, uint32_t qv, uint32_t kt, uint32_t pb, float* gsk, float (&sc)[32],
                                          int r0, int cq) {
  float g[64];
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    wgmma_bf16_n64(sc, bw_kdesc(qu, 64, ks), bw_kdesc(kt, 64, ks), ks != 0);
    wgmma_bf16_n128(g, bw_kdesc(qv, 64, ks), bw_kdesc(pb, BW_BAND, ks), ks != 0);
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs<32>(sc);
  wgmma_fence_regs<64>(g);
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int r = r0 + 8 * rr;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = 8 * j + cq + e - (BW_TILE - 1) + r;
        if (c >= 0 && c < BW_TILE) gsk[r * BW_GLD + c] = g[4 * j + 2 * rr + e];
      }
    }
  }
  __syncwarp();
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const float* grow = gsk + (r0 + 8 * rr) * BW_GLD;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 gg = *reinterpret_cast<const float2*>(grow + 8 * j + cq);
      sc[4 * j + 2 * rr] = (sc[4 * j + 2 * rr] + gg.x) * BW_SCALE;
      sc[4 * j + 2 * rr + 1] = (sc[4 * j + 2 * rr + 1] + gg.y) * BW_SCALE;
    }
  }
  __syncwarp();   // this warp's reads of gsk are done before its next writes
}

// sc (log2 scores) -> A, dp (dO.V^T) -> g, with keys j0 + c >= L masked; lse2 / dl: this thread's two rows
__device__ __forceinline__ void bw_probs(float (&sc)[32], float (&dp)[32], const float (&lse2)[2], const float (&dl)[2],
                                         int j0, int L, int cq) {
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int x = 4 * j + 2 * rr + e;
        const float a = (j0 + 8 * j + cq + e < L) ? exp2f(sc[x] - lse2[rr]) : 0.f;
        sc[x] = a;
        dp[x] = a * (dp[x] - dl[rr]) * 0.125f;
      }
}

// g -> g_band: g_band[r][c + 63 - r] = g[r][c].  Every tile writes the same positions; the rest stays zero.
__device__ __forceinline__ void bw_store_band(uint8_t* band, const float (&g)[32], int r0, int cq) {
#pragma unroll
  for (int rr = 0; rr < 2; ++rr)
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int r = r0 + 8 * rr;
        *reinterpret_cast<__nv_bfloat16*>(band + bw_off(r, 8 * j + cq + e + BW_TILE - 1 - r)) =
            __float2bfloat16_rn(g[4 * j + 2 * rr + e]);
      }
}
// ---------------------------------------------------------------- Delta_i = dctx_i . ctx_i (fp32), one warp per (b, t, h)
__global__ void attn_bwd_tc_delta_kernel(const float* __restrict__ ctx, const float* __restrict__ dctx,
                                         float* __restrict__ delta, int B, int T, int H) {
  const long w = (blockIdx.x * (long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (long)B * T * H) return;
  const int h = (int)(w % H);
  const long bt = w / H;
  const long o = bt * H * kHeadDim + h * kHeadDim;
  float s = ctx[o + lane] * dctx[o + lane];
  s = fmaf(ctx[o + lane + 32], dctx[o + lane + 32], s);
  s = warp_sum(s);
  const int b = (int)(bt / T), t = (int)(bt % T);
  if (lane == 0) delta[((long)b * H + h) * T + t] = s;
}

// ---------------------------------------------------------------- dq (and the row log-sum-exp)
__global__ void __launch_bounds__(BW_THREADS, 2) attn_bwd_tc_dq_kernel(
    const __grid_constant__ CUtensorMap tmQu, const __grid_constant__ CUtensorMap tmQv,
    const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
    const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmP, const int32_t* __restrict__ lengths,
    const float* __restrict__ delta, float* __restrict__ lse, float* __restrict__ dq_k, float* __restrict__ dq_p, int T,
    int H) {
  using S = BwDq;
  extern __shared__ uint8_t bw_smem_raw[];
  const uint32_t raw = smem_u32(bw_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gen = bw_smem_raw + (base - raw);
  const uint32_t q_full = base + S::kBars, kv_full = q_full + 8;
  float* gsk = reinterpret_cast<float*>(gen + S::kGsk);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.x, b = blockIdx.y, i0 = blockIdx.z * BW_TILE;
  const int bh = b * H + h;
  const int L = bw_len(lengths, b, T);
  const int nkt = (L + BW_TILE - 1) / BW_TILE;
  if (threadIdx.x == 0) {
    mbar_init(q_full, 1); mbar_init(kv_full, 1);
    fence_barrier_init();
  }
  bw_zero(gen + S::kGb, 2 * BW_TB);
  __syncthreads();
  const int r0 = 16 * warp + (lane >> 2), cq = 2 * (lane & 3);
  float dl[2];
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int i = i0 + r0 + 8 * rr;
    dl[rr] = i < T ? delta[(long)bh * T + i] : 0.f;
  }
  if (nkt > 0 && threadIdx.x == 0) {
    mbar_expect_tx(q_full, 3 * BW_TB);
    tma_load_2d(base + S::kQu, &tmQu, 0, bh * T + i0, q_full);
    tma_load_2d(base + S::kQv, &tmQv, 0, bh * T + i0, q_full);
    tma_load_2d(base + S::kO, &tmO, 0, bh * T + i0, q_full);
  }
  if (nkt > 0) mbar_wait(q_full, 0);
  uint32_t phase = 0;

  // pass 1: online max / sum of the rows
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
#pragma unroll 1
  for (int it = 0; it < nkt; ++it) {
    const int j0 = it * BW_TILE;
    if (threadIdx.x == 0) {
      mbar_expect_tx(kv_full, BW_TB + BW_BB);
      tma_load_2d(base + S::kK, &tmK, 0, bh * T + j0, kv_full);
      tma_load_3d(base + S::kPb, &tmP, 0, j0 - i0 - (BW_TILE - 1) + T - 1, h, kv_full);
    }
    mbar_wait(kv_full, phase);
    phase ^= 1;
    float sc[32];
    bw_scores(base + S::kQu, base + S::kQv, base + S::kK, base + S::kPb, gsk, sc, r0, cq);
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      float mx = m_run[rr];
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& s = sc[4 * j + 2 * rr + e];
          if (j0 + 8 * j + cq + e >= L) s = -INFINITY;
          mx = fmaxf(mx, s);
        }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      float l = l_run[rr] * exp2f(m_run[rr] - mx);   // first tile: exp2(-inf) = 0; every tile holds >= 1 valid key
#pragma unroll
      for (int j = 0; j < 8; ++j) l += exp2f(sc[4 * j + 2 * rr] - mx) + exp2f(sc[4 * j + 2 * rr + 1] - mx);
      m_run[rr] = mx;
      l_run[rr] = l;
    }
    __syncthreads();   // every warp is done with K and the band before the next load
  }
  float lse2[2];
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    float l = l_run[rr];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    lse2[rr] = L > 0 ? m_run[rr] + log2f(l) : INFINITY;   // len 0: every A is 0
    const int i = i0 + r0 + 8 * rr;
    if ((lane & 3) == 0 && i < T) lse[(long)bh * T + i] = lse2[rr];
  }

  // pass 2: A, g and the two parts of dq
  float ak[32], ap[32];
#pragma unroll
  for (int x = 0; x < 32; ++x) ak[x] = ap[x] = 0.f;
#pragma unroll 1
  for (int it = 0; it < nkt; ++it) {
    const int j0 = it * BW_TILE;
    if (threadIdx.x == 0) {
      mbar_expect_tx(kv_full, 2 * BW_TB + BW_BB);
      tma_load_2d(base + S::kK, &tmK, 0, bh * T + j0, kv_full);
      tma_load_2d(base + S::kV, &tmV, 0, bh * T + j0, kv_full);
      tma_load_3d(base + S::kPb, &tmP, 0, j0 - i0 - (BW_TILE - 1) + T - 1, h, kv_full);
    }
    mbar_wait(kv_full, phase);
    phase ^= 1;
    float sc[32], dp[32];
    bw_scores(base + S::kQu, base + S::kQv, base + S::kK, base + S::kPb, gsk, sc, r0, cq);
    bw_dprod(base + S::kO, base + S::kV, dp);
    bw_probs(sc, dp, lse2, dl, j0, L, cq);
    bw_store_tile(gen + S::kG, dp, r0, cq);
    bw_store_band(gen + S::kGb, dp, r0, cq);
    fence_proxy_async();   // generic-proxy smem writes -> visible to the tensor core
    __syncthreads();
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma_bf16_n64_bmn(ak, bw_kdesc(base + S::kG, 64, ks), bw_mdesc(base + S::kK, ks), 1);
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) wgmma_bf16_n64_bmn(ap, bw_kdesc(base + S::kGb, 64, ks), bw_mdesc(base + S::kPb, ks), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<32>(ak);
    wgmma_fence_regs<32>(ap);
    __syncthreads();   // K, V, the band, g and g_band are free for the next tile
  }
  const long D = (long)H * kHeadDim;
  const long o = ((long)b * T + i0) * D + h * kHeadDim;
  bw_store_out(dq_k + o, D, ak, r0, cq, T - i0);
  bw_store_out(dq_p + o, D, ap, r0, cq, T - i0);
}

// ---------------------------------------------------------------- dk, dv
__global__ void __launch_bounds__(BW_THREADS, 2) attn_bwd_tc_dkdv_kernel(
    const __grid_constant__ CUtensorMap tmQu, const __grid_constant__ CUtensorMap tmQv,
    const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
    const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmP, const int32_t* __restrict__ lengths,
    const float* __restrict__ lse, const float* __restrict__ delta, float* __restrict__ dk, float* __restrict__ dv, int T,
    int H) {
  using S = BwKv;
  extern __shared__ uint8_t bw_smem_raw[];
  const uint32_t raw = smem_u32(bw_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gen = bw_smem_raw + (base - raw);
  const uint32_t kv_full = base + S::kBars, q_full = kv_full + 8;
  float* gsk = reinterpret_cast<float*>(gen + S::kGsk);
  float* srow = reinterpret_cast<float*>(gen + S::kRows);   // [0, 64): lse, [64, 128): Delta of the query tile
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.x, b = blockIdx.y, j0 = blockIdx.z * BW_TILE;
  const int bh = b * H + h;
  const int L = bw_len(lengths, b, T);
  const long D = (long)H * kHeadDim;
  const long o = ((long)b * T + j0) * D + h * kHeadDim;
  const int r0 = 16 * warp + (lane >> 2), cq = 2 * (lane & 3);
  float ak[32], av[32];
#pragma unroll
  for (int x = 0; x < 32; ++x) ak[x] = av[x] = 0.f;
  if (j0 < L) {            // CTA-uniform: a tile without a valid key received no probability (zeros)
    if (threadIdx.x == 0) {
      mbar_init(kv_full, 1); mbar_init(q_full, 1);
      fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      mbar_expect_tx(kv_full, 2 * BW_TB);
      tma_load_2d(base + S::kK, &tmK, 0, bh * T + j0, kv_full);
      tma_load_2d(base + S::kV, &tmV, 0, bh * T + j0, kv_full);
    }
    mbar_wait(kv_full, 0);
    uint32_t phase = 0;
    const int nqt = (T + BW_TILE - 1) / BW_TILE;
#pragma unroll 1
    for (int qt = 0; qt < nqt; ++qt) {
      const int i0 = qt * BW_TILE;
      if (threadIdx.x < BW_TILE) {
        const int i = i0 + threadIdx.x;
        srow[threadIdx.x] = i < T ? lse[(long)bh * T + i] : INFINITY;   // rows past T: A = 0
        srow[BW_TILE + threadIdx.x] = i < T ? delta[(long)bh * T + i] : 0.f;
      }
      if (threadIdx.x == 0) {
        mbar_expect_tx(q_full, 3 * BW_TB + BW_BB);
        tma_load_2d(base + S::kQu, &tmQu, 0, bh * T + i0, q_full);
        tma_load_2d(base + S::kQv, &tmQv, 0, bh * T + i0, q_full);
        tma_load_2d(base + S::kO, &tmO, 0, bh * T + i0, q_full);
        tma_load_3d(base + S::kPb, &tmP, 0, j0 - i0 - (BW_TILE - 1) + T - 1, h, q_full);
      }
      mbar_wait(q_full, phase);
      phase ^= 1;
      __syncthreads();   // srow
      float sc[32], dp[32];
      bw_scores(base + S::kQu, base + S::kQv, base + S::kK, base + S::kPb, gsk, sc, r0, cq);
      bw_dprod(base + S::kO, base + S::kV, dp);
      const float lse2[2] = {srow[r0], srow[r0 + 8]}, dl[2] = {srow[BW_TILE + r0], srow[BW_TILE + r0 + 8]};
      bw_probs(sc, dp, lse2, dl, j0, L, cq);
      bw_store_tile(gen + S::kA, sc, r0, cq);
      bw_store_tile(gen + S::kG, dp, r0, cq);
      fence_proxy_async();
      __syncthreads();
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        wgmma_bf16_n64_amn_bmn(av, bw_mdesc(base + S::kA, ks), bw_mdesc(base + S::kO, ks), 1);
        wgmma_bf16_n64_amn_bmn(ak, bw_mdesc(base + S::kG, ks), bw_mdesc(base + S::kQu, ks), 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs<32>(av);
      wgmma_fence_regs<32>(ak);
      __syncthreads();   // the query tile, the band, A, g and srow are free for the next tile
    }
  }
  bw_store_out(dk + o, D, ak, r0, cq, T - j0);
  bw_store_out(dv + o, D, av, r0, cq, T - j0);
}

// ---------------------------------------------------------------- dp: band partials per (h, tile diagonal)
__global__ void __launch_bounds__(BW_THREADS, 2) attn_bwd_tc_dp_kernel(
    const __grid_constant__ CUtensorMap tmQu, const __grid_constant__ CUtensorMap tmQv,
    const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
    const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmP, const int32_t* __restrict__ lengths,
    const float* __restrict__ lse, const float* __restrict__ delta, float* __restrict__ part, int B, int T, int H,
    int per_chunk) {
  using S = BwKv;
  extern __shared__ uint8_t bw_smem_raw[];
  const uint32_t raw = smem_u32(bw_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gen = bw_smem_raw + (base - raw);
  const uint32_t pb_full = base + S::kBars, t_full = pb_full + 8;
  float* gsk = reinterpret_cast<float*>(gen + S::kGsk);
  float* srow = reinterpret_cast<float*>(gen + S::kRows);
  const uint32_t kGb = S::kA;                                // g_band: the A and g slots, [64][128]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.x, nT = (T + BW_TILE - 1) / BW_TILE, di = blockIdx.y, dd = di - (nT - 1);
  const int r0 = 16 * warp + (lane >> 2), cq = 2 * (lane & 3);
  if (threadIdx.x == 0) {
    mbar_init(pb_full, 1); mbar_init(t_full, 1);
    fence_barrier_init();
  }
  bw_zero(gen + kGb, 2 * BW_TB);
  __syncthreads();
  if (threadIdx.x == 0) {                                    // the band is the same for every tile pair of the diagonal
    mbar_expect_tx(pb_full, BW_BB);
    tma_load_3d(base + S::kPb, &tmP, 0, BW_TILE * dd + T - BW_TILE, h, pb_full);
  }
  mbar_wait(pb_full, 0);
  float da[32], db[32];                                      // band rows [0, 64) and [64, 128)
#pragma unroll
  for (int x = 0; x < 32; ++x) da[x] = db[x] = 0.f;
  uint32_t phase = 0;
  const int qlo = dd < 0 ? -dd : 0, qhi = dd > 0 ? nT - dd : nT;
#pragma unroll 1
  const int b_lo = blockIdx.z * per_chunk, b_hi = b_lo + per_chunk < B ? b_lo + per_chunk : B;
  for (int b = b_lo; b < b_hi; ++b) {
    const int L = bw_len(lengths, b, T);
    const int bh = b * H + h;
#pragma unroll 1
    for (int qt = qlo; qt < qhi; ++qt) {
      const int i0 = qt * BW_TILE, j0 = (qt + dd) * BW_TILE;
      if (j0 >= L) continue;                                 // CTA-uniform: no valid key, g = 0
      if (threadIdx.x < BW_TILE) {
        const int i = i0 + threadIdx.x;
        srow[threadIdx.x] = i < T ? lse[(long)bh * T + i] : INFINITY;
        srow[BW_TILE + threadIdx.x] = i < T ? delta[(long)bh * T + i] : 0.f;
      }
      if (threadIdx.x == 0) {
        mbar_expect_tx(t_full, 5 * BW_TB);
        tma_load_2d(base + S::kQu, &tmQu, 0, bh * T + i0, t_full);
        tma_load_2d(base + S::kQv, &tmQv, 0, bh * T + i0, t_full);
        tma_load_2d(base + S::kO, &tmO, 0, bh * T + i0, t_full);
        tma_load_2d(base + S::kK, &tmK, 0, bh * T + j0, t_full);
        tma_load_2d(base + S::kV, &tmV, 0, bh * T + j0, t_full);
      }
      mbar_wait(t_full, phase);
      phase ^= 1;
      __syncthreads();
      float sc[32], dp[32];
      bw_scores(base + S::kQu, base + S::kQv, base + S::kK, base + S::kPb, gsk, sc, r0, cq);
      bw_dprod(base + S::kO, base + S::kV, dp);
      const float lse2[2] = {srow[r0], srow[r0 + 8]}, dl[2] = {srow[BW_TILE + r0], srow[BW_TILE + r0 + 8]};
      bw_probs(sc, dp, lse2, dl, j0, L, cq);
      bw_store_band(gen + kGb, dp, r0, cq);
      fence_proxy_async();
      __syncthreads();
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        wgmma_bf16_n64_amn_bmn(da, bw_mdesc(base + kGb, ks), bw_mdesc(base + S::kQv, ks), 1);
        wgmma_bf16_n64_amn_bmn(db, bw_mdesc(base + kGb + BW_TB, ks), bw_mdesc(base + S::kQv, ks), 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs<32>(da);
      wgmma_fence_regs<32>(db);
      __syncthreads();
    }
  }
  float* dst = part + (((long)h * (2 * nT - 1) + di) * gridDim.z + blockIdx.z) * BW_BAND * kHeadDim;
  bw_store_out(dst, kHeadDim, da, r0, cq, BW_TILE);
  bw_store_out(dst + BW_TILE * kHeadDim, kHeadDim, db, r0, cq, BW_TILE);
}

// dp[m] = the band partials that hold table row m, in ascending (diagonal, chunk) order.  Diagonal index di covers the
// rows m = 64 di + T - 64 nT + r, r in [0, 127): at most two of them hold a given m.
__global__ void attn_bwd_tc_dp_fixup_kernel(const float* __restrict__ part, float* __restrict__ dp, int T, int H,
                                            int chunks) {
  const int nT = (T + BW_TILE - 1) / BW_TILE, nd = 2 * nT - 1;
  const long D = (long)H * kHeadDim, total = (long)(2 * T - 1) * D;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int m = (int)(idx / D), c = (int)(idx % D), h = c / kHeadDim, d = c % kHeadDim;
    const int off = m + BW_TILE * nT - T;                    // >= 0
    const int hi = off / BW_TILE;
    float s = 0.f;
    for (int di = hi > 0 ? hi - 1 : 0; di <= hi && di < nd; ++di) {
      const int r = off - BW_TILE * di;
      if (r < 2 * BW_TILE - 1)
        for (int z = 0; z < chunks; ++z) s += part[((((long)h * nd + di) * chunks + z) * BW_BAND + r) * kHeadDim + d];
    }
    dp[idx] = s;
  }
}

// workspace: bf16 head-major operands, lse and Delta (B,H,T), band partials (H, 2nT - 1, chunks, 128, 64)
struct BwTcWork {
  __nv_bfloat16 *qu, *qv, *kk, *vv, *dO, *pos;
  float *lse, *delta, *part;
  size_t bytes;
};
static BwTcWork bwtc_layout(void* ws, int B, int T, int H) {
  const size_t N = (size_t)B * T, D = (size_t)H * kHeadDim, R = 2 * (size_t)T - 1;
  const size_t nd = 2 * (size_t)cdiv(T, BW_TILE) - 1;
  int chunks, per_chunk;
  bw_dp_chunks(B, T, H, &chunks, &per_chunk);
  Carver cv{reinterpret_cast<char*>(ws)};
  BwTcWork w;
  w.qu = cv.take<__nv_bfloat16>(N * D);
  w.qv = cv.take<__nv_bfloat16>(N * D);
  w.kk = cv.take<__nv_bfloat16>(N * D);
  w.vv = cv.take<__nv_bfloat16>(N * D);
  w.dO = cv.take<__nv_bfloat16>(N * D);
  w.pos = cv.take<__nv_bfloat16>(R * D);
  w.lse = cv.take((size_t)B * H * T);
  w.delta = cv.take((size_t)B * H * T);
  w.part = cv.take((size_t)H * nd * chunks * BW_BAND * kHeadDim);
  w.bytes = cv.off;
  return w;
}

}  // namespace avsr

using namespace avsr;

extern "C" {

size_t avsr_relpos_attention_bwd_tc_workspace_bytes(int B, int T, int H, int precision) {
  if (precision != AVSR_PREC_BF16) return 0;
  if (B <= 0 || T <= 0 || H <= 0) return 256;
  return bwtc_layout(nullptr, B, T, H).bytes;
}

int avsr_relpos_attention_bwd_tc(const float* q, const float* k, const float* v, const float* p, const float* pos_bias_u,
                                 const float* pos_bias_v, const int32_t* lengths, const float* ctx, const float* dctx,
                                 float* dq_k, float* dq_p, float* dk, float* dv, float* dp, int B, int T, int H,
                                 int precision, void* workspace, size_t workspace_bytes, void* stream) {
  AVSR_REQUIRE(q && k && v && p && pos_bias_u && pos_bias_v && ctx && dctx && dq_k && dq_p && dk && dv && dp && workspace,
               "NULL argument");
  AVSR_REQUIRE(precision == AVSR_PREC_BF16,
               "attention backward (tensor cores): precision %d (%s) is not built; AVSR_PREC_BF16 only", precision,
               precision_name(precision));
  if (B <= 0 || T <= 0) return AVSR_OK;
  AVSR_REQUIRE(H > 0, "attention backward (tensor cores): bad H=%d", H);
  AVSR_REQUIRE_BYTES(avsr_relpos_attention_bwd_tc_workspace_bytes(B, T, H, precision), workspace_bytes,
                     "attention backward (tensor cores) workspace");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const BwTcWork w = bwtc_layout(workspace, B, T, H);
  const int R = 2 * T - 1, nT = cdiv(T, BW_TILE);
  AVSR_TRY(launch_split_heads(q, pos_bias_u, w.qu, B, T, H, T, 0, OP_BF16, st));
  AVSR_TRY(launch_split_heads(q, pos_bias_v, w.qv, B, T, H, T, 0, OP_BF16, st));
  AVSR_TRY(launch_split_heads(k, nullptr, w.kk, B, T, H, T, 0, OP_BF16, st));
  AVSR_TRY(launch_split_heads(v, nullptr, w.vv, B, T, H, T, 0, OP_BF16, st));
  AVSR_TRY(launch_split_heads(dctx, nullptr, w.dO, B, T, H, T, 0, OP_BF16, st));
  AVSR_TRY(launch_split_heads(p, nullptr, w.pos, 1, R, H, R, 0, OP_BF16, st));
  const long warps = (long)B * T * H;
  attn_bwd_tc_delta_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(ctx, dctx, w.delta, B, T, H);
  AVSR_CHECK_LAUNCH();

  CUtensorMap tmQu, tmQv, tmK, tmV, tmO, tmP;
  const uint64_t rows = (uint64_t)B * H * T;
  AVSR_TRY(make_tmap_2d(&tmQu, w.qu, rows, 64, 64, BW_TILE, OP_BF16));
  AVSR_TRY(make_tmap_2d(&tmQv, w.qv, rows, 64, 64, BW_TILE, OP_BF16));
  AVSR_TRY(make_tmap_2d(&tmK, w.kk, rows, 64, 64, BW_TILE, OP_BF16));
  AVSR_TRY(make_tmap_2d(&tmV, w.vv, rows, 64, 64, BW_TILE, OP_BF16));
  AVSR_TRY(make_tmap_2d(&tmO, w.dO, rows, 64, 64, BW_TILE, OP_BF16));
  AVSR_TRY(make_tmap_3d(&tmP, w.pos, (uint64_t)H, (uint64_t)R, 64, 64, (uint64_t)R * 64, BW_BAND, OP_BF16));

  AVSR_SET_MAX_SMEM(attn_bwd_tc_dq_kernel, BwDq::kSmem);
  attn_bwd_tc_dq_kernel<<<dim3(H, B, nT), BW_THREADS, BwDq::kSmem, st>>>(tmQu, tmQv, tmK, tmV, tmO, tmP, lengths, w.delta,
                                                                         w.lse, dq_k, dq_p, T, H);
  AVSR_CHECK_LAUNCH();
  AVSR_SET_MAX_SMEM(attn_bwd_tc_dkdv_kernel, BwKv::kSmem);
  attn_bwd_tc_dkdv_kernel<<<dim3(H, B, nT), BW_THREADS, BwKv::kSmem, st>>>(tmQu, tmQv, tmK, tmV, tmO, tmP, lengths, w.lse,
                                                                           w.delta, dk, dv, T, H);
  AVSR_CHECK_LAUNCH();
  int chunks, per_chunk;
  bw_dp_chunks(B, T, H, &chunks, &per_chunk);
  AVSR_SET_MAX_SMEM(attn_bwd_tc_dp_kernel, BwKv::kSmem);
  attn_bwd_tc_dp_kernel<<<dim3(H, 2 * nT - 1, chunks), BW_THREADS, BwKv::kSmem, st>>>(
      tmQu, tmQv, tmK, tmV, tmO, tmP, lengths, w.lse, w.delta, w.part, B, T, H, per_chunk);
  AVSR_CHECK_LAUNCH();
  attn_bwd_tc_dp_fixup_kernel<<<132 * 4, 256, 0, st>>>(w.part, dp, T, H, chunks);
  AVSR_CHECK_LAUNCH();
  return AVSR_OK;
}

}  // extern "C"
