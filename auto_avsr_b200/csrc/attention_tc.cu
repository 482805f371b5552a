// Fused rel-pos flash attention on the Hopper tensor cores (wgmma, fp32 accumulate), TF32 or fp16 operands.
//
//   scores[i,j] = ((q_i+u).k_j + (q_i+v).p[rel=i-j]) / 8 ;  keys j >= len[b] masked ;  ctx = softmax_j(scores) @ v
// (transformer/attention.py:174-189 + :59-82 of the reference).  The reference materialises the (T x 2T-1) product
// (q+v) P^T in HBM and re-lays it out with the pad/view "rel_shift" copy; here nothing of size T^2 ever leaves the SM.
//
// One CTA = one warpgroup = one (head h, utterance b, 64-query tile).  Per 64-key tile:
//   wgmma  S [64 x  64] = Qu . K_tile^T          (registers)
//   wgmma  G [64 x 128] = Qv . Pband^T           (registers, then shared memory)
//          Pband = the 127 table rows m = j-i+T-1 this (query tile, key tile) pair can touch -- a BAND of the rel-pos
//          table fetched by one TMA box; score (r, c) needs G[r][c + 63 - r]: the rel_shift is a per-row skew, read
//          from the fp32 copy of G in shared memory at the positions of this thread's S fragment.
//   softmax in the accumulator layout (the 4 threads of a quad share a row): scale, key mask, online max / sum
//          (exp2), rescale of the O accumulator, P -> shared memory in the K-major SWIZZLE_128B layout
//   wgmma  O [64 x 64] += P . V_tile             (registers)
// TF32: V arrives as v^T (B,H,64,Tp), K-major.  fp16: V keeps its natural (B,H,T,64) layout (MN-major B operand).
// Padded QUERY rows are computed like any other row (the reference masks keys only).
#include "common.cuh"
#include "sm90.cuh"

namespace avsr {

using namespace sm90;

constexpr int AT_BQ = 64;     // queries per CTA (= wgmma M)
constexpr int AT_BKV = 64;    // keys per tile
constexpr int AT_BAND = 128;  // rel-pos rows per tile (>= BQ + BKV - 1)
constexpr int AT_THREADS = 128;
constexpr int AT_GS = AT_BAND + 8;   // fp32 row stride of the G copy (8-byte aligned rows, skewed reads spread banks)

template <typename TOp>
struct AtCfg {
  static constexpr int kAtoms = 64 * (int)sizeof(TOp) / 128;   // 128-byte atoms along a 64-wide row (2 tf32 / 1 f16)
  static constexpr int kSteps = 64 * (int)sizeof(TOp) / 32;    // MMA-K steps over 64 elements
  static constexpr int kQu = 0;
  static constexpr int kQv = kQu + AT_BQ * 128 * kAtoms;
  static constexpr int kK = kQv + AT_BQ * 128 * kAtoms;
  static constexpr int kV = kK + AT_BKV * 128 * kAtoms;        // tf32: [64 d][64 keys]; f16: [64 keys][64 d]
  static constexpr int kPb = kV + 64 * 128 * kAtoms;
  static constexpr int kP = kPb + AT_BAND * 128 * kAtoms;
  static constexpr int kG = kP + AT_BQ * 128 * kAtoms;
  static constexpr int kBars = kG + AT_BQ * AT_GS * 4;
  static constexpr int kSmem = kBars + 64 + 1024;
  static constexpr uint32_t kTileBytes = (AT_BKV + AT_BAND + 64) * 128 * kAtoms;
};

// MMA-K step ks of a [ROWS][64 elements] K-major tile stored as kAtoms atoms of [ROWS][128 B]
template <typename TOp>
__device__ __forceinline__ uint64_t at_desc(uint32_t tile, int rows, int ks) {
  const int bytes = ks * 32;
  return wgmma_desc_sw128(tile + (bytes >> 7) * (rows * 128) + (bytes & 127));
}

template <typename TOp>
__global__ void __launch_bounds__(AT_THREADS, 1)
attention_wg_kernel(const __grid_constant__ CUtensorMap tmQu, const __grid_constant__ CUtensorMap tmQv,
                    const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                    const __grid_constant__ CUtensorMap tmP, const int32_t* __restrict__ lengths, TOp* __restrict__ ctx,
                    int T, int H, int round_out) {
  using Cfg = AtCfg<TOp>;
  constexpr bool kF16 = sizeof(TOp) == 2;
  extern __shared__ uint8_t at_smem_raw[];
  const uint32_t raw = smem_u32(at_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gen = at_smem_raw + (base - raw);
  const uint32_t q_full = base + Cfg::kBars, kv_full = q_full + 8;
  float* gs = reinterpret_cast<float*>(gen + Cfg::kG);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // grid = (H, B, query tiles): the query tile is the SLOWEST block index, so the partially filled last tile of every
  // utterance is scheduled last
  const int h = blockIdx.x, b = blockIdx.y, i0 = blockIdx.z * AT_BQ;
  const int bh = b * H + h;
  pdl_launch_dependents();
  int L = T;
  if (lengths) { L = lengths[b]; L = L < 0 ? 0 : (L > T ? T : L); }   // lengths: written before the graph, not by the predecessor
  const int nkt = (L + AT_BKV - 1) / AT_BKV;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQu); tma_prefetch_desc(&tmQv); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmP);
    mbar_init(q_full, 1); mbar_init(kv_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  // this thread's accumulator rows r0, r0 + 8 and first column cq of every 8-column block
  const int r0 = 16 * warp + (lane >> 2), cq = 2 * (lane & 3);
  const float kScale = 0.125f * 1.4426950408889634f;   // 1/sqrt(64) * log2(e)
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  if (nkt > 0 && threadIdx.x == 0) {
    mbar_expect_tx(q_full, 2 * AT_BQ * 128 * Cfg::kAtoms);
#pragma unroll
    for (int a = 0; a < Cfg::kAtoms; ++a) {
      tma_load_2d(base + Cfg::kQu + a * AT_BQ * 128, &tmQu, a * 32, bh * T + i0, q_full);
      tma_load_2d(base + Cfg::kQv + a * AT_BQ * 128, &tmQv, a * 32, bh * T + i0, q_full);
    }
  }
  for (int it = 0; it < nkt; ++it) {
    const int j0 = it * AT_BKV;
    if (it > 0) __syncthreads();                 // every warp's P.V(it-1) retired: K, Pband, V, P are free
    if (threadIdx.x == 0) {
      mbar_expect_tx(kv_full, Cfg::kTileBytes);
      const int m_lo = j0 - i0 - (AT_BQ - 1) + T - 1;   // first table row of the band (may be < 0: zero fill)
#pragma unroll
      for (int a = 0; a < Cfg::kAtoms; ++a) {
        tma_load_2d(base + Cfg::kK + a * AT_BKV * 128, &tmK, a * 32, bh * T + j0, kv_full);
        tma_load_3d(base + Cfg::kPb + a * AT_BAND * 128, &tmP, a * 32, m_lo, h, kv_full);
        if constexpr (kF16) tma_load_2d(base + Cfg::kV, &tmV, 0, bh * T + j0, kv_full);
        else tma_load_2d(base + Cfg::kV + a * 64 * 128, &tmV, j0 + a * 32, bh * 64, kv_full);
      }
    }
    if (it == 0) mbar_wait(q_full, 0);
    mbar_wait(kv_full, it & 1);

    float s[32], g[64];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < Cfg::kSteps; ++ks) {
      const uint64_t dq = at_desc<TOp>(base + Cfg::kQu, AT_BQ, ks), dk = at_desc<TOp>(base + Cfg::kK, AT_BKV, ks);
      const uint64_t dv = at_desc<TOp>(base + Cfg::kQv, AT_BQ, ks), dp = at_desc<TOp>(base + Cfg::kPb, AT_BAND, ks);
      if constexpr (kF16) { wgmma_f16_n64(s, dq, dk, ks != 0); wgmma_f16_n128(g, dv, dp, ks != 0); }
      else { wgmma_tf32_n64(s, dq, dk, ks != 0); wgmma_tf32_n128(g, dv, dp, ks != 0); }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<32>(s);
    wgmma_fence_regs<64>(g);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      *reinterpret_cast<float2*>(gs + r0 * AT_GS + 8 * j + cq) = make_float2(g[4 * j], g[4 * j + 1]);
      *reinterpret_cast<float2*>(gs + (r0 + 8) * AT_GS + 8 * j + cq) = make_float2(g[4 * j + 2], g[4 * j + 3]);
    }
    __syncthreads();
    // scores in the S fragment: s[4j + 2rr + e] is (row r0 + 8rr, key j0 + 8j + cq + e)
    float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int r = r0 + 8 * rr;
      const float* grow = gs + r * AT_GS + (AT_BQ - 1) - r;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * j + cq + e;
          const float v = (s[4 * j + 2 * rr + e] + grow[c]) * kScale;
          s[4 * j + 2 * rr + e] = (j0 + c < L) ? v : -INFINITY;
          mx[rr] = fmaxf(mx[rr], s[4 * j + 2 * rr + e]);
        }
      }
      mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 1));
      mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 2));
    }
    float alpha[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      alpha[rr] = exp2f(m_run[rr] - mx[rr]);     // first tile: exp2(-inf) = 0; every tile holds >= 1 valid key
      m_run[rr] = mx[rr];
      l_run[rr] *= alpha[rr];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[4 * j] *= alpha[0]; o[4 * j + 1] *= alpha[0];
      o[4 * j + 2] *= alpha[1]; o[4 * j + 3] *= alpha[1];
    }
    // P -> shared memory, K-major SWIZZLE_128B: 16-byte chunk index XOR (row & 7)
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int r = r0 + 8 * rr;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float p0 = exp2f(s[4 * j + 2 * rr] - mx[rr]);
        const float p1 = exp2f(s[4 * j + 2 * rr + 1] - mx[rr]);
        l_run[rr] += p0 + p1;
        if constexpr (kF16) {
          *reinterpret_cast<uint32_t*>(gen + Cfg::kP + r * 128 + ((j ^ (r & 7)) << 4) + cq * 2) = pack_half2_sat(p0, p1);
        } else {
          const int atom = j >> 2, chunk = 2 * (j & 3) + (cq >> 2);
          *reinterpret_cast<float2*>(gen + Cfg::kP + atom * (AT_BQ * 128) + r * 128 + ((chunk ^ (r & 7)) << 4) +
                                     (cq & 3) * 4) = make_float2(round_tf32(p0), round_tf32(p1));
        }
      }
    }
    fence_proxy_async();      // generic-proxy smem writes -> visible to the tensor core (async proxy)
    __syncthreads();
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < Cfg::kSteps; ++ks) {
      const uint64_t dp = at_desc<TOp>(base + Cfg::kP, AT_BQ, ks);
      if constexpr (kF16) wgmma_f16_n64_bmn(o, dp, wgmma_desc_sw128(base + Cfg::kV + ks * 16 * 128), 1);
      else wgmma_tf32_n64(o, dp, at_desc<TOp>(base + Cfg::kV, 64, ks), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<32>(o);
  }
  // O / l -> ctx (B*T, H*64); rows beyond T are not stored
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    float l = l_run[rr];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = l > 0.f ? 1.0f / l : 0.f;   // len == 0: zeros, like softmax(...).masked_fill(mask, 0)
    const int i = i0 + r0 + 8 * rr;
    if (i < T) {
      TOp* dst = ctx + ((long)b * T + i) * (H * kHeadDim) + h * kHeadDim;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float a = o[4 * j + 2 * rr] * inv, c = o[4 * j + 2 * rr + 1] * inv;
        if constexpr (kF16) {
          *reinterpret_cast<uint32_t*>(dst + 8 * j + cq) = pack_half2_sat(a, c);
        } else {
          if (round_out) { a = round_tf32(a); c = round_tf32(c); }
          *reinterpret_cast<float2*>(dst + 8 * j + cq) = make_float2(a, c);
        }
      }
    }
  }
}

template <typename TOp>
static int attention_wg(const TOp* qu, const TOp* qv, const TOp* kk, const TOp* v, const TOp* pos,
                        const int32_t* lengths, TOp* ctx, int B, int T, int H, int Tp, int Rp, int round_out,
                        cudaStream_t st) {
  using Cfg = AtCfg<TOp>;
  constexpr int esz = (int)sizeof(TOp);
  CUtensorMap tmQu, tmQv, tmK, tmV, tmP;
  const uint64_t rows = (uint64_t)B * H * T;
  AVSR_TRY(make_tmap_2d(&tmQu, qu, rows, 64, 64, AT_BQ, esz));
  AVSR_TRY(make_tmap_2d(&tmQv, qv, rows, 64, 64, AT_BQ, esz));
  AVSR_TRY(make_tmap_2d(&tmK, kk, rows, 64, 64, AT_BKV, esz));
  if (esz == 2) AVSR_TRY(make_tmap_2d(&tmV, v, rows, 64, 64, AT_BKV, esz));
  else AVSR_TRY(make_tmap_2d(&tmV, v, (uint64_t)B * H * 64, (uint64_t)Tp, (uint64_t)Tp, 64, esz));
  AVSR_TRY(make_tmap_3d(&tmP, pos, (uint64_t)H, (uint64_t)Rp, 64, 64, (uint64_t)Rp * 64, AT_BAND, esz));
  AVSR_SET_MAX_SMEM(attention_wg_kernel<TOp>, Cfg::kSmem);
  dim3 grid(H, B, cdiv(T, AT_BQ));
  AVSR_LAUNCH(attention_wg_kernel<TOp>, grid, AT_THREADS, Cfg::kSmem, st, tmQu, tmQv, tmK, tmV, tmP, lengths, ctx, T, H,
              round_out);
  return AVSR_OK;
}

int attention_tc(const float* qu, const float* qv, const float* kk, const float* vt, const float* pos,
                 const int32_t* lengths, float* ctx, int B, int T, int H, int Tp, int Rp, int round_out,
                 cudaStream_t st) {
  AVSR_REQUIRE(Tp % 4 == 0 && Tp >= T && Rp >= 2 * T - 1, "attention_tc: bad Tp=%d Rp=%d for T=%d", Tp, Rp, T);
  if (B <= 0 || T <= 0) return AVSR_OK;
  return attention_wg<float>(qu, qv, kk, vt, pos, lengths, ctx, B, T, H, Tp, Rp, round_out, st);
}

int attention_f16(const __half* qu, const __half* qv, const __half* kk, const __half* vv, const __half* pos,
                  const int32_t* lengths, __half* ctx, int B, int T, int H, int Rp, cudaStream_t st) {
  AVSR_REQUIRE(Rp >= 2 * T - 1, "attention_f16: bad Rp=%d for T=%d", Rp, T);
  if (B <= 0 || T <= 0) return AVSR_OK;
  return attention_wg<__half>(qu, qv, kk, vv, pos, lengths, ctx, B, T, H, T, Rp, 0, st);
}

}  // namespace avsr
