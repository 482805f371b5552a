// Backward of the decoder's masked multi-head attention core on the Hopper tensor cores (wgmma): bf16 operands, fp32
// accumulation.  The same outputs as avsr_mha_core_bwd (decoder_train_body.cuh has the notation):
//   dA_ij = (dctx_i . v_j) keep_ij s ,  Delta_i = dctx_i . ctx_i (= sum_j A_ij dA_ij) ,  dS_ij = A_ij (dA_ij - Delta_i) / 8 ,
//   dq_i = sum_j dS_ij k_j ,  dk_j = sum_i dS_ij q_i ,  dv_j = sum_i A_ij keep_ij s dctx_i .
// The probabilities A are the ones avsr_mha_core_fwd stored (fp32, 0 on every masked key), so nothing is recomputed and
// no masking is needed beyond the tensor edges: rows >= Lq and keys >= Lk of a partial tile are zero-filled.  Tiles
// that no query sees are skipped (above the causal diagonal, keys at or past the key length).  Two launches:
//   dq kernel   (h, b, 64 queries)  Delta of its rows (fp32, from ctx and dctx; kept in the workspace for the next kernel),
//                                   then over the visible key tiles: dA = dO.V^T, dS in the accumulator layout,
//                                   dq += dS.K with K read MN-major
//   dk/dv kernel (h, b, 64 keys)    over the query tiles that see the keys: dA = dO.V^T, then A' = A keep s and dS
//                                   stored as bf16 [query][key] tiles; dv += A'^T.dO and dk += dS^T.Q read both operands
//                                   MN-major
// Each CTA loads its fp32 q / k / v / dctx rows with coalesced float4 loads and writes them as bf16 into the
// 128B-swizzled tiles itself (no conversion launches); the A and keep tiles are staged through shared memory with
// coalesced loads.  One writer per output element, every sum in a fixed order: repeated calls are bit-identical.
#include "bwd_tc_tiles.cuh"
#include "decoder_train_body.cuh"

namespace avsr {
namespace dtr {

using namespace sm90;

constexpr int DB_PITCH = 65;                          // fp32 row stride of the staged A / keep tiles (conflict-free writes)
constexpr uint32_t DB_STAGE = 64 * DB_PITCH * 4;

// shared-memory layouts (offsets from a 1024-aligned base; the bf16 operand tiles 1024-aligned for the 128B swizzle)
struct DbDq {   // dO, V, K, dS | A, keep factor (fp32) | Delta of the query tile
  static constexpr uint32_t kO = 0, kV = kO + BW_TB, kK = kV + BW_TB, kG = kK + BW_TB, kP = kG + BW_TB,
                            kKf = kP + DB_STAGE, kRows = kKf + DB_STAGE, kSmem = kRows + 64 * 4 + 1024;
};
struct DbKv {   // V, dO, Q, A', dS | A, keep factor (fp32) | Delta of the query tile
  static constexpr uint32_t kV = 0, kO = kV + BW_TB, kQ = kO + BW_TB, kA = kQ + BW_TB, kG = kA + BW_TB,
                            kP = kG + BW_TB, kKf = kP + DB_STAGE, kRows = kKf + DB_STAGE, kSmem = kRows + 64 * 4 + 1024;
};

// rows [0, nrows) of a 64 x 64 fp32 block (row stride ld, 16-byte aligned rows) -> bf16 swizzled tile, later rows 0
__device__ __forceinline__ void db_load_tile(uint8_t* tile, const float* __restrict__ src, long ld, int nrows) {
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int idx = threadIdx.x + BW_THREADS * it, r = idx >> 4, c = (idx & 15) * 4;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < nrows) x = __ldg(reinterpret_cast<const float4*>(src + (long)r * ld + c));
    *reinterpret_cast<uint2*>(tile + bw_off(r, c)) = make_uint2(pack_bf162(x.x, x.y), pack_bf162(x.z, x.w));
  }
}

// db_load_tile of the dctx rows, and Delta_r = dctx_r . ctx_r in fp32 (the 16 lanes of a row summed in a fixed order)
// -> srow[r] (0 past nrows) and delta[r] (r < nrows)
__device__ __forceinline__ void db_load_dout(uint8_t* tile, float* srow, float* __restrict__ delta,
                                             const float* __restrict__ dctx, const float* __restrict__ ctx, long ld,
                                             int nrows) {
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int idx = threadIdx.x + BW_THREADS * it, r = idx >> 4, c = (idx & 15) * 4;
    float4 d = make_float4(0.f, 0.f, 0.f, 0.f), o = d;
    if (r < nrows) {
      d = __ldg(reinterpret_cast<const float4*>(dctx + (long)r * ld + c));
      o = __ldg(reinterpret_cast<const float4*>(ctx + (long)r * ld + c));
    }
    *reinterpret_cast<uint2*>(tile + bw_off(r, c)) = make_uint2(pack_bf162(d.x, d.y), pack_bf162(d.z, d.w));
    float s = fmaf(d.x, o.x, fmaf(d.y, o.y, fmaf(d.z, o.z, d.w * o.w)));
#pragma unroll
    for (int m = 8; m >= 1; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
    if ((threadIdx.x & 15) == 0) {
      srow[r] = s;
      if (r < nrows) delta[r] = s;
    }
  }
}

// A and the keep factor (keep s, or 1 without a keep-mask) of queries [i0, i0 + 64) x keys [j0, j0 + 64) -> fp32
// [64][DB_PITCH] tiles, 0 outside Lq x Lk.  `probs` / `keep` point at the (b, h) plane (Lq, Lk).
__device__ __forceinline__ void db_stage_probs(float* sp, float* skf, const float* __restrict__ probs,
                                               const uint8_t* __restrict__ keep, float kscale, int i0, int j0, int Lq,
                                               int Lk) {
  for (int idx = threadIdx.x; idx < 64 * 64; idx += BW_THREADS) {
    const int r = idx >> 6, c = idx & 63, i = i0 + r, j = j0 + c;
    float p = 0.f, kf = 0.f;
    if (i < Lq && j < Lk) {
      const long o = (long)i * Lk + j;
      p = __ldg(probs + o);
      kf = keep ? (keep[o] ? kscale : 0.f) : 1.f;
    }
    sp[r * DB_PITCH + c] = p;
    skf[r * DB_PITCH + c] = kf;
  }
}

// da (dO.V^T, accumulator layout) -> dS = A (da keep s - Delta) / 8; ap (when given) <- A keep s
template <bool kWantAp>
__device__ __forceinline__ void db_dscores(float (&da)[32], float (&ap)[32], const float* sp, const float* skf,
                                           const float (&dl)[2], int r0, int cq) {
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int x = 4 * j + 2 * rr + e, s = (r0 + 8 * rr) * DB_PITCH + 8 * j + cq + e;
        const float a = sp[s], kf = skf[s];
        if (kWantAp) ap[x] = a * kf;
        da[x] = attn_dscore(a, da[x] * kf, dl[rr]);
      }
}

__device__ __forceinline__ uint8_t* db_smem_base(uint8_t* raw_smem, uint32_t* base) {
  const uint32_t raw = smem_u32(raw_smem);
  *base = (raw + 1023u) & ~1023u;
  return raw_smem + (*base - raw);
}

// ---------------------------------------------------------------- dq (and Delta)
__global__ void __launch_bounds__(BW_THREADS) mha_bwd_tc_dq_kernel(
    const float* __restrict__ k, long ldk, const float* __restrict__ v, long ldv, int H, int Lq, int Lk, int causal,
    const int32_t* __restrict__ klen, const uint8_t* __restrict__ keep, float kscale, const float* __restrict__ probs,
    const float* __restrict__ ctx, const float* __restrict__ dctx, float* __restrict__ dq, long lddq,
    float* __restrict__ delta) {
  using S = DbDq;
  extern __shared__ uint8_t db_smem_raw[];
  uint32_t base;
  uint8_t* gen = db_smem_base(db_smem_raw, &base);
  float* sp = reinterpret_cast<float*>(gen + S::kP);
  float* skf = reinterpret_cast<float*>(gen + S::kKf);
  float* srow = reinterpret_cast<float*>(gen + S::kRows);
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.x, b = blockIdx.y, i0 = blockIdx.z * BW_TILE;
  const long bh = (long)b * H + h, D = (long)H * kHeadDim;
  const int nq = Lq - i0 < BW_TILE ? Lq - i0 : BW_TILE;
  const int L = attn_row_keys(0, Lk, 0, klen, b);
  const int kmax = causal && i0 + BW_TILE < L ? i0 + BW_TILE : L;   // keys any row of the tile sees
  const int nkt = (kmax + BW_TILE - 1) / BW_TILE;
  const long orow = ((long)b * Lq + i0) * D + h * kHeadDim;
  db_load_dout(gen + S::kO, srow, delta + bh * Lq + i0, dctx + orow, ctx + orow, D, nq);
  __syncthreads();
  const int r0 = 16 * warp + (lane >> 2), cq = 2 * (lane & 3);
  const float dl[2] = {srow[r0], srow[r0 + 8]};
  const float* pbh = probs + bh * Lq * Lk;
  const uint8_t* kbh = keep ? keep + bh * Lq * Lk : nullptr;
  float acc[32];
#pragma unroll
  for (int x = 0; x < 32; ++x) acc[x] = 0.f;
#pragma unroll 1
  for (int it = 0; it < nkt; ++it) {
    const int j0 = it * BW_TILE, nk = Lk - j0 < BW_TILE ? Lk - j0 : BW_TILE;
    const long krow = (long)b * Lk + j0;
    db_load_tile(gen + S::kV, v + krow * ldv + h * kHeadDim, ldv, nk);
    db_load_tile(gen + S::kK, k + krow * ldk + h * kHeadDim, ldk, nk);
    db_stage_probs(sp, skf, pbh, kbh, kscale, i0, j0, Lq, Lk);
    fence_proxy_async();   // generic-proxy smem writes -> visible to the tensor core
    __syncthreads();
    float da[32], unused[32];
    bw_dprod(base + S::kO, base + S::kV, da);
    db_dscores<false>(da, unused, sp, skf, dl, r0, cq);
    bw_store_tile(gen + S::kG, da, r0, cq);
    fence_proxy_async();
    __syncthreads();
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma_bf16_n64_bmn(acc, bw_kdesc(base + S::kG, 64, ks), bw_mdesc(base + S::kK, ks), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<32>(acc);
    __syncthreads();   // V, K, dS and the staged tiles are free for the next key tile
  }
  bw_store_out(dq + ((long)b * Lq + i0) * lddq + h * kHeadDim, lddq, acc, r0, cq, nq);
}

// ---------------------------------------------------------------- dk, dv
__global__ void __launch_bounds__(BW_THREADS) mha_bwd_tc_dkdv_kernel(
    const float* __restrict__ q, long ldq, const float* __restrict__ v, long ldv, int H, int Lq, int Lk, int causal,
    const int32_t* __restrict__ klen, const uint8_t* __restrict__ keep, float kscale, const float* __restrict__ probs,
    const float* __restrict__ dctx, const float* __restrict__ delta, float* __restrict__ dk, float* __restrict__ dv,
    long lddkv) {
  using S = DbKv;
  extern __shared__ uint8_t db_smem_raw[];
  uint32_t base;
  uint8_t* gen = db_smem_base(db_smem_raw, &base);
  float* sp = reinterpret_cast<float*>(gen + S::kP);
  float* skf = reinterpret_cast<float*>(gen + S::kKf);
  float* srow = reinterpret_cast<float*>(gen + S::kRows);
  pdl_launch_dependents();
  pdl_wait();                                                    // Delta comes from the dq kernel
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.x, b = blockIdx.y, j0 = blockIdx.z * BW_TILE;
  const long bh = (long)b * H + h, D = (long)H * kHeadDim;
  const int nk = Lk - j0 < BW_TILE ? Lk - j0 : BW_TILE;
  const int L = attn_row_keys(0, Lk, 0, klen, b);
  const int r0 = 16 * warp + (lane >> 2), cq = 2 * (lane & 3);
  float ak[32], av[32];
#pragma unroll
  for (int x = 0; x < 32; ++x) ak[x] = av[x] = 0.f;
  if (j0 < L) {                                                  // CTA-uniform: keys past the key length get zeros
    db_load_tile(gen + S::kV, v + ((long)b * Lk + j0) * ldv + h * kHeadDim, ldv, nk);
    const float* pbh = probs + bh * Lq * Lk;
    const uint8_t* kbh = keep ? keep + bh * Lq * Lk : nullptr;
    const int nqt = (Lq + BW_TILE - 1) / BW_TILE;
#pragma unroll 1
    for (int qt = causal ? j0 / BW_TILE : 0; qt < nqt; ++qt) {   // causal: query tiles below the diagonal see no key
      const int i0 = qt * BW_TILE, nq = Lq - i0 < BW_TILE ? Lq - i0 : BW_TILE;
      const long qrow = (long)b * Lq + i0;
      db_load_tile(gen + S::kO, dctx + qrow * D + h * kHeadDim, D, nq);
      db_load_tile(gen + S::kQ, q + qrow * ldq + h * kHeadDim, ldq, nq);
      if (threadIdx.x < BW_TILE) srow[threadIdx.x] = (int)threadIdx.x < nq ? delta[bh * Lq + i0 + threadIdx.x] : 0.f;
      db_stage_probs(sp, skf, pbh, kbh, kscale, i0, j0, Lq, Lk);
      fence_proxy_async();
      __syncthreads();
      float da[32], ap[32];
      bw_dprod(base + S::kO, base + S::kV, da);
      const float dl[2] = {srow[r0], srow[r0 + 8]};
      db_dscores<true>(da, ap, sp, skf, dl, r0, cq);
      bw_store_tile(gen + S::kA, ap, r0, cq);
      bw_store_tile(gen + S::kG, da, r0, cq);
      fence_proxy_async();
      __syncthreads();
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        wgmma_bf16_n64_amn_bmn(av, bw_mdesc(base + S::kA, ks), bw_mdesc(base + S::kO, ks), 1);
        wgmma_bf16_n64_amn_bmn(ak, bw_mdesc(base + S::kG, ks), bw_mdesc(base + S::kQ, ks), 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs<32>(av);
      wgmma_fence_regs<32>(ak);
      __syncthreads();   // the query tile, A', dS, the staged tiles and srow are free for the next query tile
    }
  }
  const long o = ((long)b * Lk + j0) * lddkv + h * kHeadDim;
  bw_store_out(dk + o, lddkv, ak, r0, cq, nk);
  bw_store_out(dv + o, lddkv, av, r0, cq, nk);
}

static bool db_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace dtr
}  // namespace avsr

using namespace avsr;
using namespace avsr::dtr;

extern "C" {

size_t avsr_mha_core_bwd_tc_workspace_bytes(int B, int H, int Lq, int Lk, int precision) {
  (void)Lk;
  if (precision != AVSR_PREC_BF16) return 0;
  if (B <= 0 || H <= 0 || Lq <= 0) return 256;
  return align_up((size_t)B * H * Lq * sizeof(float), 256);   // Delta (B, H, Lq)
}

int avsr_mha_core_bwd_tc(const float* q, long ldq, const float* k, long ldk, const float* v, long ldv, int B, int H,
                         int Lq, int Lk, int causal, const int32_t* key_lengths, const uint8_t* keep, float keep_scale,
                         const float* probs, const float* ctx, const float* dctx, float* dq, long lddq, float* dk,
                         float* dv, long lddkv, int precision, void* workspace, size_t workspace_bytes, void* stream) {
  AVSR_REQUIRE(B >= 0 && H >= 1 && Lq >= 0 && Lk >= 0, "mha_core_bwd (tensor cores): bad B=%d H=%d Lq=%d Lk=%d", B, H,
               Lq, Lk);
  const long rows = (long)B * H * Lq, keys = (long)B * H * Lk;
  // what each non-empty side reads and writes; key_lengths and keep may be NULL
  AVSR_REQUIRE(rows == 0 || (q && dq && ctx && dctx && workspace && (Lk == 0 || (k && v && probs))), "NULL argument");
  AVSR_REQUIRE(keys == 0 || (k && v && dk && dv && (Lq == 0 || (q && probs && ctx && dctx && workspace))),
               "NULL argument");
  AVSR_REQUIRE(precision == AVSR_PREC_BF16,
               "mha_core_bwd (tensor cores): precision %d (%s) is not built; AVSR_PREC_BF16 only", precision,
               precision_name(precision));
  const long D = (long)H * kHeadDim;
  AVSR_REQUIRE(ldq >= D && ldk >= D && ldv >= D && lddq >= D && lddkv >= D && ldq % 4 == 0 && ldk % 4 == 0 &&
                   ldv % 4 == 0 && lddq % 4 == 0 && lddkv % 4 == 0,
               "mha_core_bwd (tensor cores): row strides (%ld, %ld, %ld, %ld, %ld) must be multiples of 4 and >= H*64 = %ld",
               ldq, ldk, ldv, lddq, lddkv, D);
  AVSR_REQUIRE(rows == 0 || (db_aligned16(q) && db_aligned16(dq) && db_aligned16(ctx) && db_aligned16(dctx)),
               "mha_core_bwd (tensor cores): q / dq / ctx / dctx not 16-byte aligned");
  AVSR_REQUIRE(keys == 0 || (db_aligned16(k) && db_aligned16(v) && db_aligned16(dk) && db_aligned16(dv)),
               "mha_core_bwd (tensor cores): k / v / dk / dv not 16-byte aligned");
  if (rows == 0 && keys == 0) return AVSR_OK;
  if (rows > 0)   // the workspace holds Delta, which only exists with query rows
    AVSR_REQUIRE_BYTES(avsr_mha_core_bwd_tc_workspace_bytes(B, H, Lq, Lk, precision), workspace_bytes,
                       "mha_core_bwd (tensor cores) workspace");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* delta = reinterpret_cast<float*>(workspace);
  if (rows > 0) {
    AVSR_SET_MAX_SMEM(mha_bwd_tc_dq_kernel, DbDq::kSmem);
    AVSR_LAUNCH(mha_bwd_tc_dq_kernel, dim3(H, B, cdiv(Lq, BW_TILE)), BW_THREADS, DbDq::kSmem, st, k, ldk, v, ldv, H, Lq,
                Lk, causal, key_lengths, keep, keep_scale, probs, ctx, dctx, dq, lddq, delta);
  }
  if (keys > 0) {
    AVSR_SET_MAX_SMEM(mha_bwd_tc_dkdv_kernel, DbKv::kSmem);
    AVSR_LAUNCH(mha_bwd_tc_dkdv_kernel, dim3(H, B, cdiv(Lk, BW_TILE)), BW_THREADS, DbKv::kSmem, st, q, ldq, v, ldv, H, Lq,
                Lk, causal, key_lengths, keep, keep_scale, probs, dctx, delta, dk, dv, lddkv);
  }
  return AVSR_OK;
}

}  // extern "C"
