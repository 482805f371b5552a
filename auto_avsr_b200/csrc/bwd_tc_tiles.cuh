// Tile helpers shared by the tensor-core attention backwards (attention_bwd_tc.cu, decoder_attention_bwd_tc.cu): one
// warpgroup, 64 x 64 tiles of bf16 stored as 128B-swizzled rows (the layout TMA writes), read by wgmma K-major or,
// transposed, MN-major.
#pragma once
#include "common.cuh"
#include "sm90.cuh"

namespace avsr {

constexpr int BW_TILE = 64;                 // queries / keys per tile (= wgmma M)
constexpr int BW_THREADS = 128;             // one warpgroup
constexpr uint32_t BW_TB = 64 * 128;        // one [64 rows][64 bf16] 128B-swizzled tile

// MMA-K step ks (16 bf16 = 32 bytes) of a K-major [rows][K] tile stored as atoms of [rows][128 B]
__device__ __forceinline__ uint64_t bw_kdesc(uint32_t tile, int rows, int ks) {
  const int bytes = ks * 32;
  return sm90::wgmma_desc_sw128(tile + (bytes >> 7) * (rows * 128) + (bytes & 127));
}
// MMA-K step ks of an MN-major [K rows][64] tile: rows 16 ks .. 16 ks + 15
__device__ __forceinline__ uint64_t bw_mdesc(uint32_t tile, int ks) { return sm90::wgmma_desc_sw128(tile + ks * 16 * 128); }
// byte offset of element (r, c) of a [64 rows][C bf16] tile stored as 128B-swizzled atoms of 64 columns
__device__ __forceinline__ uint32_t bw_off(int r, int c) {
  return (c >> 6) * BW_TB + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4) + (c & 7) * 2;
}

// dP[64 x 64] = dO.V^T (both K-major), in the accumulator layout
__device__ __forceinline__ void bw_dprod(uint32_t o, uint32_t v, float (&dp)[32]) {
  sm90::wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) sm90::wgmma_bf16_n64(dp, bw_kdesc(o, 64, ks), bw_kdesc(v, 64, ks), ks != 0);
  sm90::wgmma_commit();
  sm90::wgmma_wait<0>();
  sm90::wgmma_fence_regs<32>(dp);
}

// a [64 x 64] accumulator -> bf16 [64 rows][64] 128B-swizzled tile (readable K-major and, transposed, MN-major)
__device__ __forceinline__ void bw_store_tile(uint8_t* tile, const float (&x)[32], int r0, int cq) {
#pragma unroll
  for (int rr = 0; rr < 2; ++rr)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int r = r0 + 8 * rr;
      *reinterpret_cast<uint32_t*>(tile + bw_off(r, 8 * j + cq)) = pack_bf162(x[4 * j + 2 * rr], x[4 * j + 2 * rr + 1]);
    }
}
__device__ __forceinline__ void bw_zero(uint8_t* p, uint32_t bytes) {
  for (uint32_t x = threadIdx.x; x < bytes / 16; x += BW_THREADS) reinterpret_cast<uint4*>(p)[x] = make_uint4(0, 0, 0, 0);
}
// accumulator rows r (+ row_off) < rows_valid of a [64 x 64] tile -> fp32 rows of `dst` (row stride ld)
__device__ __forceinline__ void bw_store_out(float* dst, long ld, const float (&x)[32], int r0, int cq, int rows_valid) {
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int r = r0 + 8 * rr;
    if (r >= rows_valid) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<float2*>(dst + (long)r * ld + 8 * j + cq) = make_float2(x[4 * j + 2 * rr], x[4 * j + 2 * rr + 1]);
  }
}

static inline const char* precision_name(int p) {
  return p == AVSR_PREC_FP32 ? "AVSR_PREC_FP32" : p == AVSR_PREC_TF32 ? "AVSR_PREC_TF32"
       : p == AVSR_PREC_F16 ? "AVSR_PREC_F16" : p == AVSR_PREC_BF16 ? "AVSR_PREC_BF16" : "unknown";
}

}  // namespace avsr
