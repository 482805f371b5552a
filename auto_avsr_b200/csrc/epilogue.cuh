// Staged (coalesced) epilogue helpers of the tensor-core GEMM (gemm_tc.cu).
#pragma once
#include "common.cuh"

namespace avsr {

// ---------------------------------------------------------------- staged (coalesced) epilogue
// Each epilogue warp drains 32 accumulator rows x CW columns at a time: lane = row of the fp32 accumulator tile, per-
// column math (bias / ReLU / GLU / pos biases, vectors read from shared memory), conversion to the destination
// storage, then a transpose through shared memory so that global memory sees, per quarter-warp, 8 lanes x 16 B = one
// full 128-byte row segment -- instead of 32 partial sectors per store instruction of direct lane-per-row stores.
// Residual reads use the same mapping.  The transpose goes through the accumulator rows the lane has just read
// (`stg` = first of the warp's 32 rows at the chunk's first column, rows `row_bytes` apart): a row stride of 4 banks
// mod 32 keeps the lane-per-row 16-byte writes conflict-free.

// lane writes its row: 32 fp32 values, optionally rounded to TF32
__device__ __forceinline__ void stage_write_f32(uint8_t* stg, int row_bytes, int lane, const float* o, bool round) {
  uint8_t* row = stg + lane * row_bytes;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float4 t = make_float4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
    if (round) { t.x = round_tf32(t.x); t.y = round_tf32(t.y); t.z = round_tf32(t.z); t.w = round_tf32(t.w); }
    *reinterpret_cast<float4*>(row + 16 * j) = t;
  }
}
// lane writes its row: 64 values converted to half (128 bytes)
__device__ __forceinline__ void stage_write_f16(uint8_t* stg, int row_bytes, int lane, const float* o) {
  uint8_t* row = stg + lane * row_bytes;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    uint4 t;
    __half2 h0 = __halves2half2(to_half_sat(o[8 * j]), to_half_sat(o[8 * j + 1]));
    __half2 h1 = __halves2half2(to_half_sat(o[8 * j + 2]), to_half_sat(o[8 * j + 3]));
    __half2 h2 = __halves2half2(to_half_sat(o[8 * j + 4]), to_half_sat(o[8 * j + 5]));
    __half2 h3 = __halves2half2(to_half_sat(o[8 * j + 6]), to_half_sat(o[8 * j + 7]));
    t.x = *reinterpret_cast<uint32_t*>(&h0); t.y = *reinterpret_cast<uint32_t*>(&h1);
    t.z = *reinterpret_cast<uint32_t*>(&h2); t.w = *reinterpret_cast<uint32_t*>(&h3);
    *reinterpret_cast<uint4*>(row + 16 * j) = t;
  }
}
// lane writes its row: 64 values converted to bfloat16 (128 bytes)
__device__ __forceinline__ void stage_write_bf16(uint8_t* stg, int row_bytes, int lane, const float* o) {
  uint8_t* row = stg + lane * row_bytes;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint4 t = make_uint4(pack_bf162(o[8 * j], o[8 * j + 1]), pack_bf162(o[8 * j + 2], o[8 * j + 3]),
                               pack_bf162(o[8 * j + 4], o[8 * j + 5]), pack_bf162(o[8 * j + 6], o[8 * j + 7]));
    *reinterpret_cast<uint4*>(row + 16 * j) = t;
  }
}
template <typename TOp> struct StageOp;
template <> struct StageOp<float> {
  static constexpr int kCols = 32;   // operand columns per 128-byte row segment
  __device__ static void write(uint8_t* stg, int row_bytes, int lane, const float* o) {
    stage_write_f32(stg, row_bytes, lane, o, true);
  }
};
template <> struct StageOp<__half> {
  static constexpr int kCols = 64;
  __device__ static void write(uint8_t* stg, int row_bytes, int lane, const float* o) {
    stage_write_f16(stg, row_bytes, lane, o);
  }
};
template <> struct StageOp<__nv_bfloat16> {
  static constexpr int kCols = 64;
  __device__ static void write(uint8_t* stg, int row_bytes, int lane, const float* o) {
    stage_write_bf16(stg, row_bytes, lane, o);
  }
};
// transposed read: iteration `it` (0..7) gives this lane the 16-byte piece (lane & 7) of row it*4 + (lane >> 3)
__device__ __forceinline__ uint4 stage_read(const uint8_t* stg, int row_bytes, int it, int lane) {
  return *reinterpret_cast<const uint4*>(stg + (it * 4 + (lane >> 3)) * row_bytes + (lane & 7) * 16);
}

// ---- per-mode emit of one 16-byte piece: row m, first column n (global indices of the GEMM) ----
// fp32 destination (LINEAR): y = [resid + alpha *] val
__device__ __forceinline__ void emit_linear_f32(const EpiParams& p, int m, int n, uint4 pay) {
  if (m >= p.M || n >= p.N) return;
  const long off = (long)m * p.ldo + n;
  float4 v = *reinterpret_cast<float4*>(&pay);
  if (p.resid) {
    const float4 r = *reinterpret_cast<const float4*>(p.resid + off);
    v.x = r.x + p.alpha * v.x; v.y = r.y + p.alpha * v.y; v.z = r.z + p.alpha * v.z; v.w = r.w + p.alpha * v.w;
  }
  *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + off) = v;
}
template <typename TOp>
__device__ __forceinline__ void emit_linear_op(const EpiParams& p, int m, int n, uint4 pay) {
  if (m >= p.M || n >= p.N) return;
  *reinterpret_cast<uint4*>(reinterpret_cast<TOp*>(p.out) + (long)m * p.ldo + n) = pay;
}
// QKV: row (b, t) and column (head h, offset d0) already decoded by the caller (no per-element divisions)
template <typename TOp>
__device__ __forceinline__ void emit_heads(const EpiParams& p, void* base, bool ok, int b, int t, int h, int d0,
                                           uint4 pay) {
  if (!ok) return;
  *reinterpret_cast<uint4*>(reinterpret_cast<TOp*>(base) + (((long)b * p.H + h) * p.T + t) * kHeadDim + d0) = pay;
}
template <typename TOp>
__device__ __forceinline__ void emit_vt(const EpiParams& p, int m, int n, uint4 pay) {  // m = feature, n = frame
  constexpr int NE = 16 / (int)sizeof(TOp);
  if (m >= p.M || n >= p.N) return;
  const int h = m >> 6, d = m & 63;
  const int b0 = n / p.T, t0 = n - b0 * p.T;
  TOp* vt = reinterpret_cast<TOp*>(p.vt);
  if (t0 + NE <= p.T && n + NE <= p.N && (t0 % NE) == 0) {
    *reinterpret_cast<uint4*>(vt + (((long)b0 * p.H + h) * kHeadDim + d) * p.Tp + t0) = pay;
  } else {   // utterance boundary / ragged T: element-wise
    const TOp* e = reinterpret_cast<const TOp*>(&pay);
#pragma unroll
    for (int i = 0; i < NE; ++i) {
      const int ne = n + i;
      if (ne < p.N) {
        const int b = ne / p.T, t = ne - b * p.T;
        vt[(((long)b * p.H + h) * kHeadDim + d) * p.Tp + t] = e[i];
      }
    }
  }
}
template <typename TOp>
__device__ __forceinline__ void emit_pos(const EpiParams& p, int m, int n, uint4 pay) {
  if (m >= p.M || n >= p.N) return;
  const int D = p.H * kHeadDim;
  const int l = n / D, r = n - l * D;
  const int h = r >> 6, d0 = r & 63;
  *reinterpret_cast<uint4*>(reinterpret_cast<TOp*>(p.out) + (((long)l * p.H + h) * p.Rp + m) * kHeadDim + d0) = pay;
}
__device__ __forceinline__ void emit_glu(const EpiParams& p, int m, int n_val, uint4 pay) {  // fp32 dest
  if (m >= p.M || n_val + 64 >= p.N) return;
  const int c = (n_val >> 7) * 64 + (n_val & 127);
  *reinterpret_cast<uint4*>(reinterpret_cast<float*>(p.out) + (long)m * p.ldo + c) = pay;
}


}  // namespace avsr
