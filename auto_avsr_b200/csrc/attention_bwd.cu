// Backward of the rel-pos attention core (SURVEY.md 8f #2): fp32 CUDA-core kernels, correctness first -- the training
// counterpart of attention_simt.cu.  Forward (transformer/attention.py:174-189 + :59-82):
//   s_ij = ((q_i + u).k_j + (q_i + v).p[m_ij]) / 8,  m_ij = j - i + T - 1 ;  keys j >= len[b] masked ;
//   A = softmax_j(s) ;  ctx_i = sum_j A_ij v_j .
// Backward, with Delta_i = dctx_i . ctx_i and g_ij = A_ij (dctx_i . v_j - Delta_i) / 8 :
//   dq_i = sum_j g_ij (k_j + p[m_ij])        (kept as two parts: their column sums are d pos_bias_u / d pos_bias_v)
//   dk_j = sum_i g_ij (q_i + u) ;  dv_j = sum_i A_ij dctx_i ;  dp[m] = sum_{b, i} g_{i, j = m + i - (T-1)} (q_i + v) .
// Nothing of size T^2 is stored: three passes recompute the scores from q, k, p --
//   rows kernel  (one warp per query row)      : log-sum-exp and Delta of the row, then the two parts of dq
//   keys kernel  (one warp per key)            : dk, dv
//   pos kernel   (one warp per (table row, h)) : dp
// A lane owns one (row, key) pair at a time; the vectors it needs are staged tile by tile in shared memory by the whole CTA
// (r02 profile of the first version, whose lanes read their rows straight from global memory: 81 % of the training
// step).  Every output element is written by exactly one warp: no atomics, deterministic.
// q, k, v, ctx, dctx and the outputs are (B, T, H*64); p / dp are (2T-1, H*64); u, v (H, 64).
#include <math.h>

#include "common.cuh"

namespace avsr {

constexpr int kAbWarps = 8;          // warps per CTA = output rows per CTA (query rows / keys / table rows)
constexpr int kAbTile = 32;          // the other index is walked in tiles of 32 (one per lane)
constexpr int kAbPitch = 68;         // floats per staged row: 64 + 4 pad -> lane-per-row float4 reads are conflict-free
constexpr int kAbBand = kAbTile + kAbWarps - 1;   // 39 rel-pos / shifted rows a (tile, 8 rows) pair touches
constexpr int kPosSmemBytes = ((3 * kAbTile + 2 * kAbBand) * kAbPitch + kAbWarps * 64 + 2 * kAbTile) * (int)sizeof(float);

// Stage `nrows` rows of 64 floats (global row r at base + r * row_stride) into shared memory, pitch kAbPitch; rows
// outside [lo, hi) are zero.  All threads of the CTA take part (coalesced: 16 float4 per row).
__device__ __forceinline__ void stage_rows(float* dst, const float* __restrict__ base, long row_stride, int first, int nrows,
                                           int lo, int hi) {
  for (int idx = threadIdx.x; idx < nrows * 16; idx += blockDim.x) {
    const int r = idx >> 4, t = idx & 15;
    const int g = first + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (g >= lo && g < hi) v = reinterpret_cast<const float4*>(base + (long)g * row_stride)[t];
    reinterpret_cast<float4*>(dst + r * kAbPitch)[t] = v;
  }
}
// the same with a bias vector (64 floats, global) added to every valid row
__device__ __forceinline__ void stage_rows_biased(float* dst, const float* __restrict__ base, long row_stride, int first,
                                                  int nrows, int lo, int hi, const float* __restrict__ bias) {
  for (int idx = threadIdx.x; idx < nrows * 16; idx += blockDim.x) {
    const int r = idx >> 4, t = idx & 15;
    const int g = first + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (g >= lo && g < hi) {
      v = reinterpret_cast<const float4*>(base + (long)g * row_stride)[t];
      const float4 c = reinterpret_cast<const float4*>(bias)[t];
      v.x += c.x; v.y += c.y; v.z += c.z; v.w += c.w;
    }
    reinterpret_cast<float4*>(dst + r * kAbPitch)[t] = v;
  }
}

// dot of two shared-memory vectors of 64 floats (a: broadcast across the warp, b: this lane's row)
__device__ __forceinline__ float sdot64(const float* a, const float* b) {
  float acc = 0.f;
#pragma unroll
  for (int t = 0; t < 16; ++t) {
    const float4 x = reinterpret_cast<const float4*>(a)[t];
    const float4 y = reinterpret_cast<const float4*>(b)[t];
    acc = fmaf(x.x, y.x, acc); acc = fmaf(x.y, y.y, acc); acc = fmaf(x.z, y.z, acc); acc = fmaf(x.w, y.w, acc);
  }
  return acc;
}
// acc[0..63] += s * row[0..63]   (row in shared memory)
__device__ __forceinline__ void saxpy64(float (&acc)[64], float s, const float* row) {
#pragma unroll
  for (int t = 0; t < 16; ++t) {
    const float4 b = reinterpret_cast<const float4*>(row)[t];
    acc[4 * t] = fmaf(s, b.x, acc[4 * t]); acc[4 * t + 1] = fmaf(s, b.y, acc[4 * t + 1]);
    acc[4 * t + 2] = fmaf(s, b.z, acc[4 * t + 2]); acc[4 * t + 3] = fmaf(s, b.w, acc[4 * t + 3]);
  }
}
// sum acc[d] over the warp's lanes; lane (d & 31) keeps element d: returns this lane's two elements (d = lane, lane + 32)
__device__ __forceinline__ float2 reduce64(float (&acc)[64], int lane) {
  float lo = 0.f, hi = 0.f;
#pragma unroll
  for (int d = 0; d < 64; ++d) {
    const float t = warp_sum(acc[d]);
    if ((d & 31) == lane) { if (d < 32) lo = t; else hi = t; }
  }
  return make_float2(lo, hi);
}

// Every kernel: a CTA owns kAbWarps consecutive output rows (one per warp) and walks the other index in tiles of 32 that
// the whole CTA stages in shared memory once (K / V / Q / dctx tiles of 32 rows, the 39-row band of the rel-pos table
// or of the shifted keys): 8x less L2 traffic than one warp streaming its own rows, and conflict-free shared reads.

// ---------------------------------------------------------------- rows: lse, Delta, dq (k part / p part)
__global__ void __launch_bounds__(32 * kAbWarps) attn_bwd_rows_kernel(
    const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, const float* __restrict__ p,
    const float* __restrict__ u, const float* __restrict__ vb, const int32_t* __restrict__ lengths,
    const float* __restrict__ ctx, const float* __restrict__ dctx, float* __restrict__ lse, float* __restrict__ delta,
    float* __restrict__ dq_k, float* __restrict__ dq_p, int T, int H) {
  __shared__ __align__(16) float Ks[kAbTile * kAbPitch], Vs[kAbTile * kAbPitch], Ps[kAbBand * kAbPitch];
  __shared__ __align__(16) float vec[kAbWarps][3][64];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i0 = blockIdx.x * kAbWarps, i = i0 + warp, h = blockIdx.y, b = blockIdx.z;
  const bool active = i < T;
  const int D = H * kHeadDim, R = 2 * T - 1;
  int L = T;
  if (lengths) { L = lengths[b]; L = L < 0 ? 0 : (L > T ? T : L); }
  const long ro = ((long)b * T + (active ? i : 0)) * D + h * kHeadDim;
  float* qu = vec[warp][0];
  float* qv = vec[warp][1];
  float* dc = vec[warp][2];
  float dl = 0.f;
  if (active) {
    for (int d = lane; d < 64; d += 32) {
      const float qq = q[ro + d];
      qu[d] = qq + u[h * 64 + d];
      qv[d] = qq + vb[h * 64 + d];
      dc[d] = dctx[ro + d];
      dl += dctx[ro + d] * ctx[ro + d];
    }
    dl = warp_sum(dl);
  }
  const float* kb = k + (long)b * T * D + h * kHeadDim;
  const float* vbase = v + (long)b * T * D + h * kHeadDim;
  const float* pb = p + h * kHeadDim;
  // pass 1: online log-sum-exp of the row
  float m = -INFINITY, ssum = 0.f;
  for (int j0 = 0; j0 < L; j0 += kAbTile) {
    const int mb = j0 - (i0 + kAbWarps - 1) + T - 1;          // table row of (key j0, last query row of the CTA)
    __syncthreads();
    stage_rows(Ks, kb, D, j0, kAbTile, 0, L);
    stage_rows(Ps, pb, D, mb, kAbBand, 0, R);
    __syncthreads();
    if (active) {
      const int j = j0 + lane;
      float s = -INFINITY;
      if (j < L) s = 0.125f * (sdot64(qu, Ks + lane * kAbPitch) + sdot64(qv, Ps + (j - i + T - 1 - mb) * kAbPitch));
      const float mn = fmaxf(m, warp_max(s));
      ssum = ssum * __expf(m - mn) + warp_sum(j < L ? __expf(s - mn) : 0.f);
      m = mn;
    }
  }
  const float row_lse = L > 0 ? m + logf(ssum) : INFINITY;     // len 0: exp(s - inf) = 0 below
  if (active && lane == 0) {
    lse[((long)b * H + h) * T + i] = row_lse;
    delta[((long)b * H + h) * T + i] = dl;
  }
  // pass 2: g_ij and the two parts of dq
  float ak[64], ap[64];
#pragma unroll
  for (int d = 0; d < 64; ++d) ak[d] = ap[d] = 0.f;
  for (int j0 = 0; j0 < L; j0 += kAbTile) {
    const int mb = j0 - (i0 + kAbWarps - 1) + T - 1;
    __syncthreads();
    stage_rows(Ks, kb, D, j0, kAbTile, 0, L);
    stage_rows(Vs, vbase, D, j0, kAbTile, 0, L);
    stage_rows(Ps, pb, D, mb, kAbBand, 0, R);
    __syncthreads();
    const int j = j0 + lane;
    if (active && j < L) {
      const float* kr = Ks + lane * kAbPitch;
      const float* pr = Ps + (j - i + T - 1 - mb) * kAbPitch;
      const float s = 0.125f * (sdot64(qu, kr) + sdot64(qv, pr));
      const float a = __expf(s - row_lse);
      const float g = a * (sdot64(dc, Vs + lane * kAbPitch) - dl) * 0.125f;
      saxpy64(ak, g, kr);
      saxpy64(ap, g, pr);
    }
  }
  if (!active) return;
  const float2 rk = reduce64(ak, lane), rp = reduce64(ap, lane);
  dq_k[ro + lane] = rk.x; dq_k[ro + lane + 32] = rk.y;
  dq_p[ro + lane] = rp.x; dq_p[ro + lane + 32] = rp.y;
}

// ---------------------------------------------------------------- keys: dk, dv
__global__ void __launch_bounds__(32 * kAbWarps) attn_bwd_keys_kernel(
    const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, const float* __restrict__ p,
    const float* __restrict__ u, const float* __restrict__ vb, const int32_t* __restrict__ lengths,
    const float* __restrict__ dctx, const float* __restrict__ lse, const float* __restrict__ delta,
    float* __restrict__ dk, float* __restrict__ dv, int T, int H) {
  __shared__ __align__(16) float Qu[kAbTile * kAbPitch], Qv[kAbTile * kAbPitch], Dc[kAbTile * kAbPitch], Ps[kAbBand * kAbPitch];
  __shared__ __align__(16) float vec[kAbWarps][2][64];
  __shared__ float ls[kAbTile], ds[kAbTile];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j0 = blockIdx.x * kAbWarps, j = j0 + warp, h = blockIdx.y, b = blockIdx.z;
  const int D = H * kHeadDim, R = 2 * T - 1;
  int L = T;
  if (lengths) { L = lengths[b]; L = L < 0 ? 0 : (L > T ? T : L); }
  const bool active = j < L;                       // a masked key (or j >= T) received no probability: zeros
  const long ko = ((long)b * T + (j < T ? j : 0)) * D + h * kHeadDim;
  float* kj = vec[warp][0];
  float* vj = vec[warp][1];
  if (j < T)
    for (int d = lane; d < 64; d += 32) { kj[d] = k[ko + d]; vj[d] = v[ko + d]; }
  const float* qb = q + (long)b * T * D + h * kHeadDim;
  const float* db_ = dctx + (long)b * T * D + h * kHeadDim;
  const float* pb = p + h * kHeadDim;
  const float* lrow = lse + ((long)b * H + h) * T;
  const float* drow = delta + ((long)b * H + h) * T;
  float ak[64], av[64];
#pragma unroll
  for (int d = 0; d < 64; ++d) ak[d] = av[d] = 0.f;
  if (j0 < L) {                                    // CTA-uniform: at least one key of this CTA is valid
    for (int i0 = 0; i0 < T; i0 += kAbTile) {
      const int mb = j0 - (i0 + kAbTile - 1) + T - 1;         // table row of (first key of the CTA, last query of the tile)
      __syncthreads();
      stage_rows_biased(Qu, qb, D, i0, kAbTile, 0, T, u + h * 64);
      stage_rows_biased(Qv, qb, D, i0, kAbTile, 0, T, vb + h * 64);
      stage_rows(Dc, db_, D, i0, kAbTile, 0, T);
      stage_rows(Ps, pb, D, mb, kAbBand, 0, R);
      if (threadIdx.x < kAbTile) {
        const int ii = i0 + threadIdx.x;
        ls[threadIdx.x] = ii < T ? lrow[ii] : INFINITY;
        ds[threadIdx.x] = ii < T ? drow[ii] : 0.f;
      }
      __syncthreads();
      const int i = i0 + lane;
      if (active && i < T) {
        const float* qur = Qu + lane * kAbPitch;
        const float* dr = Dc + lane * kAbPitch;
        const float s = 0.125f * (sdot64(kj, qur) + sdot64(Ps + (j - i + T - 1 - mb) * kAbPitch, Qv + lane * kAbPitch));
        const float a = __expf(s - ls[lane]);
        const float g = a * (sdot64(vj, dr) - ds[lane]) * 0.125f;
        saxpy64(av, a, dr);
        saxpy64(ak, g, qur);
      }
    }
  }
  if (j >= T) return;
  const float2 rk = reduce64(ak, lane), rv = reduce64(av, lane);
  dk[ko + lane] = rk.x; dk[ko + lane + 32] = rk.y;
  dv[ko + lane] = rv.x; dv[ko + lane + 32] = rv.y;
}

// ---------------------------------------------------------------- rel-pos table rows: dp
__global__ void __launch_bounds__(32 * kAbWarps) attn_bwd_pos_kernel(
    const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, const float* __restrict__ p,
    const float* __restrict__ u, const float* __restrict__ vb, const int32_t* __restrict__ lengths,
    const float* __restrict__ dctx, const float* __restrict__ lse, const float* __restrict__ delta,
    float* __restrict__ dp, int B, int T, int H) {
  extern __shared__ __align__(16) float pos_smem[];            // kPosSmemBytes (> 48 KB: opt-in, set by the launcher)
  float* Qu = pos_smem;
  float* Qv = Qu + kAbTile * kAbPitch;
  float* Dc = Qv + kAbTile * kAbPitch;
  float* Kb = Dc + kAbTile * kAbPitch;
  float* Vb = Kb + kAbBand * kAbPitch;
  float (*vec)[64] = reinterpret_cast<float (*)[64]>(Vb + kAbBand * kAbPitch);
  float* ls = &vec[kAbWarps][0];
  float* ds = ls + kAbTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * kAbWarps, m = m0 + warp, h = blockIdx.y;
  const int R = 2 * T - 1;
  const bool active = m < R;
  const int D = H * kHeadDim;
  float* pm = vec[warp];
  if (active)
    for (int d = lane; d < 64; d += 32) pm[d] = p[(long)m * D + h * 64 + d];
  float ap[64];
#pragma unroll
  for (int d = 0; d < 64; ++d) ap[d] = 0.f;
  const int shift = m - (T - 1);                   // this warp's key for query i is j = i + shift
  const int shift0 = m0 - (T - 1);                 // the CTA's first table row
  for (int b = 0; b < B; ++b) {
    int L = T;
    if (lengths) { L = lengths[b]; L = L < 0 ? 0 : (L > T ? T : L); }
    const float* qb = q + (long)b * T * D + h * kHeadDim;
    const float* kb = k + (long)b * T * D + h * kHeadDim;
    const float* vbase = v + (long)b * T * D + h * kHeadDim;
    const float* db_ = dctx + (long)b * T * D + h * kHeadDim;
    const float* lrow = lse + ((long)b * H + h) * T;
    const float* drow = delta + ((long)b * H + h) * T;
    // queries that have a valid key under ANY of the CTA's table rows: 0 <= i + shift0 + w < L for some w in [0, 8)
    int ilo = -(shift0 + kAbWarps - 1);
    if (ilo < 0) ilo = 0;
    int ihi = L - shift0;
    if (ihi > T) ihi = T;
    for (int i0 = ilo; i0 < ihi; i0 += kAbTile) {
      const int jb = i0 + shift0;                  // key of (first query of the tile, first table row of the CTA)
      __syncthreads();
      stage_rows_biased(Qu, qb, D, i0, kAbTile, 0, T, u + h * 64);
      stage_rows_biased(Qv, qb, D, i0, kAbTile, 0, T, vb + h * 64);
      stage_rows(Dc, db_, D, i0, kAbTile, 0, T);
      stage_rows(Kb, kb, D, jb, kAbBand, 0, L);
      stage_rows(Vb, vbase, D, jb, kAbBand, 0, L);
      if (threadIdx.x < kAbTile) {
        const int ii = i0 + threadIdx.x;
        ls[threadIdx.x] = ii < T ? lrow[ii] : INFINITY;
        ds[threadIdx.x] = ii < T ? drow[ii] : 0.f;
      }
      __syncthreads();
      const int i = i0 + lane, j = i + shift;
      if (active && i < T && j >= 0 && j < L) {
        const float* qvr = Qv + lane * kAbPitch;
        const float s = 0.125f * (sdot64(Qu + lane * kAbPitch, Kb + (j - jb) * kAbPitch) + sdot64(pm, qvr));
        const float a = __expf(s - ls[lane]);
        const float g = a * (sdot64(Dc + lane * kAbPitch, Vb + (j - jb) * kAbPitch) - ds[lane]) * 0.125f;
        saxpy64(ap, g, qvr);
      }
    }
  }
  if (!active) return;
  const float2 rp = reduce64(ap, lane);
  dp[(long)m * D + h * 64 + lane] = rp.x;
  dp[(long)m * D + h * 64 + lane + 32] = rp.y;
}

}  // namespace avsr

using namespace avsr;

extern "C" {

size_t avsr_relpos_attention_bwd_workspace_bytes(int B, int T, int H) {
  if (B <= 0 || T <= 0 || H <= 0) return 256;
  return align_up((size_t)2 * B * H * T * sizeof(float), 256) + 256;
}

int avsr_relpos_attention_bwd(const float* q, const float* k, const float* v, const float* p, const float* pos_bias_u,
                              const float* pos_bias_v, const int32_t* lengths, const float* ctx, const float* dctx,
                              float* dq_k, float* dq_p, float* dk, float* dv, float* dp, int B, int T, int H,
                              void* workspace, size_t workspace_bytes, void* stream) {
  AVSR_REQUIRE(q && k && v && p && pos_bias_u && pos_bias_v && ctx && dctx && dq_k && dq_p && dk && dv && dp && workspace,
               "NULL argument");
  if (B <= 0 || T <= 0) return AVSR_OK;
  AVSR_REQUIRE_BYTES(avsr_relpos_attention_bwd_workspace_bytes(B, T, H), workspace_bytes, "attention backward workspace");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* lse = reinterpret_cast<float*>(workspace);
  float* delta = lse + (size_t)B * H * T;
  dim3 block(32 * kAbWarps);
  attn_bwd_rows_kernel<<<dim3(cdiv(T, kAbWarps), H, B), block, 0, st>>>(q, k, v, p, pos_bias_u, pos_bias_v, lengths, ctx, dctx, lse,
                                                                         delta, dq_k, dq_p, T, H);
  AVSR_CHECK_LAUNCH();
  attn_bwd_keys_kernel<<<dim3(cdiv(T, kAbWarps), H, B), block, 0, st>>>(q, k, v, p, pos_bias_u, pos_bias_v, lengths, dctx, lse, delta,
                                                                         dk, dv, T, H);
  AVSR_CHECK_LAUNCH();
  static const cudaError_t pos_attr =
      cudaFuncSetAttribute(attn_bwd_pos_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPosSmemBytes);
  AVSR_REQUIRE(pos_attr == cudaSuccess, "attention backward: shared memory opt-in failed");
  attn_bwd_pos_kernel<<<dim3(cdiv(2 * T - 1, kAbWarps), H), block, kPosSmemBytes, st>>>(q, k, v, p, pos_bias_u, pos_bias_v, lengths, dctx, lse,
                                                                             delta, dp, B, T, H);
  AVSR_CHECK_LAUNCH();
  return AVSR_OK;
}

}  // extern "C"
