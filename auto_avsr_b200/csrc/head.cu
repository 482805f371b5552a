// The step behind the encoder (SURVEY.md 8f #1): row-wise log-softmax / argmax over the CTC vocabulary
// (espnet/nets/pytorch_backend/ctc.py:77-93).  The logits come from the same GEMMs as every other projection
// (avsr_linear with ctc_lo's weight padded to a multiple of 128 rows); this kernel normalises the first `n` columns.
//
// One 256-thread CTA per row.  Pass 1 keeps a running (max, sum of exp, arg max) per thread -- one read of the row,
// float4 where the padded GEMM output allows it -- then a warp-shuffle + shared-memory reduction of the triples;
// pass 2 re-reads the row (20 KB: still in L1/L2) and writes x - (max + log sum).  HBM-bound: 4 B read + 4 B
// written per logit.
#include "common.cuh"

namespace avsr {

struct MaxSum {
  float m, s;   // running max, sum of exp(x - m)
  int i;        // index of the first maximal element
};

__device__ __forceinline__ void ms_push(MaxSum& a, float x, int idx) {
  if (x > a.m) {
    a.s = a.s * __expf(a.m - x) + 1.f;   // a.m = -inf on the first element: exp(-inf) = 0
    a.m = x;
    a.i = idx;
  } else {
    a.s += (x == -INFINITY) ? 0.f : __expf(x - a.m);   // x = m = -inf would give exp(nan); F.log_softmax ignores -inf logits
  }
}

__device__ __forceinline__ MaxSum ms_merge(const MaxSum& a, const MaxSum& b) {
  MaxSum r;
  const bool take_b = b.m > a.m || (b.m == a.m && b.i < a.i);
  r.m = take_b ? b.m : a.m;
  r.i = take_b ? b.i : a.i;
  const float ea = a.m == -INFINITY ? 0.f : __expf(a.m - r.m);
  const float eb = b.m == -INFINITY ? 0.f : __expf(b.m - r.m);
  r.s = a.s * ea + b.s * eb;
  return r;
}

__global__ void __launch_bounds__(256) log_softmax_rows_kernel(const float* __restrict__ x, long ldx,
                                                               float* __restrict__ y, long ldy,
                                                               int32_t* __restrict__ best, int rows, int n) {
  pdl_launch_dependents();
  const int row = blockIdx.x;
  const float* xr = x + (long)row * ldx;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __shared__ MaxSum part[8];
  __shared__ float s_shift;
  pdl_wait();

  MaxSum acc{-INFINITY, 0.f, 0x7fffffff};
  const bool vec = ((reinterpret_cast<uintptr_t>(xr) & 15) == 0);
  const int n4 = vec ? (n & ~3) : 0;
  for (int c = threadIdx.x * 4; c < n4; c += 256 * 4) {
    const float4 v = *reinterpret_cast<const float4*>(xr + c);
    ms_push(acc, v.x, c); ms_push(acc, v.y, c + 1); ms_push(acc, v.z, c + 2); ms_push(acc, v.w, c + 3);
  }
  for (int c = n4 + threadIdx.x; c < n; c += 256) ms_push(acc, xr[c], c);

#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    MaxSum o;
    o.m = __shfl_xor_sync(0xffffffffu, acc.m, off);
    o.s = __shfl_xor_sync(0xffffffffu, acc.s, off);
    o.i = __shfl_xor_sync(0xffffffffu, acc.i, off);
    acc = ms_merge(acc, o);
  }
  if (lane == 0) part[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    MaxSum t = part[0];
    for (int w = 1; w < 8; ++w) t = ms_merge(t, part[w]);
    s_shift = t.m + logf(t.s);
    if (best) best[row] = t.i;
  }
  __syncthreads();
  if (!y) return;
  const float shift = s_shift;
  float* yr = y + (long)row * ldy;
  for (int c = threadIdx.x; c < n; c += 256) yr[c] = xr[c] - shift;
}

int launch_log_softmax_rows(const float* x, long ldx, float* y, long ldy, int32_t* best, int rows, int n, cudaStream_t st) {
  if (rows <= 0) return AVSR_OK;
  AVSR_LAUNCH(log_softmax_rows_kernel, rows, 256, 0, st, x, ldx, y, ldy, best, rows, n);
  return AVSR_OK;
}

}  // namespace avsr

using namespace avsr;

extern "C" int avsr_log_softmax(const float* x, long ldx, float* y, long ldy, int32_t* argmax, int rows, int n,
                                void* stream) {
  AVSR_REQUIRE(x && (y || argmax), "NULL argument");
  AVSR_REQUIRE(rows >= 0 && n > 0 && ldx >= n && (!y || ldy >= n), "log_softmax: bad rows=%d n=%d ldx=%ld ldy=%ld",
               rows, n, ldx, ldy);
  if (rows == 0) return AVSR_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  AVSR_LAUNCH(log_softmax_rows_kernel, rows, 256, 0, st, x, ldx, y, ldy, argmax, rows, n);
  return AVSR_OK;
}
