// The step behind the encoder (SURVEY.md 8f #1): row-wise log-softmax / argmax over the CTC vocabulary
// (espnet/nets/pytorch_backend/ctc.py:77-93).  The logits come from the same GEMMs as every other projection
// (avsr_linear with ctc_lo's weight padded to a multiple of 128 rows); this kernel normalises the first `n` columns.
//
// One 256-thread CTA per row.  Pass 1 keeps a running (max, sum of exp, arg max) per thread -- one read of the row,
// float4 where the padded GEMM output allows it -- then a warp-shuffle + shared-memory reduction of the triples;
// pass 2 re-reads the row (20 KB: still in L1/L2) and writes x - (max + log sum).  HBM-bound: 4 B read + 4 B
// written per logit.
#include "maxsum.cuh"

namespace avsr {

__global__ void __launch_bounds__(256) log_softmax_rows_kernel(const float* __restrict__ x, long ldx,
                                                               float* __restrict__ y, long ldy,
                                                               int32_t* __restrict__ best, int rows, int n) {
  pdl_launch_dependents();
  const int row = blockIdx.x;
  const float* xr = x + (long)row * ldx;
  pdl_wait();

  MaxSum acc{-INFINITY, 0.f, 0x7fffffff};
  const bool vec = ((reinterpret_cast<uintptr_t>(xr) & 15) == 0);
  const int n4 = vec ? (n & ~3) : 0;
  for (int c = threadIdx.x * 4; c < n4; c += 256 * 4) {
    const float4 v = *reinterpret_cast<const float4*>(xr + c);
    ms_push(acc, v.x, c); ms_push(acc, v.y, c + 1); ms_push(acc, v.z, c + 2); ms_push(acc, v.w, c + 3);
  }
  for (int c = n4 + threadIdx.x; c < n; c += 256) ms_push(acc, xr[c], c);

  const MaxSum t = ms_block_reduce_256(acc);
  if (best && threadIdx.x == 0) best[row] = t.i;
  if (!y) return;
  const float shift = t.m + logf(t.s);
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
