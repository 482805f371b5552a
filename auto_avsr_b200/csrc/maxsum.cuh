// Running (max, sum of exp, arg max) of a row: the one-read log-sum-exp used by the row-wise log-softmax (head.cu) and
// by the CTC loss's row passes (ctc_loss.cu).
#pragma once
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

// Combine the per-thread triples of a 256-thread CTA (warp shuffles, then warp 0's fixed-order merge of the 8 warp
// results) and hand the total to every thread.  Contains two __syncthreads(): all threads of the CTA must call it.
__device__ __forceinline__ MaxSum ms_block_reduce_256(MaxSum acc) {
  __shared__ MaxSum part[8];
  __shared__ MaxSum total;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
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
    total = t;
  }
  __syncthreads();
  return total;
}

}  // namespace avsr
