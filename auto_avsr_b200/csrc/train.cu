// Training slice of the encoder path (SURVEY.md 8f #2, first slice): backward of the HBM-bound kernels and the pieces a
// Linear's backward needs around the tensor-core GEMMs -- LayerNorm backward, bias gradients (column sums), fp32
// operand packing (so that dgrad / wgrad are the SAME wgmma GEMMs on transposed operands), ReLU backward, the depthwise
// conv's forward / backward, and the batch-statistics BatchNorm [+ SiLU] of the conformer conv module and the front-end
// convolutions, forward / backward incl. the running-statistics update.
// Reference: lightning.py:86-94 (training_step), conformer_encoder.py:26,30-35 (BatchNorm1d in train mode sees ALL B*T
// frames incl. padding), layer_norm.py:21, positionwise_feed_forward.py:28-30.  fp32 math; every cross-row reduction is
// a two-stage (per-CTA partials, fixed-order finish) sum: results do not depend on scheduling.
#include <math.h>

#include "common.cuh"

namespace avsr {

constexpr int kRedBlocks = 132;      // first-stage CTAs of every column reduction (one per SM)
constexpr int kTrMaxVec = 8;         // float4 per lane: rows of up to 1024 channels

// ------------------------------------------------------------------ LayerNorm backward
// x_hat = (x - mu) * rstd ; g = dy * gamma ; dx = rstd * (g - mean(g) - x_hat * mean(g * x_hat))
// dgamma = sum_rows dy * x_hat ; dbeta = sum_rows dy.   One warp per row (row in registers); a CTA of 8 warps walks a
// contiguous block of rows, keeps per-lane column partials of dgamma / dbeta in registers, combines its warps through
// shared memory and writes ONE partial row pair to part[blockIdx][2][d].
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                            const float* __restrict__ dy, float* __restrict__ dx,
                                                            float* __restrict__ part, int rows, int d, int rows_per_cta) {
  extern __shared__ float ln_bwd_smem[];   // [8 warps][2][d]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nvec = d >> 2;
  float4 gg[kTrMaxVec], ag[kTrMaxVec], ab[kTrMaxVec];
#pragma unroll
  for (int i = 0; i < kTrMaxVec; ++i) {
    const int c = i * 32 + lane;
    ag[i] = ab[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < nvec) gg[i] = reinterpret_cast<const float4*>(gamma)[c];
  }
  const int r0 = blockIdx.x * rows_per_cta;
  const int r1 = min(rows, r0 + rows_per_cta);
  for (int row = r0 + warp; row < r1; row += 8) {
    const float4* xr = reinterpret_cast<const float4*>(x) + (long)row * nvec;
    const float4* dr = reinterpret_cast<const float4*>(dy) + (long)row * nvec;
    float4 v[kTrMaxVec], g[kTrMaxVec];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kTrMaxVec; ++i) {
      const int c = i * 32 + lane;
      if (c < nvec) { v[i] = xr[c]; g[i] = dr[c]; s += (v[i].x + v[i].y) + (v[i].z + v[i].w); }
    }
    const float mean = warp_sum(s) / (float)d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < kTrMaxVec; ++i)
      if (i * 32 + lane < nvec) {
        v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
        q += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
      }
    const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)d + 1e-12f);
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int i = 0; i < kTrMaxVec; ++i)
      if (i * 32 + lane < nvec) {
        v[i].x *= rstd; v[i].y *= rstd; v[i].z *= rstd; v[i].w *= rstd;                      // x_hat
        ab[i].x += g[i].x; ab[i].y += g[i].y; ab[i].z += g[i].z; ab[i].w += g[i].w;          // dbeta partial
        ag[i].x += g[i].x * v[i].x; ag[i].y += g[i].y * v[i].y; ag[i].z += g[i].z * v[i].z; ag[i].w += g[i].w * v[i].w;
        g[i].x *= gg[i].x; g[i].y *= gg[i].y; g[i].z *= gg[i].z; g[i].w *= gg[i].w;          // g = dy * gamma
        sg += (g[i].x + g[i].y) + (g[i].z + g[i].w);
        sgx += (g[i].x * v[i].x + g[i].y * v[i].y) + (g[i].z * v[i].z + g[i].w * v[i].w);
      }
    const float mg = warp_sum(sg) / (float)d, mgx = warp_sum(sgx) / (float)d;
    float4* dxr = reinterpret_cast<float4*>(dx) + (long)row * nvec;
#pragma unroll
    for (int i = 0; i < kTrMaxVec; ++i) {
      const int c = i * 32 + lane;
      if (c < nvec)
        dxr[c] = make_float4(rstd * (g[i].x - mg - v[i].x * mgx), rstd * (g[i].y - mg - v[i].y * mgx),
                             rstd * (g[i].z - mg - v[i].z * mgx), rstd * (g[i].w - mg - v[i].w * mgx));
    }
  }
  float4* sm = reinterpret_cast<float4*>(ln_bwd_smem);     // [8][2][nvec]
#pragma unroll
  for (int i = 0; i < kTrMaxVec; ++i) {
    const int c = i * 32 + lane;
    if (c < nvec) { sm[(warp * 2 + 0) * nvec + c] = ag[i]; sm[(warp * 2 + 1) * nvec + c] = ab[i]; }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * nvec; c += 256) {
    const int which = c / nvec, cc = c - which * nvec;
    float4 t = sm[(0 * 2 + which) * nvec + cc];
    for (int w = 1; w < 8; ++w) {
      const float4 u = sm[(w * 2 + which) * nvec + cc];
      t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
    }
    reinterpret_cast<float4*>(part)[((long)blockIdx.x * 2 + which) * nvec + cc] = t;
  }
}

// out[j] = sum_b part[b][j], fixed order (j over `width` floats)
__global__ void reduce_partials_kernel(const float* __restrict__ part, float* __restrict__ out, int nblk, int width) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= width) return;
  float t = 0.f;
  for (int b = 0; b < nblk; ++b) t += part[(long)b * width + j];
  out[j] = t;
}

// ------------------------------------------------------------------ column sums: out[c] = sum_r y[r][c]   (bias gradients)
__global__ void __launch_bounds__(256) colsum_partial_kernel(const float* __restrict__ y, float* __restrict__ part, int rows,
                                                             int cols, int rows_per_cta) {
  const int r0 = blockIdx.x * rows_per_cta, r1 = min(rows, r0 + rows_per_cta);
  for (int c = threadIdx.x; c < cols; c += 256) {
    float t = 0.f;
    for (int r = r0; r < r1; ++r) t += y[(long)r * cols + c];
    part[(long)blockIdx.x * cols + c] = t;
  }
}

// ------------------------------------------------------------------ fp32 -> GEMM operands of kind KIND, zero padding
// (OP_F32 or OP_BF16; a compile-time kind: the runtime-kind branch per store measured 2-3 % slower)
// transposed: (rows x cols) -> (cols x ld_dst), dst[c][r]; tiles of 32 x 32 through shared memory, the padding columns
// [rows, ld_dst) written as zeros
template <int KIND>
__global__ void pack_t_kernel(const float* __restrict__ src, void* __restrict__ dst, int rows, int cols, long ld_dst) {
  __shared__ float tile[32][33];
  const int c0 = blockIdx.y * 32, r0 = blockIdx.x * 32;
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int r = r0 + j, c = c0 + threadIdx.x;
    tile[j][threadIdx.x] = (r < rows && c < cols) ? src[(long)r * cols + c] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (c < cols && r < ld_dst) store_kind1(dst, (long)c * ld_dst + r, KIND, tile[threadIdx.x][j]);
  }
}
// not transposed: (rows x cols) -> (rows x ld_dst), the padding columns [cols, ld_dst) written as zeros
template <int KIND>
__global__ void pack_kernel(const float* __restrict__ src, void* __restrict__ dst, int rows, int cols, long ld_dst) {
  const long total = (long)rows * ld_dst;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / ld_dst;
    const int c = (int)(i - r * ld_dst);
    store_kind1(dst, i, KIND, c < cols ? src[r * cols + c] : 0.f);
  }
}

// ------------------------------------------------------------------ ReLU backward: dx = dy * (y > 0)
__global__ void relu_bwd_kernel(const float4* __restrict__ y, const float4* __restrict__ dy, float4* __restrict__ dx, long n4) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    const float4 a = y[i], g = dy[i];
    dx[i] = make_float4(a.x > 0.f ? g.x : 0.f, a.y > 0.f ? g.y : 0.f, a.z > 0.f ? g.z : 0.f, a.w > 0.f ? g.w : 0.f);
  }
}

// ------------------------------------------------------------------ GLU over channels: y[r][c] = a * sigmoid(g), a = in[r][c], g = in[r][C + c]
__global__ void glu_fwd_kernel(const float* __restrict__ in, float* __restrict__ y, long rows, int C) {
  const long n = rows * C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long r = i / C;
    const int c = (int)(i - r * C);
    y[i] = in[r * 2 * C + c] * sigmoidf_acc(in[r * 2 * C + C + c]);
  }
}
// d_a = dy * sig(g) ; d_g = dy * a * sig(g) * (1 - sig(g))
__global__ void glu_bwd_kernel(const float* __restrict__ in, const float* __restrict__ dy, float* __restrict__ din, long rows, int C) {
  const long n = rows * C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long r = i / C;
    const int c = (int)(i - r * C);
    const float a = in[r * 2 * C + c], s = sigmoidf_acc(in[r * 2 * C + C + c]), g = dy[i];
    din[r * 2 * C + c] = g * s;
    din[r * 2 * C + C + c] = g * a * s * (1.0f - s);
  }
}

// ------------------------------------------------------------------ BatchNorm with batch statistics (training)
// The conformer conv module's BatchNorm1d and the front-end convolutions' BatchNorm2d share these kernels.  Statistics:
// per-tile (count, mean, M2) of every channel, merged in a fixed order with Chan's formula in fp64 (no one-pass
// variance).  Normalise [+ residual] [+ SiLU]; the backward's per-tile [sum ds, sum ds * x_hat] are summed in fp64.
// A tile is bn_tile_rows() rows of 128 channels.

// rows per tile: 256, halved (down to 32) while the grid would hold fewer than two CTAs per SM
static int bn_tile_rows(long rows, int C) {
  int h = 256;
  while (h > 32 && (rows + h - 1) / h * cdiv(C, 128) < 2 * 132) h >>= 1;
  return h;
}

// per-tile (count, mean, M2) of each channel of z (rows, C): part[tile][3][C].  Both passes sum z - (the tile's first
// row) in fp32, so a channel whose mean lies many standard deviations from 0 keeps its mean and variance.
__global__ void __launch_bounds__(128) bn_stats_partial_kernel(const float* __restrict__ z, double* __restrict__ part,
                                                               long rows, int C, int tile_rows) {
  pdl_wait();
  const int c = blockIdx.y * 128 + threadIdx.x;
  if (c >= C) return;
  const long r0 = (long)blockIdx.x * tile_rows, r1 = min(rows, r0 + tile_rows);
  const int n = (int)(r1 - r0);
  const float z0 = z[r0 * C + c];
  float s = 0.f;
  for (long r = r0; r < r1; ++r) s += z[r * C + c] - z0;
  const float dm = s / (float)n;
  float q = 0.f;
  for (long r = r0; r < r1; ++r) { const float d = (z[r * C + c] - z0) - dm; q = fmaf(d, d, q); }
  double* p = part + (long)blockIdx.x * 3 * C;
  p[c] = n; p[C + c] = (double)z0 + (double)dm; p[2 * C + c] = q;
}

__device__ __forceinline__ void chan_merge(double& n, double& m, double& q, double nb, double mb, double qb) {
  if (nb == 0.0) return;
  const double nn = n + nb, d = mb - m;
  m += d * (nb / nn);
  q += qb + d * d * (n * nb / nn);
  n = nn;
}

// one CTA per channel: thread t merges tiles t, t + 256, ... in order, then a fixed tree; out[3][C]
__global__ void __launch_bounds__(256) bn_stats_merge_kernel(const double* __restrict__ part, int tiles, int C,
                                                             double* __restrict__ out) {
  pdl_wait();
  __shared__ double sn[256], sm[256], sq[256];
  const int c = blockIdx.x, t = threadIdx.x;
  double n = 0, m = 0, q = 0;
  for (int i = t; i < tiles; i += 256) {
    const double* p = part + (long)i * 3 * C;
    chan_merge(n, m, q, p[c], p[C + c], p[2 * C + c]);
  }
  sn[t] = n; sm[t] = m; sq[t] = q;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (t < h) {
      double a = sn[t], b = sm[t], e = sq[t];
      chan_merge(a, b, e, sn[t + h], sm[t + h], sq[t + h]);
      sn[t] = a; sm[t] = b; sq[t] = e;
    }
    __syncthreads();
  }
  if (t == 0) { out[c] = sn[0]; out[C + c] = sm[0]; out[2 * C + c] = sq[0]; }
}

// merge R ranks' (count, mean, M2) in rank order; mean, 1/sqrt(var + eps) with the biased variance; running statistics
// (when given) move by `factor` toward the mean and the unbiased variance
__global__ void bn_finalize_kernel(const double* __restrict__ st, int R, int C, double eps, double factor,
                                   float* __restrict__ running_mean, float* __restrict__ running_var,
                                   float* __restrict__ mean, float* __restrict__ invstd) {
  pdl_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double n = 0, m = 0, q = 0;
  for (int r = 0; r < R; ++r) chan_merge(n, m, q, st[(long)r * 3 * C + c], st[(long)r * 3 * C + C + c],
                                         st[(long)r * 3 * C + 2 * C + c]);
  const double var = n > 0 ? q / n : 0.0;
  mean[c] = (float)m;
  invstd[c] = (float)(1.0 / sqrt(var + eps));
  if (running_mean) {
    const double unb = n > 1 ? q / (n - 1) : var;
    running_mean[c] = (float)((1.0 - factor) * running_mean[c] + factor * m);
    running_var[c] = (float)((1.0 - factor) * running_var[c] + factor * unb);
  }
}

// ds = dL/dh of y = silu(h): dy * sig(h) * (1 + h * (1 - sig(h)))
__device__ __forceinline__ float silu_grad_acc(float h, float dy) {
  const float s = sigmoidf_acc(h);
  return dy * s * (1.0f + h * (1.0f - s));
}

// y = [SiLU]((z - mean) * invstd * gamma + beta [+ resid])
__global__ void bn_act_fwd_kernel(const float* __restrict__ z, const float* __restrict__ mean,
                                  const float* __restrict__ invstd, const float* __restrict__ gamma,
                                  const float* __restrict__ beta, const float* __restrict__ resid, int act,
                                  float* __restrict__ y, long n, int C) {
  pdl_wait();
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    float h = (z[i] - mean[c]) * invstd[c] * gamma[c] + beta[c];
    if (resid) h += resid[i];
    y[i] = act ? h * sigmoidf_acc(h) : h;
  }
}

// ds = dL/d(BN output): dy, through SiLU when act; per-tile [sum ds, sum ds * x_hat]: part[tile][2][C] (fp64)
__global__ void __launch_bounds__(128) bn_bwd_partial_kernel(const float* __restrict__ z, const float* __restrict__ dy,
                                                             const float* __restrict__ mean,
                                                             const float* __restrict__ invstd,
                                                             const float* __restrict__ gamma,
                                                             const float* __restrict__ beta,
                                                             const float* __restrict__ resid, int act,
                                                             double* __restrict__ part, long rows, int C,
                                                             int tile_rows) {
  pdl_wait();
  const int c = blockIdx.y * 128 + threadIdx.x;
  if (c >= C) return;
  const long r0 = (long)blockIdx.x * tile_rows, r1 = min(rows, r0 + tile_rows);
  const float m = mean[c], is = invstd[c], g = gamma[c], b = beta[c];
  float s = 0.f, q = 0.f;
  for (long r = r0; r < r1; ++r) {
    const long i = r * C + c;
    const float xh = (z[i] - m) * is;
    float ds = dy[i];
    if (act) ds = silu_grad_acc(xh * g + b + (resid ? resid[i] : 0.f), ds);
    s += ds;
    q = fmaf(ds, xh, q);
  }
  part[(long)blockIdx.x * 2 * C + c] = s;
  part[(long)blockIdx.x * 2 * C + C + c] = q;
}

// out[j] = sum_t part[t][j] in fp64, one CTA per column j: strided per-thread sums, then a fixed tree
__global__ void __launch_bounds__(256) bn_sum_merge_kernel(const double* __restrict__ part, int tiles, int width,
                                                           float* __restrict__ out) {
  pdl_wait();
  __shared__ double sh[256];
  const int j = blockIdx.x, t = threadIdx.x;
  double s = 0;
  for (int i = t; i < tiles; i += 256) s += part[(long)i * width + j];
  sh[t] = s;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (t < h) sh[t] += sh[t + h];
    __syncthreads();
  }
  if (t == 0) out[j] = (float)sh[0];
}

// dz = gamma * invstd * (ds - (sum ds + x_hat * sum ds x_hat) / count); dres (when given) = ds
__global__ void bn_bwd_dx_kernel(const float* __restrict__ z, const float* __restrict__ dy,
                                 const float* __restrict__ mean, const float* __restrict__ invstd,
                                 const float* __restrict__ gamma, const float* __restrict__ beta,
                                 const float* __restrict__ resid, int act, const float* __restrict__ sums,
                                 float inv_count, float* __restrict__ dz, float* __restrict__ dres, long n, int C) {
  pdl_wait();
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const float g = gamma[c], is = invstd[c];
    const float xh = (z[i] - mean[c]) * is;
    float ds = dy[i];
    if (act) ds = silu_grad_acc(xh * g + beta[c] + (resid ? resid[i] : 0.f), ds);
    if (dres) dres[i] = ds;
    dz[i] = g * is * (ds - inv_count * (sums[c] + xh * sums[C + c]));
  }
}

int launch_bn_stats(const float* z, long rows, int C, double* part, double* stats, cudaStream_t st) {
  const int h = bn_tile_rows(rows, C), tiles = (int)((rows + h - 1) / h);
  AVSR_LAUNCH(bn_stats_partial_kernel, dim3(tiles, cdiv(C, 128)), 128, 0, st, z, part, rows, C, h);
  AVSR_LAUNCH(bn_stats_merge_kernel, C, 256, 0, st, (const double*)part, tiles, C, stats);
  return AVSR_OK;
}
// ------------------------------------------------------------------ depthwise conv backward: tap / bias gradients
// dw[c][k] = sum_{b,t} x[b, t+k-half, c] * dconv[b,t,c] ; db[c] = sum dconv.  part[blk][K+1][C], one CTA per block of
// (utterance, frame range); threads over channels (coalesced along C).
__global__ void __launch_bounds__(256) dwconv_wgrad_partial_kernel(const float* __restrict__ x, const float* __restrict__ dconv,
                                                                   float* __restrict__ part, int B, int T, int C, int K,
                                                                   int frames_per_cta, int ctas_per_utt) {
  const int b = blockIdx.x / ctas_per_utt, seg = blockIdx.x - b * ctas_per_utt;
  const int t0 = seg * frames_per_cta, t1 = min(T, t0 + frames_per_cta);
  const int half = (K - 1) >> 1;
  const float* xb = x + (long)b * T * C;
  const float* db_ = dconv + (long)b * T * C;
  for (int c = threadIdx.x; c < C; c += 256) {
    float bsum = 0.f;
    for (int t = t0; t < t1; ++t) bsum += db_[(long)t * C + c];
    part[((long)blockIdx.x * (K + 1) + K) * C + c] = bsum;
    for (int k = 0; k < K; ++k) {
      float acc = 0.f;
      for (int t = t0; t < t1; ++t) {
        const int ts = t + k - half;
        if (ts >= 0 && ts < T) acc += xb[(long)ts * C + c] * db_[(long)t * C + c];
      }
      part[((long)blockIdx.x * (K + 1) + k) * C + c] = acc;
    }
  }
}
// dw (C,1,K) / db (C) from part[nblk][K+1][C]
__global__ void dwconv_wgrad_finish_kernel(const float* __restrict__ part, float* __restrict__ dw, float* __restrict__ db, int nblk,
                                           int C, int K) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (K + 1) * C) return;
  const int k = i / C, c = i - k * C;
  float t = 0.f;
  for (int b = 0; b < nblk; ++b) t += part[((long)b * (K + 1) + k) * C + c];
  if (k == K) db[c] = t; else dw[(long)c * K + k] = t;
}
// taps (C,1,K) -> (K,C), optionally reversed along k (the input gradient is the correlation with the flipped taps)
__global__ void dw_taps_kernel(const float* __restrict__ w, float* __restrict__ wt, int C, int K, int flip) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= K * C) return;
  const int k = i / C, c = i - k * C;
  wt[i] = w[(long)c * K + (flip ? K - 1 - k : k)];
}
__global__ void fill_kernel(float* p, int n, float v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

static inline int grid_for(long n, int per = 256, int cap = 132 * 8) {
  long g = (n + per - 1) / per;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace avsr

using namespace avsr;

extern "C" {

size_t avsr_train_workspace_bytes(int rows, int d, int K) {
  // the largest user: dwconv_bn_silu_train_bwd = taps (K+2)*C + partials nblk*(K+1)*C (+ BN partials) + dconv rows*C
  if (rows < 0 || d <= 0 || K < 1) return 0;
  const size_t C = (size_t)d;
  return (((size_t)(K + 4) * C) + (size_t)4 * kRedBlocks * (K + 1) * C + (size_t)rows * C + 4 * C) * sizeof(float) + 1024;
}

int avsr_layernorm_bwd(const float* x, const float* gamma, const float* dy, float* dx, float* dgamma, float* dbeta,
                       int rows, int d, void* workspace, size_t workspace_bytes, void* stream) {
  AVSR_REQUIRE(gamma && dgamma && dbeta, "NULL argument");
  AVSR_REQUIRE(d > 0 && d % 4 == 0 && d <= kTrMaxVec * 128, "layernorm_bwd: d=%d must be a multiple of 4 and <= 1024", d);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (rows <= 0) {               // no rows: zero dgamma / dbeta (x, dy, dx of an empty batch may be NULL)
    AVSR_CUDA_TRY(cudaMemsetAsync(dgamma, 0, d * sizeof(float), st));
    AVSR_CUDA_TRY(cudaMemsetAsync(dbeta, 0, d * sizeof(float), st));
    return AVSR_OK;
  }
  AVSR_REQUIRE(x && dy && dx && workspace, "NULL argument");
  const int nblk = rows < kRedBlocks * 8 ? cdiv(rows, 8) : kRedBlocks;
  const int rpc = cdiv(rows, nblk);
  const int nb = cdiv(rows, rpc);
  AVSR_REQUIRE_BYTES((size_t)nb * 2 * d * sizeof(float), workspace_bytes, "layernorm_bwd workspace");
  float* part = reinterpret_cast<float*>(workspace);
  const size_t smem = (size_t)8 * 2 * d * sizeof(float);
  if (smem > 48 * 1024)
    AVSR_CUDA_TRY(cudaFuncSetAttribute(layernorm_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  layernorm_bwd_kernel<<<nb, 256, smem, st>>>(x, gamma, dy, dx, part, rows, d, rpc);
  AVSR_CHECK_LAUNCH();
  // part[b][0][:] -> dgamma, part[b][1][:] -> dbeta : reduce with width 2*d into a temporary, then split
  float* tmp = part + (size_t)nb * 2 * d;
  AVSR_REQUIRE_BYTES(((size_t)nb * 2 * d + 2 * d) * sizeof(float), workspace_bytes, "layernorm_bwd workspace");
  reduce_partials_kernel<<<cdiv(2 * d, 256), 256, 0, st>>>(part, tmp, nb, 2 * d);
  AVSR_CHECK_LAUNCH();
  AVSR_CUDA_TRY(cudaMemcpyAsync(dgamma, tmp, d * sizeof(float), cudaMemcpyDeviceToDevice, st));
  AVSR_CUDA_TRY(cudaMemcpyAsync(dbeta, tmp + d, d * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return AVSR_OK;
}

int avsr_colsum(const float* y, float* out, int rows, int cols, void* workspace, size_t workspace_bytes, void* stream) {
  AVSR_REQUIRE(y && out && workspace && cols > 0, "NULL / bad argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (rows <= 0) { AVSR_CUDA_TRY(cudaMemsetAsync(out, 0, cols * sizeof(float), st)); return AVSR_OK; }
  const int rpc = cdiv(rows, kRedBlocks), nb = cdiv(rows, rpc);
  AVSR_REQUIRE_BYTES((size_t)nb * cols * sizeof(float), workspace_bytes, "colsum workspace");
  float* part = reinterpret_cast<float*>(workspace);
  colsum_partial_kernel<<<nb, 256, 0, st>>>(y, part, rows, cols, rpc);
  AVSR_CHECK_LAUNCH();
  reduce_partials_kernel<<<cdiv(cols, 256), 256, 0, st>>>(part, out, nb, cols);
  AVSR_CHECK_LAUNCH();
  return AVSR_OK;
}

int avsr_pack_operand(const float* src, void* dst, int rows, int cols, long ld_dst, int transpose, int precision,
                      void* stream) {
  AVSR_REQUIRE(src && dst, "NULL argument");
  AVSR_REQUIRE(precision == AVSR_PREC_FP32 || precision == AVSR_PREC_BF16,
               "pack_operand: precision %d is not built; AVSR_PREC_FP32 or AVSR_PREC_BF16", precision);
  AVSR_REQUIRE(rows >= 0 && cols >= 0 && ld_dst >= (transpose ? rows : cols), "pack_operand: bad rows=%d cols=%d ld=%ld",
               rows, cols, ld_dst);
  if (rows <= 0 || cols <= 0) return AVSR_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const bool bf16 = precision == AVSR_PREC_BF16;
  if (transpose) {
    auto* k = bf16 ? pack_t_kernel<OP_BF16> : pack_t_kernel<OP_F32>;
    k<<<dim3((unsigned)((ld_dst + 31) / 32), cdiv(cols, 32)), dim3(32, 8), 0, st>>>(src, dst, rows, cols, ld_dst);
  } else {
    auto* k = bf16 ? pack_kernel<OP_BF16> : pack_kernel<OP_F32>;
    k<<<132 * 4, 256, 0, st>>>(src, dst, rows, cols, ld_dst);
  }
  AVSR_CHECK_LAUNCH();
  return AVSR_OK;
}

// The operands of a Linear's backward GEMMs in the workspace: K padded to 128 bytes (gemm_tc takes K in 128-byte
// blocks), 32 fp32 elements or 64 bf16 ones.  TF32 operands are packed as plain fp32, unrounded: the tensor core
// truncates them, as it does the forward's.  dY is read in place for dX when its rows already have that layout (fp32 /
// TF32 with n a multiple of 32), so no copy of it is made.
struct LinearBwdOperands {
  int pack_prec;          // the avsr_pack_operand precision of every operand
  long np, rp;            // n and rows padded: K of dX and of dW
  bool dy_in_place;
  void *dy, *wt, *dyt, *xt;
  LinearBwdOperands(Carver& cv, int rows, int n, int k, int precision) {
    pack_prec = precision == AVSR_PREC_BF16 ? AVSR_PREC_BF16 : AVSR_PREC_FP32;
    const size_t es = operand_bytes(operand_kind(pack_prec));
    const long e = (long)(128 / es);
    np = (n + e - 1) / e * e;
    rp = (rows + e - 1) / e * e;
    dy_in_place = np == n && pack_prec == AVSR_PREC_FP32;
    dy = dy_in_place ? nullptr : cv.take<char>((size_t)rows * np * es);
    wt = cv.take<char>((size_t)k * np * es);
    dyt = cv.take<char>((size_t)n * rp * es);
    xt = cv.take<char>((size_t)k * rp * es);
  }
};

static bool linear_bwd_precision(int precision) {
  return precision == AVSR_PREC_FP32 || precision == AVSR_PREC_TF32 || precision == AVSR_PREC_BF16;
}

size_t avsr_linear_bwd_workspace_bytes(int rows, int n, int k, int precision) {
  if (!linear_bwd_precision(precision)) return 0;
  if (rows <= 0 || n <= 0 || k <= 0) return 256;
  Carver cv{nullptr};
  const LinearBwdOperands layout(cv, rows, n, k, precision);
  return cv.off;
}

int avsr_linear_bwd(const float* dy, const float* x, const float* w, float* dx, float* dw, int rows, int n, int k,
                    int precision, void* workspace, size_t workspace_bytes, void* stream) {
  AVSR_REQUIRE(linear_bwd_precision(precision),
               "linear_bwd: precision %d: AVSR_PREC_FP32, AVSR_PREC_TF32 or AVSR_PREC_BF16 (gradients overflow f16)",
               precision);
  AVSR_REQUIRE(dy && workspace && (dx || dw) && (!dx || w) && (!dw || x), "NULL argument");
  AVSR_REQUIRE(rows > 0 && n > 0 && k > 0, "linear_bwd: bad rows=%d n=%d k=%d", rows, n, k);
  AVSR_REQUIRE_BYTES(avsr_linear_bwd_workspace_bytes(rows, n, k, precision), workspace_bytes, "linear_bwd workspace");
  Carver cv{reinterpret_cast<char*>(workspace)};
  const LinearBwdOperands o(cv, rows, n, k, precision);
  if (dx) {   // dX (rows, k) = dY W = dY (W^T)^T: K = n
    if (!o.dy_in_place) AVSR_TRY(avsr_pack_operand(dy, o.dy, rows, n, o.np, 0, o.pack_prec, stream));
    AVSR_TRY(avsr_pack_operand(w, o.wt, n, k, o.np, 1, o.pack_prec, stream));
    AVSR_TRY(avsr_linear_operands(o.dy_in_place ? dy : o.dy, o.wt, nullptr, nullptr, 1.0f, dx, rows, k, (int)o.np, 0, 0,
                                  precision, stream));
  }
  if (dw) {   // dW (n, k) = dY^T X = dY^T (X^T)^T: K = rows
    AVSR_TRY(avsr_pack_operand(dy, o.dyt, rows, n, o.rp, 1, o.pack_prec, stream));
    AVSR_TRY(avsr_pack_operand(x, o.xt, rows, k, o.rp, 1, o.pack_prec, stream));
    AVSR_TRY(avsr_linear_operands(o.dyt, o.xt, nullptr, nullptr, 1.0f, dw, n, k, (int)o.rp, 0, 0, precision, stream));
  }
  return AVSR_OK;
}

int avsr_relu_bwd(const float* y, const float* dy, float* dx, long n, void* stream) {
  AVSR_REQUIRE(y && dy && dx && n % 4 == 0, "relu_bwd: NULL argument or n %% 4 != 0");
  if (n <= 0) return AVSR_OK;
  relu_bwd_kernel<<<grid_for(n / 4), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(y), reinterpret_cast<const float4*>(dy), reinterpret_cast<float4*>(dx), n / 4);
  AVSR_CHECK_LAUNCH();
  return AVSR_OK;
}

int avsr_glu_fwd(const float* in, float* y, long rows, int C, void* stream) {
  AVSR_REQUIRE(in && y && C > 0, "NULL / bad argument");
  if (rows <= 0) return AVSR_OK;
  glu_fwd_kernel<<<grid_for(rows * C), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(in, y, rows, C);
  AVSR_CHECK_LAUNCH();
  return AVSR_OK;
}

int avsr_glu_bwd(const float* in, const float* dy, float* din, long rows, int C, void* stream) {
  AVSR_REQUIRE(in && dy && din && C > 0, "NULL / bad argument");
  if (rows <= 0) return AVSR_OK;
  glu_bwd_kernel<<<grid_for(rows * C), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(in, dy, din, rows, C);
  AVSR_CHECK_LAUNCH();
  return AVSR_OK;
}

// ---- depthwise conv of the conformer conv module (its training BatchNorm is the avsr_bn_train_* below)

// y = depthwise_conv(x) + b (raw fp32; flip != 0: taps reversed along k and b may be NULL -- the input gradient)
int avsr_dwconv_raw(const float* x, const float* w, const float* b, float* y, int B, int T, int C, int K, int flip,
                    void* workspace, size_t workspace_bytes, void* stream) {
  AVSR_REQUIRE(x && w && y && workspace, "NULL argument");
  AVSR_REQUIRE(C > 0 && C % 4 == 0 && K >= 1 && K % 2 == 1, "dwconv: bad C=%d K=%d", C, K);
  if (B <= 0 || T <= 0) return AVSR_OK;
  AVSR_REQUIRE_BYTES((size_t)(K + 2) * C * sizeof(float), workspace_bytes, "dwconv_raw workspace");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* wt = reinterpret_cast<float*>(workspace);
  float *ones = wt + (size_t)K * C, *zeros = ones + C;
  dw_taps_kernel<<<cdiv(K * C, 256), 256, 0, st>>>(w, wt, C, K, flip);
  AVSR_CHECK_LAUNCH();
  fill_kernel<<<cdiv(C, 256), 256, 0, st>>>(ones, C, 1.0f);
  AVSR_CHECK_LAUNCH();
  AVSR_CUDA_TRY(cudaMemsetAsync(zeros, 0, C * sizeof(float), st));
  return launch_dwconv_bn_silu(x, wt, ones, b ? b : zeros, y, B, T, C, K, /*out_kind=*/-1, st);
}

// dw (C,1,K), db (C) of the depthwise conv from its input x and its output gradient dconv
int avsr_dwconv_wgrad(const float* x, const float* dconv, float* dw, float* db, int B, int T, int C, int K, void* workspace,
                      size_t workspace_bytes, void* stream) {
  AVSR_REQUIRE(x && dconv && dw && db && workspace, "NULL argument");
  if (B <= 0 || T <= 0) return AVSR_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int cpu_ = cdiv(kRedBlocks, B);
  if (cpu_ < 1) cpu_ = 1;
  const int fpc = cdiv(T, cpu_);
  cpu_ = cdiv(T, fpc);
  const int nbw = B * cpu_;
  AVSR_REQUIRE_BYTES((size_t)nbw * (K + 1) * C * sizeof(float), workspace_bytes, "dwconv_wgrad workspace");
  float* partw = reinterpret_cast<float*>(workspace);
  dwconv_wgrad_partial_kernel<<<nbw, 256, 0, st>>>(x, dconv, partw, B, T, C, K, fpc, cpu_);
  AVSR_CHECK_LAUNCH();
  dwconv_wgrad_finish_kernel<<<cdiv((K + 1) * C, 256), 256, 0, st>>>(partw, dw, db, nbw, C, K);
  AVSR_CHECK_LAUNCH();
  return AVSR_OK;
}

// ---- BatchNorm with batch statistics, in the pieces a (Sync)BatchNorm needs: the per-rank statistics and the backward
// sums leave the library between the pieces, so that the host can gather / all-reduce them over the ranks
// (torch.nn.SyncBatchNorm semantics, train.py:31) before they are used.

size_t avsr_bn_train_workspace_bytes(long rows, int C) {
  if (rows < 0 || C < 1) return 0;
  const int h = bn_tile_rows(rows, C);
  return align_up((size_t)((rows + h - 1) / h) * 3 * C * sizeof(double), 256) + 256;
}

int avsr_bn_train_stats(const float* z, long rows, int C, double* stats, void* workspace, size_t workspace_bytes,
                        void* stream) {
  AVSR_REQUIRE(rows >= 0 && C >= 1, "bn_train: bad rows=%ld C=%d", rows, C);
  AVSR_REQUIRE(stats && workspace, "NULL argument");
  AVSR_REQUIRE_BYTES(avsr_bn_train_workspace_bytes(rows, C), workspace_bytes, "bn_train workspace");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (rows == 0) {               // no rows (z may be NULL): count 0, which the rank merge skips
    AVSR_CUDA_TRY(cudaMemsetAsync(stats, 0, 3 * (size_t)C * sizeof(double), st));
    return AVSR_OK;
  }
  AVSR_REQUIRE(z, "NULL argument");
  double* part = reinterpret_cast<double*>(align_up(reinterpret_cast<uintptr_t>(workspace), 256));
  return launch_bn_stats(z, rows, C, part, stats, st);
}

int avsr_bn_train_finalize(const double* stats, int ranks, int C, double eps, double factor, float* running_mean,
                           float* running_var, float* mean, float* invstd, void* stream) {
  AVSR_REQUIRE(ranks >= 1 && C >= 1 && eps >= 0.0 && factor >= 0.0 && factor <= 1.0,
               "bn_train: bad ranks=%d C=%d eps or factor", ranks, C);
  AVSR_REQUIRE(stats && mean && invstd && (running_mean != nullptr) == (running_var != nullptr), "NULL argument");
  AVSR_LAUNCH(bn_finalize_kernel, cdiv(C, 128), 128, 0, reinterpret_cast<cudaStream_t>(stream), stats, ranks, C, eps,
              factor, running_mean, running_var, mean, invstd);
  return AVSR_OK;
}

int avsr_bn_train_act_fwd(const float* z, const float* mean, const float* invstd, const float* gamma, const float* beta,
                          const float* resid, int act, float* y, long rows, int C, void* stream) {
  AVSR_REQUIRE(rows >= 0 && C >= 1, "bn_train: bad rows=%ld C=%d", rows, C);
  AVSR_REQUIRE(z && mean && invstd && gamma && beta && y, "NULL argument");
  if (rows == 0) return AVSR_OK;
  AVSR_LAUNCH(bn_act_fwd_kernel, grid_for(rows * C, 256, 8192), 256, 0, reinterpret_cast<cudaStream_t>(stream), z, mean,
              invstd, gamma, beta, resid, act, y, rows * C, C);
  return AVSR_OK;
}

int avsr_bn_train_bwd_sums(const float* z, const float* dy, const float* mean, const float* invstd, const float* gamma,
                           const float* beta, const float* resid, int act, float* sums, long rows, int C,
                           void* workspace, size_t workspace_bytes, void* stream) {
  AVSR_REQUIRE(rows >= 1 && C >= 1, "bn_train: bad rows=%ld C=%d", rows, C);
  AVSR_REQUIRE(z && dy && mean && invstd && gamma && beta && sums && workspace, "NULL argument");
  AVSR_REQUIRE_BYTES(avsr_bn_train_workspace_bytes(rows, C), workspace_bytes, "bn_train backward workspace");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  double* part = reinterpret_cast<double*>(align_up(reinterpret_cast<uintptr_t>(workspace), 256));
  const int h = bn_tile_rows(rows, C), tiles = (int)((rows + h - 1) / h);
  AVSR_LAUNCH(bn_bwd_partial_kernel, dim3(tiles, cdiv(C, 128)), 128, 0, st, z, dy, mean, invstd, gamma, beta, resid,
              act, part, rows, C, h);
  AVSR_LAUNCH(bn_sum_merge_kernel, 2 * C, 256, 0, st, (const double*)part, tiles, 2 * C, sums);
  return AVSR_OK;
}

int avsr_bn_train_bwd_dx(const float* z, const float* dy, const float* mean, const float* invstd, const float* gamma,
                         const float* beta, const float* resid, int act, const float* sums, float inv_count, float* dz,
                         float* dres, long rows, int C, void* stream) {
  AVSR_REQUIRE(rows >= 0 && C >= 1, "bn_train: bad rows=%ld C=%d", rows, C);
  AVSR_REQUIRE(z && dy && mean && invstd && gamma && beta && sums && dz, "NULL argument");
  if (rows == 0) return AVSR_OK;
  AVSR_LAUNCH(bn_bwd_dx_kernel, grid_for(rows * C, 256, 8192), 256, 0, reinterpret_cast<cudaStream_t>(stream), z, dy,
              mean, invstd, gamma, beta, resid, act, sums, inv_count, dz, dres, rows * C, C);
  return AVSR_OK;
}

}  // extern "C"
