// Training slice of the encoder path (SURVEY.md 8f #2, first slice): backward of the HBM-bound kernels and the pieces a
// Linear's backward needs around the tensor-core GEMMs -- LayerNorm backward, bias gradients (column sums), fp32
// transpose (so that dgrad / wgrad are the SAME wgmma GEMMs on transposed operands), ReLU backward, and the
// depthwise-conv + BatchNorm(batch statistics) + SiLU block forward / backward incl. the running-statistics update.
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

// ------------------------------------------------------------------ fp32 transpose (rows x cols) -> (cols x rows)
__global__ void transpose_kernel(const float* __restrict__ src, float* __restrict__ dst, int rows, int cols, long ld_dst) {
  __shared__ float tile[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int r = r0 + j, c = c0 + threadIdx.x;
    tile[j][threadIdx.x] = (r < rows && c < cols) ? src[(long)r * cols + c] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (c < cols && r < rows) dst[(long)c * ld_dst + r] = tile[threadIdx.x][j];
  }
}

// ------------------------------------------------------------------ fp32 -> bf16 GEMM operands with zero padding
// transposed: (rows x cols) -> (cols x ld_dst), dst[c][r]; tiles of 32 x 32 through shared memory, the padding columns
// [rows, ld_dst) written as zeros
__global__ void pack_bf16_t_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int rows, int cols,
                                   long ld_dst) {
  __shared__ float tile[32][33];
  const int c0 = blockIdx.y * 32, r0 = blockIdx.x * 32;
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int r = r0 + j, c = c0 + threadIdx.x;
    tile[j][threadIdx.x] = (r < rows && c < cols) ? src[(long)r * cols + c] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (c < cols && r < ld_dst) dst[(long)c * ld_dst + r] = __float2bfloat16_rn(tile[threadIdx.x][j]);
  }
}
// not transposed: (rows x cols) -> (rows x ld_dst), the padding columns [cols, ld_dst) written as zeros
__global__ void pack_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int rows, int cols,
                                 long ld_dst) {
  const long total = (long)rows * ld_dst;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / ld_dst;
    const int c = (int)(i - r * ld_dst);
    dst[i] = __float2bfloat16_rn(c < cols ? src[r * cols + c] : 0.f);
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

// ------------------------------------------------------------------ BatchNorm (batch statistics) + SiLU
// per-channel partial sums of v - shift and (v - shift)^2 over a block of rows: part[blk][2][C] (shift NULL: 0).  With
// shift = a provisional mean the sums are centred, so the variance does not come from the difference of two large sums.
__global__ void __launch_bounds__(256) chan_stats_partial_kernel(const float* __restrict__ v, const float* __restrict__ shift,
                                                                 float* __restrict__ part, int rows, int C, int rows_per_cta) {
  const int r0 = blockIdx.x * rows_per_cta, r1 = min(rows, r0 + rows_per_cta);
  for (int c = threadIdx.x; c < C; c += 256) {
    const float m = shift ? shift[c] : 0.f;
    float s = 0.f, q = 0.f;
    for (int r = r0; r < r1; ++r) { const float t = v[(long)r * C + c] - m; s += t; q += t * t; }
    part[((long)blockIdx.x * 2) * C + c] = s;
    part[((long)blockIdx.x * 2 + 1) * C + c] = q;
  }
}
// y = silu((v - mean) * invstd * gamma + beta)
__global__ void bn_silu_fwd_kernel(const float4* __restrict__ v, const float* __restrict__ mean, const float* __restrict__ invstd,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, float4* __restrict__ y,
                                   long n4, int C4) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    const float4 a = v[i], m = reinterpret_cast<const float4*>(mean)[c], s = reinterpret_cast<const float4*>(invstd)[c];
    const float4 g = reinterpret_cast<const float4*>(gamma)[c], b = reinterpret_cast<const float4*>(beta)[c];
    float4 h = make_float4((a.x - m.x) * s.x * g.x + b.x, (a.y - m.y) * s.y * g.y + b.y, (a.z - m.z) * s.z * g.z + b.z,
                           (a.w - m.w) * s.w * g.w + b.w);
    y[i] = make_float4(h.x * sigmoidf_acc(h.x), h.y * sigmoidf_acc(h.y), h.z * sigmoidf_acc(h.z), h.w * sigmoidf_acc(h.w));
  }
}
// ds = dL/dh of y = silu(h): dy * sig(h) * (1 + h * (1 - sig(h)))
__device__ __forceinline__ float silu_grad(float h, float dy) {
  const float s = sigmoidf_acc(h);
  return dy * s * (1.0f + h * (1.0f - s));
}
// per-channel partial sums of ds and ds * x_hat (h recomputed from the saved conv output): part[blk][2][C]
__global__ void __launch_bounds__(256) bn_bwd_partial_kernel(const float* __restrict__ v, const float* __restrict__ dy,
                                                             const float* __restrict__ mean, const float* __restrict__ invstd,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             float* __restrict__ part, int rows, int C, int rows_per_cta) {
  const int r0 = blockIdx.x * rows_per_cta, r1 = min(rows, r0 + rows_per_cta);
  for (int c = threadIdx.x; c < C; c += 256) {
    const float m = mean[c], is = invstd[c], g = gamma[c], b = beta[c];
    float s = 0.f, q = 0.f;
    for (int r = r0; r < r1; ++r) {
      const float xh = (v[(long)r * C + c] - m) * is;
      const float ds = silu_grad(xh * g + b, dy[(long)r * C + c]);
      s += ds; q += ds * xh;
    }
    part[((long)blockIdx.x * 2) * C + c] = s;
    part[((long)blockIdx.x * 2 + 1) * C + c] = q;
  }
}
// dconv = gamma * invstd / N * (N * ds - dbeta - x_hat * dgamma)
__global__ void bn_bwd_dx_kernel(const float* __restrict__ v, const float* __restrict__ dy, const float* __restrict__ mean,
                                 const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                                 const float* __restrict__ dgamma, const float* __restrict__ dbeta, float* __restrict__ dv, long n,
                                 int C, float inv_rows) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const float xh = (v[i] - mean[c]) * invstd[c];
    const float ds = silu_grad(xh * gamma[c] + beta[c], dy[i]);
    dv[i] = gamma[c] * invstd[c] * (ds - inv_rows * (dbeta[c] + xh * dgamma[c]));
  }
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

int avsr_transpose(const float* src, float* dst, int rows, int cols, long ld_dst, void* stream) {
  AVSR_REQUIRE(src && dst && ld_dst >= rows, "transpose: NULL argument or ld_dst < rows");
  if (rows <= 0 || cols <= 0) return AVSR_OK;
  transpose_kernel<<<dim3(cdiv(cols, 32), cdiv(rows, 32)), dim3(32, 8), 0, reinterpret_cast<cudaStream_t>(stream)>>>(src, dst, rows, cols, ld_dst);
  AVSR_CHECK_LAUNCH();
  return AVSR_OK;
}

int avsr_pack_operand(const float* src, void* dst, int rows, int cols, long ld_dst, int transpose, int precision,
                      void* stream) {
  AVSR_REQUIRE(src && dst, "NULL argument");
  AVSR_REQUIRE(precision == AVSR_PREC_BF16, "pack_operand: precision %d is not built; AVSR_PREC_BF16 only", precision);
  AVSR_REQUIRE(rows >= 0 && cols >= 0 && ld_dst >= (transpose ? rows : cols), "pack_operand: bad rows=%d cols=%d ld=%ld",
               rows, cols, ld_dst);
  if (rows <= 0 || cols <= 0) return AVSR_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(dst);
  if (transpose)
    pack_bf16_t_kernel<<<dim3((unsigned)((ld_dst + 31) / 32), cdiv(cols, 32)), dim3(32, 8), 0, st>>>(src, d, rows, cols,
                                                                                                        ld_dst);
  else
    pack_bf16_kernel<<<132 * 4, 256, 0, st>>>(src, d, rows, cols, ld_dst);
  AVSR_CHECK_LAUNCH();
  return AVSR_OK;
}

static size_t pad64(int v) { return ((size_t)v + 63) / 64 * 64; }

size_t avsr_linear_bwd_bf16_workspace_bytes(int rows, int n, int k) {
  if (rows <= 0 || n <= 0 || k <= 0) return 256;
  return align_up((size_t)rows * pad64(n) * 2, 256) + align_up((size_t)k * pad64(n) * 2, 256) +
         align_up((size_t)n * pad64(rows) * 2, 256) + align_up((size_t)k * pad64(rows) * 2, 256);
}

int avsr_linear_bwd_bf16(const float* dy, const float* x, const float* w, float* dx, float* dw, int rows, int n, int k,
                         void* workspace, size_t workspace_bytes, void* stream) {
  AVSR_REQUIRE(dy && workspace && (dx || dw) && (!dx || w) && (!dw || x), "NULL argument");
  AVSR_REQUIRE(rows > 0 && n > 0 && k > 0, "linear_bwd_bf16: bad rows=%d n=%d k=%d", rows, n, k);
  AVSR_REQUIRE_BYTES(avsr_linear_bwd_bf16_workspace_bytes(rows, n, k), workspace_bytes, "linear_bwd_bf16 workspace");
  const long np = (long)pad64(n), rp = (long)pad64(rows);
  Carver cv{reinterpret_cast<char*>(workspace)};
  __nv_bfloat16 *dy_op = cv.take<__nv_bfloat16>((size_t)rows * np), *wt_op = cv.take<__nv_bfloat16>((size_t)k * np),
                *dyt_op = cv.take<__nv_bfloat16>((size_t)n * rp), *xt_op = cv.take<__nv_bfloat16>((size_t)k * rp);
  if (dx) {   // dX (rows, k) = dY W = dY (W^T)^T: K = n
    AVSR_TRY(avsr_pack_operand(dy, dy_op, rows, n, np, 0, AVSR_PREC_BF16, stream));
    AVSR_TRY(avsr_pack_operand(w, wt_op, n, k, np, 1, AVSR_PREC_BF16, stream));
    AVSR_TRY(avsr_linear_operands(dy_op, wt_op, nullptr, nullptr, 1.0f, dx, rows, k, (int)np, 0, 0, AVSR_PREC_BF16, stream));
  }
  if (dw) {   // dW (n, k) = dY^T X = dY^T (X^T)^T: K = rows
    AVSR_TRY(avsr_pack_operand(dy, dyt_op, rows, n, rp, 1, AVSR_PREC_BF16, stream));
    AVSR_TRY(avsr_pack_operand(x, xt_op, rows, k, rp, 1, AVSR_PREC_BF16, stream));
    AVSR_TRY(avsr_linear_operands(dyt_op, xt_op, nullptr, nullptr, 1.0f, dw, n, k, (int)rp, 0, 0, AVSR_PREC_BF16, stream));
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

// ---- depthwise conv + BatchNorm (training) + SiLU, in the pieces a (Sync)BatchNorm needs: the per-channel sums leave the
// library between the pieces so that the host can all-reduce them over the ranks (torch.nn.SyncBatchNorm semantics,
// train.py:31) before the statistics are finalised.

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

// sums (2, C): dy == NULL -> [sum v, sum v^2] over the rows, or with mean given the centred [sum (v - mean),
// sum (v - mean)^2] (the second pass of the batch statistics); else the BatchNorm+SiLU backward sums [sum ds, sum ds*x_hat]
// with h = x_hat * gamma + beta, ds = dL/dh of y = silu(h)
int avsr_chan_sums(const float* v, const float* dy, const float* mean, const float* invstd, const float* gamma,
                   const float* beta, float* sums, int rows, int C, void* workspace, size_t workspace_bytes, void* stream) {
  AVSR_REQUIRE(v && sums && workspace && C > 0, "NULL / bad argument");
  AVSR_REQUIRE(!dy || (mean && invstd && gamma && beta), "chan_sums: the backward sums need mean / invstd / gamma / beta");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (rows <= 0) { AVSR_CUDA_TRY(cudaMemsetAsync(sums, 0, 2 * C * sizeof(float), st)); return AVSR_OK; }
  const int rpc = cdiv(rows, kRedBlocks), nb = cdiv(rows, rpc);
  AVSR_REQUIRE_BYTES((size_t)nb * 2 * C * sizeof(float), workspace_bytes, "chan_sums workspace");
  float* part = reinterpret_cast<float*>(workspace);
  if (dy) bn_bwd_partial_kernel<<<nb, 256, 0, st>>>(v, dy, mean, invstd, gamma, beta, part, rows, C, rpc);
  else chan_stats_partial_kernel<<<nb, 256, 0, st>>>(v, mean, part, rows, C, rpc);
  AVSR_CHECK_LAUNCH();
  reduce_partials_kernel<<<cdiv(2 * C, 256), 256, 0, st>>>(part, sums, nb, 2 * C);
  AVSR_CHECK_LAUNCH();
  return AVSR_OK;
}

// y = silu((v - mean) * invstd * gamma + beta)
int avsr_bn_silu_fwd(const float* v, const float* mean, const float* invstd, const float* gamma, const float* beta, float* y,
                     int rows, int C, void* stream) {
  AVSR_REQUIRE(v && mean && invstd && gamma && beta && y && C > 0 && C % 4 == 0, "NULL / bad argument");
  if (rows <= 0) return AVSR_OK;
  bn_silu_fwd_kernel<<<grid_for((long)rows * C / 4), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(v), mean, invstd, gamma, beta, reinterpret_cast<float4*>(y), (long)rows * C / 4, C / 4);
  AVSR_CHECK_LAUNCH();
  return AVSR_OK;
}

// dv = gamma * invstd * (ds - inv_count * (sum_ds + x_hat * sum_dsx)): sum_ds / sum_dsx (C) and inv_count are GLOBAL
// (over all ranks' rows under SyncBatchNorm)
int avsr_bn_silu_bwd_dx(const float* v, const float* dy, const float* mean, const float* invstd, const float* gamma,
                        const float* beta, const float* sum_ds, const float* sum_dsx, float inv_count, float* dv, int rows,
                        int C, void* stream) {
  AVSR_REQUIRE(v && dy && mean && invstd && gamma && beta && sum_ds && sum_dsx && dv && C > 0, "NULL / bad argument");
  if (rows <= 0) return AVSR_OK;
  bn_bwd_dx_kernel<<<grid_for((long)rows * C), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      v, dy, mean, invstd, gamma, beta, sum_dsx, sum_ds, dv, (long)rows * C, C, inv_count);
  AVSR_CHECK_LAUNCH();
  return AVSR_OK;
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

}  // extern "C"
