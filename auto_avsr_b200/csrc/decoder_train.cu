// Teacher-forced training pass of the attention decoder (transformer_decoder.py:229-258) and its LabelSmoothingLoss
// (label_smoothing_loss.py:41-63), forward and backward.  The math lives in decoder_train_body.cuh; this file is the
// launch schedule.  The GEMMs of the pass are LinearFn's (wgmma); what runs here:
//
//   mha_fwd_kernel         one warp per (b, h, query row): pass 1 the row's log-sum-exp over tiles of 32 keys (lane per
//                          key), pass 2 the probabilities (stored when a backward follows) and ctx = sum_j A'_ij v_j, the
//                          probabilities broadcast lane by lane in key order
//   mha_bwd_rows_kernel    one warp per (b, h, query row): Delta_i = sum_j A_ij dA_ij, then dq_i = sum_j dS_ij k_j
//   mha_bwd_keys_kernel    one warp per (b, h, key): dk_j = sum_i dS_ij q_i and dv_j = sum_i A'_ij dctx_i, query order
//   ls_fwd_kernel          one 256-thread CTA per logits row: ONE read of the row -> (max, sum exp) and sum x -> loss
//   ls_bwd_kernel          one 256-thread CTA per row: dscale * (softmax - t), 0 on ignored rows and padding columns
//   embed_fwd_kernel       grid-stride EmbedTrainElem
//   embed_sort_kernel      one CTA: positions grouped by token (counting sort: counts, scan, stable ranks)
//   embed_bwd_kernel       one thread per (token, column): the token's positions summed in position order
//
// fp32 CUDA cores, correctness first (attention is ~5 % of the decoder's training FLOPs).  Every output element has
// one writer and a fixed summation order: two identical calls give identical bits.
#include "decoder_train_body.cuh"
#include "maxsum.cuh"

namespace avsr {
namespace dtr {

constexpr int kMhaWarps = 8;

// dot of a 64-float vector in shared memory (broadcast across the warp) with this lane's row in global memory
__device__ __forceinline__ float dot64(const float* s, const float* __restrict__ g) {
  const float4* s4 = reinterpret_cast<const float4*>(s);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  float acc = 0.f;
#pragma unroll
  for (int t = 0; t < 16; ++t) {
    const float4 a = s4[t], b = __ldg(g4 + t);
    acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc); acc = fmaf(a.z, b.z, acc); acc = fmaf(a.w, b.w, acc);
  }
  return acc;
}

__global__ void __launch_bounds__(32 * kMhaWarps) mha_fwd_kernel(
    const float* __restrict__ q, long ldq, const float* __restrict__ k, long ldk, const float* __restrict__ v, long ldv,
    int B, int H, int Lq, int Lk, int causal, const int32_t* __restrict__ klen, const uint8_t* __restrict__ keep,
    float kscale, float* __restrict__ ctx, float* __restrict__ probs) {
  __shared__ __align__(16) float qs[kMhaWarps][64];
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long row = (long)blockIdx.x * kMhaWarps + warp;        // ((b * H + h) * Lq + i)
  if (row >= (long)B * H * Lq) return;                         // warp-uniform; only warp-level sync below
  const int i = (int)(row % Lq);
  const long bh = row / Lq;
  const int h = (int)(bh % H), b = (int)(bh / H);
  const float* qr = q + ((long)b * Lq + i) * ldq + h * 64;
  qs[warp][lane] = qr[lane];
  qs[warp][lane + 32] = qr[lane + 32];
  __syncwarp();
  const int n = attn_row_keys(i, Lk, causal, klen, b);
  const float* kb = k + (long)b * Lk * ldk + h * 64;
  const float* vb = v + (long)b * Lk * ldv + h * 64;
  float m = -INFINITY, s = 0.f;
  for (int j0 = 0; j0 < n; j0 += 32) {
    const int j = j0 + lane;
    const float sc = j < n ? dot64(qs[warp], kb + (long)j * ldk) * kAttnScale : -INFINITY;
    const float mn = fmaxf(m, warp_max(sc));
    s = s * expf(m - mn) + warp_sum(j < n ? expf(sc - mn) : 0.f);
    m = mn;
  }
  const float lse = n > 0 ? m + logf(s) : 0.f;
  const long prow = row * Lk;
  float a0 = 0.f, a1 = 0.f;
  for (int j0 = 0; j0 < n; j0 += 32) {
    const int j = j0 + lane;
    float p = 0.f, pd = 0.f;
    if (j < n) {
      p = expf(dot64(qs[warp], kb + (long)j * ldk) * kAttnScale - lse);
      pd = p * keep_factor(keep, prow + j, kscale);
      if (probs) probs[prow + j] = p;
    }
    const int cnt = n - j0 < 32 ? n - j0 : 32;
    for (int t = 0; t < cnt; ++t) {
      const float pt = __shfl_sync(0xffffffffu, pd, t);
      const float* vr = vb + (long)(j0 + t) * ldv;
      a0 = fmaf(pt, vr[lane], a0);
      a1 = fmaf(pt, vr[lane + 32], a1);
    }
  }
  if (probs)
    for (int j = n + lane; j < Lk; j += 32) probs[prow + j] = 0.f;
  float* cr = ctx + ((long)b * Lq + i) * (H * 64) + h * 64;
  cr[lane] = a0;
  cr[lane + 32] = a1;
}

__global__ void __launch_bounds__(32 * kMhaWarps) mha_bwd_rows_kernel(
    const float* __restrict__ k, long ldk, const float* __restrict__ v, long ldv, int B, int H, int Lq, int Lk,
    int causal, const int32_t* __restrict__ klen, const uint8_t* __restrict__ keep, float kscale,
    const float* __restrict__ probs, const float* __restrict__ dctx, float* __restrict__ dq, long lddq,
    float* __restrict__ delta) {
  __shared__ __align__(16) float dcs[kMhaWarps][64];
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long row = (long)blockIdx.x * kMhaWarps + warp;
  if (row >= (long)B * H * Lq) return;
  const int i = (int)(row % Lq);
  const long bh = row / Lq;
  const int h = (int)(bh % H), b = (int)(bh / H);
  const float* dr = dctx + ((long)b * Lq + i) * (H * 64) + h * 64;
  dcs[warp][lane] = dr[lane];
  dcs[warp][lane + 32] = dr[lane + 32];
  __syncwarp();
  const int n = attn_row_keys(i, Lk, causal, klen, b);
  const float* kb = k + (long)b * Lk * ldk + h * 64;
  const float* vb = v + (long)b * Lk * ldv + h * 64;
  const long prow = row * Lk;
  float acc = 0.f;
  for (int j = lane; j < n; j += 32)
    acc = fmaf(probs[prow + j], dot64(dcs[warp], vb + (long)j * ldv) * keep_factor(keep, prow + j, kscale), acc);
  const float dl = warp_sum(acc);
  if (lane == 0) delta[row] = dl;
  float g0 = 0.f, g1 = 0.f;
  for (int j0 = 0; j0 < n; j0 += 32) {
    const int j = j0 + lane;
    float ds = 0.f;
    if (j < n)
      ds = attn_dscore(probs[prow + j], dot64(dcs[warp], vb + (long)j * ldv) * keep_factor(keep, prow + j, kscale), dl);
    const int cnt = n - j0 < 32 ? n - j0 : 32;
    for (int t = 0; t < cnt; ++t) {
      const float st = __shfl_sync(0xffffffffu, ds, t);
      const float* kr = kb + (long)(j0 + t) * ldk;
      g0 = fmaf(st, kr[lane], g0);
      g1 = fmaf(st, kr[lane + 32], g1);
    }
  }
  float* o = dq + ((long)b * Lq + i) * lddq + h * 64;
  o[lane] = g0;
  o[lane + 32] = g1;
}

__global__ void __launch_bounds__(32 * kMhaWarps) mha_bwd_keys_kernel(
    const float* __restrict__ q, long ldq, const float* __restrict__ v, long ldv, int B, int H, int Lq, int Lk,
    int causal, const int32_t* __restrict__ klen, const uint8_t* __restrict__ keep, float kscale,
    const float* __restrict__ probs, const float* __restrict__ dctx, const float* __restrict__ delta,
    float* __restrict__ dk, float* __restrict__ dv, long lddkv) {
  __shared__ __align__(16) float vs[kMhaWarps][64];
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long key = (long)blockIdx.x * kMhaWarps + warp;       // ((b * H + h) * Lk + j)
  if (key >= (long)B * H * Lk) return;
  const int j = (int)(key % Lk);
  const long bh = key / Lk;
  const int h = (int)(bh % H), b = (int)(bh / H);
  const int D = H * 64;
  const float* vr = v + ((long)b * Lk + j) * ldv + h * 64;
  vs[warp][lane] = vr[lane];
  vs[warp][lane + 32] = vr[lane + 32];
  __syncwarp();
  float k0 = 0.f, k1 = 0.f, v0 = 0.f, v1 = 0.f;
  // a key below the key length is seen by every query from attn_first_query on; a masked key by none
  if (j < attn_row_keys(0, Lk, 0, klen, b)) {
    const float* qb = q + (long)b * Lq * ldq + h * 64;
    const float* db = dctx + (long)b * Lq * D + h * 64;
    const float* drow = delta + bh * Lq;
    for (int i0 = attn_first_query(j, causal); i0 < Lq; i0 += 32) {
      const int i = i0 + lane;
      float ds = 0.f, ad = 0.f;
      if (i < Lq) {
        const long pidx = (bh * Lq + i) * Lk + j;
        const float a = probs[pidx], kf = keep_factor(keep, pidx, kscale);
        ds = attn_dscore(a, dot64(vs[warp], db + (long)i * D) * kf, drow[i]);
        ad = a * kf;
      }
      const int cnt = Lq - i0 < 32 ? Lq - i0 : 32;
      for (int t = 0; t < cnt; ++t) {
        const float st = __shfl_sync(0xffffffffu, ds, t), at = __shfl_sync(0xffffffffu, ad, t);
        const float* qr = qb + (long)(i0 + t) * ldq;
        const float* dr = db + (long)(i0 + t) * D;
        k0 = fmaf(st, qr[lane], k0);
        k1 = fmaf(st, qr[lane + 32], k1);
        v0 = fmaf(at, dr[lane], v0);
        v1 = fmaf(at, dr[lane + 32], v1);
      }
    }
  }
  const long o = ((long)b * Lk + j) * lddkv + h * 64;
  dk[o + lane] = k0;
  dk[o + lane + 32] = k1;
  dv[o + lane] = v0;
  dv[o + lane + 32] = v1;
}

// fixed-order sum over a 256-thread CTA, handed to every thread (two __syncthreads: all threads must call it)
__device__ __forceinline__ float block_sum_256(float v) {
  __shared__ float part[8];
  __shared__ float total;
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = part[0];
    for (int w = 1; w < 8; ++w) t += part[w];
    total = t;
  }
  __syncthreads();
  return total;
}

__global__ void __launch_bounds__(256) ls_fwd_kernel(const float* __restrict__ x, long ld, const int64_t* __restrict__ tgt,
                                                     int odim, long long ignore_id, LsConst kc, float* __restrict__ loss,
                                                     float* __restrict__ lse_out) {
  pdl_launch_dependents();
  const long r = blockIdx.x;
  pdl_wait();
  const int kind = ls_row_kind(tgt[r], (int64_t)ignore_id, odim);     // CTA-uniform
  if (kind == 0) {
    if (threadIdx.x == 0) { loss[r] = 0.f; lse_out[r] = 0.f; }
    return;
  }
  const float* xr = x + r * ld;
  MaxSum acc{-INFINITY, 0.f, 0x7fffffff};
  float sx = 0.f;
  for (int c = threadIdx.x; c < odim; c += 256) {
    const float xv = xr[c];
    ms_push(acc, xv, c);
    sx += xv;
  }
  const MaxSum tot = ms_block_reduce_256(acc);
  const float sum_x = block_sum_256(sx);
  if (threadIdx.x == 0) {
    const float lse = tot.m + logf(tot.s);
    lse_out[r] = lse;
    loss[r] = kind < 0 ? NAN : ls_row_loss(kc, lse, sum_x, xr[tgt[r]]);
  }
}

__global__ void __launch_bounds__(256) ls_bwd_kernel(const float* __restrict__ x, long ld, const int64_t* __restrict__ tgt,
                                                     int odim, long long ignore_id, LsConst kc,
                                                     const float* __restrict__ lse, const float* __restrict__ dscale,
                                                     float* __restrict__ dx, long ldd) {
  pdl_launch_dependents();
  const long r = blockIdx.x;
  float* dr = dx + r * ldd;
  pdl_wait();
  const int64_t y = tgt[r];
  const int kind = ls_row_kind(y, (int64_t)ignore_id, odim);
  const float* xr = x + r * ld;
  const float l = lse[r], g = *dscale;
  for (int c = threadIdx.x; c < ldd; c += 256) {
    float d = 0.f;
    if (c < odim && kind != 0) d = kind < 0 ? NAN : ls_grad(kc, xr[c], l, g, c == y);
    dr[c] = d;
  }
}

__global__ void embed_fwd_kernel(EmbedTrainElem f, long count) {
  pdl_launch_dependents();
  pdl_wait();
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < count; idx += (long)gridDim.x * blockDim.x) f(idx);
}

// start (odim + 1): start[t] = first slot of token t in `order`; order (rows): positions grouped by token, each group
// in position order.  One CTA of 1024 threads.
__global__ void __launch_bounds__(1024) embed_sort_kernel(const int64_t* __restrict__ tok, int rows, int odim,
                                                          int32_t* __restrict__ start, int32_t* __restrict__ order) {
  __shared__ int32_t part[1024];
  pdl_launch_dependents();
  pdl_wait();
  const int tid = threadIdx.x;
  for (int t = tid; t <= odim; t += 1024) start[t] = 0;
  __syncthreads();
  for (int r = tid; r < rows; r += 1024)
    if (embed_token_ok(tok[r], odim)) atomicAdd(&start[tok[r] + 1], 1);      // integer counts: order-independent
  __syncthreads();
  // exclusive scan of the counts (start[0] = 0): each thread owns a contiguous chunk
  const int n = odim + 1, chunk = (n + 1023) / 1024;
  const int lo = tid * chunk < n ? tid * chunk : n, hi = lo + chunk < n ? lo + chunk : n;
  int32_t s = 0;
  for (int t = lo; t < hi; ++t) s += start[t];
  part[tid] = s;
  __syncthreads();
  if (tid == 0) {
    int32_t run = 0;
    for (int w = 0; w < 1024; ++w) { const int32_t c = part[w]; part[w] = run; run += c; }
  }
  __syncthreads();
  int32_t run = part[tid];
  for (int t = lo; t < hi; ++t) { run += start[t]; start[t] = run; }
  __syncthreads();
  // stable placement: position r goes after every earlier position with the same token
  for (int r = tid; r < rows; r += 1024) {
    const int64_t t = tok[r];
    if (!embed_token_ok(t, odim)) continue;
    int rank = 0;
    for (int m = 0; m < r; ++m) rank += tok[m] == t;
    order[start[t] + rank] = r;
  }
}

__global__ void embed_bwd_kernel(const float* __restrict__ dx, int D, int odim, float xscale,
                                 const int32_t* __restrict__ start, const int32_t* __restrict__ order,
                                 float* __restrict__ demb) {
  pdl_launch_dependents();
  pdl_wait();
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)odim * D) return;
  const int t = (int)(idx / D), c = (int)(idx - (long)t * D);
  float acc = 0.f;
  for (int e = start[t]; e < start[t + 1]; ++e) acc += dx[(long)order[e] * D + c] * xscale;
  demb[idx] = acc;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static int mha_check(const float* q, long ldq, const float* k, long ldk, const float* v, long ldv, int B, int H, int Lq,
                     int Lk) {
  AVSR_REQUIRE(B >= 0 && H >= 1 && Lq >= 0 && Lk >= 0, "mha_core: bad B=%d H=%d Lq=%d Lk=%d", B, H, Lq, Lk);
  AVSR_REQUIRE(ldq >= H * 64 && ldk >= H * 64 && ldv >= H * 64 && ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0,
               "mha_core: row strides (%ld, %ld, %ld) must be multiples of 4 and >= H*64 = %d", ldq, ldk, ldv, H * 64);
  AVSR_REQUIRE((long)B * Lq == 0 || (q && aligned16(q)), "mha_core: q NULL or not 16-byte aligned");
  AVSR_REQUIRE((long)B * Lk == 0 || (k && v && aligned16(k) && aligned16(v)), "mha_core: k / v NULL or not 16-byte aligned");
  return AVSR_OK;
}

}  // namespace dtr
}  // namespace avsr

using namespace avsr;
using namespace avsr::dtr;

extern "C" {

int avsr_mha_core_fwd(const float* q, long ldq, const float* k, long ldk, const float* v, long ldv, int B, int H, int Lq,
                      int Lk, int causal, const int32_t* key_lengths, const uint8_t* keep, float keep_scale, float* ctx,
                      float* probs, void* stream) {
  AVSR_TRY(mha_check(q, ldq, k, ldk, v, ldv, B, H, Lq, Lk));
  const long rows = (long)B * H * Lq;
  if (rows == 0) return AVSR_OK;
  AVSR_REQUIRE(ctx, "NULL argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  AVSR_LAUNCH(mha_fwd_kernel, (unsigned)((rows + kMhaWarps - 1) / kMhaWarps), 32 * kMhaWarps, 0, st, q, ldq, k, ldk, v,
              ldv, B, H, Lq, Lk, causal, key_lengths, keep, keep_scale, ctx, probs);
  return AVSR_OK;
}

size_t avsr_mha_core_bwd_workspace_bytes(int B, int H, int Lq) {
  if (B <= 0 || H <= 0 || Lq <= 0) return 256;
  return align_up((size_t)B * H * Lq * sizeof(float), 256);
}

int avsr_mha_core_bwd(const float* q, long ldq, const float* k, long ldk, const float* v, long ldv, int B, int H, int Lq,
                      int Lk, int causal, const int32_t* key_lengths, const uint8_t* keep, float keep_scale,
                      const float* probs, const float* dctx, float* dq, long lddq, float* dk, float* dv, long lddkv,
                      void* workspace, size_t workspace_bytes, void* stream) {
  AVSR_TRY(mha_check(q, ldq, k, ldk, v, ldv, B, H, Lq, Lk));
  AVSR_REQUIRE(lddq >= H * 64 && lddkv >= H * 64, "mha_core_bwd: bad output strides %ld / %ld", lddq, lddkv);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long rows = (long)B * H * Lq, keys = (long)B * H * Lk;
  if (rows > 0) {
    AVSR_REQUIRE(dq && (Lk == 0 || (probs && dctx && aligned16(dctx))) && workspace, "NULL argument");
    AVSR_REQUIRE_BYTES(avsr_mha_core_bwd_workspace_bytes(B, H, Lq), workspace_bytes, "mha_core_bwd workspace");
    AVSR_LAUNCH(mha_bwd_rows_kernel, (unsigned)((rows + kMhaWarps - 1) / kMhaWarps), 32 * kMhaWarps, 0, st, k, ldk, v,
                ldv, B, H, Lq, Lk, causal, key_lengths, keep, keep_scale, probs, dctx, dq, lddq,
                reinterpret_cast<float*>(workspace));
  }
  if (keys > 0) {
    AVSR_REQUIRE(dk && dv && (Lq == 0 || (probs && dctx && workspace)), "NULL argument");
    AVSR_LAUNCH(mha_bwd_keys_kernel, (unsigned)((keys + kMhaWarps - 1) / kMhaWarps), 32 * kMhaWarps, 0, st, q, ldq, v,
                ldv, B, H, Lq, Lk, causal, key_lengths, keep, keep_scale, probs, dctx,
                reinterpret_cast<const float*>(workspace), dk, dv, lddkv);
  }
  return AVSR_OK;
}

int avsr_label_smoothing_fwd(const float* logits, long ld, const int64_t* target, int rows, int odim, int ignore_id,
                             float smoothing, float* row_loss, float* lse, void* stream) {
  AVSR_REQUIRE(rows >= 0 && odim >= 2 && ld >= odim, "label_smoothing: bad rows=%d odim=%d ld=%ld", rows, odim, ld);
  if (rows == 0) return AVSR_OK;
  AVSR_REQUIRE(logits && target && row_loss && lse, "NULL argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  AVSR_LAUNCH(ls_fwd_kernel, rows, 256, 0, st, logits, ld, target, odim, (long long)ignore_id, ls_const(odim, smoothing),
              row_loss, lse);
  return AVSR_OK;
}

int avsr_label_smoothing_bwd(const float* logits, long ld, const int64_t* target, int rows, int odim, int ignore_id,
                             float smoothing, const float* lse, const float* dscale, float* dlogits, long ldd,
                             void* stream) {
  AVSR_REQUIRE(rows >= 0 && odim >= 2 && ld >= odim && ldd >= odim, "label_smoothing_bwd: bad rows=%d odim=%d ld=%ld ldd=%ld",
               rows, odim, ld, ldd);
  if (rows == 0) return AVSR_OK;
  AVSR_REQUIRE(logits && target && lse && dscale && dlogits, "NULL argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  AVSR_LAUNCH(ls_bwd_kernel, rows, 256, 0, st, logits, ld, target, odim, (long long)ignore_id, ls_const(odim, smoothing),
              lse, dscale, dlogits, ldd);
  return AVSR_OK;
}

int avsr_embed_fwd(const int64_t* tokens, const float* embed, int rows, int L, int D, int odim, float* x, void* stream) {
  AVSR_REQUIRE(rows >= 0 && L >= 1 && D >= 1 && odim >= 1, "embed_fwd: bad rows=%d L=%d D=%d odim=%d", rows, L, D, odim);
  if (rows == 0) return AVSR_OK;
  AVSR_REQUIRE(tokens && embed && x, "NULL argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long count = (long)rows * D;
  const EmbedTrainElem f{tokens, embed, x, D, L, odim, (float)sqrt((double)D), (float)(-(log(10000.0) / D))};
  const long blocks = (count + 255) / 256;
  AVSR_LAUNCH(embed_fwd_kernel, (unsigned)(blocks < 4096 ? blocks : 4096), 256, 0, st, f, count);
  return AVSR_OK;
}

size_t avsr_embed_bwd_workspace_bytes(int rows, int odim) {
  if (rows < 0 || odim < 0) return 0;
  return align_up((size_t)(odim + 1) * 4, 256) + align_up((size_t)(rows > 0 ? rows : 1) * 4, 256);
}

int avsr_embed_bwd(const int64_t* tokens, const float* dx, int rows, int D, int odim, float* dembed, void* workspace,
                   size_t workspace_bytes, void* stream) {
  AVSR_REQUIRE(rows >= 0 && D >= 1 && odim >= 1, "embed_bwd: bad rows=%d D=%d odim=%d", rows, D, odim);
  AVSR_REQUIRE(dembed && workspace && (rows == 0 || (tokens && dx)), "NULL argument");
  AVSR_REQUIRE_BYTES(avsr_embed_bwd_workspace_bytes(rows, odim), workspace_bytes, "embed_bwd workspace");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int32_t* start = reinterpret_cast<int32_t*>(workspace);
  int32_t* order = reinterpret_cast<int32_t*>(reinterpret_cast<char*>(workspace) + align_up((size_t)(odim + 1) * 4, 256));
  AVSR_LAUNCH(embed_sort_kernel, 1, 1024, 0, st, tokens, rows, odim, start, order);
  const long count = (long)odim * D;
  AVSR_LAUNCH(embed_bwd_kernel, (unsigned)((count + 255) / 256), 256, 0, st, dx, D, odim, (float)sqrt((double)D), start,
              order, dembed);
  return AVSR_OK;
}

}  // extern "C"
