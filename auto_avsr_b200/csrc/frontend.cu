// ResNet front-ends (Conv3dResNet for video, Conv1dResNet for audio), inference with eval-mode BatchNorm.
//
// Activations are channels-last in the precision's operand storage: (frames, H, W, C) for video and (utterances, L, C)
// for audio, which is the same layout with H = 1.  Every convolution is one implicit GEMM
//   acc[m][n] = sum_k A[m][k] * Wt[n][k],   m = output pixel of any frame, n = C_out, k = tap * C_in + c
// with the epilogue  y = [SiLU](acc * bn_scale[n] + bn_shift[n] [+ resid])  (BatchNorm stays in fp32, not folded into
// the operand weights: a channel with a tiny running_var would push folded f16 weights out of range).
//
// conv_tc_kernel (sm_90a): 128 output pixels x BN channels per CTA, two warpgroups of 64 pixels each issue
// wgmma.mma_async from a 4-stage ring of 128B-swizzled shared-memory tiles.  A K-block is 128 bytes of one filter tap
// (64 f16 / bf16 or 32 tf32 channels; every trunk C_in is a multiple of 64), so the A tile of a trunk conv is gathered with
// 16-byte cp.async copies straight from the activation (zero-filled where the tap falls into the padding); tiles of
// pixels cross frame boundaries.  The stems (C_in = 1) gather their fp32 input element by element (K = 245 -> 256
// for video, 80 -> 128 for audio), convert it to the operand type and store it with the same swizzle.
// conv_direct_kernel is the CUDA-core fp32 path (AVSR_PREC_FP32) over the same geometry.
#include "common.cuh"
#include "sm90.cuh"

namespace avsr {

using namespace sm90;

// Output pixel m = (n * Ho + oy) * Wo + ox reads input frame n (+ dt - pt inside its utterance of T frames) at
// (oy * sh - ph + ky, ox * sw - pw + kx), channel c; k = ((dt * KH + ky) * KW + kx) * Cin + c.
struct ConvGeom {
  int N, T;               // output frames; frames per utterance (temporal taps never leave an utterance)
  int H, W, Cin;          // input frame
  int Ho, Wo, Cout;
  int KT, KH, KW, sh, sw, pt, ph, pw;
  long ld_frame;          // elements between consecutive input frames
  int K, Kp;              // taps * Cin; the weights' padded row length (multiple of 64)
};

static inline long conv_rows(const ConvGeom& g) { return (long)g.N * g.Ho * g.Wo; }

__device__ __forceinline__ float silu_fast(float v) { return v * sigmoidf_fast(v); }

// ---------------------------------------------------------------- operand conversion helpers
template <typename TOp> __device__ __forceinline__ float op_ld(const TOp* p);
template <> __device__ __forceinline__ float op_ld<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float op_ld<__half>(const __half* p) { return __half2float(*p); }
template <> __device__ __forceinline__ float op_ld<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }

template <typename TOp>
__device__ __forceinline__ float4 op_ld4(const TOp* p) {
  if constexpr (sizeof(TOp) == 4) {
    return *reinterpret_cast<const float4*>(p);
  } else if constexpr (std::is_same<TOp, __nv_bfloat16>::value) {
    const uint2 u = *reinterpret_cast<const uint2*>(p);
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
    const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
  } else {
    const uint2 u = *reinterpret_cast<const uint2*>(p);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
  }
}

// kind: OP_F32 plain, OP_TF32 rounded fp32, OP_F16 half, OP_BF16 bfloat16
__global__ void cvt_to_op_kernel(const float* __restrict__ x, void* __restrict__ y, long n, int kind) {
  pdl_wait();
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    store_kind1(y, i, kind, x[i]);
}
__global__ void cvt_from_op_kernel(const void* __restrict__ x, float* __restrict__ y, long n, int kind) {
  pdl_wait();
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    y[i] = load_kind1(x, i, kind);
}

// torch conv weight (Cout, Cin, taps) -> (Cout, Kp) with k = tap * Cin + c, zero for k >= taps * Cin
__global__ void reorder_weight_kernel(const float* __restrict__ w, void* __restrict__ dst, int Cout, int Cin, int taps,
                                      int Kp, int kind) {
  pdl_wait();
  const long n = (long)Cout * Kp;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int co = (int)(i / Kp), k = (int)(i - (long)co * Kp);
    float v = 0.f;
    if (k < taps * Cin) {
      const int tap = k / Cin, c = k - tap * Cin;
      v = w[((long)co * Cin + c) * taps + tap];
    }
    store_kind1(dst, i, kind, v);
  }
}

// eval-mode BatchNorm as y = x * scale + shift, computed in double from the module's buffers and eps
__global__ void bn_fold_kernel(const float* __restrict__ g, const float* __restrict__ b, const float* __restrict__ mean,
                               const float* __restrict__ var, double eps, float* __restrict__ scale,
                               float* __restrict__ shift, int C) {
  pdl_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double s = (double)g[c] / sqrt((double)var[c] + eps);
  scale[c] = (float)s;
  shift[c] = (float)((double)b[c] - (double)mean[c] * s);
}

// ---------------------------------------------------------------- CUDA-core direct convolution (fp32 reference path)
// block (64 output channels) x (4 output pixels); taps outside the input (or outside the utterance) are skipped
__global__ void __launch_bounds__(256) conv_direct_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                          const float* __restrict__ scale,
                                                          const float* __restrict__ shift,
                                                          const float* __restrict__ resid, float* __restrict__ y,
                                                          ConvGeom g, int act) {
  pdl_wait();
  pdl_launch_dependents();
  const int co = blockIdx.y * 64 + threadIdx.x;
  const long m = (long)blockIdx.x * 4 + threadIdx.y;
  if (m >= (long)g.N * g.Ho * g.Wo || co >= g.Cout) return;
  const int hw = g.Ho * g.Wo;
  const int n = (int)(m / hw), r = (int)(m - (long)n * hw);
  const int oy = r / g.Wo, ox = r - oy * g.Wo;
  const int t = n % g.T;
  const float* wr = w + (long)co * g.Kp;
  float acc = 0.f;
  for (int dt = 0; dt < g.KT; ++dt) {
    const int tt = t + dt - g.pt;
    if (tt < 0 || tt >= g.T) continue;
    const float* xf = x + (long)(n - t + tt) * g.ld_frame;
    for (int ky = 0; ky < g.KH; ++ky) {
      const int iy = oy * g.sh - g.ph + ky;
      if (iy < 0 || iy >= g.H) continue;
      for (int kx = 0; kx < g.KW; ++kx) {
        const int ix = ox * g.sw - g.pw + kx;
        if (ix < 0 || ix >= g.W) continue;
        const float* xp = xf + ((long)iy * g.W + ix) * g.Cin;
        const float* wp = wr + ((dt * g.KH + ky) * g.KW + kx) * g.Cin;
        for (int c = 0; c < g.Cin; ++c) acc = fmaf(xp[c], wp[c], acc);
      }
    }
  }
  float v = acc * scale[co] + shift[co];
  if (resid) v += resid[m * g.Cout + co];
  if (act) v = v * sigmoidf_acc(v);
  y[m * g.Cout + co] = v;
}

// ---------------------------------------------------------------- wgmma implicit GEMM
constexpr int CV_BM = 128;
constexpr int CV_THREADS = 256;     // two warpgroups: wgmma on 64 pixels each; all 256 threads load and run the epilogue
constexpr int CV_STAGES = 4;        // ring depth; loads run CV_STAGES - 2 K-blocks ahead of the MMAs

template <int BN>
struct CvCfg {
  static constexpr int kABytes = CV_BM * 128;
  static constexpr int kStageBytes = kABytes + BN * 128;
  static constexpr int kAccLd = BN + 4;
  static constexpr int kSmem = 1024 + CV_STAGES * kStageBytes;
  static_assert(CV_BM * kAccLd * 4 <= CV_STAGES * kStageBytes, "epilogue tile must fit in the ring");
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// byte offset of 16-byte chunk c of row r in a 128B-swizzled tile (the layout TMA SWIZZLE_128B writes)
__device__ __forceinline__ uint32_t sw128(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }

template <typename TOp> struct ConvOp;
template <> struct ConvOp<float> {
  static constexpr int KE = 32;   // elements per 128-byte K-block
  template <int BN>
  __device__ static void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    if constexpr (BN == 64) wgmma_tf32_n64(d, a, b, acc); else wgmma_tf32_n128(d, a, b, acc);
  }
  __device__ static uint4 pack(const float* v) {   // 4 values
    uint4 u;
    u.x = __float_as_uint(round_tf32(v[0])); u.y = __float_as_uint(round_tf32(v[1]));
    u.z = __float_as_uint(round_tf32(v[2])); u.w = __float_as_uint(round_tf32(v[3]));
    return u;
  }
};
template <> struct ConvOp<__half> {
  static constexpr int KE = 64;
  template <int BN>
  __device__ static void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    if constexpr (BN == 64) wgmma_f16_n64(d, a, b, acc); else wgmma_f16_n128(d, a, b, acc);
  }
  __device__ static uint4 pack(const float* v) {   // 8 values
    uint4 u;
    u.x = pack_half2_sat(v[0], v[1]); u.y = pack_half2_sat(v[2], v[3]);
    u.z = pack_half2_sat(v[4], v[5]); u.w = pack_half2_sat(v[6], v[7]);
    return u;
  }
};
template <> struct ConvOp<__nv_bfloat16> {
  static constexpr int KE = 64;
  template <int BN>
  __device__ static void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    if constexpr (BN == 64) wgmma_bf16_n64(d, a, b, acc); else wgmma_bf16_n128(d, a, b, acc);
  }
  __device__ static uint4 pack(const float* v) {   // 8 values
    return make_uint4(pack_bf162(v[0], v[1]), pack_bf162(v[2], v[3]), pack_bf162(v[4], v[5]), pack_bf162(v[6], v[7]));
  }
};

// STEM: x is the fp32 clip / waveform (Cin = 1) gathered element by element; otherwise x is the TOp activation.
// RAW (training): y is fp32 and receives the accumulator itself; scale, shift, resid and act are not read.
template <typename TOp, int BN, bool STEM, bool RAW = false>
__global__ void __launch_bounds__(CV_THREADS, 1)
conv_tc_kernel(const void* __restrict__ xv, const TOp* __restrict__ w, const float* __restrict__ scale,
               const float* __restrict__ shift, const TOp* __restrict__ resid, TOp* __restrict__ y, ConvGeom g,
               int act) {
  using Op = ConvOp<TOp>;
  using Cfg = CvCfg<BN>;
  constexpr int KE = Op::KE;
  constexpr int CE = 16 / (int)sizeof(TOp);      // elements per 16-byte chunk
  constexpr int S = CV_STAGES;
  extern __shared__ uint8_t cv_smem_raw[];
  const uint32_t raw = smem_u32(cv_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gen = cv_smem_raw + (base - raw);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;
  const long M = (long)g.N * g.Ho * g.Wo;
  const long m0 = (long)blockIdx.x * CV_BM;
  const int n0 = blockIdx.y * BN;
  const int nkb = g.Kp / KE;
  const int hw = g.Ho * g.Wo;

  // this thread loads 16-byte chunk `cc` of A rows ar + 32 i (i < 4) and of B rows ar + 32 i (i < BN / 32)
  const int cc = tid & 7, ar = tid >> 3;
  long rbase[4];
  int riy[4], rix[4], rt[4];
  bool rok[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long m = m0 + ar + 32 * i;
    rok[i] = m < M;
    const long mm = rok[i] ? m : 0;
    const int n = (int)(mm / hw), r = (int)(mm - (long)n * hw);
    const int oy = r / g.Wo, ox = r - oy * g.Wo;
    rt[i] = n % g.T;
    rbase[i] = (long)(n - rt[i]) * g.ld_frame;     // first frame of the utterance (== frame n when T = 1)
    riy[i] = oy * g.sh - g.ph;
    rix[i] = ox * g.sw - g.pw;
  }

  pdl_wait();
  pdl_launch_dependents();

  auto load = [&](int kb, int s) {
    const uint32_t a_dst = base + s * Cfg::kStageBytes;
    const uint32_t b_dst = a_dst + Cfg::kABytes;
    if constexpr (STEM) {
      const float* x = reinterpret_cast<const float*>(xv);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float v[CE];
#pragma unroll
        for (int e = 0; e < CE; ++e) {
          const int k = kb * KE + cc * CE + e;
          float val = 0.f;
          if (rok[i] && k < g.K) {
            const int kx = k % g.KW, q = k / g.KW;
            const int ky = q % g.KH, dt = q / g.KH;
            const int tt = rt[i] + dt - g.pt, iy = riy[i] + ky, ix = rix[i] + kx;
            if (tt >= 0 && tt < g.T && iy >= 0 && iy < g.H && ix >= 0 && ix < g.W)
              val = __ldg(x + rbase[i] + (long)tt * g.ld_frame + (long)iy * g.W + ix);
          }
          v[e] = val;
        }
        *reinterpret_cast<uint4*>(gen + s * Cfg::kStageBytes + sw128(ar + 32 * i, cc)) = Op::pack(v);
      }
    } else {
      const TOp* x = reinterpret_cast<const TOp*>(xv);
      const int kpt = g.Cin / KE;                     // K-blocks per tap
      const int tap = kb / kpt, c0 = (kb - tap * kpt) * KE + cc * CE;
      const int ky = tap / g.KW, kx = tap - ky * g.KW;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int iy = riy[i] + ky, ix = rix[i] + kx;
        const bool ok = rok[i] && iy >= 0 && iy < g.H && ix >= 0 && ix < g.W;
        const TOp* src = ok ? x + rbase[i] + ((long)iy * g.W + ix) * g.Cin + c0 : x;
        cp_async16(a_dst + sw128(ar + 32 * i, cc), src, ok);
      }
    }
#pragma unroll
    for (int i = 0; i < BN / 32; ++i) {
      const int row = ar + 32 * i;
      const bool ok = n0 + row < g.Cout;
      const TOp* src = ok ? w + (long)(n0 + row) * g.Kp + kb * KE + cc * CE : w;
      cp_async16(b_dst + sw128(row, cc), src, ok);
    }
  };

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;

#pragma unroll 1
  for (int s = 0; s < S - 2; ++s) {
    if (s < nkb) load(s, s);
    cp_async_commit();
  }
#pragma unroll 1
  for (int kb = 0; kb < nkb; ++kb) {
    cp_async_wait<S - 3>();          // this thread's copies of K-block kb have landed
    fence_proxy_async();             // generic-proxy writes (cp.async, st.shared) -> visible to wgmma
    __syncthreads();                 // every thread's part of kb is in; both warpgroups retired the MMAs of kb - 2
    const int s = kb % S;
    const uint32_t a_addr = base + s * Cfg::kStageBytes;
    const uint64_t a_desc = wgmma_desc_sw128(a_addr + wg * (64 * 128));
    const uint64_t b_desc = wgmma_desc_sw128(a_addr + Cfg::kABytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) Op::template mma<BN>(acc, a_desc + 2 * k, b_desc + 2 * k, (kb | k) != 0);
    wgmma_commit();
    // refill the stage the MMAs of kb - 2 read, while the MMAs of kb run
    if (kb + S - 2 < nkb) load(kb + S - 2, (kb + S - 2) % S);
    cp_async_commit();
    wgmma_wait<1>();
    wgmma_fence_regs<BN / 2>(acc);
  }
  wgmma_wait<0>();
  wgmma_fence_regs<BN / 2>(acc);
  cp_async_wait<0>();
  __syncthreads();                   // the ring is free: reuse it for the fp32 accumulator tile

  constexpr int LD = Cfg::kAccLd;
  float* s_acc = reinterpret_cast<float*>(gen);
  {
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int c = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      *reinterpret_cast<float2*>(s_acc + r * LD + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(s_acc + (r + 8) * LD + 8 * j + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  __syncthreads();
  // 4 consecutive channels per thread and step: a warp covers 128 contiguous channels of one or more pixels
  constexpr int Q = BN / 4;
#pragma unroll 2
  for (int i = tid; i < CV_BM * Q; i += CV_THREADS) {
    const int r = i / Q, c = (i - r * Q) * 4;
    const long m = m0 + r;
    const int n = n0 + c;
    if (m >= M || n >= g.Cout) continue;
    const float4 a = *reinterpret_cast<const float4*>(s_acc + r * LD + c);
    if constexpr (RAW) {
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(y) + m * g.Cout + n) = a;
      continue;
    }
    const float4 sc = *reinterpret_cast<const float4*>(scale + n);
    const float4 sh = *reinterpret_cast<const float4*>(shift + n);
    float v0 = fmaf(a.x, sc.x, sh.x), v1 = fmaf(a.y, sc.y, sh.y), v2 = fmaf(a.z, sc.z, sh.z), v3 = fmaf(a.w, sc.w, sh.w);
    const long off = m * g.Cout + n;
    if (resid) {
      const float4 rr = op_ld4<TOp>(resid + off);
      v0 += rr.x; v1 += rr.y; v2 += rr.z; v3 += rr.w;
    }
    if (act) { v0 = silu_fast(v0); v1 = silu_fast(v1); v2 = silu_fast(v2); v3 = silu_fast(v3); }
    store_op4<TOp>(y + off, v0, v1, v2, v3);
  }
}

// ---------------------------------------------------------------- pooling
// MaxPool (1,3,3) / (1,2,2) / pad (0,1,1) of the video stem: (N, Hi, Wi, C) -> (N, Ho, Wo, C); padding never wins
template <typename T>
__global__ void maxpool3x3s2_kernel(const T* __restrict__ x, T* __restrict__ y, int N, int Hi, int Wi, int Ho, int Wo,
                                    int C) {
  pdl_wait();
  pdl_launch_dependents();
  const long total = (long)N * Ho * Wo * C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long p = i / C;
    const int ox = (int)(p % Wo), oy = (int)((p / Wo) % Ho);
    const long n = p / ((long)Wo * Ho);
    float best = -INFINITY;
    T keep = x[((n * Hi + 2 * oy) * Wi + 2 * ox) * C + c];     // the centre tap is always inside
    for (int dy = -1; dy <= 1; ++dy) {
      const int iy = 2 * oy + dy;
      if (iy < 0 || iy >= Hi) continue;
      for (int dx = -1; dx <= 1; ++dx) {
        const int ix = 2 * ox + dx;
        if (ix < 0 || ix >= Wi) continue;
        const T v = x[((n * Hi + iy) * Wi + ix) * C + c];
        const float f = op_ld<T>(&v);
        if (f > best) { best = f; keep = v; }
      }
    }
    y[i] = keep;
  }
}

// mean over groups of P consecutive rows: AdaptiveAvgPool2d(1) per frame (P = H*W of layer4) / AvgPool1d(20) (P = 20)
template <typename T>
__global__ void mean_rows_kernel(const T* __restrict__ x, float* __restrict__ out, long G, int P, int C) {
  pdl_wait();
  pdl_launch_dependents();
  const long total = G * C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long gi = i / C;
    const int c = (int)(i - gi * C);
    const T* p = x + gi * P * C + c;
    float s = 0.f;
    for (int j = 0; j < P; ++j) s += op_ld<T>(p + (long)j * C);
    out[i] = s / (float)P;
  }
}

// ---------------------------------------------------------------- launchers
static int grid_1d(long n) { long b = (n + 255) / 256; return (int)(b < 8192 ? (b > 0 ? b : 1) : 8192); }

template <typename TOp, int BN, bool STEM, bool RAW = false>
static int launch_conv_tc_t(const void* x, const void* w, const float* scale, const float* shift, const void* resid,
                            void* y, const ConvGeom& g, int act, cudaStream_t st) {
  auto kernel = conv_tc_kernel<TOp, BN, STEM, RAW>;
  AVSR_SET_MAX_SMEM(kernel, CvCfg<BN>::kSmem);
  const long M = conv_rows(g);
  const dim3 grid((unsigned)((M + CV_BM - 1) / CV_BM), (unsigned)cdiv(g.Cout, BN));
  AVSR_LAUNCH(kernel, grid, CV_THREADS, CvCfg<BN>::kSmem, st, x, reinterpret_cast<const TOp*>(w), scale, shift,
              reinterpret_cast<const TOp*>(resid), reinterpret_cast<TOp*>(y), g, act);
  return AVSR_OK;
}

template <typename TOp, bool STEM, bool RAW = false>
static int launch_conv_tc_bn(const void* x, const void* w, const float* scale, const float* shift, const void* resid,
                             void* y, const ConvGeom& g, int act, cudaStream_t st) {
  if (g.Cout <= 64) return launch_conv_tc_t<TOp, 64, STEM, RAW>(x, w, scale, shift, resid, y, g, act, st);
  return launch_conv_tc_t<TOp, 128, STEM, RAW>(x, w, scale, shift, resid, y, g, act, st);
}

// one conv + BN [+ resid] [+ SiLU]; x fp32 when `stem`, else operand storage of `kind`
static int run_conv(int kind, bool stem, const void* x, const void* w, const float* scale, const float* shift,
                    const void* resid, void* y, const ConvGeom& g, int act, cudaStream_t st) {
  const long M = conv_rows(g);
  if (M <= 0) return AVSR_OK;
  AVSR_REQUIRE(g.Cout % 64 == 0 && g.Kp % 64 == 0 && (stem || g.Cin % 64 == 0),
               "conv: C_out=%d, C_in=%d must be multiples of 64", g.Cout, g.Cin);
  AVSR_REQUIRE(M / CV_BM < (long)INT32_MAX, "conv: too many output pixels");
  if (kind == OP_F32) {
    const dim3 grid((unsigned)((M + 3) / 4), (unsigned)(g.Cout / 64));
    AVSR_REQUIRE(grid.x <= (unsigned)INT32_MAX, "conv: too many output pixels");
    AVSR_LAUNCH(conv_direct_kernel, grid, dim3(64, 4), 0, st, reinterpret_cast<const float*>(x),
                reinterpret_cast<const float*>(w), scale, shift, reinterpret_cast<const float*>(resid),
                reinterpret_cast<float*>(y), g, act);
    return AVSR_OK;
  }
  if (kind == OP_F16) {
    return stem ? launch_conv_tc_bn<__half, true>(x, w, scale, shift, resid, y, g, act, st)
                : launch_conv_tc_bn<__half, false>(x, w, scale, shift, resid, y, g, act, st);
  }
  if (kind == OP_BF16) {
    return stem ? launch_conv_tc_bn<__nv_bfloat16, true>(x, w, scale, shift, resid, y, g, act, st)
                : launch_conv_tc_bn<__nv_bfloat16, false>(x, w, scale, shift, resid, y, g, act, st);
  }
  return stem ? launch_conv_tc_bn<float, true>(x, w, scale, shift, resid, y, g, act, st)
              : launch_conv_tc_bn<float, false>(x, w, scale, shift, resid, y, g, act, st);
}

// ---------------------------------------------------------------- the two trunks
struct ConvSpec { int cin, cout, kt, kh, kw, stride, K, Kp; };
struct FrontendLayout {
  ConvSpec conv[AVSR_FRONTEND_CONVS];
  size_t w_off[AVSR_FRONTEND_CONVS], s_off[AVSR_FRONTEND_CONVS];   // weights; scale (shift follows at + cout floats)
  size_t total;
};

// conv index in the reference's state-dict order: 0 stem; per BasicBlock conv1, conv2 [, downsample]
static void frontend_layout(int modality, int kind, FrontendLayout* L) {
  const bool video = modality == AVSR_FRONTEND_VIDEO;
  int i = 0;
  L->conv[i++] = video ? ConvSpec{1, 64, 5, 7, 7, 2, 245, 256} : ConvSpec{1, 64, 1, 1, 80, 4, 80, 128};
  const int kh = video ? 3 : 1;
  int cin = 64;
  for (int l = 0; l < 4; ++l) {
    const int planes = 64 << l;
    for (int b = 0; b < 2; ++b) {
      const int s = (l > 0 && b == 0) ? 2 : 1;
      L->conv[i++] = ConvSpec{cin, planes, 1, kh, 3, s, kh * 3 * cin, kh * 3 * cin};
      L->conv[i++] = ConvSpec{planes, planes, 1, kh, 3, 1, kh * 3 * planes, kh * 3 * planes};
      if (l > 0 && b == 0) L->conv[i++] = ConvSpec{cin, planes, 1, 1, 1, 2, cin, cin};
      cin = planes;
    }
  }
  size_t off = 0;
  const size_t esz = operand_bytes(kind);
  for (int j = 0; j < AVSR_FRONTEND_CONVS; ++j) {
    L->w_off[j] = off;
    off = align_up(off + (size_t)L->conv[j].cout * L->conv[j].Kp * esz, 256);
    L->s_off[j] = off;
    off = align_up(off + 2 * (size_t)L->conv[j].cout * 4, 256);
  }
  L->total = off;
}

// trunk geometry with the reference's padding (k - 1) / 2; 1-D convs are H = KH = 1 (then Ho = 1 for any stride)
static ConvGeom trunk_geom(int N, int H, int W, const ConvSpec& c) {
  ConvGeom g{};
  g.N = N; g.T = 1; g.H = H; g.W = W; g.Cin = c.cin; g.Cout = c.cout;
  g.KT = 1; g.KH = c.kh; g.KW = c.kw; g.sh = c.stride; g.sw = c.stride;
  g.pt = 0; g.ph = (c.kh - 1) / 2; g.pw = (c.kw - 1) / 2;
  g.Ho = (H + 2 * g.ph - g.KH) / g.sh + 1;
  g.Wo = (W + 2 * g.pw - g.KW) / g.sw + 1;
  g.ld_frame = (long)H * W * c.cin;
  g.K = c.K; g.Kp = c.Kp;
  return g;
}

struct FrontendPlan {
  ConvGeom stem;
  int N, H0, W0;             // trunk input (after the video max-pool)
  long groups;               // output rows (B * T_out)
  size_t pre_bytes, act_bytes;
  size_t total;
};

static void frontend_plan(int modality, int kind, int B, int T_in, int H, int W, const FrontendLayout& L,
                          FrontendPlan* p) {
  const size_t esz = operand_bytes(kind);
  ConvGeom& s = p->stem;
  s = ConvGeom{};
  s.Cin = 1; s.Cout = 64; s.K = L.conv[0].K; s.Kp = L.conv[0].Kp;
  if (modality == AVSR_FRONTEND_VIDEO) {
    s.N = B * T_in; s.T = T_in; s.H = H; s.W = W;
    s.KT = 5; s.KH = 7; s.KW = 7; s.sh = 2; s.sw = 2; s.pt = 2; s.ph = 3; s.pw = 3;
    s.Ho = (H + 6 - 7) / 2 + 1; s.Wo = (W + 6 - 7) / 2 + 1;
    s.ld_frame = (long)H * W;
    p->N = s.N; p->H0 = (s.Ho + 2 - 3) / 2 + 1; p->W0 = (s.Wo + 2 - 3) / 2 + 1;
    p->groups = s.N;
  } else {
    const int Lt = T_in / 640 * 640;
    s.N = B; s.T = 1; s.H = 1; s.W = Lt;
    s.KT = 1; s.KH = 1; s.KW = 80; s.sh = 1; s.sw = 4; s.pt = 0; s.ph = 0; s.pw = 38;
    s.Ho = 1; s.Wo = Lt > 0 ? (Lt + 76 - 80) / 4 + 1 : 0;
    s.ld_frame = T_in;
    p->N = B; p->H0 = 1; p->W0 = s.Wo;
    p->groups = (long)B * (T_in / 640);
  }
  p->pre_bytes = (size_t)conv_rows(s) * 64 * esz;
  size_t act = (size_t)p->N * p->H0 * p->W0 * 64 * esz;
  int h = p->H0, w = p->W0, j = 1;
  for (int l = 0; l < 4; ++l) {
    for (int b = 0; b < 2; ++b) {
      const ConvGeom g1 = trunk_geom(p->N, h, w, L.conv[j]);     // conv2 and downsample give the same shape
      const size_t bytes = (size_t)conv_rows(g1) * g1.Cout * esz;
      if (bytes > act) act = bytes;
      h = g1.Ho; w = g1.Wo;
      j += (l > 0 && b == 0) ? 3 : 2;
    }
  }
  p->act_bytes = align_up(act, 256);
  p->pre_bytes = align_up(p->pre_bytes, 256);
  const size_t b0 = p->pre_bytes > p->act_bytes ? p->pre_bytes : p->act_bytes;
  p->total = b0 + 3 * p->act_bytes + 256;
}

}  // namespace avsr

using namespace avsr;

extern "C" size_t avsr_frontend_prepared_bytes(int modality, int precision) {
  if ((modality != AVSR_FRONTEND_VIDEO && modality != AVSR_FRONTEND_AUDIO) || !valid_precision(precision)) return 0;
  FrontendLayout L;
  frontend_layout(modality, operand_kind(precision), &L);
  return L.total;
}

extern "C" int avsr_prepare_frontend(int modality, const AvsrConvBnParams* params, void* prepared,
                                     size_t prepared_bytes, int precision, void* stream) {
  AVSR_REQUIRE(modality == AVSR_FRONTEND_VIDEO || modality == AVSR_FRONTEND_AUDIO, "frontend: bad modality %d", modality);
  AVSR_REQUIRE(valid_precision(precision), "frontend: bad precision %d", precision);
  AVSR_REQUIRE(params && prepared, "NULL argument");
  const int kind = operand_kind(precision);
  FrontendLayout L;
  frontend_layout(modality, kind, &L);
  AVSR_REQUIRE_BYTES(L.total, prepared_bytes, "frontend prepared buffer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* base = reinterpret_cast<uint8_t*>(prepared);
  for (int j = 0; j < AVSR_FRONTEND_CONVS; ++j) {
    const AvsrConvBnParams& p = params[j];
    const ConvSpec& c = L.conv[j];
    AVSR_REQUIRE(p.conv_w && p.bn_w && p.bn_b && p.bn_mean && p.bn_var && p.eps >= 0.0,
                 "frontend: conv %d has a NULL parameter or negative eps", j);
    const long n = (long)c.cout * c.Kp;
    AVSR_LAUNCH(reorder_weight_kernel, grid_1d(n), 256, 0, st, p.conv_w, (void*)(base + L.w_off[j]), c.cout, c.cin,
                c.kt * c.kh * c.kw, c.Kp, kind);
    float* sc = reinterpret_cast<float*>(base + L.s_off[j]);
    AVSR_LAUNCH(bn_fold_kernel, cdiv(c.cout, 256), 256, 0, st, p.bn_w, p.bn_b, p.bn_mean, p.bn_var, p.eps, sc,
                sc + c.cout, c.cout);
  }
  return AVSR_OK;
}

static bool frontend_shape_ok(int modality, int B, int T_in, int H, int W) {
  if (B < 0 || T_in < 0) return false;
  if (modality == AVSR_FRONTEND_VIDEO) return H >= 1 && W >= 1 && (long)B * T_in * H * W < (1L << 40);
  return true;
}

extern "C" size_t avsr_frontend_workspace_bytes(int modality, int B, int T_in, int H, int W, int precision) {
  if ((modality != AVSR_FRONTEND_VIDEO && modality != AVSR_FRONTEND_AUDIO) || !valid_precision(precision) ||
      !frontend_shape_ok(modality, B, T_in, H, W))
    return 0;
  const int kind = operand_kind(precision);
  FrontendLayout L;
  frontend_layout(modality, kind, &L);
  FrontendPlan P;
  frontend_plan(modality, kind, B, T_in, H, W, L, &P);
  return P.total;
}

// the forward of avsr_frontend_forward; taps[i] != NULL receives stage i as fp32 (avsr_frontend_tap_shape)
static int frontend_forward_body(int modality, const void* prepared, const float* x, int B, int T_in, int H, int W,
                                 float* out, void* workspace, size_t workspace_bytes, int precision, void* stream,
                                 float* const* taps) {
  AVSR_REQUIRE(modality == AVSR_FRONTEND_VIDEO || modality == AVSR_FRONTEND_AUDIO, "frontend: bad modality %d", modality);
  AVSR_REQUIRE(valid_precision(precision), "frontend: bad precision %d", precision);
  AVSR_REQUIRE(frontend_shape_ok(modality, B, T_in, H, W), "frontend: bad shape B=%d T=%d H=%d W=%d", B, T_in, H, W);
  const int kind = operand_kind(precision);
  FrontendLayout L;
  frontend_layout(modality, kind, &L);
  FrontendPlan P;
  frontend_plan(modality, kind, B, T_in, H, W, L, &P);
  if (P.groups == 0) return AVSR_OK;
  AVSR_REQUIRE(prepared && x && out && workspace, "NULL argument");
  AVSR_REQUIRE_BYTES(P.total, workspace_bytes, "frontend workspace");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const uint8_t* pb = reinterpret_cast<const uint8_t*>(prepared);
  auto wt = [&](int j) { return static_cast<const void*>(pb + L.w_off[j]); };
  auto sc = [&](int j) { return reinterpret_cast<const float*>(pb + L.s_off[j]); };
  auto sh = [&](int j) { return reinterpret_cast<const float*>(pb + L.s_off[j]) + L.conv[j].cout; };
  uint8_t* ws = reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<uintptr_t>(workspace), 256));
  const size_t b0 = P.pre_bytes > P.act_bytes ? P.pre_bytes : P.act_bytes;
  void* buf[4] = {ws, ws + b0, ws + b0 + P.act_bytes, ws + b0 + 2 * P.act_bytes};
  auto tap = [&](int i, const void* src, long n) -> int {
    if (taps && taps[i]) AVSR_LAUNCH(cvt_from_op_kernel, grid_1d(n), 256, 0, st, src, taps[i], n, kind);
    return AVSR_OK;
  };

  // stem (+ max-pool for video) -> buf[1]
  int cur = 1;
  if (modality == AVSR_FRONTEND_VIDEO) {
    AVSR_TRY(run_conv(kind, true, x, wt(0), sc(0), sh(0), nullptr, buf[0], P.stem, 1, st));
    AVSR_TRY(tap(0, buf[0], conv_rows(P.stem) * 64));
    const long n = (long)P.N * P.H0 * P.W0 * 64;
    if (kind == OP_F16)
      AVSR_LAUNCH(maxpool3x3s2_kernel<__half>, grid_1d(n), 256, 0, st, (const __half*)buf[0], (__half*)buf[1], P.N,
                  P.stem.Ho, P.stem.Wo, P.H0, P.W0, 64);
    else if (kind == OP_BF16)
      AVSR_LAUNCH(maxpool3x3s2_kernel<__nv_bfloat16>, grid_1d(n), 256, 0, st, (const __nv_bfloat16*)buf[0],
                  (__nv_bfloat16*)buf[1], P.N, P.stem.Ho, P.stem.Wo, P.H0, P.W0, 64);
    else
      AVSR_LAUNCH(maxpool3x3s2_kernel<float>, grid_1d(n), 256, 0, st, (const float*)buf[0], (float*)buf[1], P.N,
                  P.stem.Ho, P.stem.Wo, P.H0, P.W0, 64);
  } else {
    AVSR_TRY(run_conv(kind, true, x, wt(0), sc(0), sh(0), nullptr, buf[1], P.stem, 1, st));
    AVSR_TRY(tap(0, buf[1], conv_rows(P.stem) * 64));
  }
  AVSR_TRY(tap(1, buf[1], (long)P.N * P.H0 * P.W0 * 64));
  // BasicBlocks: h = SiLU(BN1(conv1 x)); r = BN(downsample x) or x; x = SiLU(BN2(conv2 h) + r)
  int h = P.H0, w = P.W0, j = 1;
  for (int l = 0; l < 4; ++l) {
    for (int b = 0; b < 2; ++b) {
      const bool ds = l > 0 && b == 0;
      int fr[3], nf = 0;
      for (int q = 0; q < 4; ++q) if (q != cur) fr[nf++] = q;
      const ConvGeom g1 = trunk_geom(P.N, h, w, L.conv[j]);
      AVSR_TRY(run_conv(kind, false, buf[cur], wt(j), sc(j), sh(j), nullptr, buf[fr[0]], g1, 1, st));
      const ConvGeom g2 = trunk_geom(P.N, g1.Ho, g1.Wo, L.conv[j + 1]);
      int res = cur;
      if (ds) {
        const ConvGeom gd = trunk_geom(P.N, h, w, L.conv[j + 2]);
        AVSR_TRY(run_conv(kind, false, buf[cur], wt(j + 2), sc(j + 2), sh(j + 2), nullptr, buf[fr[1]], gd, 0, st));
        res = fr[1];
      }
      const int dst = fr[2];
      AVSR_TRY(run_conv(kind, false, buf[fr[0]], wt(j + 1), sc(j + 1), sh(j + 1), buf[res], buf[dst], g2, 1, st));
      cur = dst;
      AVSR_TRY(tap(2 + 2 * l + b, buf[cur], conv_rows(g2) * g2.Cout));
      h = g2.Ho; w = g2.Wo;
      j += ds ? 3 : 2;
    }
  }
  // pool: per video frame over its h x w pixels; per 20 audio positions
  const int Pn = modality == AVSR_FRONTEND_VIDEO ? h * w : 20;
  const long n = P.groups * 512;
  if (kind == OP_F16)
    AVSR_LAUNCH(mean_rows_kernel<__half>, grid_1d(n), 256, 0, st, (const __half*)buf[cur], out, P.groups, Pn, 512);
  else if (kind == OP_BF16)
    AVSR_LAUNCH(mean_rows_kernel<__nv_bfloat16>, grid_1d(n), 256, 0, st, (const __nv_bfloat16*)buf[cur], out, P.groups,
                Pn, 512);
  else
    AVSR_LAUNCH(mean_rows_kernel<float>, grid_1d(n), 256, 0, st, (const float*)buf[cur], out, P.groups, Pn, 512);
  return AVSR_OK;
}

extern "C" int avsr_frontend_forward(int modality, const void* prepared, const float* x, int B, int T_in, int H, int W,
                                     float* out, void* workspace, size_t workspace_bytes, int precision, void* stream) {
  return frontend_forward_body(modality, prepared, x, B, T_in, H, W, out, workspace, workspace_bytes, precision, stream,
                               nullptr);
}

extern "C" int avsr_frontend_forward_taps(int modality, const void* prepared, const float* x, int B, int T_in, int H,
                                          int W, float* out, float* const* taps, void* workspace,
                                          size_t workspace_bytes, int precision, void* stream) {
  AVSR_REQUIRE(taps, "NULL argument");
  return frontend_forward_body(modality, prepared, x, B, T_in, H, W, out, workspace, workspace_bytes, precision, stream,
                               taps);
}

extern "C" int avsr_frontend_tap_shape(int modality, int B, int T_in, int H, int W, int tap, int* dims) {
  AVSR_REQUIRE(modality == AVSR_FRONTEND_VIDEO || modality == AVSR_FRONTEND_AUDIO, "frontend: bad modality %d", modality);
  AVSR_REQUIRE(frontend_shape_ok(modality, B, T_in, H, W), "frontend: bad shape B=%d T=%d H=%d W=%d", B, T_in, H, W);
  AVSR_REQUIRE(tap >= 0 && tap < AVSR_FRONTEND_TAPS && dims, "frontend: bad tap %d or NULL dims", tap);
  FrontendLayout L;
  frontend_layout(modality, OP_F32, &L);
  FrontendPlan P;
  frontend_plan(modality, OP_F32, B, T_in, H, W, L, &P);
  int h = P.H0, w = P.W0, c = 64, j = 1;
  if (tap == 0) { h = P.stem.Ho; w = P.stem.Wo; }
  for (int b = 0; b + 2 <= tap; ++b) {          // BasicBlock b = 2 * layer + index: conv1 sets the output geometry
    const ConvGeom g1 = trunk_geom(P.N, h, w, L.conv[j]);
    h = g1.Ho; w = g1.Wo; c = g1.Cout;
    j += (b == 2 || b == 4 || b == 6) ? 3 : 2;
  }
  if (P.W0 == 0) w = 0;                          // audio shorter than one 640-sample frame: every tap is empty
  dims[0] = P.N; dims[1] = h; dims[2] = w; dims[3] = c;
  return AVSR_OK;
}

extern "C" size_t avsr_conv_bn_act_workspace_bytes(int N, int H, int W, int C_in, int C_out, int KH, int KW, int stride,
                                                   int precision) {
  if (N < 0 || H < 1 || W < 1 || C_in < 1 || C_out < 1 || KH < 1 || KW < 1 || stride < 1 || !valid_precision(precision))
    return 0;
  const ConvSpec c{C_in, C_out, 1, KH, KW, stride, KH * KW * C_in, KH * KW * C_in};
  const ConvGeom g = trunk_geom(N, H, W, c);
  const size_t esz = operand_bytes(operand_kind(precision));
  return align_up((size_t)N * H * W * C_in * esz, 256) + align_up((size_t)C_out * g.Kp * esz, 256) +
         2 * align_up((size_t)conv_rows(g) * C_out * esz, 256) + 256;
}

extern "C" int avsr_conv_bn_act(const float* x, const float* w, const float* scale, const float* shift,
                                const float* resid, int act, float* y, int N, int H, int W, int C_in, int C_out, int KH,
                                int KW, int stride, void* workspace, size_t workspace_bytes, int precision,
                                void* stream) {
  AVSR_REQUIRE(valid_precision(precision), "conv_bn_act: bad precision %d", precision);
  AVSR_REQUIRE(N >= 0 && H >= 1 && W >= 1 && C_in % 64 == 0 && C_in > 0 && C_out % 64 == 0 && C_out > 0 &&
                   (KH == 1 || KH == 3) && (KW == 1 || KW == 3) && stride >= 1,
               "conv_bn_act: unsupported shape N=%d H=%d W=%d C_in=%d C_out=%d KH=%d KW=%d stride=%d", N, H, W, C_in,
               C_out, KH, KW, stride);
  AVSR_REQUIRE(x && w && scale && shift && y && workspace, "NULL argument");
  AVSR_REQUIRE(((reinterpret_cast<uintptr_t>(scale) | reinterpret_cast<uintptr_t>(shift)) & 15) == 0,
               "conv_bn_act: scale / shift must be 16-byte aligned");
  const size_t need = avsr_conv_bn_act_workspace_bytes(N, H, W, C_in, C_out, KH, KW, stride, precision);
  AVSR_REQUIRE_BYTES(need, workspace_bytes, "conv_bn_act workspace");
  const int kind = operand_kind(precision);
  const size_t esz = operand_bytes(kind);
  const ConvSpec c{C_in, C_out, 1, KH, KW, stride, KH * KW * C_in, KH * KW * C_in};
  const ConvGeom g = trunk_geom(N, H, W, c);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long nx = (long)N * H * W * C_in, ny = conv_rows(g) * C_out;
  uint8_t* p = reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<uintptr_t>(workspace), 256));
  void* xo = p;  p += align_up((size_t)nx * esz, 256);
  void* wo = p;  p += align_up((size_t)C_out * g.Kp * esz, 256);
  void* ro = p;  p += align_up((size_t)ny * esz, 256);
  void* yo = p;
  if (ny == 0) return AVSR_OK;
  AVSR_LAUNCH(cvt_to_op_kernel, grid_1d(nx), 256, 0, st, x, xo, nx, kind);
  AVSR_LAUNCH(reorder_weight_kernel, grid_1d((long)C_out * g.Kp), 256, 0, st, w, wo, C_out, C_in, KH * KW, g.Kp, kind);
  if (resid) AVSR_LAUNCH(cvt_to_op_kernel, grid_1d(ny), 256, 0, st, resid, ro, ny, kind);
  AVSR_TRY(run_conv(kind, false, xo, wo, scale, shift, resid ? ro : nullptr, yo, g, act, st));
  AVSR_LAUNCH(cvt_from_op_kernel, grid_1d(ny), 256, 0, st, (const void*)yo, y, ny, kind);
  return AVSR_OK;
}

// ================================================================ training (batch-statistics BatchNorm)
// The front-end's training path is a chain of library calls that auto_avsr_b200/frontend_train.py drives per conv unit
// (conv -> BatchNorm -> [+ residual] -> [SiLU]).  Activations cross the boundary as fp32 channels-last tensors.
//  - forward conv: the inference implicit GEMM (conv_tc_kernel, RAW epilogue: the fp32 accumulator) or, in fp32, the
//    direct kernel with scale 1 and shift 0; then the batch statistics of every channel (launch_bn_stats, train.cu,
//    which also holds the BatchNorm's normalise and backward: the avsr_bn_train_* entries);
//  - dgrad: stride 1 is the same implicit GEMM over dZ with the 180-degree-rotated weight; stride 2 splits the input
//    gradient into its parity classes, each a stride-1 implicit GEMM with a 1- or 2-tap sub-filter per axis (no MAC on
//    inserted zeros), scattered to the class's pixels;
//  - wgrad: a CUDA-core fp32 GEMM over output pixels, split across the SMs with partials summed in a fixed order;
//  - max-pool with a recorded winner (first maximum in scan order, NaN wins: torch's rule) and a gather backward.
namespace avsr {

__global__ void fill_f32_kernel(float* p, int n, float v) {
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// ---------------------------------------------------------------- dgrad sub-filters
// Input pixel i = s * a + r of an axis with K taps, stride s, padding p receives output o = a + d from tap
// k = r + p - s * d for every d with 0 <= k < K.  The d of one class are contiguous: [dmin, dmin + n).
struct AxisClass { int dmin, n; };
static AxisClass axis_class(int K, int s, int p, int r) {
  int lo = 1 << 30, hi = -(1 << 30);
  for (int k = 0; k < K; ++k) {
    const int t = r + p - k;
    if (t % s != 0) continue;
    const int d = t / s;
    lo = d < lo ? d : lo;
    hi = d > hi ? d : hi;
  }
  return lo > hi ? AxisClass{0, 0} : AxisClass{lo, hi - lo + 1};
}

// sub-filter of one parity class as implicit-GEMM rows: dst[ci][(ty * nx + tx) * Cout + co] = w[co][ci][ky][kx],
// ky = ry + py - s * (dy0 + ty) (likewise x); w is torch's (Cout, Cin, KH, KW)
__global__ void ft_dgrad_weight_kernel(const float* __restrict__ w, void* __restrict__ dst, int Cout, int Cin, int KH,
                                       int KW, int s, int ry, int rx, int py, int px, int dy0, int dx0, int ny, int nx,
                                       int kind) {
  pdl_wait();
  const int Kp = ny * nx * Cout;
  const long n = (long)Cin * Kp;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int ci = (int)(i / Kp), k = (int)(i - (long)ci * Kp);
    const int tap = k / Cout, co = k - tap * Cout;
    const int ty = tap / nx, tx = tap - ty * nx;
    const int ky = ry + py - s * (dy0 + ty), kx = rx + px - s * (dx0 + tx);
    float v = 0.f;
    if (ky >= 0 && ky < KH && kx >= 0 && kx < KW) v = w[(((long)co * Cin + ci) * KH + ky) * KW + kx];
    store_kind1(dst, i, kind, v);
  }
}

// dx[n][s a + ry][s b + rx][c] = sub[n][a][b][c] (sub NULL: 0)
__global__ void ft_scatter_class_kernel(const float* __restrict__ sub, float* __restrict__ dx, int N, int H, int W,
                                        int C, int s, int ry, int rx, int Hc, int Wc) {
  pdl_wait();
  const long n = (long)N * Hc * Wc * C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long p = i / C;
    const int b = (int)(p % Wc), a = (int)((p / Wc) % Hc);
    const long f = p / ((long)Wc * Hc);
    dx[((f * H + (long)s * a + ry) * W + (long)s * b + rx) * C + c] = sub ? sub[i] : 0.f;
  }
}

// ---------------------------------------------------------------- wgrad (CUDA cores, fp32)
// dw_part[split][co][k] = sum over this split's output pixels m of dz[m][co] * x[src(m, k)], k = tap * Cin + c.
// 64 x 64 outputs per CTA, 4 x 4 per thread, 16 pixels per step through shared memory.
constexpr int WG_T = 64, WG_P = 16;

__device__ __forceinline__ float ft_gather(const float* __restrict__ x, const ConvGeom& g, long m, int k) {
  if (k >= g.K) return 0.f;
  const int hw = g.Ho * g.Wo;
  const int n = (int)(m / hw), r = (int)(m - (long)n * hw);
  const int oy = r / g.Wo, ox = r - oy * g.Wo;
  const int t = n % g.T;
  const int tap = k / g.Cin, c = k - tap * g.Cin;
  const int kx = tap % g.KW, q = tap / g.KW;
  const int ky = q % g.KH, dt = q / g.KH;
  const int tt = t + dt - g.pt, iy = oy * g.sh - g.ph + ky, ix = ox * g.sw - g.pw + kx;
  if (tt < 0 || tt >= g.T || iy < 0 || iy >= g.H || ix < 0 || ix >= g.W) return 0.f;
  return x[(long)(n - t + tt) * g.ld_frame + ((long)iy * g.W + ix) * g.Cin + c];
}

__global__ void __launch_bounds__(256) ft_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dz,
                                                       float* __restrict__ part, ConvGeom g, long rows_per_split,
                                                       int Kw) {
  pdl_wait();
  __shared__ float sa[WG_P][WG_T];     // dz[pixel][co]
  __shared__ float sb[WG_P][WG_T];     // x[pixel][k]
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int k0 = blockIdx.x * WG_T, co0 = blockIdx.y * WG_T;
  const long M = (long)g.N * g.Ho * g.Wo;
  const long p0 = (long)blockIdx.z * rows_per_split, p1 = min(M, p0 + rows_per_split);
  float acc[4][4] = {};
  const int lp = tid >> 4, lc = (tid & 15) * 4;      // loader: pixel lp, columns lc .. lc + 3
  for (long pb = p0; pb < p1; pb += WG_P) {
    const long m = pb + lp;
    const bool ok = m < p1;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      sa[lp][lc + e] = ok ? dz[m * g.Cout + co0 + lc + e] : 0.f;
      sb[lp][lc + e] = ok ? ft_gather(x, g, m, k0 + lc + e) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int p = 0; p < WG_P; ++p) {
      const float4 a = *reinterpret_cast<const float4*>(&sa[p][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&sb[p][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* out = part + (long)blockIdx.z * g.Cout * Kw;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    *reinterpret_cast<float4*>(out + (long)(co0 + ty * 4 + i) * Kw + k0 + tx * 4) =
        make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
}

// The same partials on wgmma with TF32 operands: one warpgroup per 64 (co) x 64 (k) tile, 32 output pixels per K-block.
// Both operands are channels-last, so each K-block is transposed on its way into the 128B-swizzled tiles: thread t
// reads column t % 64 (a C_out channel of dz, a k of the gathered input) for pixels t / 64 + 2 i with coalesced
// loads, rounds to TF32 and stores the element at (column, pixel).  Two stages: the loads of K-block kb + 1 run under
// the MMAs of kb.  The pixel coordinates of a K-block are decoded once into shared memory.
constexpr int WGT_PB = 32;               // pixels per K-block (128 bytes of TF32)
constexpr int WGT_STAGE = 2 * 64 * 128;  // A (64 co rows) + B (64 k rows)
constexpr int WGT_SMEM = 1024 + 2 * WGT_STAGE + 2 * WGT_PB * 16;

__global__ void __launch_bounds__(128) ft_wgrad_tc_kernel(const float* __restrict__ x, const float* __restrict__ dz,
                                                          float* __restrict__ part, ConvGeom g, long rows_per_split,
                                                          int Kw) {
  pdl_wait();
  extern __shared__ uint8_t wg_smem_raw[];
  const uint32_t raw = smem_u32(wg_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gen = wg_smem_raw + (base - raw);
  int4* table = reinterpret_cast<int4*>(gen + 2 * WGT_STAGE);      // [stage][pixel]: frame base, iy0, ix0, t (-1: none)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int col = tid & 63, prow = tid >> 6;
  const int k0 = blockIdx.x * 64, co0 = blockIdx.y * 64;
  const long M = (long)g.N * g.Ho * g.Wo;
  const long p0 = (long)blockIdx.z * rows_per_split, p1 = min(M, p0 + rows_per_split);
  const int nkb = p1 > p0 ? (int)((p1 - p0 + WGT_PB - 1) / WGT_PB) : 0;
  // this thread's k column: tap and channel, decoded once
  const int k = k0 + col;
  const bool kok = k < g.K;
  const int tap = kok ? k / g.Cin : 0, cch = kok ? k - tap * g.Cin : 0;
  const int kx = tap % g.KW, ky = (tap / g.KW) % g.KH, dt = tap / (g.KW * g.KH);
  // input element of pixel (frame n, iy0, ix0) for this k: n * ld_frame + (iy0 * W + ix0) * Cin + koff
  const long koff = (long)(dt - g.pt) * g.ld_frame + ((long)ky * g.W + kx) * g.Cin + cch;
  const int hw = g.Ho * g.Wo;

  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;

#pragma unroll 1
  for (int kb = 0; kb < nkb; ++kb) {
    const int s = kb & 1;
    const long pb = p0 + (long)kb * WGT_PB;
    if (tid < WGT_PB) {
      const long m = pb + tid;
      int4 e = make_int4(0, 0, 0, -1);
      if (m < p1) {
        const int n = (int)(m / hw), r = (int)(m - (long)n * hw);
        const int oy = r / g.Wo, ox = r - oy * g.Wo;
        e = make_int4(n, oy * g.sh - g.ph, ox * g.sw - g.pw, n % g.T);
      }
      table[s * WGT_PB + tid] = e;
    }
    __syncthreads();          // the table is in; the MMAs of kb - 2 (which read stage s) retired before kb - 1's sync
    uint8_t* sa = gen + s * WGT_STAGE;
    uint8_t* sb = sa + 64 * 128;
#pragma unroll 4
    for (int i = 0; i < WGT_PB / 2; ++i) {
      const int p = prow + 2 * i;
      const int4 e = table[s * WGT_PB + p];
      float a = 0.f, b = 0.f;
      if (e.w >= 0) {
        a = dz[(pb + p) * g.Cout + co0 + col];
        const int tt = e.w + dt - g.pt, iy = e.y + ky, ix = e.z + kx;
        if (kok && tt >= 0 && tt < g.T && iy >= 0 && iy < g.H && ix >= 0 && ix < g.W)
          b = x[(long)e.x * g.ld_frame + ((long)e.y * g.W + e.z) * g.Cin + koff];
      }
      const uint32_t off = sw128(col, p >> 2) + (p & 3) * 4;
      *reinterpret_cast<float*>(sa + off) = round_tf32(a);
      *reinterpret_cast<float*>(sb + off) = round_tf32(b);
    }
    fence_proxy_async();
    __syncthreads();
    const uint64_t a_desc = wgmma_desc_sw128(base + s * WGT_STAGE);
    const uint64_t b_desc = wgmma_desc_sw128(base + s * WGT_STAGE + 64 * 128);
    wgmma_fence();
#pragma unroll
    for (int q = 0; q < 4; ++q) wgmma_tf32_n64(acc, a_desc + 2 * q, b_desc + 2 * q, (kb | q) != 0);
    wgmma_commit();
    wgmma_wait<1>();          // the MMAs of kb - 1 are done: stage s ^ 1 may be rewritten next iteration
    wgmma_fence_regs<32>(acc);
  }
  wgmma_wait<0>();
  wgmma_fence_regs<32>(acc);
  float* out = part + (long)blockIdx.z * g.Cout * Kw;
  const int r = (warp & 3) * 16 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    *reinterpret_cast<float2*>(out + (long)(co0 + r) * Kw + k0 + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2*>(out + (long)(co0 + r + 8) * Kw + k0 + 8 * j + c) =
        make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
}

// dw[co][c][tap] (torch layout) = sum over splits in order of part[split][co][tap * Cin + c]
__global__ void ft_wgrad_finish_kernel(const float* __restrict__ part, float* __restrict__ dw, int splits, int Cout,
                                       int Cin, int taps, int Kw) {
  pdl_wait();
  const long n = (long)Cout * Cin * taps;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int tap = (int)(i % taps);
    const long q = i / taps;
    const int c = (int)(q % Cin), co = (int)(q / Cin);
    const long j = (long)co * Kw + (long)tap * Cin + c;
    float s = 0.f;
    for (int sp = 0; sp < splits; ++sp) s += part[(long)sp * Cout * Kw + j];
    dw[i] = s;
  }
}

// ---------------------------------------------------------------- pooling with recorded winners
__global__ void ft_maxpool_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, uint8_t* __restrict__ idx,
                                      int N, int Hi, int Wi, int Ho, int Wo, int C) {
  pdl_wait();
  const long total = (long)N * Ho * Wo * C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long p = i / C;
    const int ox = (int)(p % Wo), oy = (int)((p / Wo) % Ho);
    const long n = p / ((long)Wo * Ho);
    float best = -INFINITY;
    int win = 4;
    for (int dy = 0; dy < 3; ++dy) {
      const int iy = 2 * oy - 1 + dy;
      if (iy < 0 || iy >= Hi) continue;
      for (int dx = 0; dx < 3; ++dx) {
        const int ix = 2 * ox - 1 + dx;
        if (ix < 0 || ix >= Wi) continue;
        const float v = x[((n * Hi + iy) * Wi + ix) * C + c];
        if (v > best || isnan(v)) { best = v; win = dy * 3 + dx; }
      }
    }
    y[i] = best;
    idx[i] = (uint8_t)win;
  }
}

// dx[pixel] = sum of dy over the (at most 4) windows whose recorded winner is this pixel, in a fixed order
__global__ void ft_maxpool_bwd_kernel(const float* __restrict__ dy, const uint8_t* __restrict__ idx,
                                      float* __restrict__ dx, int N, int Hi, int Wi, int Ho, int Wo, int C) {
  pdl_wait();
  const long total = (long)N * Hi * Wi * C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long p = i / C;
    const int ix = (int)(p % Wi), iy = (int)((p / Wi) % Hi);
    const long n = p / ((long)Wi * Hi);
    float s = 0.f;
    for (int oy = iy / 2 - 1; oy <= iy / 2 + 1; ++oy) {
      const int ky = iy - (2 * oy - 1);
      if (oy < 0 || oy >= Ho || ky < 0 || ky > 2) continue;
      for (int ox = ix / 2 - 1; ox <= ix / 2 + 1; ++ox) {
        const int kx = ix - (2 * ox - 1);
        if (ox < 0 || ox >= Wo || kx < 0 || kx > 2) continue;
        const long o = ((n * Ho + oy) * Wo + ox) * C + c;
        if (idx[o] == ky * 3 + kx) s += dy[o];
      }
    }
    dx[i] = s;
  }
}

// dx[g * P + j][c] = dout[g][c] / P
__global__ void ft_mean_rows_bwd_kernel(const float* __restrict__ dout, float* __restrict__ dx, long G, int P, int C) {
  pdl_wait();
  const long total = G * P * C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long gi = i / ((long)P * C);
    dx[i] = dout[gi * C + c] / (float)P;
  }
}

// ---------------------------------------------------------------- host side
// stem: 0 a trunk conv (x (N, H, W, C_in), padding (K - 1) / 2); 1 the video stem (x (N = B * T frames, H, W), T frames
// per utterance); 2 the audio stem (x (N, W) samples already cut to whole 640-sample frames)
static bool ft_geom(int stem, int N, int T, int H, int W, int Cin, int Cout, int KH, int KW, int stride, ConvGeom* g) {
  if (N < 0 || H < 1 || W < 1) return false;
  if (stem == 1) {
    if (T < 1 || N % T != 0) return false;
    *g = ConvGeom{};
    g->N = N; g->T = T; g->H = H; g->W = W; g->Cin = 1; g->Cout = 64;
    g->KT = 5; g->KH = 7; g->KW = 7; g->sh = 2; g->sw = 2; g->pt = 2; g->ph = 3; g->pw = 3;
    g->Ho = (H + 6 - 7) / 2 + 1; g->Wo = (W + 6 - 7) / 2 + 1;
    g->ld_frame = (long)H * W; g->K = 245; g->Kp = 256;
    return true;
  }
  if (stem == 2) {
    if (H != 1 || W % 640 != 0) return false;
    *g = ConvGeom{};
    g->N = N; g->T = 1; g->H = 1; g->W = W; g->Cin = 1; g->Cout = 64;
    g->KT = 1; g->KH = 1; g->KW = 80; g->sh = 1; g->sw = 4; g->pt = 0; g->ph = 0; g->pw = 38;
    g->Ho = 1; g->Wo = (W + 76 - 80) / 4 + 1;
    g->ld_frame = W; g->K = 80; g->Kp = 128;
    return true;
  }
  if (stem != 0 || Cin < 64 || Cin % 64 || Cout < 64 || Cout % 64 || (KH != 1 && KH != 3) || (KW != 1 && KW != 3) ||
      (stride != 1 && stride != 2))
    return false;
  const ConvSpec c{Cin, Cout, 1, KH, KW, stride, KH * KW * Cin, KH * KW * Cin};
  *g = trunk_geom(N, H, W, c);
  return true;
}

struct FtConvWs { size_t xop, wop, unit, part, total; };
static FtConvWs ft_conv_ws(const ConvGeom& g, int stem, int kind) {
  const size_t esz = operand_bytes(kind);
  FtConvWs w{};
  w.xop = stem ? 0 : align_up((size_t)g.N * g.H * g.W * g.Cin * esz, 256);
  w.wop = align_up((size_t)g.Cout * g.Kp * esz, 256);
  w.unit = align_up(2 * (size_t)g.Cout * 4, 256);
  w.part = avsr_bn_train_workspace_bytes(conv_rows(g), g.Cout);
  w.total = w.xop + w.wop + w.unit + w.part + 256;
  return w;
}

static int run_conv_raw(int kind, bool stem, const void* x, const void* w, const float* ones, const float* zeros,
                        float* z, const ConvGeom& g, cudaStream_t st) {
  if (kind == OP_F32) return run_conv(kind, stem, x, w, ones, zeros, nullptr, z, g, 0, st);
  const long M = conv_rows(g);
  if (M <= 0) return AVSR_OK;
  AVSR_REQUIRE(M / CV_BM < (long)INT32_MAX, "conv: too many output pixels");
  if (kind == OP_F16)
    return stem ? launch_conv_tc_bn<__half, true, true>(x, w, nullptr, nullptr, nullptr, z, g, 0, st)
                : launch_conv_tc_bn<__half, false, true>(x, w, nullptr, nullptr, nullptr, z, g, 0, st);
  if (kind == OP_BF16)
    return stem ? launch_conv_tc_bn<__nv_bfloat16, true, true>(x, w, nullptr, nullptr, nullptr, z, g, 0, st)
                : launch_conv_tc_bn<__nv_bfloat16, false, true>(x, w, nullptr, nullptr, nullptr, z, g, 0, st);
  return stem ? launch_conv_tc_bn<float, true, true>(x, w, nullptr, nullptr, nullptr, z, g, 0, st)
              : launch_conv_tc_bn<float, false, true>(x, w, nullptr, nullptr, nullptr, z, g, 0, st);
}

struct FtDgradWs { size_t dzop, wop, unit, sub, total; };
static FtDgradWs ft_dgrad_ws(const ConvGeom& g, int kind) {
  const size_t esz = operand_bytes(kind);
  FtDgradWs w{};
  w.dzop = align_up((size_t)conv_rows(g) * g.Cout * esz, 256);
  w.wop = align_up((size_t)g.Cin * g.KH * g.KW * g.Cout * esz, 256);     // the largest sub-filter is the whole filter
  w.unit = align_up(2 * (size_t)g.Cin * 4, 256);
  const int s = g.sh;
  const size_t hc = (size_t)(g.H + s - 1) / s, wc = (size_t)(g.W + s - 1) / s;
  w.sub = s == 1 ? 0 : align_up((size_t)g.N * hc * wc * g.Cin * 4, 256);
  w.total = w.dzop + w.wop + w.unit + w.sub + 256;
  return w;
}

static int ft_wgrad_splits(const ConvGeom& g) {
  const long M = conv_rows(g);
  const int tiles = cdiv(g.K, WG_T) * (g.Cout / WG_T);
  long s = (132L * 4 + tiles - 1) / tiles;
  const long max_s = (M + 255) / 256;              // at least 256 pixels per split
  if (s > max_s) s = max_s;
  return (int)(s < 1 ? 1 : s);
}
static size_t ft_wgrad_ws(const ConvGeom& g) {
  const int Kw = cdiv(g.K, WG_T) * WG_T;
  return align_up((size_t)ft_wgrad_splits(g) * g.Cout * Kw * 4, 256) + 256;
}

}  // namespace avsr

static bool ft_prec_ok(int precision) { return valid_precision(precision); }

extern "C" size_t avsr_frontend_train_conv_workspace_bytes(int stem, int N, int T, int H, int W, int C_in, int C_out,
                                                           int KH, int KW, int stride, int precision) {
  ConvGeom g;
  if (!ft_prec_ok(precision) || !ft_geom(stem, N, T, H, W, C_in, C_out, KH, KW, stride, &g)) return 0;
  return ft_conv_ws(g, stem, operand_kind(precision)).total;
}

extern "C" int avsr_frontend_train_conv_fwd(const float* x, const float* w, float* z, double* stats, int stem, int N,
                                            int T, int H, int W, int C_in, int C_out, int KH, int KW, int stride,
                                            void* workspace, size_t workspace_bytes, int precision, void* stream) {
  AVSR_REQUIRE(ft_prec_ok(precision), "frontend train conv: bad precision %d", precision);
  ConvGeom g;
  AVSR_REQUIRE(ft_geom(stem, N, T, H, W, C_in, C_out, KH, KW, stride, &g),
               "frontend train conv: unsupported shape stem=%d N=%d T=%d H=%d W=%d C_in=%d C_out=%d KH=%d KW=%d "
               "stride=%d", stem, N, T, H, W, C_in, C_out, KH, KW, stride);
  AVSR_REQUIRE(x && w && z && stats && workspace, "NULL argument");
  const int kind = operand_kind(precision);
  const FtConvWs L = ft_conv_ws(g, stem, kind);
  AVSR_REQUIRE_BYTES(L.total, workspace_bytes, "frontend train conv workspace");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long M = conv_rows(g);
  if (M == 0) return AVSR_OK;
  uint8_t* p = reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<uintptr_t>(workspace), 256));
  void* xo = p; p += L.xop;
  void* wo = p; p += L.wop;
  float* ones = reinterpret_cast<float*>(p); p += L.unit;
  double* part = reinterpret_cast<double*>(p);
  const int taps = g.KT * g.KH * g.KW;
  AVSR_LAUNCH(reorder_weight_kernel, grid_1d((long)g.Cout * g.Kp), 256, 0, st, w, wo, g.Cout, g.Cin, taps, g.Kp, kind);
  AVSR_LAUNCH(fill_f32_kernel, cdiv(g.Cout, 256), 256, 0, st, ones, g.Cout, 1.f);
  AVSR_LAUNCH(fill_f32_kernel, cdiv(g.Cout, 256), 256, 0, st, ones + g.Cout, g.Cout, 0.f);
  const void* xin = x;
  if (!stem) {
    const long nx = (long)g.N * g.H * g.W * g.Cin;
    AVSR_LAUNCH(cvt_to_op_kernel, grid_1d(nx), 256, 0, st, x, xo, nx, kind);
    xin = xo;
  }
  AVSR_TRY(run_conv_raw(kind, stem != 0, xin, wo, ones, ones + g.Cout, z, g, st));
  return launch_bn_stats(z, M, g.Cout, part, stats, st);
}

extern "C" size_t avsr_frontend_train_dgrad_workspace_bytes(int N, int H, int W, int C_in, int C_out, int KH, int KW,
                                                            int stride, int precision) {
  ConvGeom g;
  if (!ft_prec_ok(precision) || !ft_geom(0, N, 1, H, W, C_in, C_out, KH, KW, stride, &g)) return 0;
  return ft_dgrad_ws(g, operand_kind(precision)).total;
}

extern "C" int avsr_frontend_train_conv_dgrad(const float* dz, const float* w, float* dx, int N, int H, int W, int C_in,
                                              int C_out, int KH, int KW, int stride, void* workspace,
                                              size_t workspace_bytes, int precision, void* stream) {
  AVSR_REQUIRE(ft_prec_ok(precision), "frontend train dgrad: bad precision %d", precision);
  ConvGeom g;
  AVSR_REQUIRE(ft_geom(0, N, 1, H, W, C_in, C_out, KH, KW, stride, &g),
               "frontend train dgrad: unsupported shape N=%d H=%d W=%d C_in=%d C_out=%d KH=%d KW=%d stride=%d", N, H,
               W, C_in, C_out, KH, KW, stride);
  AVSR_REQUIRE(dz && w && dx && workspace, "NULL argument");
  const int kind = operand_kind(precision);
  const FtDgradWs L = ft_dgrad_ws(g, kind);
  AVSR_REQUIRE_BYTES(L.total, workspace_bytes, "frontend train dgrad workspace");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (N == 0) return AVSR_OK;
  uint8_t* p = reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<uintptr_t>(workspace), 256));
  void* dzo = p; p += L.dzop;
  void* wo = p; p += L.wop;
  float* ones = reinterpret_cast<float*>(p); p += L.unit;
  float* sub = reinterpret_cast<float*>(p);
  const long nz = conv_rows(g) * g.Cout;
  AVSR_LAUNCH(cvt_to_op_kernel, grid_1d(nz), 256, 0, st, dz, dzo, nz, kind);
  AVSR_LAUNCH(fill_f32_kernel, cdiv(g.Cin, 256), 256, 0, st, ones, g.Cin, 1.f);
  AVSR_LAUNCH(fill_f32_kernel, cdiv(g.Cin, 256), 256, 0, st, ones + g.Cin, g.Cin, 0.f);
  const int s = g.sh;           // both axes (a 1-D conv has H = KH = 1: its odd rows are empty)
  for (int ry = 0; ry < s; ++ry) {
    for (int rx = 0; rx < s; ++rx) {
      const AxisClass cy = axis_class(g.KH, s, g.ph, ry), cx = axis_class(g.KW, s, g.pw, rx);
      const int Hc = (g.H - ry + s - 1) / s, Wc = (g.W - rx + s - 1) / s;
      if (Hc <= 0 || Wc <= 0) continue;
      if (cy.n == 0 || cx.n == 0) {
        AVSR_LAUNCH(ft_scatter_class_kernel, grid_1d((long)N * Hc * Wc * g.Cin), 256, 0, st, (const float*)nullptr,
                    dx, N, g.H, g.W, g.Cin, s, ry, rx, Hc, Wc);
        continue;
      }
      // the class as a stride-1 conv over dz: output (Hc, Wc, C_in), taps (cy.n, cx.n) over C_out
      ConvGeom c{};
      c.N = N; c.T = 1; c.H = g.Ho; c.W = g.Wo; c.Cin = g.Cout; c.Ho = Hc; c.Wo = Wc; c.Cout = g.Cin;
      c.KT = 1; c.KH = cy.n; c.KW = cx.n; c.sh = 1; c.sw = 1; c.pt = 0; c.ph = -cy.dmin; c.pw = -cx.dmin;
      c.ld_frame = (long)g.Ho * g.Wo * g.Cout; c.K = cy.n * cx.n * g.Cout; c.Kp = c.K;
      AVSR_LAUNCH(ft_dgrad_weight_kernel, grid_1d((long)g.Cin * c.Kp), 256, 0, st, w, wo, g.Cout, g.Cin, g.KH, g.KW,
                  s, ry, rx, g.ph, g.pw, cy.dmin, cx.dmin, cy.n, cx.n, kind);
      if (s == 1) {
        AVSR_TRY(run_conv_raw(kind, false, dzo, wo, ones, ones + g.Cin, dx, c, st));
      } else {
        AVSR_TRY(run_conv_raw(kind, false, dzo, wo, ones, ones + g.Cin, sub, c, st));
        AVSR_LAUNCH(ft_scatter_class_kernel, grid_1d((long)N * Hc * Wc * g.Cin), 256, 0, st, (const float*)sub, dx,
                    N, g.H, g.W, g.Cin, s, ry, rx, Hc, Wc);
      }
    }
  }
  return AVSR_OK;
}

extern "C" size_t avsr_frontend_train_wgrad_workspace_bytes(int stem, int N, int T, int H, int W, int C_in, int C_out,
                                                            int KH, int KW, int stride) {
  ConvGeom g;
  if (!ft_geom(stem, N, T, H, W, C_in, C_out, KH, KW, stride, &g)) return 0;
  return ft_wgrad_ws(g);
}

extern "C" int avsr_frontend_train_conv_wgrad(const float* x, const float* dz, float* dw, int stem, int N, int T, int H,
                                              int W, int C_in, int C_out, int KH, int KW, int stride, void* workspace,
                                              size_t workspace_bytes, int precision, void* stream) {
  AVSR_REQUIRE(ft_prec_ok(precision), "frontend train wgrad: bad precision %d", precision);
  ConvGeom g;
  AVSR_REQUIRE(ft_geom(stem, N, T, H, W, C_in, C_out, KH, KW, stride, &g),
               "frontend train wgrad: unsupported shape stem=%d N=%d T=%d H=%d W=%d C_in=%d C_out=%d KH=%d KW=%d "
               "stride=%d", stem, N, T, H, W, C_in, C_out, KH, KW, stride);
  AVSR_REQUIRE(x && dz && dw && workspace, "NULL argument");
  AVSR_REQUIRE_BYTES(ft_wgrad_ws(g), workspace_bytes, "frontend train wgrad workspace");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* part = reinterpret_cast<float*>(align_up(reinterpret_cast<uintptr_t>(workspace), 256));
  const int Kw = cdiv(g.K, WG_T) * WG_T, splits = ft_wgrad_splits(g);
  const long M = conv_rows(g);
  const long per = ((M + splits - 1) / splits + WGT_PB - 1) / WGT_PB * WGT_PB;    // a multiple of both K-blocks
  if (operand_kind(precision) == OP_F32) {
    AVSR_LAUNCH(ft_wgrad_kernel, dim3(Kw / WG_T, g.Cout / WG_T, splits), 256, 0, st, x, dz, part, g, per, Kw);
  } else {
    AVSR_SET_MAX_SMEM(ft_wgrad_tc_kernel, WGT_SMEM);
    AVSR_LAUNCH(ft_wgrad_tc_kernel, dim3(Kw / WG_T, g.Cout / WG_T, splits), 128, WGT_SMEM, st, x, dz, part, g, per, Kw);
  }
  const int taps = g.KT * g.KH * g.KW;
  AVSR_LAUNCH(ft_wgrad_finish_kernel, grid_1d((long)g.Cout * g.Cin * taps), 256, 0, st, (const float*)part, dw, splits,
              g.Cout, g.Cin, taps, Kw);
  return AVSR_OK;
}

extern "C" int avsr_frontend_train_maxpool_fwd(const float* x, float* y, uint8_t* idx, int N, int Hi, int Wi, int C,
                                               void* stream) {
  AVSR_REQUIRE(N >= 0 && Hi >= 1 && Wi >= 1 && C >= 1, "frontend train maxpool: bad shape");
  AVSR_REQUIRE(x && y && idx, "NULL argument");
  const int Ho = (Hi - 1) / 2 + 1, Wo = (Wi - 1) / 2 + 1;
  const long n = (long)N * Ho * Wo * C;
  if (n == 0) return AVSR_OK;
  AVSR_LAUNCH(ft_maxpool_fwd_kernel, grid_1d(n), 256, 0, reinterpret_cast<cudaStream_t>(stream), x, y, idx, N, Hi, Wi,
              Ho, Wo, C);
  return AVSR_OK;
}

extern "C" int avsr_frontend_train_maxpool_bwd(const float* dy, const uint8_t* idx, float* dx, int N, int Hi, int Wi,
                                               int C, void* stream) {
  AVSR_REQUIRE(N >= 0 && Hi >= 1 && Wi >= 1 && C >= 1, "frontend train maxpool: bad shape");
  AVSR_REQUIRE(dy && idx && dx, "NULL argument");
  const int Ho = (Hi - 1) / 2 + 1, Wo = (Wi - 1) / 2 + 1;
  const long n = (long)N * Hi * Wi * C;
  if (n == 0) return AVSR_OK;
  AVSR_LAUNCH(ft_maxpool_bwd_kernel, grid_1d(n), 256, 0, reinterpret_cast<cudaStream_t>(stream), dy, idx, dx, N, Hi,
              Wi, Ho, Wo, C);
  return AVSR_OK;
}

extern "C" int avsr_frontend_train_mean_rows(const float* x, float* out, long G, int P, int C, void* stream) {
  AVSR_REQUIRE(G >= 0 && P >= 1 && C >= 1, "frontend train mean: bad shape");
  AVSR_REQUIRE(x && out, "NULL argument");
  if (G == 0) return AVSR_OK;
  AVSR_LAUNCH(mean_rows_kernel<float>, grid_1d(G * C), 256, 0, reinterpret_cast<cudaStream_t>(stream), x, out, G, P, C);
  return AVSR_OK;
}

extern "C" int avsr_frontend_train_mean_rows_bwd(const float* dout, float* dx, long G, int P, int C, void* stream) {
  AVSR_REQUIRE(G >= 0 && P >= 1 && C >= 1, "frontend train mean: bad shape");
  AVSR_REQUIRE(dout && dx, "NULL argument");
  if (G == 0) return AVSR_OK;
  AVSR_LAUNCH(ft_mean_rows_bwd_kernel, grid_1d(G * P * C), 256, 0, reinterpret_cast<cudaStream_t>(stream), dout, dx, G,
              P, C);
  return AVSR_OK;
}
