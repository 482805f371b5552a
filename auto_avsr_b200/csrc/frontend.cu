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
// (64 f16 or 32 tf32 channels; every trunk C_in is a multiple of 64), so the A tile of a trunk conv is gathered with
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

template <typename TOp>
__device__ __forceinline__ float4 op_ld4(const TOp* p) {
  if constexpr (sizeof(TOp) == 4) {
    return *reinterpret_cast<const float4*>(p);
  } else {
    const uint2 u = *reinterpret_cast<const uint2*>(p);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
  }
}

// kind: OP_F32 plain, OP_TF32 rounded fp32, OP_F16 half
__global__ void cvt_to_op_kernel(const float* __restrict__ x, void* __restrict__ y, long n, int kind) {
  pdl_wait();
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const float v = x[i];
    if (kind == OP_F16) reinterpret_cast<__half*>(y)[i] = to_half_sat(v);
    else reinterpret_cast<float*>(y)[i] = kind == OP_TF32 ? round_tf32(v) : v;
  }
}
__global__ void cvt_from_op_kernel(const void* __restrict__ x, float* __restrict__ y, long n, int kind) {
  pdl_wait();
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    y[i] = kind == OP_F16 ? __half2float(reinterpret_cast<const __half*>(x)[i]) : reinterpret_cast<const float*>(x)[i];
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
    if (kind == OP_F16) reinterpret_cast<__half*>(dst)[i] = to_half_sat(v);
    else reinterpret_cast<float*>(dst)[i] = kind == OP_TF32 ? round_tf32(v) : v;
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

// STEM: x is the fp32 clip / waveform (Cin = 1) gathered element by element; otherwise x is the TOp activation.
template <typename TOp, int BN, bool STEM>
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

template <typename TOp, int BN, bool STEM>
static int launch_conv_tc_t(const void* x, const void* w, const float* scale, const float* shift, const void* resid,
                            void* y, const ConvGeom& g, int act, cudaStream_t st) {
  auto kernel = conv_tc_kernel<TOp, BN, STEM>;
  AVSR_SET_MAX_SMEM(kernel, CvCfg<BN>::kSmem);
  const long M = conv_rows(g);
  const dim3 grid((unsigned)((M + CV_BM - 1) / CV_BM), (unsigned)cdiv(g.Cout, BN));
  AVSR_LAUNCH(kernel, grid, CV_THREADS, CvCfg<BN>::kSmem, st, x, reinterpret_cast<const TOp*>(w), scale, shift,
              reinterpret_cast<const TOp*>(resid), reinterpret_cast<TOp*>(y), g, act);
  return AVSR_OK;
}

template <typename TOp, bool STEM>
static int launch_conv_tc_bn(const void* x, const void* w, const float* scale, const float* shift, const void* resid,
                             void* y, const ConvGeom& g, int act, cudaStream_t st) {
  if (g.Cout <= 64) return launch_conv_tc_t<TOp, 64, STEM>(x, w, scale, shift, resid, y, g, act, st);
  return launch_conv_tc_t<TOp, 128, STEM>(x, w, scale, shift, resid, y, g, act, st);
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

extern "C" int avsr_frontend_forward(int modality, const void* prepared, const float* x, int B, int T_in, int H, int W,
                                     float* out, void* workspace, size_t workspace_bytes, int precision, void* stream) {
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

  // stem (+ max-pool for video) -> buf[1]
  int cur = 1;
  if (modality == AVSR_FRONTEND_VIDEO) {
    AVSR_TRY(run_conv(kind, true, x, wt(0), sc(0), sh(0), nullptr, buf[0], P.stem, 1, st));
    const long n = (long)P.N * P.H0 * P.W0 * 64;
    if (kind == OP_F16)
      AVSR_LAUNCH(maxpool3x3s2_kernel<__half>, grid_1d(n), 256, 0, st, (const __half*)buf[0], (__half*)buf[1], P.N,
                  P.stem.Ho, P.stem.Wo, P.H0, P.W0, 64);
    else
      AVSR_LAUNCH(maxpool3x3s2_kernel<float>, grid_1d(n), 256, 0, st, (const float*)buf[0], (float*)buf[1], P.N,
                  P.stem.Ho, P.stem.Wo, P.H0, P.W0, 64);
  } else {
    AVSR_TRY(run_conv(kind, true, x, wt(0), sc(0), sh(0), nullptr, buf[1], P.stem, 1, st));
  }
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
      h = g2.Ho; w = g2.Wo;
      j += ds ? 3 : 2;
    }
  }
  // pool: per video frame over its h x w pixels; per 20 audio positions
  const int Pn = modality == AVSR_FRONTEND_VIDEO ? h * w : 20;
  const long n = P.groups * 512;
  if (kind == OP_F16)
    AVSR_LAUNCH(mean_rows_kernel<__half>, grid_1d(n), 256, 0, st, (const __half*)buf[cur], out, P.groups, Pn, 512);
  else
    AVSR_LAUNCH(mean_rows_kernel<float>, grid_1d(n), 256, 0, st, (const float*)buf[cur], out, P.groups, Pn, 512);
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
