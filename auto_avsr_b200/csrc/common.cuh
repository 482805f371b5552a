// Shared internals of libavsr_b200: error plumbing, launch accounting, the GEMM epilogue family.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <cstdlib>
#include <string>
#include <tuple>
#include <type_traits>
#include <utility>

#include "../../include/avsr_b200.h"

namespace avsr {

// ---------------------------------------------------------------- errors / accounting
void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;

#define AVSR_CUDA_TRY(expr)                                                                   \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      ::avsr::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return AVSR_E_CUDA;                                                                     \
    }                                                                                         \
  } while (0)

#define AVSR_CHECK_LAUNCH()                      \
  do {                                           \
    ::avsr::g_launches.fetch_add(1);             \
    AVSR_CUDA_TRY(cudaPeekAtLastError());        \
  } while (0)

#define AVSR_REQUIRE(cond, ...)                  \
  do {                                           \
    if (!(cond)) {                               \
      ::avsr::set_error(__VA_ARGS__);            \
      return AVSR_E_INVALID;                     \
    }                                            \
  } while (0)

#define AVSR_TRY(expr)            \
  do {                            \
    int _r = (expr);              \
    if (_r != AVSR_OK) return _r; \
  } while (0)

// a caller-provided buffer of `have` bytes must hold `need`: else "<what> too small: need N bytes, got M"
#define AVSR_REQUIRE_BYTES(need, have, what)                                             \
  do {                                                                                   \
    const size_t _need = (need), _have = (have);                                         \
    if (_need > _have) {                                                                 \
      ::avsr::set_error("%s too small: need %zu bytes, got %zu", what, _need, _have);    \
      return AVSR_E_WORKSPACE;                                                           \
    }                                                                                    \
  } while (0)

constexpr int kSplitCounters = 4096;  // split-K tile counters a caller must provide (EpiParams::counters)
constexpr int kMaxSplits = 8;         // split-K slices gemm_tc may choose; sizes EpiParams::partial
constexpr int kHeadDim = 64;  // d_k of the reference encoder (768 / 12); the attention kernels are built for it

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// Lays caller-owned buffers out back to back, each in a 256-byte-aligned slot.  With a NULL base only the size is
// computed: take() returns NULL and `off` ends as the bytes the layout needs.
struct Carver {
  char* base;
  size_t off = 0;
  template <typename T = float>
  T* take(size_t n) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += align_up(n * sizeof(T), 256);
    return p;
  }
};

// ---------------------------------------------------------------- programmatic dependent launch (PDL)
// Every hot-path kernel is launched with cudaLaunchAttributeProgrammaticStreamSerialization: it may start (block
// scheduling, barrier init, tensor-map prefetch) while its predecessor in the stream / graph is
// still draining, and blocks in pdl_wait() until the predecessor has completed and flushed before it touches any
// global memory.  pdl_launch_dependents() at the top lets the successor do the same.  Without the attribute both
// are no-ops, so the same kernels work under plain launches (AVSR_B200_PDL=0).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

inline bool pdl_enabled() {
  static const bool on = [] { const char* e = getenv("AVSR_B200_PDL"); return !(e && e[0] == '0'); }();
  return on;
}

template <typename... KArgs, typename... Args, size_t... I>
inline cudaError_t launch_kernel_impl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                      unsigned cluster, std::index_sequence<I...>, Args&&... args) {
  std::tuple<KArgs...> params(static_cast<KArgs>(args)...);
  void* ptrs[] = {const_cast<void*>(static_cast<const void*>(&std::get<I>(params)))...};
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n++].val.programmaticStreamSerializationAllowed = 1;
  }
  if (cluster > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster; attr[n].val.clusterDim.y = 1; attr[n++].val.clusterDim.z = 1;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelExC(&cfg, reinterpret_cast<const void*>(kernel), ptrs);
}
// launch `kernel<<<grid, block, smem, st>>>(args...)` with the PDL attribute, in clusters of `cluster` CTAs along x
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                 unsigned cluster, Args&&... args) {
  static_assert(sizeof...(KArgs) == sizeof...(Args), "kernel argument count mismatch");
  return launch_kernel_impl(kernel, grid, block, smem, st, cluster, std::index_sequence_for<KArgs...>{},
                            std::forward<Args>(args)...);
}

// opt a kernel into > 48 KB of dynamic shared memory; remembered per device (one process may drive several GPUs)
#define AVSR_SET_MAX_SMEM(kernel, bytes)                                                                     \
  do {                                                                                                       \
    static int _done_dev = -1;                                                                               \
    int _dev = 0;                                                                                            \
    AVSR_CUDA_TRY(cudaGetDevice(&_dev));                                                                     \
    if (_done_dev != _dev) {                                                                                 \
      AVSR_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))); \
      _done_dev = _dev;                                                                                      \
    }                                                                                                        \
  } while (0)

#define AVSR_LAUNCH(kernel, grid, block, smem, st, ...)                                                \
  do {                                                                                                 \
    ::avsr::g_launches.fetch_add(1);                                                                   \
    AVSR_CUDA_TRY(::avsr::launch_kernel(kernel, dim3(grid), dim3(block), (size_t)(smem), st, 1u, __VA_ARGS__)); \
  } while (0)
// the same, in clusters of `cluster` CTAs along x (grid a multiple of it)
#define AVSR_LAUNCH_CLUSTER(kernel, grid, block, smem, st, cluster, ...)                                         \
  do {                                                                                                          \
    ::avsr::g_launches.fetch_add(1);                                                                            \
    AVSR_CUDA_TRY(::avsr::launch_kernel(kernel, dim3(grid), dim3(block), (size_t)(smem), st, (unsigned)(cluster), \
                                        __VA_ARGS__));                                                          \
  } while (0)

// ---------------------------------------------------------------- device helpers
// code shared by a kernel and the host replay the CPU tests build (tests/emu): decoder_body.cuh, ctc_loss_body.cuh
#define AVSR_HD __host__ __device__ __forceinline__

__device__ __forceinline__ float round_tf32(float x) {
  // round-to-nearest (ties away) to the 10-bit TF32 mantissa; the tensor core then truncates nothing.
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
__device__ __forceinline__ float sigmoidf_acc(float x) { return 1.0f / (1.0f + expf(-x)); }
// sigmoid through ex2.approx + fast reciprocal (relative error ~1e-6: far below the 11-bit operand rounding that
// follows in the tensor-core paths); the fp32 reference path keeps sigmoidf_acc
__device__ __forceinline__ float sigmoidf_fast(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---------------------------------------------------------------- tensor-core operand storage
// How a tensor that feeds a tensor-core contraction is stored:
//   OP_F32  : plain fp32 (CUDA-core reference path)
//   OP_TF32 : fp32 container, value rounded to TF32 (10-bit mantissa) -> wgmma .tf32
//   OP_F16  : IEEE half (same 10-bit mantissa as TF32, 5-bit exponent, saturating) -> wgmma .f16;
//             half the bytes through L2/shared memory and twice the MMA rate of .tf32
//   OP_BF16 : bfloat16 (7-bit mantissa, fp32's 8-bit exponent, round to nearest even, no saturation) -> wgmma .bf16;
//             the bytes and the rate of OP_F16, the range of fp32
enum OperandKind : int { OP_F32 = 0, OP_TF32 = 1, OP_F16 = 2, OP_BF16 = 3 };

static inline bool valid_precision(int p) {
  return p == AVSR_PREC_FP32 || p == AVSR_PREC_TF32 || p == AVSR_PREC_F16 || p == AVSR_PREC_BF16;
}
// AVSR_PREC_* -> how the operands of that precision's contractions are stored
static inline int operand_kind(int precision) {
  return precision == AVSR_PREC_F16    ? OP_F16
         : precision == AVSR_PREC_BF16 ? OP_BF16
         : precision == AVSR_PREC_TF32 ? OP_TF32
                                       : OP_F32;
}
// 2-byte operand storage (f16 or bf16): the same layouts, the same tile shapes, the same byte counts
AVSR_HD bool op16(int kind) { return kind == OP_F16 || kind == OP_BF16; }
static inline bool prec16(int precision) { return op16(operand_kind(precision)); }
static inline size_t operand_bytes(int kind) { return op16(kind) ? 2 : 4; }
// the operand kind a tensor-core kernel instantiated for element type TOp reads (float: TF32)
template <typename TOp>
constexpr int op_kind_of() {
  return sizeof(TOp) == 4 ? OP_TF32 : (std::is_same<TOp, __half>::value ? OP_F16 : OP_BF16);
}

__device__ __forceinline__ __half to_half_sat(float x) {
  unsigned short r;
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(r) : "f"(x));
  return __ushort_as_half(r);
}
// two floats -> packed IEEE halves (a in the low half), round to nearest, saturating: ONE conversion instruction
__device__ __forceinline__ uint32_t pack_half2_sat(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
// the same with ReLU folded into the conversion (F2FP.SATFINITE.RELU): negative -> +0, NaN stays NaN like torch.relu
__device__ __forceinline__ uint32_t pack_half2_sat_relu(float a, float b) {
  uint32_t r;
  asm("cvt.rn.relu.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
// two floats -> packed bfloat16s (a in the low half), round to nearest even, no saturation (beyond the largest finite
// bf16 a value rounds to +-inf like any IEEE conversion), NaN stays NaN: ONE conversion instruction
__device__ __forceinline__ uint32_t pack_bf162(float a, float b) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
// store 4 consecutive operand values (dst 16-byte aligned for float, 8-byte aligned for half / bfloat16)
template <typename TOp>
__device__ __forceinline__ void store_op4(TOp* dst, float a, float b, float c, float d);
template <>
__device__ __forceinline__ void store_op4<float>(float* dst, float a, float b, float c, float d) {
  *reinterpret_cast<float4*>(dst) = make_float4(round_tf32(a), round_tf32(b), round_tf32(c), round_tf32(d));
}
template <>
__device__ __forceinline__ void store_op4<__half>(__half* dst, float a, float b, float c, float d) {
  __half2 lo = __halves2half2(to_half_sat(a), to_half_sat(b));
  __half2 hi = __halves2half2(to_half_sat(c), to_half_sat(d));
  uint2 v;
  v.x = *reinterpret_cast<uint32_t*>(&lo);
  v.y = *reinterpret_cast<uint32_t*>(&hi);
  *reinterpret_cast<uint2*>(dst) = v;
}
template <>
__device__ __forceinline__ void store_op4<__nv_bfloat16>(__nv_bfloat16* dst, float a, float b, float c, float d) {
  *reinterpret_cast<uint2*>(dst) = make_uint2(pack_bf162(a, b), pack_bf162(c, d));
}
template <typename TOp>
__device__ __forceinline__ void store_op1(TOp* dst, float a);
template <>
__device__ __forceinline__ void store_op1<float>(float* dst, float a) { *dst = round_tf32(a); }
template <>
__device__ __forceinline__ void store_op1<__half>(__half* dst, float a) { *dst = to_half_sat(a); }
template <>
__device__ __forceinline__ void store_op1<__nv_bfloat16>(__nv_bfloat16* dst, float a) { *dst = __float2bfloat16_rn(a); }
// runtime-kind stores / loads used by the elementwise kernels (kind is warp-uniform; a negative kind is plain fp32)
__device__ __forceinline__ void store_kind1(void* base, long idx, int kind, float v) {
  if (kind == OP_F16) reinterpret_cast<__half*>(base)[idx] = to_half_sat(v);
  else if (kind == OP_BF16) reinterpret_cast<__nv_bfloat16*>(base)[idx] = __float2bfloat16_rn(v);
  else reinterpret_cast<float*>(base)[idx] = kind == OP_TF32 ? round_tf32(v) : v;
}
__device__ __forceinline__ float load_kind1(const void* base, long idx, int kind) {
  if (kind == OP_F16) return __half2float(reinterpret_cast<const __half*>(base)[idx]);
  if (kind == OP_BF16) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(base)[idx]);
  return reinterpret_cast<const float*>(base)[idx];
}
__device__ __forceinline__ void store_kind4(void* base, long idx, int kind, float a, float b, float c, float d) {
  if (kind == OP_F16) store_op4<__half>(reinterpret_cast<__half*>(base) + idx, a, b, c, d);
  else if (kind == OP_BF16) store_op4<__nv_bfloat16>(reinterpret_cast<__nv_bfloat16*>(base) + idx, a, b, c, d);
  else if (kind == OP_TF32) store_op4<float>(reinterpret_cast<float*>(base) + idx, a, b, c, d);
  else *reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + idx) = make_float4(a, b, c, d);
}

// ---------------------------------------------------------------- GEMM epilogues
// Every GEMM computes acc[m][n] = sum_k A[m][k] * Bw[n][k]  (both operands K-major, i.e. torch Linear).
enum EpiMode : int {
  EPI_LINEAR = 0,  // y = [resid + alpha *] act(acc + bias[n])                      -> out (M, ldo)
  EPI_QK = 1,      // n <  D: q -> qu = q+bias+pos_u, qv = q+bias+pos_v ; D <= n < 2D: k ; 2D <= n < 3D (when
                   // N == 3D): v into `vt` with the SAME head-major layout   -> (B,H,T,64) each
  EPI_VT = 2,      // A = W_v (m = feature), B = frames (n): v^T                     -> (B,H,64,Tp)
  EPI_GLU = 3,     // interleaved pointwise_cov1: value cols [g*128, +64), gate cols +64 -> out (M, N/2)
  EPI_POS = 4      // linear_pos of all layers: n = l*D + h*64 + d, m = table row      -> (L,H,Rp,64)
};

struct EpiParams {
  int M, N;           // logical extents of acc
  const float* bias;  // LINEAR/QK/GLU: [N]; VT: [M]; may be null (LINEAR, POS)
  void* out;          // LINEAR / GLU / POS destination: fp32, or operand-typed when round_out != 0
  long ldo;           // LINEAR / GLU row stride of out
  const float* resid; // LINEAR: optional residual (same layout as out; may alias out)
  float alpha;        // LINEAR: scale of the residual branch
  int relu;           // LINEAR
  int round_out;      // round the stored value to TF32 (it feeds a tensor-core operand)
  int T, H, Tp, Rp;   // frames per utterance, heads, padded T of v^T, padded rows of the pos table
  const float* pos_u; // QK: [H*64]
  const float* pos_v;
  float* partial;     // split-K: fp32 workspace [splits][M][ldo] for the partial tiles (deterministic fix-up)
  int* counters;      // split-K: one arrival counter per output tile, zero on entry, reset by the last arriver
  void* qu;           // operand-typed (float for OP_F32/OP_TF32, __half for OP_F16, __nv_bfloat16 for OP_BF16)
  void* qv;
  void* kk;
  void* vt;
  // Bw is a prepared weight that no kernel of the current PDL chain writes: gemm_tc may load it before
  // griddepcontrol.wait (gemm_tc.cu, "static-operand prologue").  Only the encoder forward sets it; not for EPI_VT.
  int b_static;
};

// ---------------------------------------------------------------- phase trace (diagnostic build only)
// scripts/build_trace.py compiles the library with -DAVSR_TRACE into libavsr_b200_trace.so; the product build does
// not contain any of this.  Buffer layout (64-bit words): [0] = records used, [1] = record capacity, then records of
// kTraceWords words: [0] kernel id, [1] blockIdx.x | aux << 32, [2] SM id, [3] %globaltimer at open,
// [4 + s] = clock64() at phase mark s (s < 10), [14] / [15] = %globaltimer when the dependency resolved / the CTA was done.
// One record per CTA; marks are written by whichever thread reaches the phase.
#ifdef AVSR_TRACE
constexpr int kTraceWords = 16;
// Every translation unit has its own copy of the buffer pointer (no relocatable device code in this build); each
// .cu defines a binder with AVSR_TRACE_DEFINE_BIND and avsr_trace_set (encoder.cu) calls all of them.  The kernels
// read the pointer at run time, so a CUDA graph captured before avsr_trace_set still traces.
static __device__ unsigned long long* d_trace_buf;
#define AVSR_TRACE_DEFINE_BIND(name)                                                         \
  int name(unsigned long long* p) {                                                          \
    return cudaMemcpyToSymbol(::avsr::d_trace_buf, &p, sizeof p) == cudaSuccess ? 0 : 1;     \
  }
__device__ __forceinline__ unsigned long long trace_globaltimer() {
  unsigned long long gt;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
  return gt;
}
__device__ __forceinline__ unsigned long long* trace_open(int kernel_id, unsigned aux) {
  unsigned long long* trace = d_trace_buf;
  if (!trace) return nullptr;
  const unsigned long long r = atomicAdd(trace, 1ULL);
  if (r >= trace[1]) return nullptr;
  unsigned long long* rec = trace + 2 + r * kTraceWords;
  unsigned smid;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
  rec[0] = (unsigned long long)kernel_id;
  rec[1] = (unsigned long long)blockIdx.x | ((unsigned long long)aux << 32);
  rec[2] = smid;
  rec[3] = trace_globaltimer();
  return rec;
}
__device__ __forceinline__ void trace_mark(unsigned long long* rec, int slot) {
  if (rec) rec[4 + slot] = (unsigned long long)clock64();
}
// globaltimer stamps for the launch timeline: slot 10 = dependency resolved (after griddepcontrol.wait), 11 = CTA done
__device__ __forceinline__ void trace_stamp(unsigned long long* rec, int slot) {
  if (rec) rec[4 + slot] = trace_globaltimer();
}
#define AVSR_TRACE_OPEN(slot_ptr, id, aux) do { *(slot_ptr) = ::avsr::trace_open(id, aux); } while (0)
#define AVSR_TRACE_MARK(cond, slot_ptr, s) do { if (cond) ::avsr::trace_mark(*(slot_ptr), s); } while (0)
#define AVSR_TRACE_STAMP(cond, slot_ptr, s) do { if (cond) ::avsr::trace_stamp(*(slot_ptr), s); } while (0)
// simple kernels (no shared slot): thread 0 of the CTA keeps the record pointer in a register
#define AVSR_TSPAN_OPEN(id, aux) unsigned long long* _tsp = threadIdx.x == 0 ? ::avsr::trace_open(id, aux) : nullptr
#define AVSR_TSPAN_DEP() ::avsr::trace_stamp(_tsp, 10)
#define AVSR_TSPAN_CLOSE() ::avsr::trace_stamp(_tsp, 11)
#else
#define AVSR_TRACE_DEFINE_BIND(name)
#define AVSR_TRACE_OPEN(slot_ptr, id, aux) do { } while (0)
#define AVSR_TRACE_MARK(cond, slot_ptr, s) do { } while (0)
#define AVSR_TRACE_STAMP(cond, slot_ptr, s) do { } while (0)
#define AVSR_TSPAN_OPEN(id, aux) do { } while (0)
#define AVSR_TSPAN_DEP() do { } while (0)
#define AVSR_TSPAN_CLOSE() do { } while (0)
#endif

// scalar store of one operand-or-fp32 value: `operand` says the destination is TOp-typed (rounded), else plain fp32
template <typename TOp>
__device__ __forceinline__ void put(void* base, long idx, float v, bool operand) {
  if (operand) store_op1<TOp>(reinterpret_cast<TOp*>(base) + idx, v);
  else reinterpret_cast<float*>(base)[idx] = v;
}

// Scalar (one element) epilogue: used by the CUDA-core GEMM and by the tensor-core kernel's ragged edges.
// TOp = float serves OP_F32 (round_out = 0) and OP_TF32 (round_out = 1); __half OP_F16, __nv_bfloat16 OP_BF16.
template <int MODE, typename TOp = float>
__device__ __forceinline__ void epi_store(const EpiParams& p, int m, int n, float acc) {
  if (m >= p.M || n >= p.N) return;
  if constexpr (MODE == EPI_LINEAR) {
    float v = acc + (p.bias ? p.bias[n] : 0.0f);
    if (p.relu) v = fmaxf(v, 0.0f);
    if (p.resid) v = p.resid[(long)m * p.ldo + n] + p.alpha * v;
    put<TOp>(p.out, (long)m * p.ldo + n, v, p.round_out != 0);
  } else if constexpr (MODE == EPI_QK) {
    const int D = p.H * kHeadDim;
    const int b = m / p.T, t = m - b * p.T;
    const int seg = n / D, nn = n - seg * D;          // 0: q, 1: k, 2: v (merged QKV projection)
    const int h = nn / kHeadDim, d = nn - h * kHeadDim;
    const long idx = (((long)b * p.H + h) * p.T + t) * kHeadDim + d;
    const float v = acc + p.bias[n];
    if (seg == 0) {
      put<TOp>(p.qu, idx, v + p.pos_u[nn], p.round_out != 0);
      put<TOp>(p.qv, idx, v + p.pos_v[nn], p.round_out != 0);
    } else {
      put<TOp>(seg == 1 ? p.kk : p.vt, idx, v, p.round_out != 0);
    }
  } else if constexpr (MODE == EPI_VT) {
    const int b = n / p.T, t = n - b * p.T;
    const int h = m / kHeadDim, d = m - h * kHeadDim;
    put<TOp>(p.vt, (((long)b * p.H + h) * kHeadDim + d) * p.Tp + t, acc + p.bias[m], p.round_out != 0);
  } else if constexpr (MODE == EPI_POS) {
    const int D = p.H * kHeadDim;
    const int l = n / D, r = n - l * D;
    const int h = r / kHeadDim, d = r - h * kHeadDim;
    put<TOp>(p.out, (((long)l * p.H + h) * p.Rp + m) * kHeadDim + d, acc, p.round_out != 0);
  }
}

// GLU pair: n_val is the interleaved column of the value half, the gate sits 64 columns further.  Output is fp32
// (it feeds the depthwise conv, not a tensor-core operand).
__device__ __forceinline__ void epi_store_glu(const EpiParams& p, int m, int n_val, float acc_val, float acc_gate) {
  if (m >= p.M || n_val + 64 >= p.N) return;
  const float a = acc_val + p.bias[n_val];
  const float g = acc_gate + p.bias[n_val + 64];
  const int c = (n_val >> 7) * 64 + (n_val & 63);
  reinterpret_cast<float*>(p.out)[(long)m * p.ldo + c] = a * sigmoidf_acc(g);
}

// ---------------------------------------------------------------- kernel launchers (defined in the .cu files)
// fp32 CUDA-core GEMM (gemm_simt.cu)
int gemm_simt(int mode, const float* A, const float* Bw, int M, int N, int K, const EpiParams& ep, cudaStream_t st);
// wgmma GEMM (gemm_tc.cu); opk = OP_TF32 (A, Bw are float), OP_F16 (__half) or OP_BF16 (__nv_bfloat16)
int gemm_tc(int mode, int opk, const void* A, const void* Bw, int M, int N, int K, const EpiParams& ep, cudaStream_t st);

// elementwise.cu
int launch_embed_scale(const float* xs, float* x, long n, float scale, cudaStream_t st);
// `out_kind` is an OperandKind: how y / pe is stored
int launch_layernorm(const float* x, const float* g, const float* b, void* y, int rows, int d, int out_kind,
                     cudaStream_t st);
// y_f32 = LN(x) as fp32 (may alias x) AND y_op = the same values in operand storage (after_norm feeding ctc_lo)
int launch_layernorm_dual(const float* x, const float* g, const float* b, float* y_f32, void* y_op, int rows, int d,
                          int out_kind, cudaStream_t st);
int launch_layernorm2(const float* x, const float* g1, const float* b1, const float* g2, const float* b2, float* y1,
                      void* y2, int rows, int d, int out_kind, cudaStream_t st);
int launch_sinusoid(void* pe, int T, int d, int out_kind, cudaStream_t st);
int launch_dwconv_bn_silu(const float* x, const float* wt /*(K,C)*/, const float* scale, const float* shift, void* y,
                          int B, int T, int C, int K, int out_kind, cudaStream_t st);

// train.cu: each channel's (count, mean, M2) over z (rows >= 1, C) -> stats (3, C) fp64, through the fp64 partials
// `part` (256-byte aligned, avsr_bn_train_workspace_bytes(rows, C) - 256 bytes)
int launch_bn_stats(const float* z, long rows, int C, double* part, double* stats, cudaStream_t st);

// head.cu
int launch_log_softmax_rows(const float* x, long ldx, float* y, long ldy, int32_t* best, int rows, int n, cudaStream_t st);

// attention: q-side tensors (B,H,T,64), vt (B,H,64,Tp), pos (H,Rp,64) for one layer, ctx (B*T, H*64)
int attention_simt(const float* qu, const float* qv, const float* kk, const float* vt, const float* pos,
                   const int32_t* lengths, float* ctx, int B, int T, int H, int Tp, int Rp, int round_out,
                   cudaStream_t st);
int attention_tc(const float* qu, const float* qv, const float* kk, const float* vt, const float* pos,
                 const int32_t* lengths, float* ctx, int B, int T, int H, int Tp, int Rp, int round_out,
                 cudaStream_t st);
// (B,T,H*64) fp32 [+ bias (H*64)] -> (B,H,T,64) in operand storage `kind`, or (B,H,64,Tp) when transpose != 0 (encoder.cu)
int launch_split_heads(const float* src, const float* bias, void* dst, int B, int T, int H, int Tp, int transpose, int kind,
                       cudaStream_t st);
// 2-byte operands (attention_tc.cu), kind OP_F16 or OP_BF16: qu, qv, kk, vv all (B,H,T,64) (V in its natural
// layout); ctx (B*T, H*64) in the same storage
int attention_op16(int kind, const void* qu, const void* qv, const void* kk, const void* vv, const void* pos,
                   const int32_t* lengths, void* ctx, int B, int T, int H, int Rp, cudaStream_t st);

}  // namespace avsr
