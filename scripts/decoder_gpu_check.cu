// Torch-free GPU check of the row 8f#3 entries of libavsr_b200 (decoder step over a forked beam, CTC prefix scorer)
// against oracle outputs prepared by scripts/make_decoder_check_blob.py.  Starts in seconds on a fresh box:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O2 -std=c++17 -Iinclude scripts/decoder_gpu_check.cu \
//        -Lauto_avsr_b200/csrc -lavsr_b200 -Xlinker -rpath -Xlinker '$ORIGIN/../../auto_avsr_b200/csrc' -o scripts/bin/decoder_gpu_check
//   scripts/bin/decoder_gpu_check scripts/bin/decoder_check.blob
// TEST INFRASTRUCTURE (calls the library only through include/avsr_b200.h).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <string>
#include <vector>

#include "avsr_b200.h"

#define CK(x)                                                                                   \
  do {                                                                                          \
    cudaError_t e_ = (x);                                                                       \
    if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(2); } \
  } while (0)
#define AV(x)                                                                                   \
  do {                                                                                          \
    int r_ = (x);                                                                               \
    if (r_ != 0) { printf("libavsr error %d at %s:%d: %s\n", r_, __FILE__, __LINE__, avsr_last_error()); exit(3); } \
  } while (0)

struct Arr { int dtype; std::vector<long long> shape; std::vector<char> data; size_t count() const { size_t n = 1; for (auto s : shape) n *= s; return n; } };
static std::map<std::string, Arr> g_blob;
static bool g_time = false;      // --time: after the parity pass, replay the last (widest) step / CTC call under CUDA events

static void load_blob(const char* path) {
  FILE* f = fopen(path, "rb");
  if (!f) { printf("cannot open %s\n", path); exit(1); }
  uint32_t n = 0;
  if (fread(&n, 4, 1, f) != 1) exit(1);
  for (uint32_t i = 0; i < n; ++i) {
    uint32_t len, dt, nd;
    if (fread(&len, 4, 1, f) != 1) exit(1);
    std::string name(len, ' ');
    if (fread(&name[0], 1, len, f) != len) exit(1);
    if (fread(&dt, 4, 1, f) != 1 || fread(&nd, 4, 1, f) != 1) exit(1);
    Arr a; a.dtype = dt; a.shape.resize(nd);
    if (nd && fread(a.shape.data(), 8, nd, f) != nd) exit(1);
    a.data.resize(a.count() * 4);
    if (a.count() && fread(a.data.data(), 4, a.count(), f) != a.count()) exit(1);
    g_blob[name] = std::move(a);
  }
  fclose(f);
}
static const Arr& get(const std::string& k) {
  auto it = g_blob.find(k);
  if (it == g_blob.end()) { printf("blob has no %s\n", k.c_str()); exit(1); }
  return it->second;
}
static void* to_dev(const void* h, size_t bytes) {
  void* d = nullptr;
  CK(cudaMalloc(&d, bytes ? bytes : 4));
  if (bytes) CK(cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice));
  return d;
}
static void* dev_of(const std::string& k) { const Arr& a = get(k); return to_dev(a.data.data(), a.data.size()); }

// ((i * 2654435761 + seed * 40503) mod 2^32 >> 8) / 2^24 - 0.5, * scale + offset  (make_decoder_check_blob.py hash_uniform)
static float* hashed(size_t count, int seed, float scale, float offset = 0.f) {
  std::vector<float> h(count);
  for (size_t i = 0; i < count; ++i) {
    const uint32_t u = (uint32_t)((uint64_t)i * 2654435761ull + (uint64_t)seed * 40503ull) >> 8;
    h[i] = ((float)u * (1.0f / 16777216.0f) - 0.5f) * scale + offset;
  }
  return (float*)to_dev(h.data(), count * 4);
}

static const char* kFields[26] = {"self_q_w", "self_q_b", "self_k_w", "self_k_b", "self_v_w", "self_v_b", "self_out_w", "self_out_b",
                                  "src_q_w", "src_q_b", "src_k_w", "src_k_b", "src_v_w", "src_v_b", "src_out_w", "src_out_b",
                                  "ff_w1", "ff_b1", "ff_w2", "ff_b2", "norm1_w", "norm1_b", "norm2_w", "norm2_b", "norm3_w", "norm3_b"};

static double run_decoder_case(const char* tag, bool hashed_weights, int precision) {
  const int32_t* c = (const int32_t*)get(std::string(tag) + ".cfg").data.data();
  AvsrDecoderConfig cfg{c[0], c[1], c[2], c[3], c[4]};
  const int T = c[5], steps = c[6], max_hyps = c[7];
  const size_t D = cfg.d_model, F = cfg.linear_units, O = cfg.odim;
  std::vector<AvsrDecoderLayerParams> layers(cfg.num_blocks);
  float *embed, *after_w, *after_b, *out_w, *out_b, *memory;
  int seed = 1;
  if (hashed_weights) {
    embed = hashed(O * D, seed++, 2.0f / sqrtf((float)D));
    for (int l = 0; l < cfg.num_blocks; ++l) {
      const float** p = (const float**)&layers[l];
      for (int k = 0; k < 26; ++k) {
        const std::string f = kFields[k];
        const bool is_b = f.back() == 'b' || (f.size() > 2 && f[f.size() - 2] == 'b');       // "..._b" or "ff_b1" / "ff_b2"
        if (f.rfind("norm", 0) == 0) p[k] = f.back() == 'w' ? hashed(D, seed++, 1.0f, 1.0f) : hashed(D, seed++, 0.2f);
        else if (is_b) p[k] = hashed(f == "ff_b1" ? F : D, seed++, 0.2f);
        else {
          const size_t o = f == "ff_w1" ? F : D, i = f == "ff_w2" ? F : D;
          p[k] = hashed(o * i, seed++, 2.0f / sqrtf((float)i));
        }
      }
    }
    after_w = hashed(D, seed++, 1.0f, 1.0f);
    after_b = hashed(D, seed++, 0.2f);
    out_w = hashed(O * D, seed++, 2.0f / sqrtf((float)D));
    out_b = hashed(O, seed++, 0.2f);
    memory = hashed((size_t)T * D, seed++, 3.0f);
  } else {
    const std::string t = tag;
    embed = (float*)dev_of(t + ".embed");
    for (int l = 0; l < cfg.num_blocks; ++l) {
      const float** p = (const float**)&layers[l];
      for (int k = 0; k < 26; ++k) p[k] = (const float*)dev_of(t + ".l" + std::to_string(l) + "." + kFields[k]);
    }
    after_w = (float*)dev_of(t + ".after_w"); after_b = (float*)dev_of(t + ".after_b");
    out_w = (float*)dev_of(t + ".out_w"); out_b = (float*)dev_of(t + ".out_b");
    memory = (float*)dev_of(t + ".memory");
  }
  const size_t pb = avsr_decoder_prepared_bytes(&cfg);
  void* prepared; CK(cudaMalloc(&prepared, pb));
  AV(avsr_prepare_decoder(&cfg, layers.data(), embed, after_w, after_b, out_w, out_b, prepared, pb, precision, nullptr));
  const int max_steps = steps + 1;
  const size_t sb = avsr_decoder_session_bytes(&cfg, T, max_steps, max_hyps);
  const size_t wb = avsr_decoder_step_workspace_bytes(&cfg, T, max_steps, max_hyps);
  void *session, *work; CK(cudaMalloc(&session, sb)); CK(cudaMalloc(&work, wb));
  AV(avsr_decoder_begin(&cfg, prepared, memory, T, max_steps, max_hyps, session, sb, precision, nullptr));
  double worst = 0;
  for (int s = 0; s < steps; ++s) {
    const Arr& tok = get(std::string(tag) + ".tokens" + std::to_string(s));
    const Arr& want = get(std::string(tag) + ".logp" + std::to_string(s));
    const int n = (int)tok.count();
    int32_t* d_tok = (int32_t*)dev_of(std::string(tag) + ".tokens" + std::to_string(s));
    int32_t* d_anc = s ? (int32_t*)dev_of(std::string(tag) + ".anc" + std::to_string(s)) : nullptr;
    float* d_logp; CK(cudaMalloc(&d_logp, (size_t)n * O * 4));
    AV(avsr_decoder_step(&cfg, prepared, session, sb, T, max_steps, max_hyps, d_tok, d_anc, s, n, d_logp, work, wb, precision, nullptr));
    CK(cudaDeviceSynchronize());
    std::vector<float> got((size_t)n * O);
    CK(cudaMemcpy(got.data(), d_logp, got.size() * 4, cudaMemcpyDeviceToHost));
    const float* w = (const float*)want.data.data();
    double mx = 0, sum = 0;
    for (size_t i = 0; i < got.size(); ++i) {
      const double e = fabs((double)got[i] - w[i]);
      if (!(e == e)) mx = 1e30;
      mx = e > mx ? e : mx;
    }
    for (int i = 0; i < (int)O; ++i) sum += exp((double)got[i]);
    printf("  %s prec=%d step %d n=%d  max|logp - oracle| = %.3e   sum(exp(row0)) = %.6f\n", tag, precision, s, n, mx, sum);
    worst = mx > worst ? mx : worst;
    if (g_time && s == steps - 1) {
      cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
      const unsigned long long l0 = avsr_launch_count();
      for (int it = 0; it < 5; ++it)
        AV(avsr_decoder_step(&cfg, prepared, session, sb, T, max_steps, max_hyps, d_tok, d_anc, s, n, d_logp, work, wb, precision, nullptr));
      const int reps = 50;
      CK(cudaEventRecord(e0));
      for (int it = 0; it < reps; ++it)
        AV(avsr_decoder_step(&cfg, prepared, session, sb, T, max_steps, max_hyps, d_tok, d_anc, s, n, d_logp, work, wb, precision, nullptr));
      CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
      float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
      printf("  TIMING %s prec=%d: avsr_decoder_step n=%d step=%d T=%d: %.1f us per call (CUDA events over %d back-to-back calls, %llu launches per call)\n",
             tag, precision, n, s, T, ms * 1e3 / reps, reps, (avsr_launch_count() - l0) / (reps + 5));
    }
  }
  return worst;
}

static double run_ctc_case() {
  const int32_t* c = (const int32_t*)get("ctc.cfg").data.data();
  const int T = c[0], O = c[1], n = c[2], S = c[3], steps = c[4];
  float* logp = (float*)dev_of("ctc.logp");
  float *r0, *r_prev, *s_prev, *local, *r, *log_psi, *r_next, *s_next;
  CK(cudaMalloc(&r0, T * 2 * 4)); CK(cudaMalloc(&r_prev, (size_t)T * 2 * n * 4)); CK(cudaMalloc(&s_prev, n * 4));
  CK(cudaMalloc(&local, (size_t)n * O * 4)); CK(cudaMalloc(&log_psi, (size_t)n * O * 4)); CK(cudaMalloc(&r, (size_t)T * 2 * n * S * 4));
  CK(cudaMalloc(&r_next, (size_t)T * 2 * n * 4)); CK(cudaMalloc(&s_next, n * 4));
  AV(avsr_ctc_prefix_init(logp, T, O, 0, r0, nullptr));
  std::vector<float> h0(T * 2), hp((size_t)T * 2 * n);
  CK(cudaMemcpy(h0.data(), r0, h0.size() * 4, cudaMemcpyDeviceToHost));
  for (int t = 0; t < T; ++t) for (int k = 0; k < 2; ++k) for (int i = 0; i < n; ++i) hp[((size_t)t * 2 + k) * n + i] = h0[t * 2 + k];
  CK(cudaMemcpy(r_prev, hp.data(), hp.size() * 4, cudaMemcpyHostToDevice));
  CK(cudaMemset(s_prev, 0, n * 4));
  std::vector<int32_t> lanes(n);
  for (int i = 0; i < n; ++i) lanes[i] = i;
  int32_t* d_lanes = (int32_t*)to_dev(lanes.data(), n * 4);
  double worst = 0;
  for (int s = 0; s < steps; ++s) {
    const std::string k = std::to_string(s);
    int32_t* last = (int32_t*)dev_of("ctc.last" + k);
    int32_t* cand = (int32_t*)dev_of("ctc.cand" + k);
    int32_t* keep = (int32_t*)dev_of("ctc.keep" + k);
    AV(avsr_ctc_prefix_score(logp, T, O, 0, O - 1, s, last, r_prev, s_prev, cand, n, S, local, r, log_psi, nullptr));
    AV(avsr_ctc_prefix_select(r, log_psi, cand, d_lanes, keep, T, O, n, S, n, r_next, s_next, nullptr));
    CK(cudaDeviceSynchronize());
    std::vector<float> got((size_t)n * O);
    CK(cudaMemcpy(got.data(), local, got.size() * 4, cudaMemcpyDeviceToHost));
    const float* w = (const float*)get("ctc.local" + k).data.data();
    double mx = 0;
    for (size_t i = 0; i < got.size(); ++i) {
      if (w[i] < -1e9f || w[i] > 1e9f) { if (!(got[i] < -1e9f || got[i] > 1e9f)) mx = 1e30; continue; }
      const double e = fabs((double)got[i] - w[i]);
      if (!(e == e)) mx = 1e30;
      mx = e > mx ? e : mx;
    }
    printf("  ctc step %d  max|local - oracle| (live entries) = %.3e\n", s, mx);
    worst = mx > worst ? mx : worst;
    CK(cudaMemcpy(r_prev, r_next, (size_t)T * 2 * n * 4, cudaMemcpyDeviceToDevice));
    CK(cudaMemcpy(s_prev, s_next, n * 4, cudaMemcpyDeviceToDevice));
  }
  return worst;
}

static void time_ctc(int T, int O, int n, int S) {
  std::vector<float> h((size_t)T * O);
  for (size_t i = 0; i < h.size(); ++i) h[i] = -8.5f + 0.001f * (float)(i % 977);        // plausible log-posteriors
  float* logp = (float*)to_dev(h.data(), h.size() * 4);
  std::vector<int32_t> cand((size_t)n * S), last(n, O - 1);
  for (int i = 0; i < n; ++i) for (int c = 0; c < S; ++c) cand[(size_t)i * S + c] = 1 + ((i * 131 + c * 17) % (O - 2));
  int32_t* d_cand = (int32_t*)to_dev(cand.data(), cand.size() * 4);
  int32_t* d_last = (int32_t*)to_dev(last.data(), n * 4);
  float *r_prev, *s_prev, *local, *r, *log_psi;
  CK(cudaMalloc(&r_prev, (size_t)T * 2 * n * 4)); CK(cudaMemset(r_prev, 0, (size_t)T * 2 * n * 4));
  CK(cudaMalloc(&s_prev, n * 4)); CK(cudaMemset(s_prev, 0, n * 4));
  CK(cudaMalloc(&local, (size_t)n * O * 4)); CK(cudaMalloc(&log_psi, (size_t)n * O * 4)); CK(cudaMalloc(&r, (size_t)T * 2 * n * S * 4));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  for (int it = 0; it < 3; ++it) AV(avsr_ctc_prefix_score(logp, T, O, 0, O - 1, 5, d_last, r_prev, s_prev, d_cand, n, S, local, r, log_psi, nullptr));
  const int reps = 50;
  CK(cudaEventRecord(e0));
  for (int it = 0; it < reps; ++it) AV(avsr_ctc_prefix_score(logp, T, O, 0, O - 1, 5, d_last, r_prev, s_prev, d_cand, n, S, local, r, log_psi, nullptr));
  CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
  float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
  printf("  TIMING avsr_ctc_prefix_score T=%d O=%d n=%d S=%d: %.1f us per call\n", T, O, n, S, ms * 1e3 / reps);
}

int main(int argc, char** argv) {
  const char* blob = "scripts/bin/decoder_check.blob";
  bool only_time = false;
  for (int i = 1; i < argc; ++i) {
    if (!strcmp(argv[i], "--time")) g_time = true;
    else if (!strcmp(argv[i], "--only-time")) g_time = only_time = true;
    else blob = argv[i];
  }
  load_blob(blob);
  if (only_time) {            // the two full-size decoder passes (they carry the timing hook) and the CTC call, nothing else
    cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
    printf("device: %s\n", p.name);
    run_decoder_case("full", true, AVSR_PREC_F16);
    run_decoder_case("full", true, AVSR_PREC_FP32);
    time_ctc(100, 5049, 40, 60);
    time_ctc(400, 5049, 40, 60);
    return 0;
  }
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  printf("device: %s (sm_%d%d), libavsr ABI %d\n", prop.name, prop.major, prop.minor, avsr_abi_version());
  int bad = 0;
  const double c = run_ctc_case();
  printf("CTC prefix scorer: worst %.3e (bound 1e-3)\n", c); bad |= !(c < 1e-3);
  const double t32 = run_decoder_case("tiny", false, AVSR_PREC_FP32);
  printf("decoder tiny fp32: worst %.3e (bound 2e-4)\n", t32); bad |= !(t32 < 2e-4);
  const double t16 = run_decoder_case("tiny", false, AVSR_PREC_F16);
  printf("decoder tiny f16: worst %.3e (bound 5e-2)\n", t16); bad |= !(t16 < 5e-2);
  const double ttf = run_decoder_case("tiny", false, AVSR_PREC_TF32);
  printf("decoder tiny tf32: worst %.3e (bound 5e-2)\n", ttf); bad |= !(ttf < 5e-2);
  const double f16 = run_decoder_case("full", true, AVSR_PREC_F16);
  printf("decoder full f16: worst %.3e (bound 1e-1)\n", f16); bad |= !(f16 < 1e-1);
  const double f32 = run_decoder_case("full", true, AVSR_PREC_FP32);
  printf("decoder full fp32: worst %.3e (bound 5e-4)\n", f32); bad |= !(f32 < 5e-4);
  printf("launches: %llu\nDECODER_GPU_CHECK %s\n", (unsigned long long)avsr_launch_count(), bad ? "FAILED" : "PASSED");
  return bad;
}
