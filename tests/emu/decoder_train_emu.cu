// HOST replay of the decoder's training kernels (csrc/decoder_train.cu) -- TEST INFRASTRUCTURE ONLY
// (tests/emu/build_decoder_train.py builds it into tests/emu/_build/libavsr_decoder_train_emu.so; nothing under
// auto_avsr_b200/ knows it exists).
//
// The CPU suite checks the masks, dropout factors, softmax / backward combination and the label-smoothing and embedding
// math of csrc/decoder_train_body.cuh by compiling that same header into plain loops that follow the kernels' schedule
// (per query row: log-sum-exp, probabilities, ctx; backward: Delta and dq per row, dk / dv per key; per logits row the
// one-pass (max, sum exp, sum x)).  Same extern "C" names and signatures as include/avsr_b200.h, HOST pointers.
#include <stdarg.h>

#include <vector>

#include "../../auto_avsr_b200/csrc/decoder_train_body.cuh"

namespace avsr {
static thread_local std::string g_emu_err;
void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_emu_err = buf;
}
}  // namespace avsr

using namespace avsr;
using namespace avsr::dtr;

static float dot64h(const float* a, const float* b) {
  float acc = 0.f;
  for (int d = 0; d < 64; ++d) acc = fmaf(a[d], b[d], acc);
  return acc;
}

extern "C" {
const char* avsr_last_error(void) { return g_emu_err.c_str(); }

int avsr_mha_core_fwd(const float* q, long ldq, const float* k, long ldk, const float* v, long ldv, int B, int H, int Lq,
                      int Lk, int causal, const int32_t* key_lengths, const uint8_t* keep, float keep_scale, float* ctx,
                      float* probs, void*) {
  AVSR_REQUIRE(B >= 0 && H >= 1 && Lq >= 0 && Lk >= 0 && ldq >= H * 64 && ldk >= H * 64 && ldv >= H * 64, "emu: bad shape");
  std::vector<float> sc(Lk > 0 ? Lk : 1);
  for (int b = 0; b < B; ++b)
    for (int h = 0; h < H; ++h)
      for (int i = 0; i < Lq; ++i) {
        const long row = ((long)b * H + h) * Lq + i, prow = row * Lk;
        const int n = attn_row_keys(i, Lk, causal, key_lengths, b);
        const float* qr = q + ((long)b * Lq + i) * ldq + h * 64;
        float m = -INFINITY;
        for (int j = 0; j < n; ++j) {
          sc[j] = dot64h(qr, k + ((long)b * Lk + j) * ldk + h * 64) * kAttnScale;
          m = fmaxf(m, sc[j]);
        }
        float s = 0.f;
        for (int j = 0; j < n; ++j) s += expf(sc[j] - m);
        const float lse = n > 0 ? m + logf(s) : 0.f;
        float* cr = ctx + ((long)b * Lq + i) * (H * 64) + h * 64;
        for (int d = 0; d < 64; ++d) cr[d] = 0.f;
        for (int j = 0; j < Lk; ++j) {
          const float p = j < n ? expf(sc[j] - lse) : 0.f;
          if (probs) probs[prow + j] = p;
          if (j >= n) continue;
          const float pd = p * keep_factor(keep, prow + j, keep_scale);
          const float* vr = v + ((long)b * Lk + j) * ldv + h * 64;
          for (int d = 0; d < 64; ++d) cr[d] = fmaf(pd, vr[d], cr[d]);
        }
      }
  return AVSR_OK;
}

size_t avsr_mha_core_bwd_workspace_bytes(int B, int H, int Lq) {
  if (B <= 0 || H <= 0 || Lq <= 0) return 256;
  return align_up((size_t)B * H * Lq * sizeof(float), 256);
}

int avsr_mha_core_bwd(const float* q, long ldq, const float* k, long ldk, const float* v, long ldv, int B, int H, int Lq,
                      int Lk, int causal, const int32_t* key_lengths, const uint8_t* keep, float keep_scale,
                      const float* probs, const float* dctx, float* dq, long lddq, float* dk, float* dv, long lddkv,
                      void* workspace, size_t workspace_bytes, void*) {
  if (avsr_mha_core_bwd_workspace_bytes(B, H, Lq) > workspace_bytes) return AVSR_E_WORKSPACE;
  float* delta = reinterpret_cast<float*>(workspace);
  const int D = H * 64;
  auto da = [&](int b, int h, int i, int j) {
    const long pidx = (((long)b * H + h) * Lq + i) * Lk + j;
    return dot64h(dctx + ((long)b * Lq + i) * D + h * 64, v + ((long)b * Lk + j) * ldv + h * 64) *
           keep_factor(keep, pidx, keep_scale);
  };
  for (int b = 0; b < B; ++b)
    for (int h = 0; h < H; ++h) {
      for (int i = 0; i < Lq; ++i) {                      // rows: Delta, dq
        const long row = ((long)b * H + h) * Lq + i, prow = row * Lk;
        const int n = attn_row_keys(i, Lk, causal, key_lengths, b);
        float dl = 0.f;
        for (int j = 0; j < n; ++j) dl = fmaf(probs[prow + j], da(b, h, i, j), dl);
        delta[row] = dl;
        float* o = dq + ((long)b * Lq + i) * lddq + h * 64;
        for (int d = 0; d < 64; ++d) o[d] = 0.f;
        for (int j = 0; j < n; ++j) {
          const float ds = attn_dscore(probs[prow + j], da(b, h, i, j), dl);
          const float* kr = k + ((long)b * Lk + j) * ldk + h * 64;
          for (int d = 0; d < 64; ++d) o[d] = fmaf(ds, kr[d], o[d]);
        }
      }
      for (int j = 0; j < Lk; ++j) {                      // keys: dk, dv
        float* ko = dk + ((long)b * Lk + j) * lddkv + h * 64;
        float* vo = dv + ((long)b * Lk + j) * lddkv + h * 64;
        for (int d = 0; d < 64; ++d) ko[d] = vo[d] = 0.f;
        if (j >= attn_row_keys(0, Lk, 0, key_lengths, b)) continue;
        for (int i = attn_first_query(j, causal); i < Lq; ++i) {
          const long row = ((long)b * H + h) * Lq + i, pidx = row * Lk + j;
          const float a = probs[pidx], kf = keep_factor(keep, pidx, keep_scale);
          const float ds = attn_dscore(a, da(b, h, i, j), delta[row]);
          const float* qr = q + ((long)b * Lq + i) * ldq + h * 64;
          const float* dr = dctx + ((long)b * Lq + i) * D + h * 64;
          for (int d = 0; d < 64; ++d) {
            ko[d] = fmaf(ds, qr[d], ko[d]);
            vo[d] = fmaf(a * kf, dr[d], vo[d]);
          }
        }
      }
    }
  return AVSR_OK;
}

int avsr_label_smoothing_fwd(const float* logits, long ld, const int64_t* target, int rows, int odim, int ignore_id,
                             float smoothing, float* row_loss, float* lse, void*) {
  AVSR_REQUIRE(rows >= 0 && odim >= 2 && ld >= odim, "emu: bad shape");
  const LsConst kc = ls_const(odim, smoothing);
  for (long r = 0; r < rows; ++r) {
    const int kind = ls_row_kind(target[r], ignore_id, odim);
    if (kind == 0) { row_loss[r] = lse[r] = 0.f; continue; }
    const float* xr = logits + r * ld;
    float m = -INFINITY, sx = 0.f;
    for (int c = 0; c < odim; ++c) { m = fmaxf(m, xr[c]); sx += xr[c]; }
    float s = 0.f;
    for (int c = 0; c < odim; ++c) s += expf(xr[c] - m);
    lse[r] = m + logf(s);
    row_loss[r] = kind < 0 ? NAN : ls_row_loss(kc, lse[r], sx, xr[target[r]]);
  }
  return AVSR_OK;
}

int avsr_label_smoothing_bwd(const float* logits, long ld, const int64_t* target, int rows, int odim, int ignore_id,
                             float smoothing, const float* lse, const float* dscale, float* dlogits, long ldd, void*) {
  AVSR_REQUIRE(rows >= 0 && odim >= 2 && ld >= odim && ldd >= odim, "emu: bad shape");
  const LsConst kc = ls_const(odim, smoothing);
  for (long r = 0; r < rows; ++r) {
    const int kind = ls_row_kind(target[r], ignore_id, odim);
    for (long c = 0; c < ldd; ++c) {
      float d = 0.f;
      if (c < odim && kind != 0) d = kind < 0 ? NAN : ls_grad(kc, logits[r * ld + c], lse[r], *dscale, c == target[r]);
      dlogits[r * ldd + c] = d;
    }
  }
  return AVSR_OK;
}

int avsr_embed_fwd(const int64_t* tokens, const float* embed, int rows, int L, int D, int odim, float* x, void*) {
  AVSR_REQUIRE(rows >= 0 && L >= 1 && D >= 1 && odim >= 1, "emu: bad shape");
  const EmbedTrainElem f{tokens, embed, x, D, L, odim, (float)sqrt((double)D), (float)(-(log(10000.0) / D))};
  for (long idx = 0; idx < (long)rows * D; ++idx) f(idx);
  return AVSR_OK;
}

size_t avsr_embed_bwd_workspace_bytes(int rows, int odim) {
  if (rows < 0 || odim < 0) return 0;
  return align_up((size_t)(odim + 1) * 4, 256) + align_up((size_t)(rows > 0 ? rows : 1) * 4, 256);
}

int avsr_embed_bwd(const int64_t* tokens, const float* dx, int rows, int D, int odim, float* dembed, void*, size_t, void*) {
  const float xscale = (float)sqrt((double)D);
  for (long idx = 0; idx < (long)odim * D; ++idx) dembed[idx] = 0.f;
  for (int t = 0; t < odim; ++t)                          // per token, its positions in position order
    for (int r = 0; r < rows; ++r)
      if (embed_token_ok(tokens[r], odim) && tokens[r] == t)
        for (int c = 0; c < D; ++c) dembed[(long)t * D + c] += dx[(long)r * D + c] * xscale;
  return AVSR_OK;
}
}  // extern "C"
