// sae_optim.cuh -- the SAE optimizer, defined once for the single-GPU (sae.cu, sae_dense.cu) and peer-memory (p2p.cu) kernels:
// the device scalars of a step, the clip coefficient, Adam, the dead-feature counters and the per-feature row update.
//   clip -> remove decoder-parallel gradient -> Adam -> unit-norm decoder rows (+ counters)
//   (train_sae.py:394-401, sae.py:275-297, torch.optim.Adam defaults betas (0.9, 0.999), eps 1e-8, no weight decay)
//   The row renorm is the *next* step's set_decoder_norm_to_unit_norm() (train_sae.py:307) applied early; forward
//   and backward of every later step see identical numbers.
#pragma once
#include <stddef.h>
#include "common.cuh"

// ---------------------------------------------------------------------------------------------
// device scalars of one step (pb_abi_sizeof_sae(7) reports the size; Python reads clip_coef at its offset)
struct SaeScalars {
  float loss_sum;      // sum_b sum_c (out-x)^2 / nf[b]            (mse = loss_sum / (Bt*d))
  float gnorm_sq;      // sum of squares of all gradient entries (pre-clip)
  float clip_coef;     // min(1, max_norm / (norm + 1e-6))
  float mse;           // loss_sum / (Bt*d)
  float l0;            // mean number of positive activations per token
  unsigned pos_count;  // accumulator for l0: an integer, since an fp32 sum stops being exact past 2^24 positives
  float grad_norm;     // sqrt(gnorm_sq)
  float reserved;
};
static_assert(sizeof(SaeScalars) == 32, "SaeScalars is 8 floats");
static_assert(offsetof(SaeScalars, clip_coef) == 8, "SaeScalars.clip_coef is float 2");

// clip_grad_norm_ (train_sae.py:394-397)
__device__ __forceinline__ float sae_clip_coef(float norm, float max_norm) {
  return max_norm > 0.f ? fminf(1.f, max_norm / (norm + 1e-6f)) : 1.f;
}

// total gradient norm -> grad_norm, clip coefficient; accumulated loss / activation counts -> mse, l0
__device__ __forceinline__ void sae_publish_scalars(SaeScalars* sc, float gnorm_sq, float max_norm, float inv_elems, float inv_rows) {
  const float norm = sqrtf(gnorm_sq);
  sc->gnorm_sq = gnorm_sq;
  sc->grad_norm = norm;
  sc->clip_coef = sae_clip_coef(norm, max_norm);
  sc->mse = sc->loss_sum * inv_elems;
  sc->l0 = (float)sc->pos_count * inv_rows;
}

// ---------------------------------------------------------------------------------------------
struct AdamHyper { float lr, beta1, beta2, eps, bc1, bc2_sqrt; };  // bc1 = 1-beta1^t, bc2_sqrt = sqrt(1-beta2^t)

static inline AdamHyper adam_hyper(float lr, float beta1, float beta2, float eps, int step) {
  AdamHyper h;
  h.lr = lr; h.beta1 = beta1; h.beta2 = beta2; h.eps = eps;
  h.bc1 = 1.f - powf(beta1, (float)step);
  h.bc2_sqrt = sqrtf(1.f - powf(beta2, (float)step));
  return h;
}

// torch.optim.Adam (single tensor, no amsgrad / weight decay): m, v exactly as torch computes them; the parameter update
// -(lr / bc1) m / (sqrt(v) / bc2_sqrt + eps) uses MUFU sqrt / reciprocal approximations (relative error ~1e-7 of an update that is
// itself ~lr relative to the parameter: 1e-10 on the parameter, against a 1e-4 parity bar).  The IEEE sqrt + two divisions of the
// first version were ~30 of the ~45 instructions per element and made the optimizer issue-bound.  The moment updates are written
// as fmaf: left to contraction, the compiler fused a different product of `beta2 * v + (1 - beta2) * gr * gr` in different
// kernels, and the single-GPU and peer-memory optimizers differed in the last bit of v.
__device__ __forceinline__ float adam_update(float p, float gr, float& m, float& v, const AdamHyper& h) {
  m = fmaf(h.beta1, m, (1.f - h.beta1) * gr);
  v = fmaf(h.beta2, v, (1.f - h.beta2) * gr * gr);
  float sq, rc;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(sq) : "f"(v));
  const float denom = fmaf(sq, __frcp_rn(h.bc2_sqrt), h.eps);
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(denom));
  return fmaf(-(h.lr * __frcp_rn(h.bc1)) * m, rc, p);
}

// dead-feature bookkeeping of feature f (train_sae.py:356-361): sf / af are the counters' current values; either array may be absent
__device__ __forceinline__ void dead_feature_counters(float* since_fired, float* act_freq, int f, float fired, float sf, float af) {
  if (since_fired) since_fired[f] = fired > 0.f ? 0.f : sf + 1.f;
  if (act_freq) act_freq[f] = af + fired;
}

// ---------------------------------------------------------------------------------------------
// Who holds a row.  WarpRow: one warp (d <= 1536, the narrow kernels).  CtaRow: the SAE_WIDE_THREADS threads of a CTA (the wide
// kernels, 1536 < d <= 8192); its sums go through shared memory (red: SAE_WIDE_WARPS floats) and end in a barrier, so every
// thread of the CTA must reach each one.  Thread t() of a row holds columns 4 (i * kThreads + t()) .. +3 of chunk i.
constexpr int SAE_WIDE_THREADS = 256;
constexpr int SAE_WIDE_WARPS = SAE_WIDE_THREADS / 32;
constexpr int SAE_NARROW_MAX_D = 1536;
constexpr int SAE_WIDE_MAX_D = 8192;

// sum of v over the CTA (every thread gets it, added in the same warp order)
__device__ __forceinline__ float cta_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();                        // every thread has read the previous sum out of red
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < SAE_WIDE_WARPS; ++w) s += red[w];
  return s;
}

struct WarpRow {
  static constexpr int kThreads = 32;
  __device__ __forceinline__ int t() const { return threadIdx.x & 31; }
  __device__ __forceinline__ float sum(float v) const { return warp_sum(v); }
};
struct CtaRow {
  float* red;
  static constexpr int kThreads = SAE_WIDE_THREADS;
  __device__ __forceinline__ int t() const { return threadIdx.x; }
  __device__ __forceinline__ float sum(float v) const { return cta_sum(v, red); }
};

// ---------------------------------------------------------------------------------------------
// The update of one feature by one row holder (a warp, or with CtaRow a CTA; below "lane" is the holder's thread index t()).  The row pointers (parameters,
// gradients, Adam moments; global or shared memory) are read; the moments are written back in place; the updated parameter rows
// go to out.dec(c4, w) / out.enc(c4, p, lo, p16) (lo = tf32 residual of p, p16 = fp16 copy of p, packed), which decide where they
// are stored.  Returns this lane's partials of ||w_enc||^2, ||w_enc - trunc(w_enc)||^2 and ||w_enc - fp16(w_enc)||^2 (the fused
// encoder's error bounds) in esq / elo / e16; a caller that stores no fp16 copy ignores e16 and the compiler drops its arithmetic.
template <int CHUNKS, class Out, class Row = WarpRow>
__device__ __forceinline__ void sae_adam_feature(const float* wd, const float* gd, float* md, float* vd, const float* we, const float* ge,
                                                 float* me, float* ve, float clip, const AdamHyper& h, int nvec, bool renorm,
                                                 const Out& out, float& esq, float& elo, float& e16, const Row& row = Row()) {
  const int lane = row.t();
  // ---- decoder row: clip, remove the component parallel to the (unit-norm) row, Adam, renormalise
  float w[CHUNKS][4], gq[CHUNKS][4];
  float par = 0.f;
#pragma unroll
  for (int i = 0; i < CHUNKS; ++i) {
    const int c4 = i * Row::kThreads + lane;
    if (c4 < nvec) {
      ld4(wd + 4 * c4, w[i]);
      ld4(gd + 4 * c4, gq[i]);
#pragma unroll
      for (int q = 0; q < 4; ++q) { gq[i][q] *= clip; par = fmaf(gq[i][q], w[i][q], par); }
    } else {
      w[i][0] = w[i][1] = w[i][2] = w[i][3] = gq[i][0] = gq[i][1] = gq[i][2] = gq[i][3] = 0.f;
    }
  }
  par = row.sum(par);
  float nsq = 0.f;
#pragma unroll
  for (int i = 0; i < CHUNKS; ++i) {
    const int c4 = i * Row::kThreads + lane;
    if (c4 < nvec) {
      float mm[4], vv[4];
      ld4(md + 4 * c4, mm);
      ld4(vd + 4 * c4, vv);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        w[i][q] = adam_update(w[i][q], gq[i][q] - par * w[i][q], mm[q], vv[q], h);
        nsq += w[i][q] * w[i][q];
      }
      st4(md + 4 * c4, mm);
      st4(vd + 4 * c4, vv);
    }
  }
  const float inv_nrm = 1.f / sqrtf(row.sum(nsq));
#pragma unroll
  for (int i = 0; i < CHUNKS; ++i) {
    const int c4 = i * Row::kThreads + lane;
    if (c4 < nvec) {
      if (renorm) {
#pragma unroll
        for (int q = 0; q < 4; ++q) w[i][q] = w[i][q] * inv_nrm;
      }
      out.dec(c4, w[i]);
    }
  }
  // ---- encoder row (feature-major)
  esq = 0.f;
  elo = 0.f;
  e16 = 0.f;
#pragma unroll
  for (int i = 0; i < CHUNKS; ++i) {
    const int c4 = i * Row::kThreads + lane;
    if (c4 < nvec) {
      float p[4], gr[4], mm[4], vv[4], lo[4];
      ld4(we + 4 * c4, p);
      ld4(ge + 4 * c4, gr);
      ld4(me + 4 * c4, mm);
      ld4(ve + 4 * c4, vv);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        p[q] = adam_update(p[q], gr[q] * clip, mm[q], vv[q], h);
        lo[q] = tf32_lo(p[q]);
        esq = fmaf(p[q], p[q], esq);
        const float tl = p[q] - tf32_trunc(p[q]);
        elo = fmaf(tl, tl, elo);
      }
      st4(me + 4 * c4, mm);
      st4(ve + 4 * c4, vv);
      out.enc(c4, p, lo, f16x4(p, e16));
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side: the narrow row kernels are instantiated per CHUNKS = ceil(d / 128) rounded up to a built width (d <= 1536,
// d % 4 == 0), the wide ones per CHUNKS = ceil(d / 1024) rounded up to a built width (1536 < d <= 8192, d % 4 == 0)
static inline int chunks_for(int d) {
  if (d % 4 != 0) return -1;
  const int nvec = d / 4;
  if (nvec <= 32) return 1;
  if (nvec <= 64) return 2;
  if (nvec <= 128) return 4;
  if (nvec <= 192) return 6;
  if (nvec <= 256) return 8;
  if (nvec <= 384) return 12;
  return -1;
}
static inline int wide_chunks_for(int d) {
  if (d % 4 != 0 || d <= SAE_NARROW_MAX_D || d > SAE_WIDE_MAX_D) return -1;
  const int nvec = d / 4;
  if (nvec <= 2 * SAE_WIDE_THREADS) return 2;
  if (nvec <= 4 * SAE_WIDE_THREADS) return 4;
  if (nvec <= 6 * SAE_WIDE_THREADS) return 6;
  return 8;
}
#define PB_SAE_D_UNSUPPORTED()                                                                                      \
  do {                                                                                                              \
    pb_set_error("sae: d_in=%d unsupported (needs d %% 4 == 0 and d <= 8192)", d);                                  \
    return PB_EUNSUPPORTED;                                                                                         \
  } while (0)
#define PB_DISPATCH_CHUNKS(CH, ...)                                                    \
  switch (CH) {                                                                        \
    case 1: { constexpr int C_ = 1; __VA_ARGS__; } break;                              \
    case 2: { constexpr int C_ = 2; __VA_ARGS__; } break;                              \
    case 4: { constexpr int C_ = 4; __VA_ARGS__; } break;                              \
    case 6: { constexpr int C_ = 6; __VA_ARGS__; } break;                              \
    case 8: { constexpr int C_ = 8; __VA_ARGS__; } break;                              \
    case 12: { constexpr int C_ = 12; __VA_ARGS__; } break;                            \
    default: PB_SAE_D_UNSUPPORTED();                                                   \
  }
#define PB_DISPATCH_WIDE(CH, ...)                                                      \
  switch (CH) {                                                                        \
    case 2: { constexpr int C_ = 2; __VA_ARGS__; } break;                              \
    case 4: { constexpr int C_ = 4; __VA_ARGS__; } break;                              \
    case 6: { constexpr int C_ = 6; __VA_ARGS__; } break;                              \
    case 8: { constexpr int C_ = 8; __VA_ARGS__; } break;                              \
    default: PB_SAE_D_UNSUPPORTED();                                                   \
  }
