// sae_dense.cu -- the pieces of the SAE training step that are dense in d_sae:
//   * activation_fn_str = "relu" (+ L1 sparsity term), the reference's default activation (sae/sae.py:617-626, 810-839):
//     feature_acts, the decoder product and all four weight gradients are dense [tokens, d_sae] / [d_sae, d_in] GEMMs; they
//     run on pb_gemm (wgmma, 3xTF32) and the kernels here are the glue between them -- transposes (pb_gemm takes K-major
//     operands), statistics, loss / dL/d(out), the ReLU + L1 backward mask, bias gradients, the global gradient norm;
//   * the ghost-grad auxiliary loss on dead features (sae/sae.py:151-179; train_sae.py:330-332), for either activation:
//     column gather exp(hidden_pre[:, dead]), the per-row residual / rescale / loss / dL/dG kernel, row gathers and
//     scatter-adds that fold the dead-feature gradient blocks into the [d_sae, d_in] gradient arrays.
// Everything is fp32, HBM-bound streaming work (one read + one write per element unless stated).
#include <algorithm>

#include "common.cuh"
#include "sae_optim.cuh"

namespace {

// ---- out[c][r] = in[r][c] (+ tf32 residual plane of the transposed values)
__global__ void __launch_bounds__(256) k_transpose32(const float* __restrict__ in, float* __restrict__ out, float* __restrict__ out_lo, int rows,
                                                     int cols) {
  __shared__ float tile[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
#pragma unroll
  for (int j = 0; j < 32; j += 8) {
    const int r = r0 + ty + j, c = c0 + tx;
    tile[ty + j][tx] = (r < rows && c < cols) ? in[(int64_t)r * cols + c] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 32; j += 8) {
    const int c = c0 + ty + j, r = r0 + tx;
    if (c < cols && r < rows) {
      const float v = tile[tx][ty + j];
      out[(int64_t)c * rows + r] = v;
      if (out_lo) out_lo[(int64_t)c * rows + r] = tf32_lo(v);
    }
  }
}

// ---- out[c] += sum over a chunk of rows of x[r][c]   (out zeroed by the launcher unless accumulate)
__global__ void __launch_bounds__(256) k_colsum_any(const float* __restrict__ x, float* __restrict__ out, int rows, int cols, int rows_per_cta) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= cols) return;
  const int r0 = blockIdx.y * rows_per_cta, r1 = min(rows, r0 + rows_per_cta);
  float s = 0.f;
  for (int r = r0; r < r1; ++r) s += x[(int64_t)r * cols + c];
  atomicAdd(out + c, s);
}

// ---- out[c] += sum_f v[f] * W[f][c]
__global__ void __launch_bounds__(256) k_gemv_rows(const float* __restrict__ W, const float* __restrict__ v, float* __restrict__ out, int F, int d,
                                                   int f_per_cta) {
  const int f0 = blockIdx.x * f_per_cta, f1 = min(F, f0 + f_per_cta);
  for (int c = threadIdx.x; c < d; c += 256) {
    float s = 0.f;
    for (int f = f0; f < f1; ++f) s = fmaf(v[f], W[(int64_t)f * d + c], s);
    atomicAdd(out + c, s);
  }
}

// ---- dense activation statistics (train_sae.py:356-365): fired[f] += #{tokens: acts > 0}; l1_sum += sum |acts|; pos_count
__global__ void __launch_bounds__(256) k_dense_stats(const float* __restrict__ acts, int rows, int F, int rows_per_cta, float* __restrict__ fired,
                                                     float* __restrict__ l1_sum, SaeScalars* __restrict__ sc) {
  __shared__ float red[2][8];
  const int f = blockIdx.x * 256 + threadIdx.x;
  float cnt = 0.f, l1 = 0.f;
  if (f < F) {
    const int r0 = blockIdx.y * rows_per_cta, r1 = min(rows, r0 + rows_per_cta);
    for (int r = r0; r < r1; ++r) {
      const float a = acts[(int64_t)r * F + f];
      cnt += a > 0.f ? 1.f : 0.f;
      l1 += fabsf(a);
    }
    if (cnt > 0.f) atomicAdd(fired + f, cnt);
  }
  const float c = warp_sum(cnt), l = warp_sum(l1);
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = c; red[1][threadIdx.x >> 5] = l; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int i = 0; i < 8; ++i) { a += red[0][i]; b += red[1][i]; }
    if (a != 0.f) atomicAdd(&sc->pos_count, (unsigned)a);     // a: a whole count below 2^24, exact in fp32
    if (b != 0.f) atomicAdd(l1_sum, b);
  }
}

// ---- loss / dL/d(out_n) from the dense decoder output (sae.py:144-149, 584-592); one warp per token row
__global__ void __launch_bounds__(256) k_dense_loss(const float* __restrict__ x, const float* __restrict__ out_n, const float* __restrict__ mu,
                                                    const float* __restrict__ sd, const float* __restrict__ xsum, float* __restrict__ sae_out,
                                                    float* __restrict__ g, float* __restrict__ resid, SaeScalars* __restrict__ sc, int rows, int d,
                                                    int norm_mode, float inv_rows) {
  __shared__ float red[8];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int row = blockIdx.x * 8 + w;
  float loss_part = 0.f;
  if (row < rows) {
    const float m = norm_mode == 1 ? mu[row] : 0.f;
    const float s = norm_mode ? sd[row] : 1.f;
    const float* xr = x + (int64_t)row * d;
    const float* orow = out_n + (int64_t)row * d;
    float nsq = 0.f, esq = 0.f;
    for (int c = lane; c < d; c += 32) {
      const float o = norm_mode == 1 ? orow[c] * s + m : (norm_mode == 2 ? orow[c] * s : orow[c]);
      const float xc = xr[c] - xsum[c] * inv_rows;
      const float e = o - xr[c];
      nsq += xc * xc;
      esq += e * e;
      if (sae_out) sae_out[(int64_t)row * d + c] = o;
      if (resid) resid[(int64_t)row * d + c] = -e;
    }
    const float nf = sqrtf(warp_sum(nsq));
    loss_part = warp_sum(esq) / nf;
    if (g) {
      const float gs = 2.f * s * inv_rows / ((float)d * nf);
      for (int c = lane; c < d; c += 32) {
        const float o = norm_mode == 1 ? orow[c] * s + m : (norm_mode == 2 ? orow[c] * s : orow[c]);
        g[(int64_t)row * d + c] = (o - xr[c]) * gs;
      }
    }
  }
  if (lane == 0) red[w] = loss_part;
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f;
    for (int i = 0; i < 8; ++i) a += red[i];
    atomicAdd(&sc->loss_sum, a);
  }
}

// ---- d_hid = (d_acts + l1_grad) * [acts > 0]  (ReLU backward with the L1 term folded in), in place, + tf32 residual
__global__ void __launch_bounds__(256) k_dense_dhid(float* __restrict__ d_acts, const float* __restrict__ acts, float* __restrict__ lo, float l1_grad,
                                                    int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
    const float v = acts[i] > 0.f ? d_acts[i] + l1_grad : 0.f;
    d_acts[i] = v;
    if (lo) lo[i] = tf32_lo(v);
  }
}

// ---- sum of squares of an array into *acc
__global__ void __launch_bounds__(256) k_sumsq(const float* __restrict__ a, int64_t n, float* __restrict__ acc) {
  __shared__ float red[8];
  float s = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) s = fmaf(a[i], a[i], s);
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i];
    atomicAdd(acc, t);
  }
}
__global__ void k_grad_finish(SaeScalars* sc, float max_norm, float inv_elems, float inv_rows) {
  sae_publish_scalars(sc, sc->gnorm_sq, max_norm, inv_elems, inv_rows);
}

// ---- ghost grads ------------------------------------------------------------------------------------------------
// E[r][j] = exp(hidden_pre[r][dead[j]]) for j < nd, 0 for the padding columns nd <= j < ldE   (sae.py:164)
__global__ void __launch_bounds__(256) k_ghost_gather(const float* __restrict__ hp, const int* __restrict__ dead, int nd, int rows, int F,
                                                      float* __restrict__ E, int ldE) {
  const int64_t n = (int64_t)rows * ldE;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
    const int r = (int)(i / ldE), j = (int)(i - (int64_t)r * ldE);
    E[i] = j < nd ? expf(hp[(int64_t)r * F + dead[j]]) : 0.f;
  }
}
// out[j][:] = W[idx[j]][:] (j < n), zero rows up to n_pad
__global__ void __launch_bounds__(256) k_gather_rows(const float* __restrict__ W, const int* __restrict__ idx, int n, int n_pad, int d,
                                                     float* __restrict__ out) {
  const int64_t tot = (int64_t)n_pad * d;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < tot; i += (int64_t)gridDim.x * 256) {
    const int j = (int)(i / d), c = (int)(i - (int64_t)j * d);
    out[i] = j < n ? W[(int64_t)idx[j] * d + c] : 0.f;
  }
}
// dst[idx[j]][:] += scale * src[j][:]   (indices are distinct: plain read-modify-write)
__global__ void __launch_bounds__(256) k_scatter_add_rows(float* __restrict__ dst, const int* __restrict__ idx, int n, int d,
                                                          const float* __restrict__ src, float scale) {
  const int64_t tot = (int64_t)n * d;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < tot; i += (int64_t)gridDim.x * 256) {
    const int j = (int)(i / d), c = (int)(i - (int64_t)j * d);
    dst[(int64_t)idx[j] * d + c] += scale * src[i];
  }
}
// y[i] *= x[i]
__global__ void __launch_bounds__(256) k_mul_inplace(float* __restrict__ y, const float* __restrict__ x, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) y[i] *= x[i];
}

// _compute_ghost_residual_loss (sae.py:151-179), one warp per token row.  In: r = x - sae_out, rsum = column sums of r,
// G0 = exp(hidden_pre[:, dead]) @ W_dec[dead].  Out (in place of G0): dL_ghost/dG0; ghost_sum += sum_c c * Lel.
//   rcn = ||r - mean_batch r||, s = ||r|| / (1e-6 + 2 ||G0||)  [detached], G = s G0, Lel = (G - r)^2 / rcn,
//   c = mse / (Lel + 1e-6) [detached], loss = mean(c * Lel)  =>  dL/dG0 = c * 2 (G - r) / rcn / (rows * d) * s
__global__ void __launch_bounds__(256) k_ghost_rows(const float* __restrict__ r, const float* __restrict__ rsum, float* __restrict__ G0,
                                                    const SaeScalars* __restrict__ sc, float* __restrict__ ghost_sum, int rows, int d,
                                                    float inv_rows, float inv_elems) {
  __shared__ float red[8];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int row = blockIdx.x * 8 + w;
  float part = 0.f;
  if (row < rows) {
    const float mse = sc->loss_sum * inv_elems;
    const float* rr = r + (int64_t)row * d;
    float* gr = G0 + (int64_t)row * d;
    float rc2 = 0.f, r2 = 0.f, g2 = 0.f;
    for (int c = lane; c < d; c += 32) {
      const float rv = rr[c], rc = rv - rsum[c] * inv_rows, gv = gr[c];
      rc2 += rc * rc; r2 += rv * rv; g2 += gv * gv;
    }
    const float rcn = sqrtf(warp_sum(rc2)), l2r = sqrtf(warp_sum(r2)), l2g = sqrtf(warp_sum(g2));
    const float s = l2r / (1e-6f + l2g * 2.f);
    for (int c = lane; c < d; c += 32) {
      const float diff = gr[c] * s - rr[c];
      const float lel = diff * diff / rcn;
      const float cc = mse / (lel + 1e-6f);
      part += cc * lel;
      gr[c] = cc * 2.f * diff / rcn * inv_elems * s;
    }
    part = warp_sum(part);
  }
  if (lane == 0) red[w] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f;
    for (int i = 0; i < 8; ++i) a += red[i];
    atomicAdd(ghost_sum, a);
  }
}

inline int stream_grid(int64_t n) { return (int)std::min<int64_t>((n + 255) / 256, (int64_t)pb_sm_count() * 16); }

}  // namespace

extern "C" int pb_transpose(const float* in, float* out, float* out_lo, int32_t rows, int32_t cols, pb_stream_t stream) {
  PB_CHECK_ARG(in && out && rows >= 0 && cols >= 0, "pb_transpose: bad arguments");
  if (rows == 0 || cols == 0) return PB_OK;
  PB_CHECK_ARG((rows + 31) / 32 <= 65535, "pb_transpose: rows %d too large", rows);
  dim3 grid((cols + 31) / 32, (rows + 31) / 32);
  k_transpose32<<<grid, 256, 0, (cudaStream_t)stream>>>(in, out, out_lo, rows, cols);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_colsum(const float* x, float* out, int32_t rows, int32_t cols, int32_t accumulate, pb_stream_t stream) {
  PB_CHECK_ARG(x && out && rows >= 0 && cols > 0, "pb_colsum: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (!accumulate) PB_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * cols, st));
  if (rows == 0) return PB_OK;
  const int gx = (cols + 255) / 256;
  const int chunks = std::max(1, std::min(rows, (pb_sm_count() * 8 + gx - 1) / gx));
  const int rpc = (rows + chunks - 1) / chunks;
  k_colsum_any<<<dim3(gx, (rows + rpc - 1) / rpc), 256, 0, st>>>(x, out, rows, cols, rpc);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_gemv_rows(const float* W, const float* v, float* out, int32_t F, int32_t d, int32_t accumulate, pb_stream_t stream) {
  PB_CHECK_ARG(W && v && out && F >= 0 && d > 0, "pb_gemv_rows: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (!accumulate) PB_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * d, st));
  if (F == 0) return PB_OK;
  const int ctas = std::max(1, std::min(F, pb_sm_count() * 4));
  const int fpc = (F + ctas - 1) / ctas;
  k_gemv_rows<<<(F + fpc - 1) / fpc, 256, 0, st>>>(W, v, out, F, d, fpc);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_sae_dense_stats(const float* acts, int32_t rows, int32_t F, float* fired, float* l1_sum, void* scalars, pb_stream_t stream) {
  PB_CHECK_ARG(acts && fired && l1_sum && scalars && rows >= 0 && F > 0, "pb_sae_dense_stats: bad arguments");
  if (rows == 0) return PB_OK;
  const int gx = (F + 255) / 256;
  const int chunks = std::max(1, std::min(rows, (pb_sm_count() * 8 + gx - 1) / gx));
  const int rpc = (rows + chunks - 1) / chunks;
  k_dense_stats<<<dim3(gx, (rows + rpc - 1) / rpc), 256, 0, (cudaStream_t)stream>>>(acts, rows, F, rpc, fired, l1_sum, (SaeScalars*)scalars);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_sae_dense_loss(const float* x, const float* out_n, const float* mu, const float* sd, const float* xsum, float* sae_out,
                                 float* g, float* resid, void* scalars, int32_t rows, int32_t global_rows, int32_t d, int32_t norm_mode,
                                 pb_stream_t stream) {
  PB_CHECK_ARG(x && out_n && xsum && scalars && rows >= 0 && d > 0, "pb_sae_dense_loss: bad arguments");
  PB_CHECK_ARG(norm_mode == 0 || (mu && sd), "pb_sae_dense_loss: normalised modes need mu / sd");
  if (rows == 0) return PB_OK;
  const float inv_rows = 1.f / (float)(global_rows > 0 ? global_rows : rows);
  k_dense_loss<<<(rows + 7) / 8, 256, 0, (cudaStream_t)stream>>>(x, out_n, mu, sd, xsum, sae_out, g, resid, (SaeScalars*)scalars, rows, d,
                                                                 norm_mode, inv_rows);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_sae_dense_dhid(float* d_acts, const float* acts, float* lo, float l1_grad, int64_t n, pb_stream_t stream) {
  PB_CHECK_ARG(d_acts && acts && n >= 0, "pb_sae_dense_dhid: bad arguments");
  if (n == 0) return PB_OK;
  k_dense_dhid<<<stream_grid(n), 256, 0, (cudaStream_t)stream>>>(d_acts, acts, lo, l1_grad, n);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_sae_ghost_gather(const float* hidden_pre, const int32_t* dead_idx, int32_t nd, int32_t rows, int32_t F, float* E, int32_t ldE,
                                   pb_stream_t stream) {
  PB_CHECK_ARG(hidden_pre && E && (nd == 0 || dead_idx) && nd >= 0 && ldE >= nd && rows >= 0, "pb_sae_ghost_gather: bad arguments");
  const int64_t n = (int64_t)rows * ldE;
  if (n == 0) return PB_OK;
  k_ghost_gather<<<stream_grid(n), 256, 0, (cudaStream_t)stream>>>(hidden_pre, dead_idx, nd, rows, F, E, ldE);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_gather_rows(const float* W, const int32_t* idx, int32_t n, int32_t n_pad, int32_t d, float* out, pb_stream_t stream) {
  PB_CHECK_ARG(W && out && (n == 0 || idx) && n >= 0 && n_pad >= n && d > 0, "pb_gather_rows: bad arguments");
  const int64_t tot = (int64_t)n_pad * d;
  if (tot == 0) return PB_OK;
  k_gather_rows<<<stream_grid(tot), 256, 0, (cudaStream_t)stream>>>(W, idx, n, n_pad, d, out);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_scatter_add_rows(float* dst, const int32_t* idx, int32_t n, int32_t d, const float* src, float scale, pb_stream_t stream) {
  PB_CHECK_ARG(dst && src && (n == 0 || idx) && n >= 0 && d > 0, "pb_scatter_add_rows: bad arguments");
  const int64_t tot = (int64_t)n * d;
  if (tot == 0) return PB_OK;
  k_scatter_add_rows<<<stream_grid(tot), 256, 0, (cudaStream_t)stream>>>(dst, idx, n, d, src, scale);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_mul_inplace(float* y, const float* x, int64_t n, pb_stream_t stream) {
  PB_CHECK_ARG(y && x && n >= 0, "pb_mul_inplace: bad arguments");
  if (n == 0) return PB_OK;
  k_mul_inplace<<<stream_grid(n), 256, 0, (cudaStream_t)stream>>>(y, x, n);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_sae_ghost_rows(const float* resid, const float* rsum, float* G0, const void* scalars, float* ghost_sum, int32_t rows,
                                 int32_t d, pb_stream_t stream) {
  PB_CHECK_ARG(resid && rsum && G0 && scalars && ghost_sum && rows > 0 && d > 0, "pb_sae_ghost_rows: bad arguments");
  k_ghost_rows<<<(rows + 7) / 8, 256, 0, (cudaStream_t)stream>>>(resid, rsum, G0, (const SaeScalars*)scalars, ghost_sum, rows, d,
                                                                 1.f / (float)rows, 1.f / ((float)rows * (float)d));
  PB_LAUNCH_CHECK();
  return PB_OK;
}

// ================================================================================================ Gated SAE (sae/sae.py:648-792)
// The magnitude path shares the encoder matrix: sae_in @ (W_enc * exp(r_mag)) + b_mag = (pi - b_gate) * exp(r_mag) + b_mag with
// pi = sae_in @ W_enc + b_gate, so one encoder GEMM feeds both paths and everything else below is element-wise in [tokens, d_sae].
namespace {

// forward: acts = [pi > 0] * relu(mag_pre), pi_act = relu(pi) (+ tf32 residual planes); column statistics for the step
__global__ void __launch_bounds__(256) k_gated_fwd(const float* __restrict__ pi, const float* __restrict__ b_gate, const float* __restrict__ r_mag,
                                                   const float* __restrict__ b_mag, float* __restrict__ acts, float* __restrict__ acts_lo,
                                                   float* __restrict__ pi_act, float* __restrict__ pi_act_lo, float* __restrict__ fired,
                                                   float* __restrict__ piact_colsum, SaeScalars* __restrict__ sc, int rows, int F, int rows_per_cta) {
  __shared__ float red[8];
  const int f = blockIdx.x * 256 + threadIdx.x;
  float cnt = 0.f;
  if (f < F) {
    const float bg = b_gate[f], er = expf(r_mag[f]), bm = b_mag[f];
    const int r0 = blockIdx.y * rows_per_cta, r1 = min(rows, r0 + rows_per_cta);
    float psum = 0.f;
    for (int r = r0; r < r1; ++r) {
      const int64_t i = (int64_t)r * F + f;
      const float p = pi[i];
      const float mag = fmaf(p - bg, er, bm);
      const float a = (p > 0.f && mag > 0.f) ? mag : 0.f;
      const float pa = fmaxf(p, 0.f);
      acts[i] = a;
      pi_act[i] = pa;
      if (acts_lo) acts_lo[i] = tf32_lo(a);
      if (pi_act_lo) pi_act_lo[i] = tf32_lo(pa);
      cnt += a > 0.f ? 1.f : 0.f;
      psum += pa;
    }
    if (cnt > 0.f) atomicAdd(fired + f, cnt);
    if (psum != 0.f) atomicAdd(piact_colsum + f, psum);
  }
  const float c = warp_sum(cnt);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f;
    for (int i = 0; i < 8; ++i) a += red[i];
    if (a != 0.f) atomicAdd(&sc->pos_count, (unsigned)a);     // a: a whole count below 2^24, exact in fp32
  }
}

// aux reconstruction: ga = 2 (via - sae_in) / rows; *aux_sum += sum (via - sae_in)^2          (sae.py:783-788)
__global__ void __launch_bounds__(256) k_gated_aux(const float* __restrict__ via, const float* __restrict__ sae_in, float* __restrict__ ga,
                                                   float* __restrict__ aux_sum, int64_t n, float scale) {
  __shared__ float red[8];
  float s = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
    const float e = via[i] - sae_in[i];
    ga[i] = e * scale;
    s = fmaf(e, e, s);
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i];
    atomicAdd(aux_sum, t);
  }
}

// backward through both encoder paths.  In: d_acts = g @ W_dec^T, d_pia = ga @ W_dec^T + (added here) l1_grad * ||W_dec[f]||.
// Out (over d_acts): D = d_pi + d_mag * exp(r_mag) = dL/d(sae_in @ W_enc); column sums gb_gate, gb_mag, gr_mag, dsum = colsum(D).
__global__ void __launch_bounds__(256) k_gated_bwd(float* __restrict__ d_acts, float* __restrict__ D_lo, const float* __restrict__ d_pia,
                                                   const float* __restrict__ pi, const float* __restrict__ b_gate, const float* __restrict__ r_mag,
                                                   const float* __restrict__ b_mag, const float* __restrict__ wnorm, float l1_grad,
                                                   float* __restrict__ gb_gate, float* __restrict__ gb_mag, float* __restrict__ gr_mag,
                                                   float* __restrict__ dsum, int rows, int F, int rows_per_cta) {
  const int f = blockIdx.x * 256 + threadIdx.x;
  if (f >= F) return;
  const float bg = b_gate[f], er = expf(r_mag[f]), bm = b_mag[f], l1w = l1_grad * wnorm[f];
  const int r0 = blockIdx.y * rows_per_cta, r1 = min(rows, r0 + rows_per_cta);
  float sg = 0.f, sm = 0.f, sr = 0.f, sD = 0.f;
  for (int r = r0; r < r1; ++r) {
    const int64_t i = (int64_t)r * F + f;
    const float p = pi[i], u = p - bg;
    const float mag = fmaf(u, er, bm);
    const bool on = p > 0.f;
    const float dm = (on && mag > 0.f) ? d_acts[i] : 0.f;     // through [pi > 0] * relu(mag_pre); the Heaviside gate has no gradient
    const float dp = on ? d_pia[i] + l1w : 0.f;               // through relu(pi): aux reconstruction + L1
    const float D = fmaf(dm, er, dp);
    d_acts[i] = D;
    if (D_lo) D_lo[i] = tf32_lo(D);
    sg += dp; sm += dm; sr = fmaf(dm * u, er, sr); sD += D;
  }
  atomicAdd(gb_gate + f, sg);
  atomicAdd(gb_mag + f, sm);
  atomicAdd(gr_mag + f, sr);
  atomicAdd(dsum + f, sD);
}

// out[f] = ||W[f,:]||
__global__ void __launch_bounds__(256) k_row_norms(const float* __restrict__ W, float* __restrict__ out, int F, int d) {
  const int lane = threadIdx.x & 31;
  const int f = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (f >= F) return;
  float s = 0.f;
  for (int c = lane; c < d; c += 32) { const float w = W[(int64_t)f * d + c]; s = fmaf(w, w, s); }
  s = warp_sum(s);
  if (lane == 0) out[f] = sqrtf(s);
}

// L1 term of the Gated SAE: l1 = coeff * mean_b sum_f pi_act[b,f] ||W_dec[f]|| (sae.py:776-781, W_dec.norm is part of the graph):
// gW_dec[f,:] += l1_grad * colsum(pi_act)[f] * W_dec[f,:] / ||W_dec[f]|| ;  *l1_sum += colsum(pi_act)[f] * ||W_dec[f]||
__global__ void __launch_bounds__(256) k_gated_l1_rows(float* __restrict__ gW_dec, const float* __restrict__ W_dec, const float* __restrict__ piact_colsum,
                                                       const float* __restrict__ wnorm, float l1_grad, float* __restrict__ l1_sum, int F, int d) {
  const int lane = threadIdx.x & 31;
  const int f = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (f >= F) return;
  const float cs = piact_colsum[f], wn = wnorm[f];
  const float coef = l1_grad * cs / wn;
  for (int c = lane; c < d; c += 32) gW_dec[(int64_t)f * d + c] = fmaf(coef, W_dec[(int64_t)f * d + c], gW_dec[(int64_t)f * d + c]);
  if (lane == 0 && cs != 0.f) atomicAdd(l1_sum, cs * wn);
}

inline void col_grid(int rows, int F, dim3& grid, int& rpc) {
  const int gx = (F + 255) / 256;
  const int chunks = std::max(1, std::min(rows, (pb_sm_count() * 8 + gx - 1) / gx));
  rpc = (rows + chunks - 1) / chunks;
  grid = dim3(gx, (rows + rpc - 1) / rpc);
}

}  // namespace

extern "C" int pb_gated_fwd(const float* pi, const float* b_gate, const float* r_mag, const float* b_mag, float* acts, float* acts_lo,
                            float* pi_act, float* pi_act_lo, float* fired, float* piact_colsum, void* scalars, int32_t rows, int32_t F,
                            pb_stream_t stream) {
  PB_CHECK_ARG(pi && b_gate && r_mag && b_mag && acts && pi_act && fired && piact_colsum && scalars && rows >= 0 && F > 0,
               "pb_gated_fwd: bad arguments");
  if (rows == 0) return PB_OK;
  dim3 grid; int rpc;
  col_grid(rows, F, grid, rpc);
  k_gated_fwd<<<grid, 256, 0, (cudaStream_t)stream>>>(pi, b_gate, r_mag, b_mag, acts, acts_lo, pi_act, pi_act_lo, fired, piact_colsum,
                                                      (SaeScalars*)scalars, rows, F, rpc);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_gated_aux(const float* via, const float* sae_in, float* ga, float* aux_sum, int32_t rows, int32_t d, pb_stream_t stream) {
  PB_CHECK_ARG(via && sae_in && ga && aux_sum && rows > 0 && d > 0, "pb_gated_aux: bad arguments");
  const int64_t n = (int64_t)rows * d;
  k_gated_aux<<<stream_grid(n), 256, 0, (cudaStream_t)stream>>>(via, sae_in, ga, aux_sum, n, 2.f / (float)rows);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_gated_bwd(float* d_acts, float* D_lo, const float* d_pia, const float* pi, const float* b_gate, const float* r_mag,
                            const float* b_mag, const float* wnorm, float l1_grad, float* gb_gate, float* gb_mag, float* gr_mag, float* dsum,
                            int32_t rows, int32_t F, pb_stream_t stream) {
  PB_CHECK_ARG(d_acts && d_pia && pi && b_gate && r_mag && b_mag && wnorm && gb_gate && gb_mag && gr_mag && dsum && rows >= 0 && F > 0,
               "pb_gated_bwd: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  PB_CUDA(cudaMemsetAsync(gb_gate, 0, sizeof(float) * F, st));
  PB_CUDA(cudaMemsetAsync(gb_mag, 0, sizeof(float) * F, st));
  PB_CUDA(cudaMemsetAsync(gr_mag, 0, sizeof(float) * F, st));
  PB_CUDA(cudaMemsetAsync(dsum, 0, sizeof(float) * F, st));
  if (rows == 0) return PB_OK;
  dim3 grid; int rpc;
  col_grid(rows, F, grid, rpc);
  k_gated_bwd<<<grid, 256, 0, st>>>(d_acts, D_lo, d_pia, pi, b_gate, r_mag, b_mag, wnorm, l1_grad, gb_gate, gb_mag, gr_mag, dsum, rows, F, rpc);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_row_norms(const float* W, float* out, int32_t F, int32_t d, pb_stream_t stream) {
  PB_CHECK_ARG(W && out && F >= 0 && d > 0, "pb_row_norms: bad arguments");
  if (F == 0) return PB_OK;
  k_row_norms<<<(F + 7) / 8, 256, 0, (cudaStream_t)stream>>>(W, out, F, d);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_gated_l1_rows(float* gW_dec, const float* W_dec, const float* piact_colsum, const float* wnorm, float l1_grad, float* l1_sum,
                                int32_t F, int32_t d, pb_stream_t stream) {
  PB_CHECK_ARG(gW_dec && W_dec && piact_colsum && wnorm && l1_sum && F >= 0 && d > 0, "pb_gated_l1_rows: bad arguments");
  if (F == 0) return PB_OK;
  k_gated_l1_rows<<<(F + 7) / 8, 256, 0, (cudaStream_t)stream>>>(gW_dec, W_dec, piact_colsum, wnorm, l1_grad, l1_sum, F, d);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_sumsq(const float* a, int64_t n, float* acc, pb_stream_t stream) {
  PB_CHECK_ARG(a && acc && n >= 0, "pb_sumsq: bad arguments");
  if (n == 0) return PB_OK;
  k_sumsq<<<stream_grid(n), 256, 0, (cudaStream_t)stream>>>(a, n, acc);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_sae_clip_finish(void* scalars, float max_grad_norm, int32_t rows, int32_t d, pb_stream_t stream) {
  PB_CHECK_ARG(scalars && rows > 0 && d > 0, "pb_sae_clip_finish: bad arguments");
  k_grad_finish<<<1, 1, 0, (cudaStream_t)stream>>>((SaeScalars*)scalars, max_grad_norm, 1.f / ((float)rows * (float)d), 1.f / (float)rows);
  PB_LAUNCH_CHECK();
  return PB_OK;
}
