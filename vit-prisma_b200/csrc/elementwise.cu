// elementwise.cu -- HBM-bound glue kernels of the hooked ViT path.
//
// All of these are pure streaming kernels (1 read + 1 write per element or close to it):
// the rule is 16-byte vector accesses, grid sized to a multiple of the SM count, grid-stride
// loops.  Reference call sites are cited at each entry point.
#include "common.cuh"
#include <stdlib.h>
#include <stdarg.h>

// ------------------------------------------------------------------ library
static thread_local char g_err[512] = "";
void pb_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
extern "C" const char* pb_last_error(void) { return g_err; }
extern "C" int pb_version(void) { return 100; }
unsigned long long g_pb_launches = 0;
extern "C" unsigned long long pb_launch_count(void) { return g_pb_launches; }

bool pb_pdl_enabled() {
  static int on = -1;
  if (on < 0) { const char* e = getenv("PB_PDL"); on = (e && e[0] == '0') ? 0 : 1; }
  return on == 1;
}

int pb_sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

extern "C" int pb_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0, n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    pb_set_error("no CUDA device visible: libprisma_b200 has no CPU path");
    return PB_ENODEVICE;
  }
  PB_CUDA(cudaGetDevice(&dev));
  if (sm_count) PB_CUDA(cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, dev));
  if (cc_major) PB_CUDA(cudaDeviceGetAttribute(cc_major, cudaDevAttrComputeCapabilityMajor, dev));
  if (cc_minor) PB_CUDA(cudaDeviceGetAttribute(cc_minor, cudaDevAttrComputeCapabilityMinor, dev));
  return PB_OK;
}

static inline int stream_grid(int64_t work_items, int threads) {
  int64_t blocks = ceil_div64(work_items, threads);
  int64_t cap = (int64_t)pb_sm_count() * 8;  // 8 resident CTAs of 256 threads per SM
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

// ----------------------------------------------------------- binary / unary
enum { OP_ADD = 0, OP_MUL = 1 };

template <typename T, int OP>
__global__ void __launch_bounds__(256) k_binary(const T* __restrict__ a, const T* __restrict__ b,
                                                T* __restrict__ out, int64_t n) {
  const int64_t n4 = n >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float x[4], y[4], r[4];
    ld4(a + 4 * i, x);
    ld4(b + 4 * i, y);
#pragma unroll
    for (int j = 0; j < 4; ++j) r[j] = OP == OP_ADD ? x[j] + y[j] : x[j] * y[j];
    st4(out + 4 * i, r);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    int64_t i = (n4 << 2) + threadIdx.x;
    float x = ld_as_float(a + i), y = ld_as_float(b + i);
    st_from_float(out + i, OP == OP_ADD ? x + y : x * y);
  }
}

template <int OP>
static int launch_binary(const void* a, const void* b, void* out, int64_t n, int32_t dtype, pb_stream_t s) {
  PB_CHECK_ARG(a && b && out && n >= 0, "pb_add/pb_mul: null pointer or negative size");
  if (n == 0) return PB_OK;
  PB_CHECK_ARG((((uintptr_t)a | (uintptr_t)b | (uintptr_t)out) & 15) == 0, "pb_add/pb_mul: pointers must be 16B aligned");
  int grid = stream_grid(n / 4 + 1, 256);
  if (dtype == PB_F32)
    k_binary<float, OP><<<grid, 256, 0, (cudaStream_t)s>>>((const float*)a, (const float*)b, (float*)out, n);
  else if (dtype == PB_BF16)
    k_binary<bf16, OP><<<grid, 256, 0, (cudaStream_t)s>>>((const bf16*)a, (const bf16*)b, (bf16*)out, n);
  else
    PB_CHECK_ARG(false, "pb_add/pb_mul: unknown dtype %d", dtype);
  PB_LAUNCH_CHECK();
  return PB_OK;
}
// residual adds: models/layers/transformer_block.py:121-134, models/base_vit.py:179
extern "C" int pb_add(const void* a, const void* b, void* out, int64_t n, int32_t dtype, pb_stream_t s) {
  return launch_binary<OP_ADD>(a, b, out, n, dtype, s);
}
// solu(x) = x * softmax(x): models/activation_fns.py:50-57
extern "C" int pb_mul(const void* a, const void* b, void* out, int64_t n, int32_t dtype, pb_stream_t s) {
  return launch_binary<OP_MUL>(a, b, out, n, dtype, s);
}

template <typename T>
__global__ void __launch_bounds__(256) k_act(const T* __restrict__ x, T* __restrict__ y, int64_t n, int act) {
  const int64_t n4 = n >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float v[4];
    ld4(x + 4 * i, v);
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = apply_act(v[j], act);
    st4(y + 4 * i, v);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    int64_t i = (n4 << 2) + threadIdx.x;
    st_from_float(y + i, apply_act(ld_as_float(x + i), act));
  }
}
// MLP activation on the hooked path: models/layers/mlp.py:71-75
extern "C" int pb_activation(const void* x, void* y, int64_t n, int32_t act, int32_t dtype, pb_stream_t s) {
  PB_CHECK_ARG(x && y && n >= 0, "pb_activation: null pointer or negative size");
  if (n == 0) return PB_OK;
  PB_CHECK_ARG((((uintptr_t)x | (uintptr_t)y) & 15) == 0, "pb_activation: pointers must be 16B aligned");
  int grid = stream_grid(n / 4 + 1, 256);
  if (dtype == PB_F32)
    k_act<float><<<grid, 256, 0, (cudaStream_t)s>>>((const float*)x, (float*)y, n, act);
  else if (dtype == PB_BF16)
    k_act<bf16><<<grid, 256, 0, (cudaStream_t)s>>>((const bf16*)x, (bf16*)y, n, act);
  else
    PB_CHECK_ARG(false, "pb_activation: unknown dtype %d", dtype);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

// --------------------------------------------------------------------- cast
template <typename TI, typename TO>
__global__ void __launch_bounds__(256) k_cast(const TI* __restrict__ x, TO* __restrict__ y, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    st_from_float(y + i, ld_as_float(x + i));
}
// fp32 <-> bf16, eight elements per thread and trip (two 16-byte loads / one 16-byte store, or the reverse)
__global__ void __launch_bounds__(256) k_cast_f32_bf16_v8(const float4* __restrict__ x, uint4* __restrict__ y, int64_t n8) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += stride) {
    const float4 a = x[2 * i], b = x[2 * i + 1];
    __nv_bfloat162 p0 = __floats2bfloat162_rn(a.x, a.y), p1 = __floats2bfloat162_rn(a.z, a.w);
    __nv_bfloat162 p2 = __floats2bfloat162_rn(b.x, b.y), p3 = __floats2bfloat162_rn(b.z, b.w);
    uint4 o;
    o.x = *reinterpret_cast<uint32_t*>(&p0); o.y = *reinterpret_cast<uint32_t*>(&p1);
    o.z = *reinterpret_cast<uint32_t*>(&p2); o.w = *reinterpret_cast<uint32_t*>(&p3);
    y[i] = o;
  }
}
__global__ void __launch_bounds__(256) k_cast_bf16_f32_v8(const uint4* __restrict__ x, float4* __restrict__ y, int64_t n8) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += stride) {
    const uint4 v = x[i];
    y[2 * i] = make_float4(__uint_as_float(v.x << 16), __uint_as_float(v.x & 0xffff0000u), __uint_as_float(v.y << 16), __uint_as_float(v.y & 0xffff0000u));
    y[2 * i + 1] = make_float4(__uint_as_float(v.z << 16), __uint_as_float(v.z & 0xffff0000u), __uint_as_float(v.w << 16), __uint_as_float(v.w & 0xffff0000u));
  }
}
extern "C" int pb_cast(const void* x, int32_t dtype_in, void* y, int32_t dtype_out, int64_t n, pb_stream_t s) {
  PB_CHECK_ARG(x && y && n >= 0, "pb_cast: null pointer or negative size");
  if (n == 0) return PB_OK;
  int grid = stream_grid(n, 256);
  cudaStream_t st = (cudaStream_t)s;
  const bool vec8 = n % 8 == 0 && n >= 4096 && (((uintptr_t)x | (uintptr_t)y) & 15) == 0;
  if (vec8 && dtype_in == PB_F32 && dtype_out == PB_BF16)
    k_cast_f32_bf16_v8<<<stream_grid(n / 8, 256), 256, 0, st>>>((const float4*)x, (uint4*)y, n / 8);
  else if (vec8 && dtype_in == PB_BF16 && dtype_out == PB_F32)
    k_cast_bf16_f32_v8<<<stream_grid(n / 8, 256), 256, 0, st>>>((const uint4*)x, (float4*)y, n / 8);
  else if (dtype_in == PB_F32 && dtype_out == PB_BF16) k_cast<float, bf16><<<grid, 256, 0, st>>>((const float*)x, (bf16*)y, n);
  else if (dtype_in == PB_BF16 && dtype_out == PB_F32) k_cast<bf16, float><<<grid, 256, 0, st>>>((const bf16*)x, (float*)y, n);
  else if (dtype_in == PB_F32 && dtype_out == PB_F32) k_cast<float, float><<<grid, 256, 0, st>>>((const float*)x, (float*)y, n);
  else if (dtype_in == PB_BF16 && dtype_out == PB_BF16) k_cast<bf16, bf16><<<grid, 256, 0, st>>>((const bf16*)x, (bf16*)y, n);
  else PB_CHECK_ARG(false, "pb_cast: unknown dtype pair %d -> %d", dtype_in, dtype_out);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

// --------------------------------------------------------------- tf32 split
__global__ void __launch_bounds__(256) k_split_tf32(const float* __restrict__ x, float* __restrict__ lo, int64_t n) {
  const int64_t n4 = n >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 v = reinterpret_cast<const float4*>(x)[i];
    float4 r = make_float4(tf32_lo(v.x), tf32_lo(v.y), tf32_lo(v.z), tf32_lo(v.w));
    reinterpret_cast<float4*>(lo)[i] = r;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    int64_t i = (n4 << 2) + threadIdx.x;
    lo[i] = tf32_lo(x[i]);
  }
}
extern "C" int pb_split_tf32(const float* x, float* lo, int64_t n, pb_stream_t s) {
  PB_CHECK_ARG(x && lo && n >= 0, "pb_split_tf32: null pointer or negative size");
  if (n == 0) return PB_OK;
  PB_CHECK_ARG((((uintptr_t)x | (uintptr_t)lo) & 15) == 0, "pb_split_tf32: pointers must be 16B aligned");
  k_split_tf32<<<stream_grid(n / 4 + 1, 256), 256, 0, (cudaStream_t)s>>>(x, lo, n);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

// ------------------------------------------------------------- L2 normalise
// one warp per row; F.normalize(x, dim=-1): x / max(||x||_2, eps)
template <typename T>
__global__ void __launch_bounds__(256) k_l2norm(const T* __restrict__ x, T* __restrict__ out, int64_t rows, int cols, float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const T* xr = x + row * cols;
  float ss = 0.f;
  for (int c = lane; c < cols; c += 32) { float v = ld_as_float(xr + c); ss += v * v; }
  ss = warp_sum(ss);
  // torch computes the norm in the tensor dtype: round it the same way for bf16
  float denom = fmaxf(round_to<T>(sqrtf(ss)), eps);
  T* orow = out + row * cols;
  for (int c = lane; c < cols; c += 32) st_from_float(orow + c, ld_as_float(xr + c) / denom);
}
extern "C" int pb_l2_normalize_rows(const void* x, void* out, int64_t rows, int32_t cols, float eps, int32_t dtype, pb_stream_t s) {
  PB_CHECK_ARG(x && out && rows >= 0 && cols > 0, "pb_l2_normalize_rows: bad arguments");
  if (rows == 0) return PB_OK;
  int grid = (int)ceil_div64(rows, 8);
  if (dtype == PB_F32) k_l2norm<float><<<grid, 256, 0, (cudaStream_t)s>>>((const float*)x, (float*)out, rows, cols, eps);
  else if (dtype == PB_BF16) k_l2norm<bf16><<<grid, 256, 0, (cudaStream_t)s>>>((const bf16*)x, (bf16*)out, rows, cols, eps);
  else PB_CHECK_ARG(false, "pb_l2_normalize_rows: unknown dtype %d", dtype);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

// -------------------------------------------------------------- token mean
template <typename T>
__global__ void __launch_bounds__(256) k_mean_tokens(const T* __restrict__ x, T* __restrict__ out, int B, int Tn, int d) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)B * d) return;
  const int b = (int)(idx / d), c = (int)(idx % d);
  float acc = 0.f;
  for (int t = 0; t < Tn; ++t) acc += ld_as_float(x + ((int64_t)b * Tn + t) * d + c);
  st_from_float(out + idx, acc / (float)Tn);
}
extern "C" int pb_mean_tokens(const void* x, void* out, int32_t B, int32_t Tn, int32_t d, int32_t dtype, pb_stream_t s) {
  PB_CHECK_ARG(x && out && B >= 0 && Tn > 0 && d > 0, "pb_mean_tokens: bad arguments");
  if (B == 0) return PB_OK;
  int grid = (int)ceil_div64((int64_t)B * d, 256);
  if (dtype == PB_F32) k_mean_tokens<float><<<grid, 256, 0, (cudaStream_t)s>>>((const float*)x, (float*)out, B, Tn, d);
  else if (dtype == PB_BF16) k_mean_tokens<bf16><<<grid, 256, 0, (cudaStream_t)s>>>((const bf16*)x, (bf16*)out, B, Tn, d);
  else PB_CHECK_ARG(false, "pb_mean_tokens: unknown dtype %d", dtype);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

// ------------------------------------------------------------------ im2col
// Tubelets of D frames x P x P pixels (nt = F / D tubelets in time, g = S / P patches per side); images are F = D = 1:
//   patches[((b*nt + t)*g + py)*g + px, ((c*D + dt)*P + i)*P + j] = x[b, c, t*D + dt, py*P + i, px*P + j]
// Frames past nt*D are not read, as Conv3d with stride D drops them.
// One thread moves VEC contiguous pixels of one patch row (j..j+VEC-1): reads and writes are both
// contiguous runs of P elements, so with P % 4 == 0 every access is a 16 B (fp32) / 8 B (bf16) vector.
template <typename T, int VEC>
__global__ void __launch_bounds__(256) k_im2col(const T* __restrict__ img, T* __restrict__ out, int B, int C, int F, int S, int P, int D) {
  const int g = S / P, nt = F / D;
  const int pv = P / VEC;                                          // vectors per patch row
  const int64_t total = (int64_t)B * nt * g * g * C * D * P * pv;  // one item = one vector
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < total; it += stride) {
    int64_t r = it;
    const int jv = (int)(r % pv); r /= pv;
    const int i = (int)(r % P);   r /= P;
    const int dt = (int)(r % D);  r /= D;
    const int c = (int)(r % C);   r /= C;
    const int px = (int)(r % g);  r /= g;
    const int py = (int)(r % g);  r /= g;
    const int t = (int)(r % nt);  r /= nt;
    const int b = (int)r;
    const T* src = img + ((((int64_t)b * C + c) * F + (t * D + dt)) * S + (py * P + i)) * S + px * P + jv * VEC;
    T* dst = out + ((((int64_t)b * nt + t) * g + py) * g + px) * ((int64_t)C * D * P * P) + (((int64_t)c * D + dt) * P + i) * P + jv * VEC;
    if (VEC == 4) {
      float v[4];
      ld4(src, v);
      st4(dst, v);
    } else {
      *dst = *src;
    }
  }
}
static int launch_im2col(const void* images, void* patches, int B, int C, int F, int S, int P, int D, int dtype, pb_stream_t s) {
  if (B == 0) return PB_OK;
  const bool vec = (P % 4 == 0) && (S % 4 == 0) && (((uintptr_t)images | (uintptr_t)patches) & 15) == 0;
  const int g = S / P;
  int64_t items = (int64_t)B * (F / D) * g * g * C * D * P * (vec ? P / 4 : P);
  int grid = stream_grid(items, 256);
  cudaStream_t st = (cudaStream_t)s;
  if (dtype == PB_F32) {
    if (vec) k_im2col<float, 4><<<grid, 256, 0, st>>>((const float*)images, (float*)patches, B, C, F, S, P, D);
    else k_im2col<float, 1><<<grid, 256, 0, st>>>((const float*)images, (float*)patches, B, C, F, S, P, D);
  } else if (dtype == PB_BF16) {
    if (vec) k_im2col<bf16, 4><<<grid, 256, 0, st>>>((const bf16*)images, (bf16*)patches, B, C, F, S, P, D);
    else k_im2col<bf16, 1><<<grid, 256, 0, st>>>((const bf16*)images, (bf16*)patches, B, C, F, S, P, D);
  } else PB_CHECK_ARG(false, "pb_im2col: unknown dtype %d", dtype);
  PB_LAUNCH_CHECK();
  return PB_OK;
}
extern "C" int pb_im2col_patches(const void* images, void* patches, int32_t B, int32_t C, int32_t S, int32_t P, int32_t dtype, pb_stream_t s) {
  PB_CHECK_ARG(images && patches && B >= 0 && C > 0 && S > 0 && P > 0 && S % P == 0, "pb_im2col_patches: bad geometry (S=%d P=%d)", S, P);
  return launch_im2col(images, patches, B, C, 1, S, P, 1, dtype, s);
}
// video tubelets (reference models/layers/patch_embedding.py:36-62, Conv3d with kernel = stride = (D, P, P))
extern "C" int pb_im2col_tubelets(const void* images, void* patches, int32_t B, int32_t C, int32_t F, int32_t S, int32_t P, int32_t D,
                                  int32_t dtype, pb_stream_t s) {
  PB_CHECK_ARG(images && patches && B >= 0 && C > 0 && S > 0 && P > 0 && S % P == 0 && D > 0 && F >= D,
               "pb_im2col_tubelets: bad geometry (F=%d D=%d S=%d P=%d)", F, D, S, P);
  return launch_im2col(images, patches, B, C, F, S, P, D, dtype, s);
}

// ---------------------------------------------------------- embed assemble
template <typename T>
__global__ void __launch_bounds__(256) k_embed_assemble(const T* __restrict__ embed, const T* __restrict__ cls, const T* __restrict__ pos,
                                                        T* __restrict__ full, int B, int np, int d, int use_cls) {
  const int Tn = np + (use_cls ? 1 : 0);
  const int d4 = d >> 2;  // host guarantees d % 4 == 0 on this path
  const int64_t total = (int64_t)B * Tn * d4;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < total; it += stride) {
    const int c4 = (int)(it % d4);
    const int64_t bt = it / d4;
    const int t = (int)(bt % Tn);
    const int b = (int)(bt / Tn);
    float a[4], p[4], r[4];
    ld4(pos + (int64_t)t * d + 4 * c4, p);
    if (use_cls && t == 0) ld4(cls + 4 * c4, a);
    else ld4(embed + ((int64_t)b * np + (t - (use_cls ? 1 : 0))) * d + 4 * c4, a);
#pragma unroll
    for (int j = 0; j < 4; ++j) r[j] = a[j] + p[j];
    st4(full + bt * d + 4 * c4, r);
  }
}
template <typename T>
__global__ void __launch_bounds__(256) k_embed_assemble_scalar(const T* __restrict__ embed, const T* __restrict__ cls, const T* __restrict__ pos,
                                                               T* __restrict__ full, int B, int np, int d, int use_cls) {
  const int Tn = np + (use_cls ? 1 : 0);
  const int64_t total = (int64_t)B * Tn * d;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < total; it += stride) {
    const int c = (int)(it % d);
    const int64_t bt = it / d;
    const int t = (int)(bt % Tn);
    const int b = (int)(bt / Tn);
    float a = (use_cls && t == 0) ? ld_as_float(cls + c) : ld_as_float(embed + ((int64_t)b * np + (t - (use_cls ? 1 : 0))) * d + c);
    st_from_float(full + it, a + ld_as_float(pos + (int64_t)t * d + c));
  }
}
extern "C" int pb_embed_assemble(const void* embed, const void* cls, const void* pos, void* full, int32_t B, int32_t np, int32_t d,
                                 int32_t use_cls, int32_t dtype, pb_stream_t s) {
  PB_CHECK_ARG(embed && pos && full && (cls || !use_cls) && B >= 0 && np > 0 && d > 0, "pb_embed_assemble: bad arguments");
  if (B == 0) return PB_OK;
  const int Tn = np + (use_cls ? 1 : 0);
  const bool vec = (d % 4 == 0) && (((uintptr_t)embed | (uintptr_t)pos | (uintptr_t)full | (uintptr_t)cls) & 15) == 0;
  int grid = stream_grid((int64_t)B * Tn * (vec ? d / 4 : d), 256);
  cudaStream_t st = (cudaStream_t)s;
#define PB_EA(T)                                                                                                        \
  if (vec) k_embed_assemble<T><<<grid, 256, 0, st>>>((const T*)embed, (const T*)cls, (const T*)pos, (T*)full, B, np, d, use_cls); \
  else k_embed_assemble_scalar<T><<<grid, 256, 0, st>>>((const T*)embed, (const T*)cls, (const T*)pos, (T*)full, B, np, d, use_cls)
  if (dtype == PB_F32) { PB_EA(float); }
  else if (dtype == PB_BF16) { PB_EA(bf16); }
  else PB_CHECK_ARG(false, "pb_embed_assemble: unknown dtype %d", dtype);
#undef PB_EA
  PB_LAUNCH_CHECK();
  return PB_OK;
}

// ------------------------------------------------------------- text towers
// embed[b,t,:] = W_E[ids[b,t],:]  (nn.Embedding, base_text_transformer.py:125)
// full[b,t,:]  = round(embed[b,t,:] + pos[t,:])  (:139-141; pos is pos_embed[:T], broadcast over the batch)
// One 16-byte vector per thread and step.  Ids outside [0, vocab) are never dereferenced: their rows are filled with NaN
// (the host checks the range and raises before any launch, as nn.Embedding raises).
template <typename T, int VEC>
__global__ void __launch_bounds__(256) k_embed_tokens(const int64_t* __restrict__ ids, const T* __restrict__ W_E, const T* __restrict__ pos,
                                                      T* __restrict__ embed, T* __restrict__ full, int Tn, int d, int vocab, int64_t total) {
  const int nv = d / VEC;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < total; it += stride) {
    const int c = (int)(it % nv) * VEC;
    const int64_t bt = it / nv;
    const int t = (int)(bt % Tn);
    const int64_t id = ids[bt];
    T e[VEC], f[VEC];
    if (id >= 0 && id < vocab) {
      if constexpr (VEC * sizeof(T) == 16) {
        *reinterpret_cast<uint4*>(e) = *reinterpret_cast<const uint4*>(W_E + id * d + c);
        uint4 pu = *reinterpret_cast<const uint4*>(pos + (int64_t)t * d + c);
        const T* p = reinterpret_cast<const T*>(&pu);
#pragma unroll
        for (int j = 0; j < VEC; ++j) st_from_float(f + j, ld_as_float(e + j) + ld_as_float(p + j));
      } else {
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          e[j] = W_E[id * d + c + j];
          st_from_float(f + j, ld_as_float(e + j) + ld_as_float(pos + (int64_t)t * d + c + j));
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < VEC; ++j) { st_from_float(e + j, __int_as_float(0x7fc00000)); f[j] = e[j]; }
    }
    if constexpr (VEC * sizeof(T) == 16) {
      *reinterpret_cast<uint4*>(embed + bt * d + c) = *reinterpret_cast<const uint4*>(e);
      *reinterpret_cast<uint4*>(full + bt * d + c) = *reinterpret_cast<const uint4*>(f);
    } else {
#pragma unroll
      for (int j = 0; j < VEC; ++j) { embed[bt * d + c + j] = e[j]; full[bt * d + c + j] = f[j]; }
    }
  }
}
extern "C" int pb_embed_tokens(const int64_t* ids, const void* W_E, const void* pos, void* embed, void* full, int32_t B, int32_t T,
                               int32_t d, int32_t vocab, int32_t dtype, pb_stream_t s) {
  PB_CHECK_ARG(ids && W_E && pos && embed && full && B >= 0 && T > 0 && d > 0 && vocab > 0, "pb_embed_tokens: bad arguments");
  PB_CHECK_ARG(dtype == PB_F32 || dtype == PB_BF16, "pb_embed_tokens: unknown dtype %d", dtype);
  if (B == 0) return PB_OK;
  const int es = dtype == PB_F32 ? 4 : 2;
  const bool vec = ((int64_t)d * es) % 16 == 0 && (((uintptr_t)W_E | (uintptr_t)pos | (uintptr_t)embed | (uintptr_t)full) & 15) == 0;
  const int VEC = vec ? 16 / es : 1;
  const int64_t total = (int64_t)B * T * (d / VEC);
  const int grid = stream_grid(total, 256);
  cudaStream_t st = (cudaStream_t)s;
  if (dtype == PB_F32) {
    if (vec) k_embed_tokens<float, 4><<<grid, 256, 0, st>>>(ids, (const float*)W_E, (const float*)pos, (float*)embed, (float*)full, T, d, vocab, total);
    else k_embed_tokens<float, 1><<<grid, 256, 0, st>>>(ids, (const float*)W_E, (const float*)pos, (float*)embed, (float*)full, T, d, vocab, total);
  } else {
    if (vec) k_embed_tokens<bf16, 8><<<grid, 256, 0, st>>>(ids, (const bf16*)W_E, (const bf16*)pos, (bf16*)embed, (bf16*)full, T, d, vocab, total);
    else k_embed_tokens<bf16, 1><<<grid, 256, 0, st>>>(ids, (const bf16*)W_E, (const bf16*)pos, (bf16*)embed, (bf16*)full, T, d, vocab, total);
  }
  PB_LAUNCH_CHECK();
  return PB_OK;
}

// out[b,:] = x[b, argmax_t ids[b,t], :] with the first maximal index on ties, as torch.argmax
// (base_text_transformer.py:151: x[arange(B), input.argmax(-1)]).  One CTA per batch row: a block argmax, then a row copy.
template <typename T>
__global__ void __launch_bounds__(256) k_gather_argmax_rows(const int64_t* __restrict__ ids, const T* __restrict__ x, T* __restrict__ out,
                                                            int Tn, int d) {
  __shared__ int64_t s_val[8];
  __shared__ int s_idx[8];
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t* row = ids + (int64_t)b * Tn;
  int64_t best = INT64_MIN;
  int bi = INT32_MAX;
  for (int t = threadIdx.x; t < Tn; t += blockDim.x) {
    const int64_t v = row[t];
    if (v > best) { best = v; bi = t; }                     // strided ascending t: first maximum of this thread's share
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const int64_t ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if (lane == 0) { s_val[warp] = best; s_idx[warp] = bi; }
  __syncthreads();
  best = s_val[0]; bi = s_idx[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
    if (s_val[w] > best || (s_val[w] == best && s_idx[w] < bi)) { best = s_val[w]; bi = s_idx[w]; }
  const T* src = x + ((int64_t)b * Tn + bi) * d;
  T* dst = out + (int64_t)b * d;
  for (int c = threadIdx.x; c < d; c += blockDim.x) dst[c] = src[c];
}
extern "C" int pb_gather_argmax_rows(const int64_t* ids, const void* x, void* out, int32_t B, int32_t T, int32_t d, int32_t dtype,
                                     pb_stream_t s) {
  PB_CHECK_ARG(ids && x && out && B >= 0 && T > 0 && d > 0, "pb_gather_argmax_rows: bad arguments");
  if (B == 0) return PB_OK;
  cudaStream_t st = (cudaStream_t)s;
  if (dtype == PB_F32) k_gather_argmax_rows<float><<<B, 256, 0, st>>>(ids, (const float*)x, (float*)out, T, d);
  else if (dtype == PB_BF16) k_gather_argmax_rows<bf16><<<B, 256, 0, st>>>(ids, (const bf16*)x, (bf16*)out, T, d);
  else PB_CHECK_ARG(false, "pb_gather_argmax_rows: unknown dtype %d", dtype);
  PB_LAUNCH_CHECK();
  return PB_OK;
}
