// attention.cu -- hooked attention core (reference models/layers/attention.py:126-184, 246-281).
//
//   scores[b,h,i,j] = <q[b,i,h,:], k[b,j,h,:]> / attn_scale      -> hook_attn_scores
//   pattern         = softmax_j(scores), NaN -> 0                 -> hook_pattern
//   z[b,i,h,:]      = sum_j pattern[b,h,i,j] v[b,j,h,:]           -> hook_z
//
// Both [B,H,T,T] tensors are hook points, so when they are requested this op is bound by the HBM
// write of 2*B*H*T*T elements plus the q/k/v read and the z write (algorithmic bytes in DESIGN.md);
// flash-style non-materialisation is what happens automatically when scores/pattern are NULL.
// Tokens per image are small (50 / 197 / 257), so one CTA keeps a whole head's K (transposed) and V
// in shared memory and each warp walks 4 query rows at a time with register tiles:
//   QK^T : lane owns keys {lane, lane+32, ...}; per feature e one LDS.128 broadcast of the 4 q values
//          + KPL conflict-free LDS of K^T  -> 4*KPL FMAs
//   PV   : lane owns features {lane, lane+32, ...}; per key one LDS.128 broadcast of 4 probabilities
//          + EPL conflict-free LDS of V    -> 4*EPL FMAs
// Arithmetic is fp32; in bf16 mode values are rounded to bf16 exactly where the reference
// materialises a bf16 tensor (scores, pattern, z).
#include "common.cuh"

// the d_head == 64 tensor-core kernels; callers guarantee d_head == 64 and 16-byte aligned operands
int pb_attention_mma(const PbAttention* p, cudaStream_t st);     // attention_mma.cu: T <= 128
int pb_attention_long(const PbAttention* p, cudaStream_t st);    // attention_long.cu: any T
int pb_attn_scores_long(const PbAttention* p, cudaStream_t st);
int pb_attn_pv_long(const PbAttention* p, cudaStream_t st);

// every pointer 16-byte aligned: the tensor-core kernels move head rows in 16-byte vectors
template <typename... P> static bool aligned16(const P*... p) { return !((reinterpret_cast<uintptr_t>(p) | ...) & 15); }

enum { ATT_FUSED = 0, ATT_SCORES = 1, ATT_PV = 2 };

// CAUSAL (ATT_FUSED only): keys j > query i score -inf, as scores / scale + mask does; they drop out of the max and get e = 0
template <typename T, int KPL, int EPL, int MODE, bool CAUSAL>
__global__ void __launch_bounds__(256) k_attention(const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v,
                                                   T* __restrict__ scores, T* __restrict__ pattern, T* __restrict__ z, int B, int Tn,
                                                   int H, int dh, float attn_scale, int rows_per_cta) {
  constexpr int TP = KPL * 32;   // padded key count
  constexpr int TPS = TP + 1;    // K^T row stride (odd -> conflict-free transposed stores)
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int nwarps = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x / H, h = blockIdx.x % H;
  const int row0 = blockIdx.y * rows_per_cta;
  const int row_end = min(Tn, row0 + rows_per_cta);

  // carve: [q4: nwarps*dh float4][p4: nwarps*TP float4][Kt: dh*TPS float][Vs: Tn*dh float]
  float4* q4_all = reinterpret_cast<float4*>(smem_raw);
  float4* p4_all = q4_all + (size_t)nwarps * dh;
  float* Kt = reinterpret_cast<float*>(p4_all + (size_t)nwarps * TP);
  float* Vs = Kt + (size_t)dh * TPS;

  const int64_t tok_stride = (int64_t)H * dh;
  const int64_t head_base = (int64_t)b * Tn * tok_stride + (int64_t)h * dh;
  if (MODE != ATT_PV) {
    for (int idx = threadIdx.x; idx < dh * TP; idx += blockDim.x) {
      const int j = idx / dh, e = idx - j * dh;
      Kt[e * TPS + j] = j < Tn ? ld_as_float(k + head_base + (int64_t)j * tok_stride + e) : 0.f;
    }
  }
  if (MODE != ATT_SCORES) {
    for (int idx = threadIdx.x; idx < Tn * dh; idx += blockDim.x) {
      const int j = idx / dh, e = idx - j * dh;
      Vs[idx] = ld_as_float(v + head_base + (int64_t)j * tok_stride + e);
    }
  }
  __syncthreads();

  float4* q4 = q4_all + (size_t)warp * dh;
  float4* p4 = p4_all + (size_t)warp * TP;
  float* p4f = reinterpret_cast<float*>(p4);
  const int64_t sc_base = ((int64_t)b * H + h) * Tn * (int64_t)Tn;

  for (int r0 = row0 + warp * 4; r0 < row_end; r0 += nwarps * 4) {
    const int nrows = min(4, row_end - r0);
    if (MODE != ATT_PV) {
      for (int e = lane; e < dh; e += 32) {
        float qq[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) qq[r] = r < nrows ? ld_as_float(q + head_base + (int64_t)(r0 + r) * tok_stride + e) : 0.f;
        q4[e] = make_float4(qq[0], qq[1], qq[2], qq[3]);
      }
      __syncwarp();
      float acc[KPL][4];
#pragma unroll
      for (int m = 0; m < KPL; ++m) acc[m][0] = acc[m][1] = acc[m][2] = acc[m][3] = 0.f;
      for (int e = 0; e < dh; ++e) {
        const float4 qv = q4[e];
        const float* krow = Kt + e * TPS + lane;
#pragma unroll
        for (int m = 0; m < KPL; ++m) {
          const float kv = krow[m * 32];
          acc[m][0] = fmaf(kv, qv.x, acc[m][0]);
          acc[m][1] = fmaf(kv, qv.y, acc[m][1]);
          acc[m][2] = fmaf(kv, qv.z, acc[m][2]);
          acc[m][3] = fmaf(kv, qv.w, acc[m][3]);
        }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        if (r < nrows) {  // warp-uniform
          const int64_t ob = sc_base + (int64_t)(r0 + r) * Tn;
          float mx = -INFINITY;
#pragma unroll
          for (int m = 0; m < KPL; ++m) {
            const int j = m * 32 + lane;
            if (j < Tn) {
              float s = round_to<T>(round_to<T>(acc[m][r]) / attn_scale);  // einsum -> tensor, then "/ attn_scale" -> tensor
              if (CAUSAL && j > r0 + r) s = -INFINITY;
              acc[m][r] = s;
              if (scores) st_from_float(scores + ob + j, s);
              mx = fmaxf(mx, s);
            }
          }
          if (MODE == ATT_FUSED) {
            mx = warp_max(mx);
            float sum = 0.f;
#pragma unroll
            for (int m = 0; m < KPL; ++m) {
              const int j = m * 32 + lane;
              if (j < Tn) {
                const float ex = expf(acc[m][r] - mx);
                acc[m][r] = ex;
                sum += ex;
              }
            }
            sum = warp_sum(sum);
#pragma unroll
            for (int m = 0; m < KPL; ++m) {
              const int j = m * 32 + lane;
              if (j < Tn) {
                float p = acc[m][r] / sum;
                if (isnan(p)) p = 0.f;  // torch.where(isnan(pattern), 0, pattern)
                p = round_to<T>(p);
                if (pattern) st_from_float(pattern + ob + j, p);
                p4f[j * 4 + r] = p;
              }
            }
          }
        } else if (MODE == ATT_FUSED) {
#pragma unroll
          for (int m = 0; m < KPL; ++m) {
            const int j = m * 32 + lane;
            if (j < Tn) p4f[j * 4 + r] = 0.f;
          }
        }
      }
    }
    if (MODE == ATT_PV) {
      for (int j = lane; j < Tn; j += 32) {
        float pp[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) pp[r] = r < nrows ? ld_as_float(pattern + sc_base + (int64_t)(r0 + r) * Tn + j) : 0.f;
        p4[j] = make_float4(pp[0], pp[1], pp[2], pp[3]);
      }
    }
    if (MODE != ATT_SCORES) {
      __syncwarp();
      float zacc[EPL][4];
#pragma unroll
      for (int m = 0; m < EPL; ++m) zacc[m][0] = zacc[m][1] = zacc[m][2] = zacc[m][3] = 0.f;
      for (int j = 0; j < Tn; ++j) {
        const float4 pv = p4[j];
        const float* vrow = Vs + j * dh + lane;
#pragma unroll
        for (int m = 0; m < EPL; ++m) {
          const float vv = (m * 32 + lane < dh) ? vrow[m * 32] : 0.f;
          zacc[m][0] = fmaf(pv.x, vv, zacc[m][0]);
          zacc[m][1] = fmaf(pv.y, vv, zacc[m][1]);
          zacc[m][2] = fmaf(pv.z, vv, zacc[m][2]);
          zacc[m][3] = fmaf(pv.w, vv, zacc[m][3]);
        }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        if (r < nrows) {
#pragma unroll
          for (int m = 0; m < EPL; ++m) {
            const int e = m * 32 + lane;
            if (e < dh) st_from_float(z + head_base + (int64_t)(r0 + r) * tok_stride + e, zacc[m][r]);
          }
        }
      }
    }
    __syncwarp();
  }
}

template <typename T, int KPL, int EPL, int MODE, bool CAUSAL>
static int launch_att_inst(const PbAttention* p, cudaStream_t st) {
  const int TP = KPL * 32;
  const int threads = p->T <= 64 ? 128 : 256;
  const int nwarps = threads / 32;
  // query rows per CTA: whole head for short sequences, 64-row slabs otherwise (more CTAs, K/V reloaded per slab)
  const int rows_per_cta = p->T <= 64 ? p->T : 64;
  const size_t smem = (size_t)nwarps * p->dh * 16 + (size_t)nwarps * TP * 16 + (size_t)p->dh * (TP + 1) * 4 + (size_t)p->T * p->dh * 4;
  if (smem > 227 * 1024) {
    pb_set_error("pb_attention: T=%d dh=%d needs %zu B of shared memory (> 227 KB); sequence too long for this kernel", p->T, p->dh, smem);
    return PB_EUNSUPPORTED;
  }
  auto kern = k_attention<T, KPL, EPL, MODE, CAUSAL>;
  if (smem > 48 * 1024) PB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(p->B * p->H, (p->T + rows_per_cta - 1) / rows_per_cta);
  kern<<<grid, threads, smem, st>>>((const T*)p->q, (const T*)p->k, (const T*)p->v, (T*)p->scores, (T*)p->pattern, (T*)p->z, p->B, p->T,
                                    p->H, p->dh, p->attn_scale, rows_per_cta);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

template <typename T, int MODE, bool CAUSAL = false>
static int launch_att(const PbAttention* p, cudaStream_t st) {
  const int kpl = (p->T + 31) / 32, epl = (p->dh + 31) / 32;
#define PB_ATT_E(KPL)                                                                       \
  do {                                                                                      \
    if (epl <= 1) return launch_att_inst<T, KPL, 1, MODE, CAUSAL>(p, st);                   \
    if (epl <= 2) return launch_att_inst<T, KPL, 2, MODE, CAUSAL>(p, st);                   \
    if (epl <= 4) return launch_att_inst<T, KPL, 4, MODE, CAUSAL>(p, st);                   \
  } while (0)
  if (epl > 4) { pb_set_error("pb_attention: d_head=%d > 128 unsupported", p->dh); return PB_EUNSUPPORTED; }
  if (kpl <= 1) PB_ATT_E(1);
  else if (kpl <= 2) PB_ATT_E(2);
  else if (kpl <= 4) PB_ATT_E(4);
  else if (kpl <= 7) PB_ATT_E(7);
  else if (kpl <= 9) PB_ATT_E(9);
  else if (kpl <= 19) PB_ATT_E(19);
#undef PB_ATT_E
  pb_set_error("pb_attention: T=%d > 608 tokens unsupported", p->T);
  return PB_EUNSUPPORTED;
}

static int check_att(const PbAttention* p, const char* who) {
  PB_CHECK_ARG(p && p->B >= 0 && p->T > 0 && p->H > 0 && p->dh > 0, "%s: bad geometry", who);
  PB_CHECK_ARG(p->dtype == PB_F32 || p->dtype == PB_BF16, "%s: unknown dtype %d", who, p->dtype);
  PB_CHECK_ARG(p->attn_scale != 0.f, "%s: attn_scale must be non-zero", who);
  return PB_OK;
}

// Beyond the 608 tokens of the FFMA kernel the split stages run the tensor-core modes of attention_long.cu, which exist for
// d_head == 64 only.  Up to 608 tokens the FFMA kernel keeps serving them, so shorter sequences keep their results.
constexpr int ATT_SIMT_MAX_T = 608;
static int split_long(int (*fn)(const PbAttention*, cudaStream_t), const PbAttention* p, cudaStream_t st, const char* who, bool aligned) {
  if (p->dh != 64) {
    pb_set_error("%s: T=%d with d_head=%d unsupported: beyond %d tokens only d_head 64 is supported", who, p->T, p->dh, ATT_SIMT_MAX_T);
    return PB_EUNSUPPORTED;
  }
  if (!aligned) {
    pb_set_error("%s: T=%d d_head=%d needs 16-byte aligned q/k/v/z pointers", who, p->T, p->dh);
    return PB_EUNSUPPORTED;
  }
  return fn(p, st);
}

extern "C" int pb_attention(const PbAttention* p, pb_stream_t stream) {
  PB_TRY(check_att(p, "pb_attention"));
  PB_CHECK_ARG(p->q && p->k && p->v && p->z, "pb_attention: q, k, v, z are required");
  if (p->B == 0) return PB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  // d_head == 64 with 16-byte aligned q / k / v / z: tensor cores, whole rows up to 128 tokens, 64-key chunks beyond;
  // anything else: the FFMA kernel
  if (p->dh == 64 && aligned16(p->q, p->k, p->v, p->z)) return p->T <= 128 ? pb_attention_mma(p, st) : pb_attention_long(p, st);
  if (p->causal) return p->dtype == PB_F32 ? launch_att<float, ATT_FUSED, true>(p, st) : launch_att<bf16, ATT_FUSED, true>(p, st);
  return p->dtype == PB_F32 ? launch_att<float, ATT_FUSED>(p, st) : launch_att<bf16, ATT_FUSED>(p, st);
}
extern "C" int pb_attn_scores(const PbAttention* p, pb_stream_t stream) {
  PB_TRY(check_att(p, "pb_attn_scores"));
  PB_CHECK_ARG(p->q && p->k && p->scores, "pb_attn_scores: q, k, scores are required");
  if (p->B == 0) return PB_OK;
  if (p->T > ATT_SIMT_MAX_T) return split_long(pb_attn_scores_long, p, (cudaStream_t)stream, "pb_attn_scores", aligned16(p->q, p->k));
  return p->dtype == PB_F32 ? launch_att<float, ATT_SCORES>(p, (cudaStream_t)stream) : launch_att<bf16, ATT_SCORES>(p, (cudaStream_t)stream);
}
extern "C" int pb_attn_pv(const PbAttention* p, pb_stream_t stream) {
  PB_TRY(check_att(p, "pb_attn_pv"));
  PB_CHECK_ARG(p->pattern && p->v && p->z, "pb_attn_pv: pattern, v, z are required");
  if (p->B == 0) return PB_OK;
  if (p->T > ATT_SIMT_MAX_T) return split_long(pb_attn_pv_long, p, (cudaStream_t)stream, "pb_attn_pv", aligned16(p->v, p->z));
  return p->dtype == PB_F32 ? launch_att<float, ATT_PV>(p, (cudaStream_t)stream) : launch_att<bf16, ATT_PV>(p, (cudaStream_t)stream);
}

// ------------------------------------------------------------ row softmax
// F.softmax(x, -1) then NaN -> 0 (attention.py:148-149); also the softmax inside solu
// (activation_fns.py:50-57).  One warp per row, three passes served by L1/L2 after the first.
template <typename T>
__global__ void __launch_bounds__(256) k_softmax_rows(const T* __restrict__ x, T* __restrict__ y, int64_t rows, int cols) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const T* xr = x + row * cols;
  T* yr = y + row * cols;
  float mx = -INFINITY;
  for (int c = lane; c < cols; c += 32) mx = fmaxf(mx, ld_as_float(xr + c));
  mx = warp_max(mx);
  float sum = 0.f;
  for (int c = lane; c < cols; c += 32) sum += expf(ld_as_float(xr + c) - mx);
  sum = warp_sum(sum);
  for (int c = lane; c < cols; c += 32) {
    float p = expf(ld_as_float(xr + c) - mx) / sum;
    if (isnan(p)) p = 0.f;
    st_from_float(yr + c, p);
  }
}
extern "C" int pb_softmax_rows(const void* x, void* y, int64_t rows, int32_t cols, int32_t dtype, pb_stream_t s) {
  PB_CHECK_ARG(x && y && rows >= 0 && cols > 0, "pb_softmax_rows: bad arguments");
  if (rows == 0) return PB_OK;
  int grid = (int)ceil_div64(rows, 8);
  if (dtype == PB_F32) k_softmax_rows<float><<<grid, 256, 0, (cudaStream_t)s>>>((const float*)x, (float*)y, rows, cols);
  else if (dtype == PB_BF16) k_softmax_rows<bf16><<<grid, 256, 0, (cudaStream_t)s>>>((const bf16*)x, (bf16*)y, rows, cols);
  else PB_CHECK_ARG(false, "pb_softmax_rows: unknown dtype %d", dtype);
  PB_LAUNCH_CHECK();
  return PB_OK;
}
