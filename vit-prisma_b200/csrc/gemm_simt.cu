// gemm_simt.cu -- exact-fp32 FFMA GEMM with the hooked epilogue; any shape, any stride.
//
// Role: (1) the fp32 parity path (bit-for-bit fp32 products, fp32 accumulation -- what the
// reference's CPU bmm computes up to summation order); (2) the shape-agnostic path for problems the
// wgmma kernel (gemm_tc.cu) does not take (tiny d_model in unit tests, K not a multiple of the
// swizzle atom, unaligned leading dimensions); (3) the on-device cross-check for gemm_tc.cu.
// 128x128x16 CTA tile, 256 threads, 8x8 register tile per thread (as 2x2 blocks of 4x4 so shared
// loads are LDS.128 and global stores are 16 B), register-staged double buffering of the next k-slab.
#include "common.cuh"
#include "gemm_epi.cuh"

namespace {

constexpr int BM = 128, BN = 128, BK = 16, LDS_PAD = 4;
constexpr int LDT = BM + LDS_PAD;  // smem row stride (floats), keeps float4 alignment

// load 4 consecutive k of one row into v (zero beyond bounds)
template <typename T, bool VEC>
__device__ __forceinline__ void load_k4(const T* __restrict__ base, int64_t ld, int row, int nrows, int k, int K, float (&v)[4]) {
  if (row < nrows) {
    const T* p = base + (int64_t)row * ld + k;
    if (VEC && k + 3 < K) {
      ld4(p, v);
      return;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = (k + j < K) ? ld_as_float(p + j) : 0.f;
  } else {
    v[0] = v[1] = v[2] = v[3] = 0.f;
  }
}

template <typename T, bool VEC>
__global__ void __launch_bounds__(256) k_gemm_simt(const T* __restrict__ A, int64_t lda, const T* __restrict__ B, int64_t ldb, int K,
                                                   EpiParams ep) {
  __shared__ __align__(16) float As[2][BK][LDT];
  __shared__ __align__(16) float Bs[2][BK][LDT];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  // global->smem mapping: thread moves rows {lr, lr+64}, 4 consecutive k starting at lk
  const int lr = tid >> 2, lk = (tid & 3) * 4;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float ra[2][4], rb[2][4];
  const int ktiles = (K + BK - 1) / BK;
  auto gload = [&](int kt) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      load_k4<T, VEC>(A, lda, m0 + lr + 64 * i, ep.M, kt * BK + lk, K, ra[i]);
      load_k4<T, VEC>(B, ldb, n0 + lr + 64 * i, ep.N, kt * BK + lk, K, rb[i]);
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        As[buf][lk + j][lr + 64 * i] = ra[i][j];
        Bs[buf][lk + j][lr + 64 * i] = rb[i][j];
      }
  };

  gload(0);
  sstore(0);
  __syncthreads();
  for (int kt = 0; kt < ktiles; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < ktiles) gload(kt + 1);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[8], b[8];
      *reinterpret_cast<float4*>(&a[0]) = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      *reinterpret_cast<float4*>(&a[4]) = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
      *reinterpret_cast<float4*>(&b[0]) = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      *reinterpret_cast<float4*>(&b[4]) = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < ktiles) {
      sstore(buf ^ 1);
      __syncthreads();
    }
  }

#pragma unroll
  for (int ih = 0; ih < 2; ++ih)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = m0 + ih * 64 + ty * 4 + i;
      if (row >= ep.M) continue;
#pragma unroll
      for (int jh = 0; jh < 2; ++jh) {
        const int col = n0 + jh * 64 + tx * 4;
        if (col >= ep.N) continue;
        float v[4] = {acc[ih * 4 + i][jh * 4 + 0], acc[ih * 4 + i][jh * 4 + 1], acc[ih * 4 + i][jh * 4 + 2], acc[ih * 4 + i][jh * 4 + 3]};
        epilogue_store4<T>(ep, row, col, v);
      }
    }
}

}  // namespace

int pb_gemm_simt(const PbGemm* g, cudaStream_t st) {
  EpiParams ep = pb_make_epi(g);
  const bool in_vec = pb_aligned16(g->A) && pb_aligned16(g->B) && (g->lda % 4 == 0) && (g->ldb % 4 == 0);
  dim3 grid((g->N + BN - 1) / BN, (g->M + BM - 1) / BM);
  if (g->dtype == PB_F32) {
    if (in_vec) k_gemm_simt<float, true><<<grid, 256, 0, st>>>((const float*)g->A, g->lda, (const float*)g->B, g->ldb, g->K, ep);
    else k_gemm_simt<float, false><<<grid, 256, 0, st>>>((const float*)g->A, g->lda, (const float*)g->B, g->ldb, g->K, ep);
  } else {
    if (in_vec) k_gemm_simt<bf16, true><<<grid, 256, 0, st>>>((const bf16*)g->A, g->lda, (const bf16*)g->B, g->ldb, g->K, ep);
    else k_gemm_simt<bf16, false><<<grid, 256, 0, st>>>((const bf16*)g->A, g->lda, (const bf16*)g->B, g->ldb, g->K, ep);
  }
  PB_LAUNCH_CHECK();
  return PB_OK;
}
