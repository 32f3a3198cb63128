// gemm_tc.cu -- wgmma / TMA GEMM with the hooked epilogue (sm_90a).
//
//   out = A[M,K] @ B[N,K]^T, both operands K-major in HBM, fp32 accumulation in registers.
//
// Persistent kernel, one CTA per SM, 128 x 128 output tiles walked with a grid stride:
//   warpgroup 0   TMA producer : one thread issues cp.async.bulk.tensor.2d (128B-swizzled boxes, one k-slab of 128 bytes per row)
//                                into a STAGES-deep shared-memory ring, completion on "full" mbarriers;
//   warpgroups 1-2 consumers   : each owns 64 rows of the tile and issues wgmma.mma_async m64n128 (32 bytes of K per
//                                instruction) straight from the swizzled tiles through shared-memory descriptors; a slot is
//                                handed back ("empty") once the wgmma group that read it has retired.  After the last k-slab
//                                the accumulators go through a shared-memory transposer to the hooked epilogue (bias /
//                                activation / residual, hook-point spill to up to two destinations) while the producer
//                                already fills the ring with the next tile.
//
// Precision modes
//   bf16  : wgmma .bf16, bf16 operands.                      1 MMA per k-step
//   tf32x3: wgmma .tf32 on fp32 operands split as x = hi + lo with hi = tf32_trunc(x) (the tensor core
//           ignores the 13 low mantissa bits, so the unsplit fp32 array *is* hi) and lo = x - hi stored
//           separately:  A@B ~= Alo@Bhi + Ahi@Blo + Ahi@Bhi (lo*lo ~ 2^-22 relative is dropped).
//           3 MMAs per k-step into the same accumulator -> fp32-grade products for the 1e-4 parity bar.
#include "common.cuh"
#include "gemm_epi.cuh"
#include <cuda.h>

#include "tc_common.cuh"

namespace {

template <typename T>
__device__ __forceinline__ void epi_rows_scalar(const EpiParams& ep, const float* stage, int lane, int row0, int nrows, int col) {
  // one column per lane, rows walked sequentially: every warp store is one contiguous 32-element row segment
  const T* bias = (const T*)ep.bias;
  const bool has_bias = bias != nullptr;
  const float bv = has_bias ? ld_as_float(bias + col) : 0.f;
  T* o0 = nullptr;
  if (ep.n_split > 1) {
    const int blk = col / ep.split_n;
    o0 = (T*)(blk == 0 ? ep.out_split[0] : blk == 1 ? ep.out_split[1] : blk == 2 ? ep.out_split[2] : ep.out_split[3]) + (col - blk * ep.split_n);
  } else if (ep.out0) {
    o0 = (T*)ep.out0 + col;
  }
  if (o0) o0 += (int64_t)row0 * ep.ld0;
  T* o1 = ep.out1 ? (T*)ep.out1 + (int64_t)row0 * ep.ld1 + col : nullptr;
  float* o1lo = ep.out1_lo ? ep.out1_lo + (int64_t)row0 * ep.ld1 + col : nullptr;
  const T* res = ep.residual ? (const T*)ep.residual + (int64_t)row0 * ep.ldr + col : nullptr;
  for (int rr = 0; rr < nrows; ++rr) {
    const float a = stage[rr * 33 + lane];
    const float v = has_bias ? round_to<T>(round_to<T>(a) + bv) : round_to<T>(a);
    if (o0) { st_from_float(o0, v); o0 += ep.ld0; }
    if (o1) {
      float o;
      if (res) { o = ld_as_float(res) + v; res += ep.ldr; }
      else o = apply_act(v, ep.act);
      st_from_float(o1, o);
      o1 += ep.ld1;
      if (o1lo) { *o1lo = tf32_lo(o); o1lo += ep.ld1; }
    }
  }
}

__device__ __forceinline__ void st2(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }
__device__ __forceinline__ void st2(bf16* p, float a, float b) { *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(a, b); }
__device__ __forceinline__ void ld2(const float* p, float& a, float& b) { float2 t = *reinterpret_cast<const float2*>(p); a = t.x; b = t.y; }
__device__ __forceinline__ void ld2(const bf16* p, float& a, float& b) {
  float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
  a = t.x; b = t.y;
}

// GELU(x) = x/2 (1 + erf(x/sqrt2)) with erf from Abramowitz-Stegun 7.1.26 (|erf error| <= 1.5e-7, branch-free, one
// MUFU.EX2 + one MUFU.RCP): the epilogue of the MLP-in GEMM evaluates it B*T*d_mlp times per block and was issue-bound
// on libdevice's branchy erff.  Absolute error of the result <= 0.75e-7 |x|.
__device__ __forceinline__ float mufu_rcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float mufu_ex2(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float gelu_fast(float x) {
  // single MUFU.RCP / MUFU.EX2, no IEEE fix-up branches: __frcp_rn's slow path put a BSSY/BSYNC pair around every element,
  // which serialised the 32 unrolled evaluations
  const float ax = fabsf(x) * 0.70710678118654752440f;
  const float t = mufu_rcp(fmaf(0.3275911f, ax, 1.f));
  float p = fmaf(t, 1.061405429f, -1.453152027f);
  p = fmaf(t, p, 1.421413741f);
  p = fmaf(t, p, -0.284496736f);
  p = fmaf(t, p, 0.254829592f);
  const float erf_abs = fmaf(-p * t, mufu_ex2(ax * ax * -1.4426950408889634f), 1.f);
  return 0.5f * x * (1.f + copysignf(erf_abs, x));
}

// out1 flavour of one 32-column chunk, fixed at compile time so the row loop carries no activation switch
enum { EPI_NONE = 0, EPI_RESID = 1, EPI_GELU = 2, EPI_ACT = 3 };

template <typename T, int MODE, bool HAS_BIAS, bool HAS_OUT0>
__device__ __forceinline__ void epi_pair_loop(const float* __restrict__ stage, int hi, int cp, int nrows, float b0, float b1, T* o0,
                                              int64_t ld0, T* o1, float* o1lo, int64_t ld1, const T* res, int64_t ldr, int act) {
  // rows hi, hi+2, ...: pointers advance by two rows per trip (no per-row multiplies), trips independent -> unrolled for ILP
  const float* sp = stage + hi * 33 + 2 * cp;
  if (HAS_OUT0) o0 += hi * ld0;
  if (MODE != EPI_NONE) { o1 += hi * ld1; if (o1lo) o1lo += hi * ld1; }
  if (MODE == EPI_RESID) res += hi * ldr;
#pragma unroll 4
  for (int rr = hi; rr < nrows; rr += 2) {
    const float a0 = sp[0], a1 = sp[1];
    sp += 66;
    const float v0 = HAS_BIAS ? round_to<T>(round_to<T>(a0) + b0) : round_to<T>(a0);
    const float v1 = HAS_BIAS ? round_to<T>(round_to<T>(a1) + b1) : round_to<T>(a1);
    if (HAS_OUT0) { st2(o0, v0, v1); o0 += 2 * ld0; }
    if (MODE != EPI_NONE) {
      float x0, x1;
      if (MODE == EPI_RESID) { ld2(res, x0, x1); x0 += v0; x1 += v1; res += 2 * ldr; }
      else if (MODE == EPI_GELU) { x0 = gelu_fast(v0); x1 = gelu_fast(v1); }
      else { x0 = apply_act(v0, act); x1 = apply_act(v1, act); }
      st2(o1, x0, x1);
      o1 += 2 * ld1;
      if (o1lo) { st2(o1lo, tf32_lo(x0), tf32_lo(x1)); o1lo += 2 * ld1; }
    }
  }
}

template <typename T>
__device__ __forceinline__ void epi_rows_pair(const EpiParams& ep, const float* stage, int lane, int row0, int nrows, int col0) {
  // two adjacent columns per lane, two rows per warp instruction (lanes 0-15: even row, 16-31: odd row):
  // half the load/store instructions of the scalar walk, still whole 32-column row segments per half-warp.
  const int hi = lane >> 4, cp = lane & 15;
  const int col = col0 + 2 * cp;
  if (col >= ep.N) return;   // N % 4 == 0 on this path, so the pair is either fully inside or fully outside
  const T* bias = (const T*)ep.bias;
  float b0 = 0.f, b1 = 0.f;
  if (bias) ld2(bias + col, b0, b1);
  T* o0 = nullptr;
  if (ep.n_split > 1) {       // no dynamic indexing of the parameter struct (it would be copied to local memory)
    const int blk = col / ep.split_n;
    void* base = blk == 0 ? ep.out_split[0] : blk == 1 ? ep.out_split[1] : blk == 2 ? ep.out_split[2] : ep.out_split[3];
    o0 = (T*)base + (col - blk * ep.split_n);
  } else if (ep.out0) {
    o0 = (T*)ep.out0 + col;
  }
  const int64_t ld0 = ep.ld0, ld1 = ep.ld1, ldr = ep.ldr;
  if (o0) o0 += (int64_t)row0 * ld0;
  T* o1 = ep.out1 ? (T*)ep.out1 + (int64_t)row0 * ld1 + col : nullptr;
  float* o1lo = ep.out1_lo ? ep.out1_lo + (int64_t)row0 * ld1 + col : nullptr;
  const T* res = ep.residual ? (const T*)ep.residual + (int64_t)row0 * ldr + col : nullptr;
  const int mode = !o1 ? EPI_NONE : res ? EPI_RESID : ep.act == PB_ACT_GELU ? EPI_GELU : EPI_ACT;
#define PB_EPI(MODE_)                                                                                                             \
  do {                                                                                                                            \
    if (bias) { if (o0) epi_pair_loop<T, MODE_, true, true>(stage, hi, cp, nrows, b0, b1, o0, ld0, o1, o1lo, ld1, res, ldr, ep.act); \
                else epi_pair_loop<T, MODE_, true, false>(stage, hi, cp, nrows, b0, b1, o0, ld0, o1, o1lo, ld1, res, ldr, ep.act); } \
    else { if (o0) epi_pair_loop<T, MODE_, false, true>(stage, hi, cp, nrows, b0, b1, o0, ld0, o1, o1lo, ld1, res, ldr, ep.act);    \
           else epi_pair_loop<T, MODE_, false, false>(stage, hi, cp, nrows, b0, b1, o0, ld0, o1, o1lo, ld1, res, ldr, ep.act); }   \
  } while (0)
  if (mode == EPI_NONE) PB_EPI(EPI_NONE);
  else if (mode == EPI_RESID) PB_EPI(EPI_RESID);
  else if (mode == EPI_GELU) PB_EPI(EPI_GELU);
  else PB_EPI(EPI_ACT);
#undef PB_EPI
}

// ---- row-per-lane epilogue: shared memory only as a 16-byte-vector transposer --------------------------------------
// The caller gives thread t row t of a 32x32 chunk.  Bias / rounding / GELU / residual are applied right there (constant
// register indices, no per-element address arithmetic); the packed results are written as the thread's row into a padded
// stage (row stride 32*sizeof(T)+16 B: conflict-free for 128-bit accesses) and copied out with 16 B loads/stores where
// consecutive lanes cover consecutive 16 B of a row.  ~20 instructions per element against ~56 for the per-element walk
// and every global access is a full 16 B vector of a contiguous row segment.
template <typename T> struct EpiStage {
  static constexpr int VPR = 32 * (int)sizeof(T) / 16;        // 16-byte vectors per 32-column row: 4 (bf16) / 8 (fp32)
  static constexpr int ROW_BYTES = 32 * (int)sizeof(T) + 16;
};

__device__ __forceinline__ void stage_put_row(uint8_t* row, const float (&v)[32], float) {   // fp32 rows
#pragma unroll
  for (int q = 0; q < 8; ++q) *reinterpret_cast<float4*>(row + 16 * q) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
}
__device__ __forceinline__ void stage_put_row(uint8_t* row, const float (&v)[32], bf16) {    // bf16 rows
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint4 u;
    __nv_bfloat162 p0 = __floats2bfloat162_rn(v[8 * q], v[8 * q + 1]), p1 = __floats2bfloat162_rn(v[8 * q + 2], v[8 * q + 3]);
    __nv_bfloat162 p2 = __floats2bfloat162_rn(v[8 * q + 4], v[8 * q + 5]), p3 = __floats2bfloat162_rn(v[8 * q + 6], v[8 * q + 7]);
    u.x = *reinterpret_cast<uint32_t*>(&p0); u.y = *reinterpret_cast<uint32_t*>(&p1);
    u.z = *reinterpret_cast<uint32_t*>(&p2); u.w = *reinterpret_cast<uint32_t*>(&p3);
    *reinterpret_cast<uint4*>(row + 16 * q) = u;
  }
}
__device__ __forceinline__ void stage_get_row(const uint8_t* row, float (&v)[32], float) {
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 t = *reinterpret_cast<const float4*>(row + 16 * q);
    v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
  }
}
__device__ __forceinline__ void stage_get_row(const uint8_t* row, float (&v)[32], bf16) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + 16 * q);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v[8 * q + 2 * j] = __uint_as_float(w[j] << 16);
      v[8 * q + 2 * j + 1] = __uint_as_float(w[j] & 0xFFFF0000u);
    }
  }
}

// stage (32 rows x 32 cols of T) -> global rows [row0, row0+nrows) x cols [col, col+32): 16 B per lane per trip
template <typename T>
__device__ __forceinline__ void stage_copy_out(const uint8_t* stage, T* __restrict__ gbase, int64_t ld, int lane, int nrows) {
  constexpr int VPR = EpiStage<T>::VPR;
#pragma unroll
  for (int i = 0; i < VPR; ++i) {
    const int vidx = lane + 32 * i, row = vidx / VPR, vin = vidx % VPR;
    if (row < nrows)
      *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(gbase + (int64_t)row * ld) + 16 * vin) =
          *reinterpret_cast<const uint4*>(stage + row * EpiStage<T>::ROW_BYTES + 16 * vin);
  }
}
template <typename T>
__device__ __forceinline__ void stage_copy_in(uint8_t* stage, const T* __restrict__ gbase, int64_t ld, int lane, int nrows) {
  constexpr int VPR = EpiStage<T>::VPR;
#pragma unroll
  for (int i = 0; i < VPR; ++i) {
    const int vidx = lane + 32 * i, row = vidx / VPR, vin = vidx % VPR;
    if (row < nrows)
      *reinterpret_cast<uint4*>(stage + row * EpiStage<T>::ROW_BYTES + 16 * vin) =
          *reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(gbase + (int64_t)row * ld) + 16 * vin);
  }
}

template <typename T>
__device__ __forceinline__ void epi_chunk_vec(const EpiParams& ep, const uint32_t (&r)[32], uint8_t* stage, int lane, int row0, int nrows,
                                              int col0) {
  uint8_t* my_row = stage + lane * EpiStage<T>::ROW_BYTES;
  float v[32];
  const T* bias = (const T*)ep.bias;
  if (bias) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      float bb[4];
      ld4(bias + col0 + 4 * q, bb);                              // same address in every lane: one broadcast transaction
#pragma unroll
      for (int j = 0; j < 4; ++j) v[4 * q + j] = round_to<T>(__uint_as_float(r[4 * q + j]) + bb[j]);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = round_to<T>(__uint_as_float(r[j]));
  }
  // ---- out0 (or the q / k / v block this chunk falls into)
  T* o0 = nullptr;
  if (ep.n_split > 1) {
    const int blk = col0 / ep.split_n;
    void* base = blk == 0 ? ep.out_split[0] : blk == 1 ? ep.out_split[1] : blk == 2 ? ep.out_split[2] : ep.out_split[3];
    o0 = (T*)base + (col0 - blk * ep.split_n);
  } else if (ep.out0) {
    o0 = (T*)ep.out0 + col0;
  }
  if (o0) {
    stage_put_row(my_row, v, T());
    __syncwarp();
    stage_copy_out<T>(stage, o0 + (int64_t)row0 * ep.ld0, ep.ld0, lane, nrows);
    __syncwarp();
  }
  if (!ep.out1) return;
  // ---- out1 = residual + v  |  act(v)
  if (ep.residual) {
    stage_copy_in<T>(stage, (const T*)ep.residual + (int64_t)row0 * ep.ldr + col0, ep.ldr, lane, nrows);
    __syncwarp();
    float rs[32];
    stage_get_row(my_row, rs, T());
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = rs[j] + v[j];
  } else if (ep.act == PB_ACT_GELU) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = gelu_fast(v[j]);
  } else {
    const int act = ep.act;
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = apply_act(v[j], act);
  }
  stage_put_row(my_row, v, T());
  __syncwarp();
  stage_copy_out<T>(stage, (T*)ep.out1 + (int64_t)row0 * ep.ld1 + col0, ep.ld1, lane, nrows);
  __syncwarp();
  if (sizeof(T) == 4 && ep.out1_lo) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = tf32_lo(v[j]);
    stage_put_row(my_row, v, T());
    __syncwarp();
    stage_copy_out<T>(stage, (T*)ep.out1_lo + (int64_t)row0 * ep.ld1 + col0, ep.ld1, lane, nrows);
    __syncwarp();
  }
}


// Epilogue transposer: per consumer warp one 32 x 32 fp32 block (row stride 33, conflict-free when a lane reads its row),
// sized for the 16-byte-vector stage of epi_chunk_vec (32 rows x 144 B) that reuses it once the block is in registers.
constexpr int EPI_WARP_BYTES = 32 * 36 * 4;
template <typename T, int NPASS, int STAGES>
struct TcSmem {
  using C = TcCfg<T, NPASS, STAGES>;
  static constexpr int EPI_BYTES = 8 * EPI_WARP_BYTES;
  static constexpr int SMEM_BYTES = C::RING_BYTES + EPI_BYTES + 1024 /*alignment slack*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 232448, "shared memory budget exceeded");
};

template <typename T, int NPASS>
__device__ __forceinline__ void wgmma_step(float (&acc)[64], uint32_t sa, uint32_t sb, uint32_t koff, uint32_t a_lo_off, uint32_t b_lo_off,
                                           uint32_t first) {
  const uint64_t a_hi = make_smem_desc(sa + koff);
  const uint64_t b_hi = make_smem_desc(sb + koff);
  if (sizeof(T) == 2) {
    wgmma_bf16_n128(acc, a_hi, b_hi, first);
  } else if (NPASS == 3) {
    wgmma_tf32_n128(acc, make_smem_desc(sa + a_lo_off + koff), b_hi, first);
    wgmma_tf32_n128(acc, a_hi, make_smem_desc(sb + b_lo_off + koff), 1u);
    wgmma_tf32_n128(acc, a_hi, b_hi, 1u);
  } else {
    wgmma_tf32_n128(acc, a_hi, b_hi, first);
  }
}

template <typename T, int NPASS, int STAGES>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_gemm_tc(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmAlo,
          const __grid_constant__ CUtensorMap tmBlo, int K, EpiParams ep, int num_m_tiles, int num_n_tiles, int m_fast) {
  using C = TcCfg<T, NPASS, STAGES>;
  // raster order of the persistent tile walk: the ~132 tiles in flight share one operand through L2 and stream the other.
  // n-fastest (default) streams A once and wants B (the weights) L2-resident; m_fast streams B once and keeps A resident --
  // a large dictionary against a few thousand tokens (the SAE products) needs the latter.
  auto tile_m = [&](int tile) { return m_fast ? tile % num_m_tiles : tile / num_n_tiles; };
  auto tile_n = [&](int tile) { return m_fast ? tile / num_m_tiles : tile % num_n_tiles; };
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem0 = smem_u32(smem_raw);
  const uint32_t ring = (smem0 + 1023u) & ~1023u;     // SWIZZLE_128B tiles need 1024 B alignment
  const uint32_t epi_stage = ring + C::RING_BYTES;
  const uint32_t bar_base = epi_stage + 8 * EPI_WARP_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int num_kb = (K + C::BK - 1) / C::BK;
  const int num_tiles = num_m_tiles * num_n_tiles;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    if (NPASS == 3) { prefetch_tmap(&tmAlo); prefetch_tmap(&tmBlo); }
    for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 2); }   // empty: one arrival per consumer warpgroup
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = tile_m(tile) * TC_BM, n0 = tile_n(tile) * TC_BN;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          mbar_wait<false>(empty_bar(s), ph ^ 1);
          mbar_expect_tx(full_bar(s), C::STAGE_BYTES);
          const uint32_t sa = ring + s * C::STAGE_BYTES;
          const int kc = kb * C::BK;
          tma_load_2d(sa, &tmA, full_bar(s), kc, m0);
          if (NPASS == 3) tma_load_2d(sa + C::A_BYTES, &tmAlo, full_bar(s), kc, m0);
          const uint32_t sb = sa + C::NOP * C::A_BYTES;
          tma_load_2d(sb, &tmB, full_bar(s), kc, n0);
          if (NPASS == 3) tma_load_2d(sb + C::B_BYTES, &tmBlo, full_bar(s), kc, n0);
        }
      }
    }
    return;
  }
  // ===================== consumers: warpgroup c owns rows [64 c, 64 c + 64) of each tile =====================
  reg_alloc<232>();
  const int c = wg - 1;
  const int wq = warp & 3;                 // warp inside the warpgroup
  const int tid = threadIdx.x & 127;
  uint8_t* stage_wg = smem_raw + (epi_stage - smem0) + c * 4 * EPI_WARP_BYTES;
  float* region = reinterpret_cast<float*>(stage_wg + wq * EPI_WARP_BYTES);
  // bf16: every 64-wide k-slab goes into a fresh wgmma accumulator that is then added into `acc` with FADD.  The tensor core's own
  // fp32 accumulation over the whole K chain rounded the bf16 outputs measurably further from the exact sum than the reference's
  // fp32 GEMM.  The slab's group is waited for at once; the other consumer warpgroup's MMAs keep the tensor core busy meanwhile.
  constexpr bool PROMOTE = sizeof(T) == 2;
  float acc[64], part[PROMOTE ? 64 : 1];
  uint32_t it = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m0 = tile_m(tile) * TC_BM, n0 = tile_n(tile) * TC_BN;
    int prev_s = -1;
    if constexpr (PROMOTE) {
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    }
    for (int kb = 0; kb < num_kb; ++kb, ++it) {
      const int s = it % STAGES;
      const uint32_t ph = (it / STAGES) & 1;
      mbar_wait<false>(full_bar(s), ph);
      const uint32_t sa = ring + s * C::STAGE_BYTES + c * 64 * 128;       // this warpgroup's 64 rows of A
      const uint32_t sb = ring + s * C::STAGE_BYTES + C::NOP * C::A_BYTES;
      wgmma_fence();
      if constexpr (PROMOTE) {
#pragma unroll
        for (int k = 0; k < C::KSTEPS; ++k) wgmma_step<T, NPASS>(part, sa, sb, 32u * k, C::A_BYTES, C::B_BYTES, k != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(part);
        if (tid == 0) mbar_arrive(empty_bar(s));
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] += part[i];
      } else {
#pragma unroll
        for (int k = 0; k < C::KSTEPS; ++k)
          wgmma_step<T, NPASS>(acc, sa, sb, 32u * k, C::A_BYTES, C::B_BYTES, (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();                      // the group of the previous k-slab has retired: its slot may be refilled
        if (prev_s >= 0 && tid == 0) mbar_arrive(empty_bar(prev_s));
        prev_s = s;
      }
    }
    if constexpr (!PROMOTE) {
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (tid == 0) mbar_arrive(empty_bar(prev_s));
    }

    // ---- epilogue, 64 columns at a time.  Accumulator element i of thread (warp w, lane l) is row 16 w + l / 4 + 8 ((i >> 1) & 1),
    // column 8 (i >> 2) + 2 (l % 4) + (i & 1) of the warpgroup's 64 x 128 block.  Warp q of the warpgroup then takes the 32 x 32
    // block q (rows 32 (q & 1) .., columns 32 (q >> 1) .. of the 64-column half) with one row per lane.
#pragma unroll
    for (int half = 0; half < 2; ++half) {
#pragma unroll
      for (int i = 32 * half; i < 32 * half + 32; ++i) {
        const int r = 16 * wq + (lane >> 2) + 8 * ((i >> 1) & 1);
        const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1) - 64 * half;
        float* dst = reinterpret_cast<float*>(stage_wg + ((r >> 5) | ((col >> 5) << 1)) * EPI_WARP_BYTES);
        dst[(r & 31) * 33 + (col & 31)] = acc[i];
      }
      wg_sync(1 + c);
      const int row0 = m0 + 64 * c + 32 * (wq & 1);
      const int nrows = min(32, ep.M - row0);
      const int col0 = n0 + 64 * half + 32 * (wq >> 1);
      if (nrows > 0 && col0 < ep.N) {
        if (ep.vec16_ok && col0 + 32 <= ep.N) {     // whole chunk inside the matrix: row-per-lane epilogue with 16-byte stores
          uint32_t r[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) r[j] = __float_as_uint(region[lane * 33 + j]);
          __syncwarp();
          epi_chunk_vec<T>(ep, r, reinterpret_cast<uint8_t*>(region), lane, row0, nrows, col0);
        } else {                                     // ragged edge / unaligned operands: per-element walk
          if (ep.vec_ok) epi_rows_pair<T>(ep, region, lane, row0, nrows, col0);
          else if (col0 + lane < ep.N) epi_rows_scalar<T>(ep, region, lane, row0, nrows, col0 + lane);
        }
      }
      wg_sync(1 + c);                                // every warp is done with the blocks before the next half lands in them
    }
  }
}

// ---------------------------------------------------------------- host side
template <typename T, int NPASS, int STAGES>
int launch_tc(const PbGemm* g, cudaStream_t st) {
  using S = TcSmem<T, NPASS, STAGES>;
  CUtensorMap tmA, tmB, tmAlo, tmBlo;
  PB_TRY(make_map(&tmA, g->A, g->dtype, g->M, g->K, g->lda, TC_BM));
  PB_TRY(make_map(&tmB, g->B, g->dtype, g->N, g->K, g->ldb, TC_BN));
  if (NPASS == 3) {
    PB_TRY(make_map(&tmAlo, g->A_lo, g->dtype, g->M, g->K, g->lda, TC_BM));
    PB_TRY(make_map(&tmBlo, g->B_lo, g->dtype, g->N, g->K, g->ldb, TC_BN));
  } else {
    tmAlo = tmA;
    tmBlo = tmB;
  }
  auto kern = k_gemm_tc<T, NPASS, STAGES>;
  static bool attr_done = false;  // per instantiation
  if (!attr_done) {
    PB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::SMEM_BYTES));
    attr_done = true;
  }
  EpiParams ep = pb_make_epi(g);
  const int num_m = (g->M + TC_BM - 1) / TC_BM, num_n = (g->N + TC_BN - 1) / TC_BN;
  int grid = pb_sm_count();
  if (grid > num_m * num_n) grid = num_m * num_n;
  const size_t planes = NPASS > 1 ? 2 : 1;
  const size_t a_bytes = (size_t)g->M * g->K * sizeof(T) * planes, b_bytes = (size_t)g->N * g->K * sizeof(T) * planes;
  const int m_fast = (b_bytes > ((size_t)24 << 20) && a_bytes < b_bytes) ? 1 : 0;   // B no longer fits half of the 50 MB L2
  kern<<<grid, TC_THREADS, S::SMEM_BYTES, st>>>(tmA, tmB, tmAlo, tmBlo, g->K, ep, num_m, num_n, m_fast);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

}  // namespace

// shape / alignment gate for the tensor-core path
bool pb_gemm_tc_eligible(const PbGemm* g) {
  const int es = g->dtype == PB_BF16 ? 2 : 4;
  if (g->M < 1 || g->N < 16 || g->K < 128 / es) return false;
  if (!pb_aligned16(g->A) || !pb_aligned16(g->B)) return false;
  if ((g->lda * es) % 16 != 0 || (g->ldb * es) % 16 != 0) return false;
  if (g->dtype == PB_F32) {
    if (!g->A_lo || !g->B_lo) return false;
    if (!pb_aligned16(g->A_lo) || !pb_aligned16(g->B_lo)) return false;
  }
  return true;
}

int pb_gemm_tc(const PbGemm* g, cudaStream_t st) {
  if (!pb_gemm_tc_eligible(g)) {
    pb_set_error("pb_gemm: tensor-core path refused M=%d N=%d K=%d dtype=%d lda=%lld ldb=%lld (alignment / missing *_lo)", g->M, g->N, g->K,
                 g->dtype, (long long)g->lda, (long long)g->ldb);
    return PB_EUNSUPPORTED;
  }
  // ring depth: bf16 4 x 32 KB, 3xTF32 (hi + lo planes of both operands) 2 x 64 KB; the 36 KB epilogue transposer sits beside it
  if (g->dtype == PB_BF16) return launch_tc<bf16, 1, 4>(g, st);
  return launch_tc<float, 3, 2>(g, st);
}
