// attention_frag.cuh -- the mma.sync fragment layer of the d_head == 64 tensor-core attention: attention_mma.cu (whole
// rows, T <= 128) and attention_long.cu (K / V in 64-key chunks) build their kernels from these wrappers and layouts.
//   bf16 : mma.sync.m16n8k16 bf16 (fp32 accumulate); fragments come from ldmatrix (.trans for V, so the PV operand
//          needs no transposed copy of V -- the transposing 2-byte stores of a first version were bank-conflict bound).
//   fp32 : mma.sync.m16n8k8 tf32 in 3 passes (x = hi + lo, hi = what the tensor core reads of x, lo = x - hi:
//          lo*hi + hi*lo + hi*hi) -> fp32-grade products for the 1e-4 parity bar.
// Rounding points follow the reference graph: scores = round(round(q.k) / scale); pattern = round(softmax);
// z = round(pattern @ v) with the rounded pattern as the operand.
#pragma once
#include "common.cuh"

namespace {

__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// 3xTF32 with the A operand already split (Q fragments live in registers across all key tiles)
__device__ __forceinline__ void mma_tf32x3_presplit(float (&d)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], const float (&b)[2]) {
  uint32_t bh[2], bl[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) { bh[i] = __float_as_uint(b[i]); bl[i] = __float_as_uint(tf32_lo(b[i])); }
  mma_tf32(d, al, bh);
  mma_tf32(d, ah, bl);
  mma_tf32(d, ah, bh);
}
// 3xTF32: operands given as fp32 values (mma.sync reads the tf32 part of the word)
__device__ __forceinline__ void mma_tf32x3(float (&d)[4], const float (&a)[4], const float (&b)[2]) {
  uint32_t ah[4], al[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { ah[i] = __float_as_uint(a[i]); al[i] = __float_as_uint(tf32_lo(a[i])); }
  mma_tf32x3_presplit(d, ah, al, b);
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* smem_row) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem_row);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem_row) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem_row);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}

constexpr int DH = 64;

// shared-memory row stride of Q / K / V in elements: 144 B (bf16) / 272 B (fp32) -- 16-byte aligned rows whose 16 B
// pieces rotate through the banks (ldmatrix, 128-bit copies and the scalar tf32 fragment loads are all conflict-free)
template <typename T> struct Lay { static constexpr int LD = DH + (sizeof(T) == 2 ? 8 : 4); };

// ---------------------------------------------------------------- host side
// the kernels' inv_scale argument: 1 / attn_scale when attn_scale is a power of two, 0 (divide) otherwise
float pow2_inv_scale(float attn_scale) {
  int ex = 0;
  return frexpf(attn_scale, &ex) == 0.5f ? 1.f / attn_scale : 0.f;
}

// lets KERN use smem bytes of dynamic shared memory (a one-time opt-in above 48 KB)
template <auto KERN>
int smem_opt_in(size_t smem) {
  static bool done = false;
  if (!done && smem > 48 * 1024) {
    PB_CUDA(cudaFuncSetAttribute(KERN, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    done = true;
  }
  return PB_OK;
}

}  // namespace
