// attention_mma.cu -- fused hooked attention for d_head == 64 on warp-level tensor-core MMAs.
//
// Why not wgmma here: one head is a 50..257-token problem (S = Q K^T is 50x50 for ViT-B/32) and the op is bound by
// the HBM traffic of its hook points (scores + pattern = 2*B*H*T*T elements written) -- a 64-row wgmma tile with a register
// round trip would be mostly padding.  Warp-level mma.sync keeps S and P in registers between QK^T, softmax and PV.
//
// One CTA = one (batch, head) x one slab of NW*16 query rows; K, V (and the Q slab) of the head sit in shared memory,
// row-major, copied in with 16-byte vectors (no conversion, no transposition on the way in); the mma.sync wrappers, operand
// layouts and rounding points are those of attention_frag.cuh.  Hook points leave through a per-warp stage that holds the
// warp's 16 rows packed exactly as they lie in global memory ([16][T] elements of T, already rounded), so the copy-out is a
// linear vector memcpy of one contiguous run.
#include "attention_frag.cuh"

namespace {

// two adjacent columns (c even) of one stage row; only columns < Tn exist in the packed layout
template <typename T> __device__ __forceinline__ void stage_put2(T* stage, int r, int c, int Tn, float a, float b);
template <> __device__ __forceinline__ void stage_put2<float>(float* stage, int r, int c, int Tn, float a, float b) {
  float* p = stage + r * Tn + c;
  if (!(Tn & 1)) { if (c < Tn) *reinterpret_cast<float2*>(p) = make_float2(a, b); }
  else { if (c < Tn) p[0] = a; if (c + 1 < Tn) p[1] = b; }
}
template <> __device__ __forceinline__ void stage_put2<bf16>(bf16* stage, int r, int c, int Tn, float a, float b) {
  bf16* p = stage + r * Tn + c;
  if (!(Tn & 1)) { if (c < Tn) *reinterpret_cast<uint32_t*>(p) = pack_bf16(a, b); }
  else { if (c < Tn) p[0] = __float2bfloat16_rn(a); if (c + 1 < Tn) p[1] = __float2bfloat16_rn(b); }
}

// contiguous run: shared -> global, vb-byte vectors (vb chosen on the host from the alignment of every run start)
template <typename T>
__device__ __forceinline__ void copy_run(T* __restrict__ g, const T* s, int n_elems, int vb, int lane) {
  uint8_t* gb = reinterpret_cast<uint8_t*>(g);
  const uint8_t* sb = reinterpret_cast<const uint8_t*>(s);
  const int nbytes = n_elems * (int)sizeof(T);
  int done = 0;
  if (vb == 16) {
    done = nbytes & ~15;
    for (int i = lane * 16; i < done; i += 512) *reinterpret_cast<uint4*>(gb + i) = *reinterpret_cast<const uint4*>(sb + i);
  } else if (vb == 8) {
    done = nbytes & ~7;
    for (int i = lane * 8; i < done; i += 256) *reinterpret_cast<uint2*>(gb + i) = *reinterpret_cast<const uint2*>(sb + i);
  } else if (vb == 4) {
    done = nbytes & ~3;
    for (int i = lane * 4; i < done; i += 128) *reinterpret_cast<uint32_t*>(gb + i) = *reinterpret_cast<const uint32_t*>(sb + i);
  }
  for (int i = done / (int)sizeof(T) + lane; i < n_elems; i += 32) g[i] = s[i];
}

// NT = key tiles of 8 (TPAD = 8*NT, multiple of 16), NW warps of 16 query rows; CAUSAL: keys j > query i score -inf
template <typename T, int NT, int NW, bool CAUSAL>
__global__ void __launch_bounds__(NW * 32) k_attention_mma(const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v,
                                                          T* __restrict__ scores, T* __restrict__ pattern, T* __restrict__ z, int Tn, int H,
                                                          float attn_scale, float inv_scale, int vb) {
  constexpr int TPAD = NT * 8;
  constexpr bool BF = sizeof(T) == 2;
  constexpr int LD = Lay<T>::LD;
  constexpr int VEC = 16 / (int)sizeof(T);                // elements per 16-byte vector
  constexpr int VPR = DH / VEC;                           // vectors per head row
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* Ks = reinterpret_cast<T*>(smem_raw);                 // [TPAD][LD]
  T* Vs = Ks + (size_t)TPAD * LD;                         // [TPAD][LD]
  T* Qs = Vs + (size_t)TPAD * LD;                         // [NW*16][LD]
  T* stage_all = Qs + (size_t)NW * 16 * LD;               // [NW][16*TPAD] packed rows

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int b = blockIdx.x / H, h = blockIdx.x % H;
  const int row0 = blockIdx.y * (NW * 16);
  const int64_t tok_stride = (int64_t)H * DH;
  const int64_t head_base = (int64_t)b * Tn * tok_stride + (int64_t)h * DH;

  // ---- stage K, V (whole head) and the Q slab with 16-byte copies; rows >= Tn are zero
  const uint4 zero4 = make_uint4(0u, 0u, 0u, 0u);
  for (int idx = threadIdx.x; idx < TPAD * VPR; idx += NW * 32) {
    const int j = idx / VPR, e = (idx % VPR) * VEC;
    uint4 kv = zero4, vv = zero4;
    if (j < Tn) {
      kv = *reinterpret_cast<const uint4*>(k + head_base + (int64_t)j * tok_stride + e);
      vv = *reinterpret_cast<const uint4*>(v + head_base + (int64_t)j * tok_stride + e);
    }
    *reinterpret_cast<uint4*>(Ks + (size_t)j * LD + e) = kv;
    *reinterpret_cast<uint4*>(Vs + (size_t)j * LD + e) = vv;
  }
  for (int idx = threadIdx.x; idx < NW * 16 * VPR; idx += NW * 32) {
    const int r = idx / VPR, e = (idx % VPR) * VEC;
    uint4 qv = zero4;
    if (row0 + r < Tn) qv = *reinterpret_cast<const uint4*>(q + head_base + (int64_t)(row0 + r) * tok_stride + e);
    *reinterpret_cast<uint4*>(Qs + (size_t)r * LD + e) = qv;
  }
  __syncthreads();

  const int wrow0 = row0 + warp * 16;                     // first query row of this warp
  if (wrow0 >= Tn) return;
  const int nvalid = min(16, Tn - wrow0);
  T* stage = stage_all + (size_t)warp * 16 * TPAD;
  const T* Qw = Qs + (size_t)warp * 16 * LD;

  // ---- S = Q K^T
  float acc[NT][4];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
  if constexpr (BF) {
    // A (16 x 16 slice of Q): matrices [rows 0-7 | 8-15] x [k 0-7 | 8-15]; lane l addresses row (l & 15), k half (l >> 4)
    uint32_t a[DH / 16][4];
#pragma unroll
    for (int kk = 0; kk < DH / 16; ++kk) ldmatrix_x4(a[kk], Qw + (size_t)(lane & 15) * LD + kk * 16 + 8 * (lane >> 4));
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      // B (keys nt*8..+7): four 8x8 blocks along d_head per ldmatrix -> {b0, b1} of two k-steps
#pragma unroll
      for (int kp = 0; kp < DH / 32; ++kp) {
        uint32_t bb[4];
        ldmatrix_x4(bb, Ks + (size_t)(nt * 8 + (lane & 7)) * LD + kp * 32 + 8 * (lane >> 3));
        mma_bf16(acc[nt], a[2 * kp], bb[0], bb[1]);
        mma_bf16(acc[nt], a[2 * kp + 1], bb[2], bb[3]);
      }
    }
  } else {
    const float* Qf = reinterpret_cast<const float*>(Qw);
    const float* Kf = reinterpret_cast<const float*>(Ks);
#pragma unroll
    for (int kk = 0; kk < DH / 8; ++kk) {
      float a[4];
      a[0] = Qf[g * LD + kk * 8 + t];
      a[1] = Qf[(g + 8) * LD + kk * 8 + t];
      a[2] = Qf[g * LD + kk * 8 + 4 + t];
      a[3] = Qf[(g + 8) * LD + kk * 8 + 4 + t];
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        float bb[2];
        bb[0] = Kf[(nt * 8 + g) * LD + kk * 8 + t];
        bb[1] = Kf[(nt * 8 + g) * LD + kk * 8 + 4 + t];
        mma_tf32x3(acc[nt], a, bb);
      }
    }
  }

  // ---- scores: scale + round; row max over valid keys. rows: lo = g, hi = g + 8; cols nt*8 + 2t + {0,1}
  // inv_scale != 0 <=> attn_scale is a power of two, where x / scale == x * (1 / scale) bit for bit (no IEEE divide)
  if (inv_scale != 0.f) {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[nt][c] = round_to<T>(round_to<T>(acc[nt][c]) * inv_scale);
  } else {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[nt][c] = round_to<T>(round_to<T>(acc[nt][c]) / attn_scale);
  }
  if constexpr (CAUSAL) {   // scores / scale + mask with mask = -inf above the diagonal: -inf there, out of the max, e = 0
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (nt * 8 + 2 * t + (c & 1) > wrow0 + g + (c < 2 ? 0 : 8)) acc[nt][c] = -INFINITY;
  }
  float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int col = nt * 8 + 2 * t + (c & 1);
      if (col < Tn) { if (c < 2) mx_lo = fmaxf(mx_lo, acc[nt][c]); else mx_hi = fmaxf(mx_hi, acc[nt][c]); }
    }
  }
  const int64_t sc_base = (((int64_t)b * H + h) * Tn + wrow0) * (int64_t)Tn;   // warp's rows are one contiguous run
  if (scores) {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      stage_put2<T>(stage, g, nt * 8 + 2 * t, Tn, acc[nt][0], acc[nt][1]);
      if (g + 8 < nvalid) stage_put2<T>(stage, g + 8, nt * 8 + 2 * t, Tn, acc[nt][2], acc[nt][3]);
    }
    __syncwarp();
    copy_run<T>(scores + sc_base, stage, nvalid * Tn, vb, lane);
    __syncwarp();
  }
  // ---- softmax (NaN -> 0), rounded to T
  mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
  mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
  mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
  mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
  float sum_lo = 0.f, sum_hi = 0.f;
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int col = nt * 8 + 2 * t + (c & 1);
      const float x = acc[nt][c] - (c < 2 ? mx_lo : mx_hi);
      // libdevice expf in both modes: with MUFU.EX2 (2 ulp) the bf16 pattern rounded the other way near half-ulp boundaries
      // often enough to put hook_pattern / hook_z measurably further from the fp32 truth than the reference's own bf16 path
      const float e = col < Tn ? expf(x) : 0.f;
      acc[nt][c] = e;
      if (c < 2) sum_lo += e; else sum_hi += e;
    }
  }
  sum_lo += __shfl_xor_sync(0xffffffffu, sum_lo, 1);
  sum_lo += __shfl_xor_sync(0xffffffffu, sum_lo, 2);
  sum_hi += __shfl_xor_sync(0xffffffffu, sum_hi, 1);
  sum_hi += __shfl_xor_sync(0xffffffffu, sum_hi, 2);
  const float rs_lo = 1.f / sum_lo, rs_hi = 1.f / sum_hi;   // one IEEE divide per row, then multiplies (<= 1.5 ulp of e / sum)
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int col = nt * 8 + 2 * t + (c & 1);
      float p = acc[nt][c] * (c < 2 ? rs_lo : rs_hi);
      if (isnan(p)) p = 0.f;
      acc[nt][c] = col < Tn ? round_to<T>(p) : 0.f;
    }
  }
  if (pattern) {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      stage_put2<T>(stage, g, nt * 8 + 2 * t, Tn, acc[nt][0], acc[nt][1]);
      if (g + 8 < nvalid) stage_put2<T>(stage, g + 8, nt * 8 + 2 * t, Tn, acc[nt][2], acc[nt][3]);
    }
    __syncwarp();
    copy_run<T>(pattern + sc_base, stage, nvalid * Tn, vb, lane);
    __syncwarp();
  }

  // ---- Z = P V  (P straight from the accumulator registers)
  float o[DH / 8][4];
#pragma unroll
  for (int nn = 0; nn < DH / 8; ++nn) o[nn][0] = o[nn][1] = o[nn][2] = o[nn][3] = 0.f;
  if constexpr (BF) {
#pragma unroll
    for (int kk = 0; kk < TPAD / 16; ++kk) {
      uint32_t a[4];
      a[0] = pack_bf16(acc[2 * kk][0], acc[2 * kk][1]);
      a[1] = pack_bf16(acc[2 * kk][2], acc[2 * kk][3]);
      a[2] = pack_bf16(acc[2 * kk + 1][0], acc[2 * kk + 1][1]);
      a[3] = pack_bf16(acc[2 * kk + 1][2], acc[2 * kk + 1][3]);
      // B (k = key, n = d_head) from row-major V through ldmatrix.trans: blocks [keys 0-7 | 8-15] x [d_head 8-column pair]
#pragma unroll
      for (int np = 0; np < DH / 16; ++np) {
        uint32_t bb[4];
        ldmatrix_x4_trans(bb, Vs + (size_t)(kk * 16 + (lane & 15)) * LD + np * 16 + 8 * (lane >> 4));
        mma_bf16(o[2 * np], a, bb[0], bb[1]);
        mma_bf16(o[2 * np + 1], a, bb[2], bb[3]);
      }
    }
  } else {
    const float* Vf = reinterpret_cast<const float*>(Vs);
#pragma unroll
    for (int kk = 0; kk < TPAD / 8; ++kk) {
      // k-slot t <-> key kk*8 + 2t, k-slot t+4 <-> key kk*8 + 2t + 1 (same permutation on A and B: the sum over k is unchanged)
      float a[4] = {acc[kk][0], acc[kk][2], acc[kk][1], acc[kk][3]};
#pragma unroll
      for (int nn = 0; nn < DH / 8; ++nn) {
        float bb[2];
        bb[0] = Vf[(kk * 8 + 2 * t) * LD + nn * 8 + g];
        bb[1] = Vf[(kk * 8 + 2 * t + 1) * LD + nn * 8 + g];
        mma_tf32x3(o[nn], a, bb);
      }
    }
  }
  // ---- z rows through the stage: [16][DH] packed -> each token row is 64 contiguous elements in [B,T,H,dh]
#pragma unroll
  for (int nn = 0; nn < DH / 8; ++nn) {
    stage_put2<T>(stage, g, nn * 8 + 2 * t, DH, o[nn][0], o[nn][1]);
    stage_put2<T>(stage, g + 8, nn * 8 + 2 * t, DH, o[nn][2], o[nn][3]);
  }
  __syncwarp();
  for (int i = lane; i < nvalid * VPR; i += 32) {
    const int r = i / VPR, e = (i % VPR) * VEC;
    *reinterpret_cast<uint4*>(z + head_base + (int64_t)(wrow0 + r) * tok_stride + e) = *reinterpret_cast<const uint4*>(stage + r * DH + e);
  }
}

int pow2_align(uint64_t x) {   // largest power of two <= 16 dividing x
  int a = 16;
  while (a > 1 && (x % (uint64_t)a)) a >>= 1;
  return a;
}

template <typename T, int NT, bool CAUSAL>
int launch_mma(const PbAttention* p, cudaStream_t st) {
  constexpr int NW = 4, TPAD = NT * 8;
  constexpr size_t es = sizeof(T);
  constexpr size_t smem = ((size_t)2 * TPAD * Lay<T>::LD + (size_t)NW * 16 * Lay<T>::LD + (size_t)NW * 16 * TPAD) * es;
  static_assert(smem <= 227 * 1024, "K, V, the Q slab and the stages must fit in shared memory");
  constexpr auto kern = k_attention_mma<T, NT, NW, CAUSAL>;
  PB_TRY(smem_opt_in<kern>(smem));
  // vector width of the score / pattern copy-out: every warp run starts at base + ((bh*T + 16*w) * T) elements
  int vb = pow2_align((uint64_t)p->T * p->T * es);
  vb = min(vb, pow2_align((uint64_t)16 * p->T * es));
  if (p->scores) vb = min(vb, pow2_align((uint64_t)(uintptr_t)p->scores));
  if (p->pattern) vb = min(vb, pow2_align((uint64_t)(uintptr_t)p->pattern));
  if (vb < 4) vb = 0;
  dim3 grid(p->B * p->H, (p->T + NW * 16 - 1) / (NW * 16));
  kern<<<grid, NW * 32, smem, st>>>((const T*)p->q, (const T*)p->k, (const T*)p->v, (T*)p->scores, (T*)p->pattern, (T*)p->z, p->T, p->H,
                                    p->attn_scale, pow2_inv_scale(p->attn_scale), vb);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

template <typename T, bool CAUSAL>
int dispatch_mma(const PbAttention* p, cudaStream_t st) {
  return p->T <= 64 ? launch_mma<T, 8, CAUSAL>(p, st) : launch_mma<T, 16, CAUSAL>(p, st);
}

}  // namespace

// d_head == 64, T <= 128, q / k / v / z 16-byte aligned: pb_attention (attention.cu) routes only such calls here
int pb_attention_mma(const PbAttention* p, cudaStream_t st) {
  if (p->causal) return p->dtype == PB_F32 ? dispatch_mma<float, true>(p, st) : dispatch_mma<bf16, true>(p, st);
  return p->dtype == PB_F32 ? dispatch_mma<float, false>(p, st) : dispatch_mma<bf16, false>(p, st);
}
