// attention_long.cu -- fused hooked attention for d_head == 64 and LONG sequences (T > 128: ViT-B/16 197, ViT-L/14 257 tokens).
//
// attention_mma.cu keeps a whole score row block in registers (NT key tiles) and the whole K / V of the head in shared memory.
// At T = 257 that is 136 accumulator registers per thread, 148 KB of fp32 K / V per CTA, two warps per CTA and one CTA per SM:
// the L/14 fp32 forward spent two thirds of its time there (DESIGN.md section 6).  This kernel streams K / V through shared
// memory in chunks of 64 keys and walks them twice:
//   pass 1: S_chunk = Q K_chunk^T -> scale, round -> [scores hook point] -> running row max m and sum l (online rescale);
//   pass 2: the same S_chunk again (bit-identical), P = round(exp(S - m) / l) -> [pattern hook point] -> Z += P V_chunk.
// QK^T is computed twice (7.7 MFLOP per image and layer more) in exchange for 32 accumulator registers, 3-6 CTAs per SM and
// K / V traffic that no longer scales with the number of query slabs per head beyond L2.  Rounding points are the reference's:
// scores = round(round(q.k) / scale), pattern = round(softmax), z = round(pattern @ v) with the rounded pattern as operand.
//
// Two more modes serve the split hooked stages (pb_attn_scores / pb_attn_pv) beyond the 608 tokens of the FFMA kernel:
//   LONG_SCORES: pass 1 alone, without the softmax statistics -> scores;
//   LONG_PV:     pass 2 with P read from a [B,H,T,T] pattern in 64-key chunks instead of computed -> z.
// Both share the fused mode's arithmetic and rounding points, so the scores equal the fused kernel's scores spill bit for bit, and
// the z of LONG_PV fed the fused kernel's own spilled pattern equals the fused kernel's z bit for bit.
//
// CAUSAL (fused mode only, the text towers' mask): keys j > query i score -inf, as scores / scale + mask does.  A CTA's query
// slab is one 64-row chunk, so key chunks past the slab lie wholly above the diagonal: neither pass loads or multiplies them,
// and a requested spill gets -inf / 0 there.  Every processed chunk has key kc0 <= each row of the slab, so the running max of
// a row is finite from chunk 0 on; masked entries are still kept out of the running sum explicitly.
#include "attention_frag.cuh"

namespace {

constexpr int KC = 64;                                    // keys per chunk
enum { LONG_FUSED = 0, LONG_SCORES = 1, LONG_PV = 2 };
__device__ __forceinline__ void stage_put(float* p, float a, float b) { p[0] = a; p[1] = b; }
__device__ __forceinline__ void stage_put(bf16* p, float a, float b) { *reinterpret_cast<uint32_t*>(p) = pack_bf16(a, b); }

// one warp's [16][KC] stage -> ncols columns of nvalid global rows (row stride Tn elements)
template <typename T>
__device__ __forceinline__ void copy_rows_out(T* __restrict__ gbase, int64_t row_stride, const T* stage, int nvalid, int ncols, int lane) {
  for (int r = 0; r < nvalid; ++r) {
    T* g = gbase + (int64_t)r * row_stride;
    const T* s = stage + r * KC;
    if (sizeof(T) == 4 || ((reinterpret_cast<uintptr_t>(g) & 3) == 0 && (ncols & 1) == 0)) {
      const int nw = ncols * (int)sizeof(T) / 4;             // 4-byte words
      for (int i = lane; i < nw; i += 32) reinterpret_cast<uint32_t*>(g)[i] = reinterpret_cast<const uint32_t*>(s)[i];
    } else {
      for (int i = lane; i < ncols; i += 32) g[i] = s[i];
    }
  }
}

// nvalid global rows of ncols columns (row stride Tn elements) -> one warp's [16][KC] stage; the rest of the stage is left as is
template <typename T>
__device__ __forceinline__ void copy_rows_in(T* stage, const T* __restrict__ gbase, int64_t row_stride, int nvalid, int ncols, int lane) {
  for (int r = 0; r < nvalid; ++r) {
    const T* g = gbase + (int64_t)r * row_stride;
    T* s = stage + r * KC;
    if (sizeof(T) == 4 || ((reinterpret_cast<uintptr_t>(g) & 3) == 0 && (ncols & 1) == 0)) {
      const int nw = ncols * (int)sizeof(T) / 4;
      for (int i = lane; i < nw; i += 32) reinterpret_cast<uint32_t*>(s)[i] = reinterpret_cast<const uint32_t*>(g)[i];
    } else {
      for (int i = lane; i < ncols; i += 32) s[i] = g[i];
    }
  }
}

template <typename T, int NW, int MODE, bool CAUSAL>
__global__ void __launch_bounds__(NW * 32) k_attention_long(const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v,
                                                           T* __restrict__ scores, T* __restrict__ pattern, T* __restrict__ z, int Tn, int H,
                                                           float attn_scale, float inv_scale) {
  constexpr bool BF = sizeof(T) == 2;
  constexpr int LD = Lay<T>::LD;
  constexpr int VEC = 16 / (int)sizeof(T);
  constexpr int VPR = DH / VEC;
  constexpr int NTC = KC / 8;                              // key tiles of 8 per chunk
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* Qs = reinterpret_cast<T*>(smem_raw);                  // [NW*16][LD]
  T* Ks = Qs + (size_t)NW * 16 * LD;                       // [KC][LD]
  T* Vs = Ks + (size_t)KC * LD;                            // [KC][LD]
  T* stage_all = Vs + (size_t)KC * LD;                     // [NW][16*KC]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int b = blockIdx.x / H, h = blockIdx.x % H;
  const int row0 = blockIdx.y * (NW * 16);
  const int64_t tok_stride = (int64_t)H * DH;
  const int64_t head_base = (int64_t)b * Tn * tok_stride + (int64_t)h * DH;
  const uint4 zero4 = make_uint4(0u, 0u, 0u, 0u);

  if (MODE != LONG_PV) {
    for (int idx = threadIdx.x; idx < NW * 16 * VPR; idx += NW * 32) {
      const int r = idx / VPR, e = (idx % VPR) * VEC;
      uint4 qv = zero4;
      if (row0 + r < Tn) qv = *reinterpret_cast<const uint4*>(q + head_base + (int64_t)(row0 + r) * tok_stride + e);
      *reinterpret_cast<uint4*>(Qs + (size_t)r * LD + e) = qv;
    }
    __syncthreads();
  }

  const int wrow0 = row0 + warp * 16;
  const bool active = wrow0 < Tn;                          // inactive warps still load chunks and hit the barriers
  const int nvalid = active ? min(16, Tn - wrow0) : 0;
  T* stage = stage_all + (size_t)warp * 16 * KC;
  const T* Qw = Qs + (size_t)warp * 16 * LD;

  // ---- Q fragments of this warp, kept in registers for both passes
  uint32_t qa[BF ? DH / 16 : DH / 8][4];                   // bf16: packed pairs; fp32: tf32 hi words
  uint32_t qal[BF ? 1 : DH / 8][4];                        // fp32: tf32 lo words
  if constexpr (MODE == LONG_PV) {
  } else if constexpr (BF) {
#pragma unroll
    for (int kk = 0; kk < DH / 16; ++kk) ldmatrix_x4(qa[kk], Qw + (size_t)(lane & 15) * LD + kk * 16 + 8 * (lane >> 4));
  } else {
    const float* Qf = reinterpret_cast<const float*>(Qw);
#pragma unroll
    for (int kk = 0; kk < DH / 8; ++kk) {
      const float a[4] = {Qf[g * LD + kk * 8 + t], Qf[(g + 8) * LD + kk * 8 + t], Qf[g * LD + kk * 8 + 4 + t], Qf[(g + 8) * LD + kk * 8 + 4 + t]};
#pragma unroll
      for (int i = 0; i < 4; ++i) { qa[kk][i] = __float_as_uint(a[i]); qal[kk][i] = __float_as_uint(tf32_lo(a[i])); }
    }
  }

  // causal: chunks starting past the slab's last query row are all -inf (written below when spilled) and are never loaded
  const int nchunks = CAUSAL ? min((Tn + KC - 1) / KC, (row0 + NW * 16 - 1) / KC + 1) : (Tn + KC - 1) / KC;
  const int64_t sc_row0 = ((int64_t)b * H + h) * Tn + wrow0;   // first score / pattern row of this warp
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
  float inv_lo = 0.f, inv_hi = 0.f;
  float o[DH / 8][4];
#pragma unroll
  for (int nn = 0; nn < DH / 8; ++nn) o[nn][0] = o[nn][1] = o[nn][2] = o[nn][3] = 0.f;

  // LONG_FUSED: passes 0 and 1; LONG_SCORES: pass 0 alone; LONG_PV: pass 1 alone
  constexpr int PASS_BEGIN = MODE == LONG_PV ? 1 : 0, PASS_END = MODE == LONG_SCORES ? 1 : 2;
#pragma unroll 1
  for (int pass = PASS_BEGIN; pass < PASS_END; ++pass) {
#pragma unroll 1
    for (int c = 0; c < nchunks; ++c) {
      const int kc0 = c * KC;
      __syncthreads();                                     // everyone is done with the previous chunk
      for (int idx = threadIdx.x; idx < KC * VPR; idx += NW * 32) {
        const int j = idx / VPR, e = (idx % VPR) * VEC;
        uint4 kv = zero4, vv = zero4;
        if (kc0 + j < Tn) {
          if (MODE != LONG_PV) kv = *reinterpret_cast<const uint4*>(k + head_base + (int64_t)(kc0 + j) * tok_stride + e);
          if (pass == 1) vv = *reinterpret_cast<const uint4*>(v + head_base + (int64_t)(kc0 + j) * tok_stride + e);
        }
        if (MODE != LONG_PV) *reinterpret_cast<uint4*>(Ks + (size_t)j * LD + e) = kv;
        if (pass == 1) *reinterpret_cast<uint4*>(Vs + (size_t)j * LD + e) = vv;
      }
      __syncthreads();
      if (!active) continue;

      // ---- S chunk = Q K_chunk^T (identical arithmetic in both passes); LONG_PV: the P chunk from the pattern instead
      float acc[NTC][4];
#pragma unroll
      for (int nt = 0; nt < NTC; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
      if constexpr (MODE == LONG_PV) {
        const int pcols = min(KC, Tn - kc0);
        copy_rows_in<T>(stage, pattern + sc_row0 * Tn + kc0, Tn, nvalid, pcols, lane);
        __syncwarp();
#pragma unroll
        for (int nt = 0; nt < NTC; ++nt)
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int row = g + (i < 2 ? 0 : 8), col = nt * 8 + 2 * t + (i & 1);
            acc[nt][i] = (row < nvalid && col < pcols) ? ld_as_float(stage + row * KC + col) : 0.f;
          }
        __syncwarp();
      } else if constexpr (BF) {
#pragma unroll
        for (int nt = 0; nt < NTC; ++nt) {
#pragma unroll
          for (int kp = 0; kp < DH / 32; ++kp) {
            uint32_t bb[4];
            ldmatrix_x4(bb, Ks + (size_t)(nt * 8 + (lane & 7)) * LD + kp * 32 + 8 * (lane >> 3));
            mma_bf16(acc[nt], qa[2 * kp], bb[0], bb[1]);
            mma_bf16(acc[nt], qa[2 * kp + 1], bb[2], bb[3]);
          }
        }
      } else {
        const float* Kf = reinterpret_cast<const float*>(Ks);
#pragma unroll
        for (int kk = 0; kk < DH / 8; ++kk) {
#pragma unroll
          for (int nt = 0; nt < NTC; ++nt) {
            const float bb[2] = {Kf[(nt * 8 + g) * LD + kk * 8 + t], Kf[(nt * 8 + g) * LD + kk * 8 + 4 + t]};
            mma_tf32x3_presplit(acc[nt], qa[kk], qal[kk], bb);
          }
        }
      }
      if (MODE == LONG_PV) {
      } else if (inv_scale != 0.f) {
#pragma unroll
        for (int nt = 0; nt < NTC; ++nt)
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[nt][i] = round_to<T>(round_to<T>(acc[nt][i]) * inv_scale);
      } else {
#pragma unroll
        for (int nt = 0; nt < NTC; ++nt)
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[nt][i] = round_to<T>(round_to<T>(acc[nt][i]) / attn_scale);
      }
      if constexpr (CAUSAL) {
#pragma unroll
        for (int nt = 0; nt < NTC; ++nt)
#pragma unroll
          for (int i = 0; i < 4; ++i)
            if (kc0 + nt * 8 + 2 * t + (i & 1) > wrow0 + g + (i < 2 ? 0 : 8)) acc[nt][i] = -INFINITY;
      }
      const int ncols = min(KC, Tn - kc0);

      if (pass == 0) {
        if (MODE == LONG_FUSED) {
          // ---- running max / sum over the valid keys of this chunk
          float cm_lo = -INFINITY, cm_hi = -INFINITY;
#pragma unroll
          for (int nt = 0; nt < NTC; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int col = nt * 8 + 2 * t + (i & 1);
              if (col < ncols) { if (i < 2) cm_lo = fmaxf(cm_lo, acc[nt][i]); else cm_hi = fmaxf(cm_hi, acc[nt][i]); }
            }
          cm_lo = fmaxf(cm_lo, __shfl_xor_sync(0xffffffffu, cm_lo, 1));
          cm_lo = fmaxf(cm_lo, __shfl_xor_sync(0xffffffffu, cm_lo, 2));
          cm_hi = fmaxf(cm_hi, __shfl_xor_sync(0xffffffffu, cm_hi, 1));
          cm_hi = fmaxf(cm_hi, __shfl_xor_sync(0xffffffffu, cm_hi, 2));
          const float mn_lo = fmaxf(m_lo, cm_lo), mn_hi = fmaxf(m_hi, cm_hi);
          // exp(-inf - finite) = 0 on the first chunk; a row of all -inf keeps m = -inf and l = NaN -> pattern 0 below, as the reference
          l_lo *= (m_lo == mn_lo) ? 1.f : (BF ? __expf(m_lo - mn_lo) : expf(m_lo - mn_lo));
          l_hi *= (m_hi == mn_hi) ? 1.f : (BF ? __expf(m_hi - mn_hi) : expf(m_hi - mn_hi));
          m_lo = mn_lo; m_hi = mn_hi;
#pragma unroll
          for (int nt = 0; nt < NTC; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int col = nt * 8 + 2 * t + (i & 1);
              if (col < ncols && (!CAUSAL || acc[nt][i] != -INFINITY)) {
                const float x = acc[nt][i] - (i < 2 ? m_lo : m_hi);
                const float e = BF ? __expf(x) : expf(x);
                if (i < 2) l_lo += e; else l_hi += e;
              }
            }
        }
        if (scores) {
#pragma unroll
          for (int nt = 0; nt < NTC; ++nt) {
            stage_put(stage + g * KC + nt * 8 + 2 * t, acc[nt][0], acc[nt][1]);
            stage_put(stage + (g + 8) * KC + nt * 8 + 2 * t, acc[nt][2], acc[nt][3]);
          }
          __syncwarp();
          copy_rows_out<T>(scores + sc_row0 * Tn + kc0, Tn, stage, nvalid, ncols, lane);
          __syncwarp();
        }
      } else {
        if (MODE == LONG_FUSED) {
          if (c == 0) {                                        // finish pass 1: per-row sum over the quad, one divide per row
            l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
            l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
            l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
            l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
            inv_lo = 1.f / l_lo; inv_hi = 1.f / l_hi;
          }
          // ---- P chunk = round(exp(S - m) / l), NaN -> 0 (attention.py:149), keys past T -> 0
#pragma unroll
          for (int nt = 0; nt < NTC; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int col = nt * 8 + 2 * t + (i & 1);
              const float x = acc[nt][i] - (i < 2 ? m_lo : m_hi);
              float p = (BF ? __expf(x) : expf(x)) * (i < 2 ? inv_lo : inv_hi);
              if (isnan(p)) p = 0.f;
              acc[nt][i] = col < ncols ? round_to<T>(p) : 0.f;
            }
          if (pattern) {
#pragma unroll
            for (int nt = 0; nt < NTC; ++nt) {
              stage_put(stage + g * KC + nt * 8 + 2 * t, acc[nt][0], acc[nt][1]);
              stage_put(stage + (g + 8) * KC + nt * 8 + 2 * t, acc[nt][2], acc[nt][3]);
            }
            __syncwarp();
            copy_rows_out<T>(pattern + sc_row0 * Tn + kc0, Tn, stage, nvalid, ncols, lane);
            __syncwarp();
          }
        }
        // ---- Z += P_chunk V_chunk
        if constexpr (BF) {
#pragma unroll
          for (int kk = 0; kk < KC / 16; ++kk) {
            uint32_t a[4];
            a[0] = pack_bf16(acc[2 * kk][0], acc[2 * kk][1]);
            a[1] = pack_bf16(acc[2 * kk][2], acc[2 * kk][3]);
            a[2] = pack_bf16(acc[2 * kk + 1][0], acc[2 * kk + 1][1]);
            a[3] = pack_bf16(acc[2 * kk + 1][2], acc[2 * kk + 1][3]);
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
          for (int kk = 0; kk < KC / 8; ++kk) {
            // k-slot t <-> key kk*8 + 2t, k-slot t+4 <-> key kk*8 + 2t + 1 (same permutation on A and B)
            const float a[4] = {acc[kk][0], acc[kk][2], acc[kk][1], acc[kk][3]};
#pragma unroll
            for (int nn = 0; nn < DH / 8; ++nn) {
              const float bb[2] = {Vf[(kk * 8 + 2 * t) * LD + nn * 8 + g], Vf[(kk * 8 + 2 * t + 1) * LD + nn * 8 + g]};
              mma_tf32x3(o[nn], a, bb);
            }
          }
        }
      }
    }
  }
  if constexpr (CAUSAL) {                                   // spilled regions of the skipped chunks: scores -inf, pattern 0
    const int c0 = nchunks * KC;
    if (active && c0 < Tn) {
      for (int r = 0; r < nvalid; ++r) {
        const int64_t rb = (sc_row0 + r) * Tn;
        for (int j = c0 + lane; j < Tn; j += 32) {
          if (scores) st_from_float(scores + rb + j, -INFINITY);
          if (pattern) st_from_float(pattern + rb + j, 0.f);
        }
      }
    }
  }
  if constexpr (MODE != LONG_SCORES) {
    if (!active) return;
    // ---- z rows: [16][DH] through the stage, 16-byte vectors per token row
#pragma unroll
    for (int nn = 0; nn < DH / 8; ++nn) {
      stage_put(stage + g * KC + nn * 8 + 2 * t, o[nn][0], o[nn][1]);
      stage_put(stage + (g + 8) * KC + nn * 8 + 2 * t, o[nn][2], o[nn][3]);
    }
    __syncwarp();
    for (int i = lane; i < nvalid * VPR; i += 32) {
      const int r = i / VPR, e = (i % VPR) * VEC;
      *reinterpret_cast<uint4*>(z + head_base + (int64_t)(wrow0 + r) * tok_stride + e) = *reinterpret_cast<const uint4*>(stage + r * KC + e);
    }
  }
}

template <typename T, int MODE, bool CAUSAL = false>
int launch_long(const PbAttention* p, cudaStream_t st) {
  constexpr int NW = 4;
  const size_t smem = ((size_t)(NW * 16 + 2 * KC) * Lay<T>::LD + (size_t)NW * 16 * KC) * sizeof(T);
  constexpr auto kern = k_attention_long<T, NW, MODE, CAUSAL>;
  PB_TRY(smem_opt_in<kern>(smem));
  dim3 grid(p->B * p->H, (p->T + NW * 16 - 1) / (NW * 16));
  kern<<<grid, NW * 32, smem, st>>>((const T*)p->q, (const T*)p->k, (const T*)p->v, (T*)p->scores, (T*)p->pattern, (T*)p->z, p->T, p->H,
                                    p->attn_scale, pow2_inv_scale(p->attn_scale));
  PB_LAUNCH_CHECK();
  return PB_OK;
}

}  // namespace

// d_head == 64 and 16-byte aligned q / k / v / z, any T: pb_attention (attention.cu) routes T > 128 here.
int pb_attention_long(const PbAttention* p, cudaStream_t st) {
  if (p->causal) return p->dtype == PB_F32 ? launch_long<float, LONG_FUSED, true>(p, st) : launch_long<bf16, LONG_FUSED, true>(p, st);
  return p->dtype == PB_F32 ? launch_long<float, LONG_FUSED>(p, st) : launch_long<bf16, LONG_FUSED>(p, st);
}

// The split stages for d_head == 64 with 16-byte aligned q / k (scores) or v / z (pv); attention.cu routes T > 608 here.
int pb_attn_scores_long(const PbAttention* p, cudaStream_t st) {
  return p->dtype == PB_F32 ? launch_long<float, LONG_SCORES>(p, st) : launch_long<bf16, LONG_SCORES>(p, st);
}
int pb_attn_pv_long(const PbAttention* p, cudaStream_t st) {
  return p->dtype == PB_F32 ? launch_long<float, LONG_PV>(p, st) : launch_long<bf16, LONG_PV>(p, st);
}
