// sae_fused.cu -- fused SAE encoder -> TopK for sm_90a: the dense pre-activation matrix hidden_pre [tokens, d_sae] is never
// written to HBM (reference sae/sae.py:557-581 `sae_in @ W_enc + b_enc` followed by TopK.forward :795-808 `torch.topk`).
//
// Approximate-then-rescore, exact by construction:
//   1. k_enc_cand     persistent wgmma GEMM, ONE pass at 11 significant bits, 128 x 256 tiles: a tile's columns are two 128-feature
//                     segments.  Either on the fp32 operands, read as tf32 (the tensor core ignores their 13 low mantissa bits), or
//                     on fp16 copies of them (round to nearest, clamped to +-65504): the same precision at half the bytes.  The
//                     GEMM is bound by the operand stream from L2 (3.6 GB per call at the bench shape in fp32), so the fp16 pass,
//                     which also runs at twice the tensor rate, takes about half the time.  The epilogue never stores the tile:
//                     per segment, every thread turns the 32 values it holds of each of its two token rows into packed keys (order-preserving int of the value, the low 7 bits replaced by the column inside the segment)
//                     and keeps the 8 largest with sorting networks, the four threads sharing a row merge their lists by
//                     shuffles, and one of them writes the first C_KEEP x 4 bytes.  Per token: d_sae / 128 segments x C_KEEP keys
//                     (6 KB at d_sae = 24576) instead of a 98 KB dense row.
//   2. k_cand_select  one CTA per token: the m_cand best keys of the row (threshold from per-thread bests, rank by counting),
//                     EXACT fp32 re-evaluation of those m_cand pre-activations (FFMA dot products against W_encT rows),
//                     exact top-k of the re-scored values (ties -> lower index, sorted descending), and a proof that no
//                     feature outside the candidate set can belong to the exact top-k:
//                         ub(best key not selected, or last kept key of a segment whose keys were all selected) + E_row < tau_k
//                     where E_row bounds |one-pass product - exact| by Cauchy-Schwarz on the operand residuals (a - read(a),
//                     w - read(w); each < 2^-10 relative for tf32 truncation, 2^-11 for fp16 rounding) plus the fp32 accumulation
//                     of the wgmma chain.  Rows that fail the proof go on a list.
//   3. k_topk_fallback  persistent, normally finds the list empty: recomputes a listed row's 'd_sae' pre-activations exactly and
//                     selects from all of them.  Correctness therefore never depends on the approximation; only speed does.
// Outputs are those of pb_sae_topk: idx int32 / val fp32 [rows][k] sorted by value, feat_count[f] += selections.
#include "tc_common.cuh"
#include "gemm_epi.cuh"
#include <limits.h>

namespace {

__device__ __forceinline__ int f2ord(float v) {           // monotone float -> signed int
  const int k = __float_as_int(v);
  return k ^ ((k >> 31) & 0x7fffffff);
}
__device__ __forceinline__ float ord2f(int k) { return __int_as_float(k ^ ((k >> 31) & 0x7fffffff)); }
__device__ __forceinline__ bool key_gt_f(float va, int ia, float vb, int ib) { return va > vb || (va == vb && ia < ib); }

constexpr int FZ_SEG = 128;                       // features per segment: the keys of a segment carry the column in 7 bits
constexpr int FZ_BM = 128;                        // tile rows: two consumer warpgroups of 64 tokens
constexpr int FZ_BN = 2 * FZ_SEG;                 // tile columns: two segments, one m64n256 accumulator (128 registers) per thread
constexpr int FZ_KSTEPS = 4;                      // one wgmma consumes 32 bytes of K per row: 8 fp32 (tf32 k8) or 16 fp16 (k16)
constexpr int FZ_A_BYTES = FZ_BM * 128;           // 16 KB
constexpr int FZ_STAGE_BYTES = FZ_A_BYTES + FZ_BN * 128;   // + 32 KB of W_encT
constexpr int FZ_STAGES = 4;                      // 4 x 48 KB = 192 KB operand ring
constexpr int FZ_SMEM = FZ_STAGES * FZ_STAGE_BYTES + 1024 + 256;

// ---- top-8 of a thread's keys by sorting networks (keys are distinct: the column sits in the low 7 bits)
__device__ __forceinline__ void key_cas(int& a, int& b) {   // a >= b afterwards
  const int hi = max(a, b);
  b = min(a, b);
  a = hi;
}
// v[0, 8) sorted descending: the optimal 19-comparator network for 8 inputs
__device__ __forceinline__ void key_sort8(int* v) {
  key_cas(v[0], v[2]); key_cas(v[1], v[3]); key_cas(v[4], v[6]); key_cas(v[5], v[7]);
  key_cas(v[0], v[4]); key_cas(v[1], v[5]); key_cas(v[2], v[6]); key_cas(v[3], v[7]);
  key_cas(v[0], v[1]); key_cas(v[2], v[3]); key_cas(v[4], v[5]); key_cas(v[6], v[7]);
  key_cas(v[2], v[4]); key_cas(v[3], v[5]);
  key_cas(v[1], v[4]); key_cas(v[3], v[6]);
  key_cas(v[1], v[2]); key_cas(v[3], v[4]); key_cas(v[5], v[6]);
}
// a, b sorted descending -> a = the 8 largest of both, sorted descending: a half-cleaner against reversed b leaves the top 8 as a
// bitonic sequence, which 12 comparators sort
__device__ __forceinline__ void key_merge8(int* a, const int* b) {
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = max(a[i], b[7 - i]);
  key_cas(a[0], a[4]); key_cas(a[1], a[5]); key_cas(a[2], a[6]); key_cas(a[3], a[7]);
  key_cas(a[0], a[2]); key_cas(a[1], a[3]); key_cas(a[4], a[6]); key_cas(a[5], a[7]);
  key_cas(a[0], a[1]); key_cas(a[2], a[3]); key_cas(a[4], a[5]); key_cas(a[6], a[7]);
}
// v[0, 32) -> v[0, 8) = the 8 largest, sorted descending
__device__ __forceinline__ void key_top8_of32(int (&v)[32]) {
  key_sort8(v); key_sort8(v + 8); key_sort8(v + 16); key_sort8(v + 24);
  key_merge8(v, v + 8);
  key_merge8(v + 16, v + 24);
  key_merge8(v, v + 16);
}

// T = float: tf32 wgmma on the fp32 operands; T = __half: fp16 wgmma on their fp16 copies.  A stage is a 128-byte k-slab of
// both operands either way (32 fp32 or 64 fp16 elements of K).
template <int C_KEEP, typename T>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_enc_cand(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int K, int M, int N,
           const float* __restrict__ bias, int* __restrict__ cand, int num_m_tiles, int num_n_tiles) {
  constexpr int FZ_BK = 128 / sizeof(T);
  pb_pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem0 = smem_u32(smem_raw);
  const uint32_t ring = (smem0 + 1023u) & ~1023u;
  const uint32_t bar_base = ring + FZ_STAGES * FZ_STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (FZ_STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int num_kb = (K + FZ_BK - 1) / FZ_BK;
  const int num_tiles = num_m_tiles * num_n_tiles;
  const int nseg = N / FZ_SEG;
  // m-fastest raster: the CTAs in flight share one 256-feature slab of the dictionary and walk the token tiles, so W_encT
  // (75 MB at d_sae = 24576) streams from HBM once while sae_in (12.6 MB) stays L2-resident.
  auto tile_m = [&](int tile) { return tile % num_m_tiles; };
  auto tile_n = [&](int tile) { return tile / num_m_tiles; };

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < FZ_STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pb_pdl_wait();            // barriers initialised, tensor maps prefetched: now the prep kernel's sae_in must be complete

  if (wg == 0) {
    // ===================== TMA producer =====================
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = tile_m(tile) * FZ_BM, n0 = tile_n(tile) * FZ_BN;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % FZ_STAGES;
          const uint32_t ph = (it / FZ_STAGES) & 1;
          mbar_wait<false>(empty_bar(s), ph ^ 1);
          mbar_expect_tx(full_bar(s), FZ_STAGE_BYTES);       // a box reaching past M or F still delivers (zero-filled) full bytes
          const uint32_t sa = ring + s * FZ_STAGE_BYTES;
          tma_load_2d(sa, &tmA, full_bar(s), kb * FZ_BK, m0);
          tma_load_2d(sa + FZ_A_BYTES, &tmB, full_bar(s), kb * FZ_BK, n0);
        }
      }
    }
    return;
  }
  // ===================== consumers: one pass, then per-row top-C_KEEP of each segment as packed keys =====================
  reg_alloc<232>();
  const int c = wg - 1, wq = warp & 3, tid = threadIdx.x & 127;
  float acc[128];
  uint32_t it = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m0 = tile_m(tile) * FZ_BM, n0 = tile_n(tile) * FZ_BN;
    int prev_s = -1;
    for (int kb = 0; kb < num_kb; ++kb, ++it) {
      const int s = it % FZ_STAGES;
      const uint32_t ph = (it / FZ_STAGES) & 1;
      mbar_wait<false>(full_bar(s), ph);
      const uint32_t sa = ring + s * FZ_STAGE_BYTES + c * 64 * 128;
      const uint32_t sb = ring + s * FZ_STAGE_BYTES + FZ_A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < FZ_KSTEPS; ++k) {
        if constexpr (sizeof(T) == 2) wgmma_f16_n256(acc, make_smem_desc(sa + 32 * k), make_smem_desc(sb + 32 * k), (kb | k) != 0 ? 1u : 0u);
        else wgmma_tf32_n256(acc, make_smem_desc(sa + 32 * k), make_smem_desc(sb + 32 * k), (kb | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev_s >= 0 && tid == 0) mbar_arrive(empty_bar(prev_s));
      prev_s = s;
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    if (tid == 0) mbar_arrive(empty_bar(prev_s));

    // accumulator element i of this thread: row 16 wq + lane / 4 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (lane % 4) + (i & 1);
    // segment g of the tile is elements [64 g, 64 g + 64).  Only one segment's key lists are live at a time.
    const int row = m0 + 64 * c + 16 * wq + (lane >> 2);
#pragma unroll
    for (int g = 0; g < 2; ++g) {
      const int f0 = n0 + g * FZ_SEG;
      if (f0 >= N) break;                            // F is a multiple of 128, not of 256: the last tile's second half is empty
      int s0[32], s1[32];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
        const float2 bb = *reinterpret_cast<const float2*>(bias + f0 + col);
        const float* a = acc + 64 * g + 4 * j;
        s0[2 * j] = (f2ord(a[0] + bb.x) & ~127) | col;
        s0[2 * j + 1] = (f2ord(a[1] + bb.y) & ~127) | (col + 1);
        s1[2 * j] = (f2ord(a[2] + bb.x) & ~127) | col;
        s1[2 * j + 1] = (f2ord(a[3] + bb.y) & ~127) | (col + 1);
      }
      key_top8_of32(s0);
      key_top8_of32(s1);
      // the four lanes of a quad hold disjoint columns of the same two rows: merge their lists (keys are distinct)
#pragma unroll
      for (int off = 1; off <= 2; off <<= 1) {
        int t0[8], t1[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) { t0[i] = __shfl_xor_sync(0xffffffffu, s0[i], off); t1[i] = __shfl_xor_sync(0xffffffffu, s1[i], off); }
        key_merge8(s0, t0);
        key_merge8(s1, t1);
      }
      if ((lane & 3) == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int* sv = h == 0 ? s0 : s1;
          if (row + 8 * h < M) {
            int* dst = cand + ((int64_t)(row + 8 * h) * nseg + f0 / FZ_SEG) * C_KEEP;
            if (C_KEEP % 4 == 0) {
#pragma unroll
              for (int i = 0; i < C_KEEP / 4; ++i) reinterpret_cast<int4*>(dst)[i] = make_int4(sv[4 * i], sv[4 * i + 1], sv[4 * i + 2], sv[4 * i + 3]);
            } else {
#pragma unroll
              for (int i = 0; i < C_KEEP / 2; ++i) reinterpret_cast<int2*>(dst)[i] = make_int2(sv[2 * i], sv[2 * i + 1]);
            }
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// exact fp32 dot products of one shared-memory row with rows of W (16-byte loads, one warp per dot, two dots in flight)
__device__ __forceinline__ float warp_dot(const float4* __restrict__ a4, const float4* __restrict__ w4, int nvec, int lane) {
  float acc = 0.f;
  for (int i = lane; i < nvec; i += 32) {
    const float4 a = a4[i], w = __ldg(w4 + i);
    acc = fmaf(a.x, w.x, acc); acc = fmaf(a.y, w.y, acc); acc = fmaf(a.z, w.z, acc); acc = fmaf(a.w, w.w, acc);
  }
  return warp_sum(acc);
}
__device__ __forceinline__ void warp_dot2(const float4* __restrict__ a4, const float4* __restrict__ w0, const float4* __restrict__ w1, int nvec,
                                          int lane, float& o0, float& o1) {
  float x = 0.f, y = 0.f;
  for (int i = lane; i < nvec; i += 32) {
    const float4 a = a4[i], u = __ldg(w0 + i), v = __ldg(w1 + i);
    x = fmaf(a.x, u.x, x); x = fmaf(a.y, u.y, x); x = fmaf(a.z, u.z, x); x = fmaf(a.w, u.w, x);
    y = fmaf(a.x, v.x, y); y = fmaf(a.y, v.y, y); y = fmaf(a.z, v.z, y); y = fmaf(a.w, v.w, y);
  }
  o0 = warp_sum(x);
  o1 = warp_sum(y);
}

constexpr int SEL_MAX_CAND = 128;   // most candidates one row may re-score before it gives up and takes the exact path
constexpr int SEL_EXTEND = 16;      // candidates added per extension round
constexpr int SEL_TAU_RANK = 96;    // the gather threshold keeps at least this many keys (typically 1.2-1.5x as many)
constexpr int SEL_SLOTS = 512;      // gathered keys that can be sorted; more (massive ties) -> exact path

__device__ __forceinline__ unsigned long long sel_pack(int key, int pos) {    // orders like (key descending-first, pos ascending-first)
  return ((unsigned long long)((unsigned)key ^ 0x80000000u) << 32) | (unsigned)(0xFFFFFFFFu - (unsigned)pos);
}
__device__ __forceinline__ int sel_key(unsigned long long it) { return (int)((unsigned)(it >> 32) ^ 0x80000000u); }
__device__ __forceinline__ int sel_pos(unsigned long long it) { return (int)(0xFFFFFFFFu - (unsigned)it); }

// One CTA (256 threads) per token row.  dynamic smem: a_row[d]
//   1. threshold: every warp bitonic-sorts its 32 per-thread bests (= segment maxima) in registers and reports its q-th largest;
//      the smallest report is a key with at least SEL_TAU_RANK keys of the row at or above it;
//   2. gather the keys >= threshold (packed with their position) and bitonic-sort them in shared memory (256 or 512 slots);
//   3. rounds: exactly re-score the first m_cur sorted candidates (m_cand, then +16 per round), take the exact top-k of those,
//      and try to prove no other feature can beat the k-th:   ub(best key not yet re-scored) + E_row < tau_k.  Most rows are
//      proven in the first round; a row that runs out of sorted candidates (or whose segment kept-lists saturate) is listed.
// (A first version ranked by counting -- 256^2 + G^2 shared-memory compares per row -- and was ALU-bound.)
template <int SPT>
__global__ void __launch_bounds__(256) k_cand_select(const int* __restrict__ cand, int nseg, int c_keep, const float* __restrict__ sae_in,
                                                     const float* __restrict__ W_encT, const float* __restrict__ b_enc,
                                                     const float* __restrict__ wnorm_max, const float* __restrict__ wlo_max, int f16,
                                                     float acc_units, float err_scale, int d, int k, int m_cand,
                                                     int* __restrict__ out_idx, float* __restrict__ out_val, float* __restrict__ feat_count,
                                                     int* __restrict__ fb_count, int* __restrict__ fb_rows, int* __restrict__ stats) {
  pb_pdl();
  extern __shared__ __align__(16) unsigned char sm_raw[];
  float* a_row = reinterpret_cast<float*>(sm_raw);
  __shared__ unsigned long long items[SEL_SLOTS];
  __shared__ int ex_idx[SEL_MAX_CAND], win_idx[64], warp_tau[8];
  __shared__ float ex_val[SEL_MAX_CAND];
  __shared__ float red[2][8];
  __shared__ int g_n, u_below, sat_key;
  __shared__ float tau_exact, a_norm, a_lo_norm;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int row = blockIdx.x;
  const int nvec = d >> 2;
  const int nkeys = nseg * c_keep;

  // ---- the token's encoder input -> shared memory; ||a|| and ||a - read(a)|| (tf32 truncation or fp16 rounding) for the error bound
  {
    const float4* src = reinterpret_cast<const float4*>(sae_in + (int64_t)row * d);
    float4* dst = reinterpret_cast<float4*>(a_row);
    float nsq = 0.f, lsq = 0.f;
    for (int i = t; i < nvec; i += 256) {
      const float4 v = src[i];
      dst[i] = v;
      nsq += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
      if (f16) {
        const float q[4] = {v.x, v.y, v.z, v.w};
        f16x4(q, lsq);
      } else {
        const float lx = v.x - tf32_trunc(v.x), ly = v.y - tf32_trunc(v.y), lz = v.z - tf32_trunc(v.z), lw = v.w - tf32_trunc(v.w);
        lsq += lx * lx + ly * ly + lz * lz + lw * lw;
      }
    }
    nsq = warp_sum(nsq);
    lsq = warp_sum(lsq);
    if (lane == 0) { red[0][warp] = nsq; red[1][warp] = lsq; }
  }
  // ---- keys of this row.  Thread t owns WHOLE segments t, t + 256, ... (their c_keep keys, sorted descending by the GEMM
  // epilogue), so a thread's best key is the largest segment maximum it holds.
  int key[SPT][8];
  int bk = INT_MIN;
  const int* kr = cand + (int64_t)row * nkeys;
#pragma unroll
  for (int i = 0; i < SPT; ++i) {
    const int sg = t + 256 * i;
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
      int2 v = make_int2(INT_MIN, INT_MIN);
      if (sg < nseg && j < c_keep) v = *reinterpret_cast<const int2*>(kr + sg * c_keep + j);
      key[i][j] = v.x;
      key[i][j + 1] = v.y;
    }
    bk = max(bk, key[i][0]);
  }
  // ---- threshold.  Warp w holds cnt_w = clamp(nthr - 32 w, 0, 32) valid bests (nthr = threads that own a segment); its quota
  // q_w = ceil(m_tau cnt_w / nthr) of them are >= its q_w-th largest, and the quotas add up to >= m_tau.
  {
    int v = bk;                                     // bitonic sort across the warp, descending: lane i ends with the i-th largest
#pragma unroll
    for (int kk = 2; kk <= 32; kk <<= 1) {
#pragma unroll
      for (int j = kk >> 1; j > 0; j >>= 1) {
        const int o = __shfl_xor_sync(0xffffffffu, v, j);
        const bool keep_max = ((lane & kk) == 0) == ((lane & j) == 0);
        v = keep_max ? max(v, o) : min(v, o);
      }
    }
    const int nthr = min(256, nseg);
    const int m_tau = min(SEL_TAU_RANK, nthr);
    const int cnt_w = max(0, min(32, nthr - 32 * warp));
    const int q_w = (m_tau * cnt_w + nthr - 1) / nthr;
    const int rep = __shfl_sync(0xffffffffu, v, max(q_w - 1, 0));
    if (lane == 0) warp_tau[warp] = q_w > 0 ? rep : INT_MAX;
  }
  if (t == 0) { g_n = 0; u_below = INT_MIN; }
  __syncthreads();
  if (t == 0) {
    float s0 = 0.f, s1 = 0.f;
    for (int i = 0; i < 8; ++i) { s0 += red[0][i]; s1 += red[1][i]; }
    a_norm = sqrtf(s0);
    a_lo_norm = sqrtf(s1);
  }
  int tau = INT_MAX;
#pragma unroll
  for (int w = 0; w < 8; ++w) tau = min(tau, warp_tau[w]);
  // ---- gather
  int lower = INT_MIN;                              // best key of this thread below tau
#pragma unroll
  for (int i = 0; i < SPT; ++i) {
    const int sg = t + 256 * i;
    if (sg < nseg) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (j < c_keep) {
          if (key[i][j] >= tau) {
            const int slot = atomicAdd(&g_n, 1);
            if (slot < SEL_SLOTS) items[slot] = sel_pack(key[i][j], sg * c_keep + j);
          } else {
            lower = max(lower, key[i][j]);
          }
        }
      }
    }
  }
  if (lower != INT_MIN) atomicMax(&u_below, lower);
  __syncthreads();
  const bool overflow = g_n > SEL_SLOTS;            // only with massive ties (e.g. constant rows): such rows take the exact path
  const int G = min(g_n, SEL_SLOTS);
  const int n_sort = G <= 256 ? 256 : SEL_SLOTS;
  for (int i = G + t; i < n_sort; i += 256) items[i] = 0ull;     // padding sorts last
  __syncthreads();
  // ---- bitonic sort of items[0, n_sort), descending
  for (int kk = 2; kk <= n_sort; kk <<= 1) {
    for (int j = kk >> 1; j > 0; j >>= 1) {
      for (int p = t; p < (n_sort >> 1); p += 256) {
        const int i = 2 * j * (p / j) + (p % j);
        const int o = i + j;
        const unsigned long long x = items[i], y = items[o];
        const bool desc = (i & kk) == 0;
        if ((x < y) == desc) { items[i] = y; items[o] = x; }
      }
      __syncthreads();
    }
  }
  const int Gs = min(G, SEL_MAX_CAND);
  const float4* a4 = reinterpret_cast<const float4*>(a_row);
  int m_prev = 0, m_cur = min(m_cand, Gs);
  bool ok = false;
  for (;;) {
    if (t == 0) sat_key = INT_MIN;
    // ---- exact re-evaluation of candidates [m_prev, m_cur): hidden_pre[f] = <sae_in, W_enc[:, f]> + b_enc[f]   (sae.py:568-574)
    for (int c = m_prev + 2 * warp; c < m_cur; c += 16) {
      const unsigned long long it0 = items[c];
      const int f0 = (sel_pos(it0) / c_keep) * FZ_SEG + (sel_key(it0) & 127);
      if (c + 1 < m_cur) {
        const unsigned long long it1 = items[c + 1];
        const int f1 = (sel_pos(it1) / c_keep) * FZ_SEG + (sel_key(it1) & 127);
        float v0, v1;
        warp_dot2(a4, reinterpret_cast<const float4*>(W_encT + (int64_t)f0 * d), reinterpret_cast<const float4*>(W_encT + (int64_t)f1 * d), nvec,
                  lane, v0, v1);
        if (lane == 0) { ex_val[c] = v0 + b_enc[f0]; ex_idx[c] = f0; ex_val[c + 1] = v1 + b_enc[f1]; ex_idx[c + 1] = f1; }
      } else {
        const float v0 = warp_dot(a4, reinterpret_cast<const float4*>(W_encT + (int64_t)f0 * d), nvec, lane);
        if (lane == 0) { ex_val[c] = v0 + b_enc[f0]; ex_idx[c] = f0; }
      }
    }
    __syncthreads();
    // ---- exact top-k among the first m_cur candidates (sorted descending, ties -> lower index)
    if (t < m_cur) {
      const float v = ex_val[t];
      const int f = ex_idx[t];
      int rank = 0;
      for (int j = 0; j < m_cur; ++j) rank += key_gt_f(ex_val[j], ex_idx[j], v, f) ? 1 : 0;
      if (rank < k) {
        out_idx[(int64_t)row * k + rank] = f;
        out_val[(int64_t)row * k + rank] = v;
        win_idx[rank] = f;
        if (rank == k - 1) tau_exact = v;
      }
    }
    // a segment whose c_keep kept keys were ALL re-scored may have dropped a value as large as its last kept key
    if (m_cur > 0) {
      const int key_m = sel_key(items[m_cur - 1]);
      int sat = INT_MIN;
#pragma unroll
      for (int i = 0; i < SPT; ++i) {
        if (t + 256 * i < nseg) {
          int last = key[i][3];                    // last kept key of the segment: slot c_keep - 1
          if (c_keep == 6) last = key[i][5];
          if (c_keep == 8) last = key[i][7];
          if (last >= key_m) sat = max(sat, last);
        }
      }
      if (sat != INT_MIN) atomicMax(&sat_key, sat);
    }
    __syncthreads();
    // ---- proof of completeness for this round
    {
      const int u_rest = m_cur < G ? sel_key(items[m_cur]) : u_below;                      // best key not re-scored
      const int u = max(u_rest, sat_key);
      const float u_val = u == INT_MIN ? -INFINITY : ord2f((u & ~127) | 127);               // upper end of the key's value bucket
      // |one-pass product - exact| = |a_lo.w + a_hi.w_lo| <= ||a_lo|| max||w|| + ||a|| max||w_lo||   (Cauchy-Schwarz, per row;
      // a_hi / w_hi = what the tensor core reads, a_lo / w_lo = the residuals)
      // + the fp32 accumulation of the wgmma chain: acc_units = ceil(d / 8) tf32 k-steps x 4 units of 2^-23, or ceil(d / 16) fp16
      //   k-steps x 8 units, of the magnitudes entering a step (accumulator and 8 or 16 products: an alignment that truncates
      //   instead of rounding costs 2 units, the rest is margin), every one of them bounded by sum_i |a_i w_i| <= ||a|| max||w||
      const float acc_err = acc_units * 1.19209290e-7f * a_norm * wnorm_max[0];
      const float E = err_scale * (a_lo_norm * wnorm_max[0] + a_norm * wlo_max[0]) + acc_err + fabsf(tau_exact) * 1.2207031e-4f;
      ok = !overflow && m_cur >= k && (u_val + E < tau_exact);
    }
    if (ok || m_cur >= Gs) break;
    __syncthreads();                                // everybody has read sat_key / tau_exact of this round
    m_prev = m_cur;
    m_cur = min(m_cur + SEL_EXTEND, Gs);
  }
  if (ok) {
    if (t < k && feat_count) atomicAdd(feat_count + win_idx[t], 1.0f);
    if (stats && t == 0) atomicAdd(stats, m_cur);                 // candidates re-scored, summed over the proven rows
  } else if (t == 0) {
    fb_rows[atomicAdd(fb_count, 1)] = row;
  }
}

// Exact path for listed rows: hidden row recomputed with FFMA into this CTA's scratch row, then exact selection from all F values.
// dynamic smem: a_row[d] | cand_v[cap] | cand_i[cap]
__global__ void __launch_bounds__(256) k_topk_fallback(const int* __restrict__ fb_count, const int* __restrict__ fb_rows,
                                                       const float* __restrict__ sae_in, const float* __restrict__ W_encT,
                                                       const float* __restrict__ b_enc, float* __restrict__ scratch, int d, int F, int k, int cap,
                                                       int* __restrict__ out_idx, float* __restrict__ out_val, float* __restrict__ feat_count) {
  pb_pdl();
  const int n_items = *fb_count;
  if (n_items == 0) return;
  extern __shared__ __align__(16) unsigned char sm_raw[];
  float* a_row = reinterpret_cast<float*>(sm_raw);
  float* cand_v = a_row + d;
  int* cand_i = reinterpret_cast<int*>(cand_v + cap);
  __shared__ float best_v[256];
  __shared__ int best_i[256];
  __shared__ float tau_v;
  __shared__ int tau_i, cand_n;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int nvec = d >> 2;
  float* h = scratch + (int64_t)blockIdx.x * F;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int row = fb_rows[item];
    __syncthreads();
    for (int i = t; i < nvec; i += 256) reinterpret_cast<float4*>(a_row)[i] = reinterpret_cast<const float4*>(sae_in + (int64_t)row * d)[i];
    if (t == 0) cand_n = 0;
    __syncthreads();
    const float4* a4 = reinterpret_cast<const float4*>(a_row);
    for (int f = 2 * warp; f < F; f += 16) {
      float v0, v1;
      warp_dot2(a4, reinterpret_cast<const float4*>(W_encT + (int64_t)f * d), reinterpret_cast<const float4*>(W_encT + (int64_t)(f + 1) * d), nvec, lane,
                v0, v1);
      if (lane == 0) { h[f] = v0 + b_enc[f]; h[f + 1] = v1 + b_enc[f + 1]; }
    }
    __syncthreads();
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int p = t; p < F; p += 256) {
      const float v = h[p];
      if (key_gt_f(v, p, bv, bi)) { bv = v; bi = p; }
    }
    best_v[t] = bv;
    best_i[t] = bi;
    __syncthreads();
    {
      int rank = 0;
      for (int j = 0; j < 256; ++j) rank += key_gt_f(best_v[j], best_i[j], bv, bi) ? 1 : 0;
      if (rank == min(k, 256) - 1) { tau_v = bv; tau_i = bi; }
    }
    __syncthreads();
    const float tv = tau_v;
    const int ti = tau_i;
    for (int p = t; p < F; p += 256) {
      const float v = h[p];
      if (!key_gt_f(tv, ti, v, p)) {
        const int slot = atomicAdd(&cand_n, 1);
        if (slot < cap) { cand_v[slot] = v; cand_i[slot] = p; }
      }
    }
    __syncthreads();
    const int C = min(cand_n, cap);
    for (int c = t; c < C; c += 256) {
      const float cv = cand_v[c];
      const int ci = cand_i[c];
      int rank = 0;
      for (int j = 0; j < C; ++j) rank += key_gt_f(cand_v[j], cand_i[j], cv, ci) ? 1 : 0;
      if (rank < k) {
        out_idx[(int64_t)row * k + rank] = ci;
        out_val[(int64_t)row * k + rank] = cv;
        if (feat_count) atomicAdd(feat_count + ci, 1.0f);
      }
    }
  }
}

// out[0] = max_f ||W[f, :]||_2, out[1] = max_f ||W[f, :] - tf32_trunc(W[f, :])||_2 (atomic max on the bit patterns: norms are
// non-negative); out must be zeroed by the caller
__global__ void __launch_bounds__(256) k_rownorm_max(const float* __restrict__ W, int F, int d, float* __restrict__ out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int nvec = d >> 2;
  float best = 0.f, best_lo = 0.f;
  for (int f = blockIdx.x * nw + warp; f < F; f += gridDim.x * nw) {
    const float4* w4 = reinterpret_cast<const float4*>(W + (int64_t)f * d);
    float s = 0.f, l = 0.f;
    for (int i = lane; i < nvec; i += 32) {
      const float4 v = w4[i];
      s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
      const float lx = v.x - tf32_trunc(v.x), ly = v.y - tf32_trunc(v.y), lz = v.z - tf32_trunc(v.z), lw = v.w - tf32_trunc(v.w);
      l += lx * lx + ly * ly + lz * lz + lw * lw;
    }
    best = fmaxf(best, warp_sum(s));
    best_lo = fmaxf(best_lo, warp_sum(l));
  }
  if (lane == 0 && best > 0.f) {
    atomicMax(reinterpret_cast<unsigned int*>(out), __float_as_uint(sqrtf(best)));
    atomicMax(reinterpret_cast<unsigned int*>(out) + 1, __float_as_uint(sqrtf(best_lo)));
  }
}

// W16 = fp16 copy of W [rows][d]; lo_max[0] = max_r ||W[r,:] - W16[r,:]|| (atomic max on the bit patterns; zeroed by the caller)
__global__ void __launch_bounds__(256) k_f16_copy(const float* __restrict__ W, int64_t rows, int d, __half* __restrict__ W16, float* __restrict__ lo_max) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int nvec = d >> 2;
  float best = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * nw + warp; r < rows; r += (int64_t)gridDim.x * nw) {
    float l = 0.f;
    for (int i = lane; i < nvec; i += 32) {
      float v[4];
      ld4(W + r * d + 4 * i, v);
      *reinterpret_cast<uint2*>(W16 + r * d + 4 * i) = f16x4(v, l);
    }
    best = fmaxf(best, warp_sum(l));
  }
  if (lo_max && lane == 0 && best > 0.f) atomicMax(reinterpret_cast<unsigned int*>(lo_max), __float_as_uint(sqrtf(best)));
}

template <int C_KEEP, typename T>
int launch_enc_cand(const PbSaeEncode* e, cudaStream_t st) {
  constexpr bool F16 = sizeof(T) == 2;
  CUtensorMap tmA, tmB;
  PB_TRY(make_map(&tmA, F16 ? e->sae_in16 : (const void*)e->sae_in, F16 ? PB_F16 : PB_F32, e->rows, e->d, e->d, FZ_BM));
  PB_TRY(make_map(&tmB, F16 ? e->W_encT16 : (const void*)e->W_encT, F16 ? PB_F16 : PB_F32, e->F, e->d, e->d, FZ_BN));
  auto kern = k_enc_cand<C_KEEP, T>;
  static bool attr_done = false;
  if (!attr_done) {
    PB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, FZ_SMEM));
    attr_done = true;
  }
  const int num_m = (e->rows + FZ_BM - 1) / FZ_BM, num_n = (e->F + FZ_BN - 1) / FZ_BN;
  int grid = pb_sm_count();
  if (grid > num_m * num_n) grid = num_m * num_n;
  PB_LAUNCH_PDL(kern, grid, TC_THREADS, FZ_SMEM, st, tmA, tmB, e->d, e->rows, e->F, e->b_enc, e->cand, num_m, num_n);
  return PB_OK;
}

template <int SPT>
int launch_select(const PbSaeEncode* e, bool f16, int nseg, float scale, cudaStream_t st) {
  const size_t smem = sizeof(float) * e->d;
  const float acc_units = f16 ? 8.f * (float)((e->d + 15) / 16) : 4.f * (float)((e->d + 7) / 8);
  PB_LAUNCH_PDL(k_cand_select<SPT>, e->rows, 256, smem, st, (const int*)e->cand, nseg, e->c_keep, e->sae_in, e->W_encT, e->b_enc, e->enc_norm_max,
                f16 ? e->enc16_lo_max : e->enc_norm_max + 1, (int)f16, acc_units, scale, e->d, e->k, e->m_cand, e->idx, e->val, e->feat_count,
                e->fb_count, e->fb_rows, e->fb_count + 1);
  return PB_OK;
}

}  // namespace

extern "C" int pb_sae_fused_workspace(int32_t rows, int32_t F, int32_t c_keep, int64_t* cand_bytes, int64_t* fb_scratch_bytes) {
  PB_CHECK_ARG(rows >= 0 && F > 0 && F % FZ_SEG == 0 && (c_keep == 4 || c_keep == 6 || c_keep == 8) && cand_bytes && fb_scratch_bytes,
               "pb_sae_fused_workspace: needs d_sae %% 128 == 0 and c_keep in {4, 6, 8}");
  *cand_bytes = (int64_t)rows * (F / FZ_SEG) * c_keep * 4;
  *fb_scratch_bytes = (int64_t)2 * pb_sm_count() * F * 4;
  return PB_OK;
}

extern "C" int pb_sae_encode_topk_fused(const PbSaeEncode* e, pb_stream_t stream) {
  PB_CHECK_ARG(e && e->sae_in && e->W_encT && e->b_enc && e->cand && e->enc_norm_max && e->idx && e->val && e->fb_count && e->fb_rows,
               "pb_sae_encode_topk_fused: missing pointers");
  PB_CHECK_ARG(e->rows >= 0 && e->d >= 32 && e->d % 4 == 0 && e->d <= 8192 && e->F % FZ_SEG == 0 && e->F >= FZ_SEG,
               "pb_sae_encode_topk_fused: needs d_in %% 4 == 0, 32 <= d_in <= 8192, d_sae %% 128 == 0 (d=%d F=%d)", e->d, e->F);
  PB_CHECK_ARG(e->c_keep == 4 || e->c_keep == 6 || e->c_keep == 8, "pb_sae_encode_topk_fused: c_keep must be 4, 6 or 8");
  PB_CHECK_ARG(e->k >= 1 && e->k <= 64 && e->k <= e->m_cand && e->m_cand <= SEL_MAX_CAND && e->k <= e->F,
               "pb_sae_encode_topk_fused: needs k <= 64 and k <= m_cand <= %d", SEL_MAX_CAND);
  PB_CHECK_ARG(pb_aligned16(e->sae_in) && pb_aligned16(e->W_encT) && pb_aligned16(e->b_enc) && pb_aligned16(e->cand),
               "pb_sae_encode_topk_fused: operands must be 16-byte aligned");
  const int nkeys = e->F / FZ_SEG * e->c_keep;
  PB_CHECK_ARG(e->F / FZ_SEG <= 256 * 4, "pb_sae_encode_topk_fused: d_sae=%d too large for the selection kernel (max 131072)", e->F);
  PB_CHECK_ARG(e->cand_bytes >= (int64_t)e->rows * nkeys * 4, "pb_sae_encode_topk_fused: candidate buffer too small");
  const bool f16 = e->sae_in16 != nullptr;
  PB_CHECK_ARG(f16 == (e->W_encT16 != nullptr) && f16 == (e->enc16_lo_max != nullptr),
               "pb_sae_encode_topk_fused: sae_in16, W_encT16 and enc16_lo_max go together");
  PB_CHECK_ARG(!f16 || (e->d % 8 == 0 && pb_aligned16(e->sae_in16) && pb_aligned16(e->W_encT16)),
               "pb_sae_encode_topk_fused: the fp16 candidate GEMM needs d_in %% 8 == 0 and 16-byte aligned fp16 operands (d=%d)", e->d);
  if (e->rows == 0) return PB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int phases = (e->phases & 7) ? e->phases : (e->phases | 7);
  if (phases & 1) {
    if (f16) {
      if (e->c_keep == 4) PB_TRY((launch_enc_cand<4, __half>(e, st)));
      else if (e->c_keep == 6) PB_TRY((launch_enc_cand<6, __half>(e, st)));
      else PB_TRY((launch_enc_cand<8, __half>(e, st)));
    } else {
      if (e->c_keep == 4) PB_TRY((launch_enc_cand<4, float>(e, st)));
      else if (e->c_keep == 6) PB_TRY((launch_enc_cand<6, float>(e, st)));
      else PB_TRY((launch_enc_cand<8, float>(e, st)));
    }
  }
  if (phases & 2) {
    if (!(phases & 8)) PB_CUDA(cudaMemsetAsync(e->fb_count, 0, 2 * sizeof(int), st));    // [0] rows on the exact path, [1] candidates re-scored
    const float coef = e->err_coef > 0.f ? e->err_coef : 1.05f;       // safety factor on the Cauchy-Schwarz bound (norms evaluated in fp32)
    const int nseg = e->F / FZ_SEG, spt = (nseg + 255) / 256;
    if (spt <= 1) PB_TRY(launch_select<1>(e, f16, nseg, coef, st));
    else if (spt <= 2) PB_TRY(launch_select<2>(e, f16, nseg, coef, st));
    else PB_TRY(launch_select<4>(e, f16, nseg, coef, st));
  }
  if (phases & 4) {
    PB_CHECK_ARG(e->fb_scratch && e->fb_scratch_bytes >= (int64_t)e->F * 4, "pb_sae_encode_topk_fused: fallback scratch missing");
    int grid = (int)(e->fb_scratch_bytes / ((int64_t)e->F * 4));
    if (grid > 2 * pb_sm_count()) grid = 2 * pb_sm_count();
    int cap = ((e->F + 255) / 256) * e->k;
    if (cap > e->F) cap = e->F;
    const size_t smem = sizeof(float) * e->d + 8 * (size_t)cap;
    PB_CHECK_ARG(smem <= 200 * 1024, "pb_sae_encode_topk_fused: k=%d x d_sae=%d too large for the exact-path candidate buffer", e->k, e->F);
    static size_t attr_smem = 0;
    if (smem > 48 * 1024 && smem > attr_smem) {
      PB_CUDA(cudaFuncSetAttribute(k_topk_fallback, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      attr_smem = smem;
    }
    PB_LAUNCH_PDL(k_topk_fallback, grid, 256, smem, st, (const int*)e->fb_count, (const int*)e->fb_rows, e->sae_in, e->W_encT, e->b_enc, e->fb_scratch,
                  e->d, e->F, e->k, cap, e->idx, e->val, e->feat_count);
  }
  return PB_OK;
}

extern "C" int pb_rownorm_max(const float* W, int32_t F, int32_t d, float* out, pb_stream_t stream) {
  PB_CHECK_ARG(W && out && F >= 0 && d > 0 && d % 4 == 0, "pb_rownorm_max: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  PB_CUDA(cudaMemsetAsync(out, 0, 2 * sizeof(float), st));
  if (F == 0) return PB_OK;
  int grid = pb_sm_count() * 4;
  if (grid > (F + 7) / 8) grid = (F + 7) / 8;
  k_rownorm_max<<<grid, 256, 0, st>>>(W, F, d, out);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

extern "C" int pb_f16_copy(const float* W, int64_t rows, int32_t d, void* W16, float* lo_max, pb_stream_t stream) {
  PB_CHECK_ARG(W && W16 && rows >= 0 && d > 0 && d % 4 == 0 && pb_aligned16(W) && ((uintptr_t)W16 & 7) == 0, "pb_f16_copy: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (lo_max) PB_CUDA(cudaMemsetAsync(lo_max, 0, sizeof(float), st));
  if (rows == 0) return PB_OK;
  int64_t grid = (rows + 7) / 8;
  if (grid > pb_sm_count() * 4) grid = pb_sm_count() * 4;
  k_f16_copy<<<(int)grid, 256, 0, st>>>(W, rows, d, (__half*)W16, lo_max);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

int pb_abi_sizeof_fused(int which) { return which == 9 ? (int)sizeof(PbSaeEncode) : -1; }
