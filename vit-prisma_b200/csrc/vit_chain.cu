// vit_chain.cu -- pb_vit_forward: the fused HookedViT forward (reference models/base_vit.py:152-217,
// layers/transformer_block.py:80-138) as one native launch sequence on one stream.
//
// Per block (M = batch * tokens rows):
//   LN1                      -> ln1.hook_scale, ln1.hook_normalized
//   QKV GEMM  (N = 3*H*dh)   -> attn.hook_q / hook_k / hook_v          (one launch, split epilogue)
//   attention core           -> attn.hook_attn_scores, hook_pattern, hook_z
//   O GEMM + residual        -> hook_attn_out, hook_resid_mid          (dual epilogue)
//   LN2                      -> ln2.hook_scale, ln2.hook_normalized
//   MLP-in GEMM + activation -> mlp.hook_pre, mlp.hook_post            (dual epilogue)
//   MLP-out GEMM + residual  -> hook_mlp_out, hook_resid_post          (dual epilogue)
// 7 kernels per block, no host round trip, nothing written to HBM that was not requested or is not an
// operand of a later kernel.  hook_resid_pre(l) aliases hook_resid_post(l-1) exactly as in the
// reference cache (the HookPoint is an identity on the same tensor), so it costs no traffic.
//
// In fp32 mode with *_lo weight packs present the GEMMs run wgmma 3xTF32: the A-operand residuals are
// produced by the kernel that produces the operand (LayerNorm out_lo, GEMM out1_lo) or by one
// pb_split_tf32 pass (patches, z), into f->lo_scratch.
#include "common.cuh"

template <typename T>
__global__ void __launch_bounds__(256) k_gather_rows(const T* __restrict__ src, int64_t src_ld, T* __restrict__ dst, int rows, int cols) {
  const int64_t total = (int64_t)rows * cols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / cols), c = (int)(i % cols);
    dst[i] = src[(int64_t)r * src_ld + c];
  }
}

static int gather_rows(const void* src, int64_t src_ld, void* dst, int rows, int cols, int dtype, cudaStream_t st) {
  int grid = (int)ceil_div64((int64_t)rows * cols, 256);
  if (grid > pb_sm_count() * 8) grid = pb_sm_count() * 8;
  if (grid < 1) grid = 1;
  if (dtype == PB_F32) k_gather_rows<float><<<grid, 256, 0, st>>>((const float*)src, src_ld, (float*)dst, rows, cols);
  else k_gather_rows<bf16><<<grid, 256, 0, st>>>((const bf16*)src, src_ld, (bf16*)dst, rows, cols);
  PB_LAUNCH_CHECK();
  return PB_OK;
}

static void gemm_init(PbGemm* g, const PbVitForward* f, int M, int N, int K) {
  memset(g, 0, sizeof(*g));
  g->M = M; g->N = N; g->K = K;
  g->dtype = f->dtype;
  g->impl = f->gemm_impl;
  g->act = PB_ACT_NONE;
  g->lda = K; g->ldb = K; g->ld0 = N; g->ld1 = N; g->ldr = N;
}

extern "C" int pb_vit_forward(const PbVitForward* f, pb_stream_t stream) {
  PB_CHECK_ARG(f, "pb_vit_forward: null descriptor");
  PB_CHECK_ARG(f->dtype == PB_F32 || f->dtype == PB_BF16, "pb_vit_forward: unknown dtype %d", f->dtype);
  PB_CHECK_ARG(f->batch >= 0 && f->n_tokens > 0 && f->d_model > 0 && f->n_heads > 0 && f->d_head > 0, "pb_vit_forward: bad geometry");
  PB_CHECK_ARG(f->n_tokens == f->n_patches + (f->use_cls ? 1 : 0), "pb_vit_forward: n_tokens != n_patches + cls");
  PB_CHECK_ARG(f->images && f->patch_w && f->patch_b && f->pos && f->patches && f->embed && f->full_embed, "pb_vit_forward: embed stage pointers missing");
  PB_CHECK_ARG(f->n_layers_run == 0 || (f->layers_host && f->spills_host), "pb_vit_forward: layer tables missing");
  if (f->batch == 0) return PB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int B = f->batch, T = f->n_tokens, d = f->d_model, HD = f->n_heads * f->d_head, dm = f->d_mlp;
  const int64_t M64 = (int64_t)B * T;
  PB_CHECK_ARG(M64 < (1ll << 31), "pb_vit_forward: batch*tokens overflows int32");
  const int M = (int)M64;
  PB_CHECK_ARG(f->tubelet_depth >= 0, "pb_vit_forward: tubelet_depth %d < 0", f->tubelet_depth);
  const int D = f->tubelet_depth > 0 ? f->tubelet_depth : 1;     // video: tubelets of D frames; image: one frame
  if (f->tubelet_depth > 0) {
    const int g = f->patch_size > 0 ? f->image_size / f->patch_size : 0;
    PB_CHECK_ARG(f->n_frames >= D && f->n_patches == g * g * (f->n_frames / D),
                 "pb_vit_forward: n_patches %d != (S/P)^2 * (n_frames %d / tubelet_depth %d)", f->n_patches, f->n_frames, D);
  }
  const int CPP = f->n_channels * D * f->patch_size * f->patch_size;   // patch GEMM K
  const bool x3 = f->dtype == PB_F32 && f->gemm_impl != PB_GEMM_SIMT && f->lo_scratch != nullptr;
  float* lo_a = f->lo_scratch;                                   // [M, d] or [M, HD] or patches
  float* lo_b = f->lo_scratch ? f->lo_scratch + (int64_t)M * d : nullptr;  // [M, max(dm, HD)]
  PbGemm g;

  // ---- patch (or tubelet) embedding: im2col + GEMM (+bias) -> hook_embed; cls/pos assembly -> hook_full_embed
  if (f->tubelet_depth > 0)
    PB_TRY(pb_im2col_tubelets(f->images, f->patches, B, f->n_channels, f->n_frames, f->image_size, f->patch_size, D, f->dtype, stream));
  else
    PB_TRY(pb_im2col_patches(f->images, f->patches, B, f->n_channels, f->image_size, f->patch_size, f->dtype, stream));
  gemm_init(&g, f, B * f->n_patches, d, CPP);
  g.A = f->patches; g.B = f->patch_w; g.bias = f->patch_b; g.out0 = f->embed;
  if (x3 && f->patch_w_lo) {
    PB_TRY(pb_split_tf32((const float*)f->patches, lo_a, (int64_t)B * f->n_patches * CPP, stream));
    g.A_lo = lo_a; g.B_lo = f->patch_w_lo;
  }
  PB_TRY(pb_gemm(&g, stream));
  PB_TRY(pb_embed_assemble(f->embed, f->cls, f->pos, f->full_embed, B, f->n_patches, d, f->use_cls, f->dtype, stream));

  const void* resid = f->full_embed;
  PbLayerNorm ln;
  if (f->layer_norm_pre) {
    PB_CHECK_ARG(f->lnpre_out, "pb_vit_forward: lnpre_out missing");
    memset(&ln, 0, sizeof(ln));
    ln.rows = M; ln.cols = d; ln.dtype_in = f->dtype; ln.dtype_out = f->dtype; ln.eps = f->eps;
    ln.x = resid; ln.w = f->lnpre_w; ln.b = f->lnpre_b;
    ln.scale = f->lnpre_scale; ln.norm_f32 = f->lnpre_norm_f32; ln.out = f->lnpre_out;
    PB_TRY(pb_layernorm(&ln, stream));
    resid = f->lnpre_out;
  }

  for (int l = 0; l < f->n_layers_run; ++l) {
    const PbVitLayerW& W = f->layers_host[l];
    const PbVitLayerSpill& S = f->spills_host[l];
    PB_CHECK_ARG(S.ln1_out && S.q && S.k && S.v && S.z && S.resid_mid && S.ln2_out && S.post && S.resid_post,
                 "pb_vit_forward: layer %d: a compute-required buffer is NULL", l);
    const bool lx3 = x3 && W.wqkv_lo && W.wo_lo && W.win_lo && W.wout_lo;

    // LN1
    memset(&ln, 0, sizeof(ln));
    ln.rows = M; ln.cols = d; ln.dtype_in = f->dtype; ln.dtype_out = f->dtype; ln.eps = f->eps;
    ln.x = resid; ln.w = W.ln1_w; ln.b = W.ln1_b;
    ln.scale = S.ln1_scale; ln.norm_f32 = S.ln1_norm_f32; ln.out = S.ln1_out; ln.out_lo = lx3 ? lo_a : nullptr;
    PB_TRY(pb_layernorm(&ln, stream));

    // QKV
    gemm_init(&g, f, M, 3 * HD, d);
    g.A = S.ln1_out; g.B = W.wqkv; g.bias = W.bqkv;
    g.n_split = 3; g.split_n = HD; g.ld0 = HD;
    g.out_split[0] = S.q; g.out_split[1] = S.k; g.out_split[2] = S.v;
    if (lx3) { g.A_lo = lo_a; g.B_lo = W.wqkv_lo; }
    PB_TRY(pb_gemm(&g, stream));

    // attention core
    PbAttention at;
    memset(&at, 0, sizeof(at));
    at.B = B; at.T = T; at.H = f->n_heads; at.dh = f->d_head; at.dtype = f->dtype; at.attn_scale = f->attn_scale;
    at.q = S.q; at.k = S.k; at.v = S.v; at.scores = S.scores; at.pattern = S.pattern; at.z = S.z;
    PB_TRY(pb_attention(&at, stream));

    // O projection + residual
    gemm_init(&g, f, M, d, HD);
    g.A = S.z; g.B = W.wo; g.bias = W.bo;
    g.out0 = S.attn_out; g.residual = resid; g.out1 = S.resid_mid;
    if (lx3) {
      PB_TRY(pb_split_tf32((const float*)S.z, lo_b, (int64_t)M * HD, stream));
      g.A_lo = lo_b; g.B_lo = W.wo_lo;
    }
    PB_TRY(pb_gemm(&g, stream));

    // LN2
    memset(&ln, 0, sizeof(ln));
    ln.rows = M; ln.cols = d; ln.dtype_in = f->dtype; ln.dtype_out = f->dtype; ln.eps = f->eps;
    ln.x = S.resid_mid; ln.w = W.ln2_w; ln.b = W.ln2_b;
    ln.scale = S.ln2_scale; ln.norm_f32 = S.ln2_norm_f32; ln.out = S.ln2_out; ln.out_lo = lx3 ? lo_a : nullptr;
    PB_TRY(pb_layernorm(&ln, stream));

    // MLP in + activation
    gemm_init(&g, f, M, dm, d);
    g.A = S.ln2_out; g.B = W.win; g.bias = W.bin;
    g.out0 = S.pre; g.act = f->act; g.out1 = S.post;
    if (lx3) { g.A_lo = lo_a; g.B_lo = W.win_lo; g.out1_lo = lo_b; }
    PB_TRY(pb_gemm(&g, stream));

    // MLP out + residual
    gemm_init(&g, f, M, d, dm);
    g.A = S.post; g.B = W.wout; g.bias = W.bout;
    g.out0 = S.mlp_out; g.residual = S.resid_mid; g.out1 = S.resid_post;
    if (lx3) { g.A_lo = lo_b; g.B_lo = W.wout_lo; }
    PB_TRY(pb_gemm(&g, stream));

    resid = S.resid_post;
  }
  if (!f->run_head) return PB_OK;

  // ---- ln_final -> pool -> head -> normalise
  PB_CHECK_ARG(f->lnf_out && f->pre_normalize && f->out, "pb_vit_forward: head stage pointers missing");
  memset(&ln, 0, sizeof(ln));
  ln.rows = M; ln.cols = d; ln.dtype_in = f->dtype; ln.dtype_out = f->dtype; ln.eps = f->eps;
  ln.x = resid; ln.w = f->lnf_w; ln.b = f->lnf_b;
  ln.scale = f->lnf_scale; ln.norm_f32 = f->lnf_norm_f32; ln.out = f->lnf_out;
  PB_TRY(pb_layernorm(&ln, stream));

  // pooling: cls token = row b*T of the ln_final output (a strided view, lda = T*d); gaap = token mean
  const void* pooled = f->lnf_out;
  int64_t pooled_ld = (int64_t)T * d;
  if (f->pool_gaap) {
    PB_CHECK_ARG(f->pooled, "pb_vit_forward: pooled buffer missing for gaap");
    PB_TRY(pb_mean_tokens(f->lnf_out, f->pooled, B, T, d, f->dtype, stream));
    pooled = f->pooled;
    pooled_ld = d;
  }
  int out_cols = d;
  if (f->head_proj) {
    PB_CHECK_ARG(f->head_w && f->head_b, "pb_vit_forward: head weights missing");
    out_cols = f->n_classes;
    gemm_init(&g, f, B, f->n_classes, d);
    g.A = pooled; g.lda = pooled_ld; g.B = f->head_w; g.bias = f->head_b; g.out0 = f->pre_normalize;
    if (f->dtype == PB_F32) g.impl = PB_GEMM_SIMT;  // 2*B*d*n_classes flops: negligible, keep it exact
    PB_TRY(pb_gemm(&g, stream));
  } else {
    PB_TRY(gather_rows(pooled, pooled_ld, f->pre_normalize, B, d, f->dtype, st));
  }
  if (f->normalize_output) {
    PB_TRY(pb_l2_normalize_rows(f->pre_normalize, f->out, B, out_cols, 1e-12f, f->dtype, stream));
  } else if (f->out != f->pre_normalize) {
    PB_TRY(gather_rows(f->pre_normalize, out_cols, f->out, B, out_cols, f->dtype, st));
  }
  return PB_OK;
}

int pb_abi_sizeof_sae(int which);  // sae.cu
extern "C" int pb_abi_sizeof(int which) {
  switch (which) {
    case 0: return (int)sizeof(PbGemm);
    case 1: return (int)sizeof(PbLayerNorm);
    case 2: return (int)sizeof(PbAttention);
    case 3: return (int)sizeof(PbVitLayerW);
    case 4: return (int)sizeof(PbVitLayerSpill);
    case 5: return (int)sizeof(PbVitForward);
    default: return pb_abi_sizeof_sae(which);
  }
}
