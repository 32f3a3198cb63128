// vit_chain.cu -- pb_vit_forward: the fused HookedViT forward (reference models/base_vit.py:152-217,
// layers/transformer_block.py:80-138) as one native launch sequence on one stream; pb_text_forward: the same block
// stack and head tail behind a token embedding, with the causal mask and end-of-text pooling
// (models/base_text_transformer.py:119-160).
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

// What the block stack and the head tail read from either descriptor (PbVitForward, PbTextForward).
struct Chain {
  int B, T, d, H, dh, dm;
  int dtype, gemm_impl, act, causal;
  float eps, attn_scale;
  bool x3;                 // fp32 3xTF32 GEMMs with tf32 residuals in lo_a / lo_b
  float* lo_a;             // [M, d] or [M, HD] or patches
  float* lo_b;             // [M, max(dm, HD)]
};

static Chain chain_init(int B, int T, int d, int H, int dh, int dm, int dtype, int gemm_impl, int act, float eps, float attn_scale,
                        float* lo_scratch) {
  Chain c;
  c.B = B; c.T = T; c.d = d; c.H = H; c.dh = dh; c.dm = dm;
  c.dtype = dtype; c.gemm_impl = gemm_impl; c.act = act; c.causal = 0;
  c.eps = eps; c.attn_scale = attn_scale;
  c.x3 = dtype == PB_F32 && gemm_impl != PB_GEMM_SIMT && lo_scratch != nullptr;
  c.lo_a = lo_scratch;
  c.lo_b = lo_scratch ? lo_scratch + (int64_t)B * T * d : nullptr;
  return c;
}

static void gemm_init(PbGemm* g, const Chain& c, int M, int N, int K) {
  memset(g, 0, sizeof(*g));
  g->M = M; g->N = N; g->K = K;
  g->dtype = c.dtype;
  g->impl = c.gemm_impl;
  g->act = PB_ACT_NONE;
  g->lda = K; g->ldb = K; g->ld0 = N; g->ld1 = N; g->ldr = N;
}

static int layernorm_rows(const Chain& c, const void* x, const void* w, const void* b, float* scale, float* norm_f32, void* out,
                          float* out_lo, pb_stream_t stream) {
  PbLayerNorm ln;
  memset(&ln, 0, sizeof(ln));
  ln.rows = (int64_t)c.B * c.T; ln.cols = c.d; ln.dtype_in = c.dtype; ln.dtype_out = c.dtype; ln.eps = c.eps;
  ln.x = x; ln.w = w; ln.b = b;
  ln.scale = scale; ln.norm_f32 = norm_f32; ln.out = out; ln.out_lo = out_lo;
  return pb_layernorm(&ln, stream);
}

// The transformer blocks (layers/transformer_block.py:80-138): *resid is the block-0 input on entry and the last
// hook_resid_post on return.
static int run_blocks(const Chain& c, const PbVitLayerW* layers, const PbVitLayerSpill* spills, int n_layers, const void** resid,
                      const char* who, pb_stream_t stream) {
  const int M = c.B * c.T, d = c.d, HD = c.H * c.dh, dm = c.dm;
  PbGemm g;
  for (int l = 0; l < n_layers; ++l) {
    const PbVitLayerW& W = layers[l];
    const PbVitLayerSpill& S = spills[l];
    PB_CHECK_ARG(S.ln1_out && S.q && S.k && S.v && S.z && S.resid_mid && S.ln2_out && S.post && S.resid_post,
                 "%s: layer %d: a compute-required buffer is NULL", who, l);
    const bool lx3 = c.x3 && W.wqkv_lo && W.wo_lo && W.win_lo && W.wout_lo;

    // LN1
    PB_TRY(layernorm_rows(c, *resid, W.ln1_w, W.ln1_b, S.ln1_scale, S.ln1_norm_f32, S.ln1_out, lx3 ? c.lo_a : nullptr, stream));

    // QKV
    gemm_init(&g, c, M, 3 * HD, d);
    g.A = S.ln1_out; g.B = W.wqkv; g.bias = W.bqkv;
    g.n_split = 3; g.split_n = HD; g.ld0 = HD;
    g.out_split[0] = S.q; g.out_split[1] = S.k; g.out_split[2] = S.v;
    if (lx3) { g.A_lo = c.lo_a; g.B_lo = W.wqkv_lo; }
    PB_TRY(pb_gemm(&g, stream));

    // attention core
    PbAttention at;
    memset(&at, 0, sizeof(at));
    at.B = c.B; at.T = c.T; at.H = c.H; at.dh = c.dh; at.dtype = c.dtype; at.attn_scale = c.attn_scale;
    at.q = S.q; at.k = S.k; at.v = S.v; at.scores = S.scores; at.pattern = S.pattern; at.z = S.z;
    at.causal = c.causal;
    PB_TRY(pb_attention(&at, stream));

    // O projection + residual
    gemm_init(&g, c, M, d, HD);
    g.A = S.z; g.B = W.wo; g.bias = W.bo;
    g.out0 = S.attn_out; g.residual = *resid; g.out1 = S.resid_mid;
    if (lx3) {
      PB_TRY(pb_split_tf32((const float*)S.z, c.lo_b, (int64_t)M * HD, stream));
      g.A_lo = c.lo_b; g.B_lo = W.wo_lo;
    }
    PB_TRY(pb_gemm(&g, stream));

    // LN2
    PB_TRY(layernorm_rows(c, S.resid_mid, W.ln2_w, W.ln2_b, S.ln2_scale, S.ln2_norm_f32, S.ln2_out, lx3 ? c.lo_a : nullptr, stream));

    // MLP in + activation
    gemm_init(&g, c, M, dm, d);
    g.A = S.ln2_out; g.B = W.win; g.bias = W.bin;
    g.out0 = S.pre; g.act = c.act; g.out1 = S.post;
    if (lx3) { g.A_lo = c.lo_a; g.B_lo = W.win_lo; g.out1_lo = c.lo_b; }
    PB_TRY(pb_gemm(&g, stream));

    // MLP out + residual
    gemm_init(&g, c, M, d, dm);
    g.A = S.post; g.B = W.wout; g.bias = W.bout;
    g.out0 = S.mlp_out; g.residual = S.resid_mid; g.out1 = S.resid_post;
    if (lx3) { g.A_lo = c.lo_b; g.B_lo = W.wout_lo; }
    PB_TRY(pb_gemm(&g, stream));

    *resid = S.resid_post;
  }
  return PB_OK;
}

// pooled [B, d] (row stride pooled_ld) -> head (unless pre_logits) -> hook_post_head_pre_normalize -> F.normalize
// (base_vit.py:210-215, base_text_transformer.py:153-158)
static int run_head(const Chain& c, const void* pooled, int64_t pooled_ld, int head_proj, int n_classes, const void* head_w,
                    const void* head_b, int normalize_output, void* pre_normalize, void* out, const char* who, pb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int B = c.B, d = c.d;
  int out_cols = d;
  PbGemm g;
  if (head_proj) {
    PB_CHECK_ARG(head_w && head_b, "%s: head weights missing", who);
    out_cols = n_classes;
    gemm_init(&g, c, B, n_classes, d);
    g.A = pooled; g.lda = pooled_ld; g.B = head_w; g.bias = head_b; g.out0 = pre_normalize;
    if (c.dtype == PB_F32) g.impl = PB_GEMM_SIMT;  // 2*B*d*n_classes flops: negligible, keep it exact
    PB_TRY(pb_gemm(&g, stream));
  } else {
    PB_TRY(gather_rows(pooled, pooled_ld, pre_normalize, B, d, c.dtype, st));
  }
  if (normalize_output) {
    PB_TRY(pb_l2_normalize_rows(pre_normalize, out, B, out_cols, 1e-12f, c.dtype, stream));
  } else if (out != pre_normalize) {
    PB_TRY(gather_rows(pre_normalize, out_cols, out, B, out_cols, c.dtype, st));
  }
  return PB_OK;
}

extern "C" int pb_vit_forward(const PbVitForward* f, pb_stream_t stream) {
  PB_CHECK_ARG(f, "pb_vit_forward: null descriptor");
  PB_CHECK_ARG(f->dtype == PB_F32 || f->dtype == PB_BF16, "pb_vit_forward: unknown dtype %d", f->dtype);
  PB_CHECK_ARG(f->batch >= 0 && f->n_tokens > 0 && f->d_model > 0 && f->n_heads > 0 && f->d_head > 0, "pb_vit_forward: bad geometry");
  PB_CHECK_ARG(f->n_tokens == f->n_patches + (f->use_cls ? 1 : 0), "pb_vit_forward: n_tokens != n_patches + cls");
  PB_CHECK_ARG(f->images && f->patch_w && f->patch_b && f->pos && f->patches && f->embed && f->full_embed, "pb_vit_forward: embed stage pointers missing");
  PB_CHECK_ARG(f->n_layers_run == 0 || (f->layers_host && f->spills_host), "pb_vit_forward: layer tables missing");
  if (f->batch == 0) return PB_OK;
  const int B = f->batch, T = f->n_tokens, d = f->d_model;
  const int64_t M64 = (int64_t)B * T;
  PB_CHECK_ARG(M64 < (1ll << 31), "pb_vit_forward: batch*tokens overflows int32");
  PB_CHECK_ARG(f->tubelet_depth >= 0, "pb_vit_forward: tubelet_depth %d < 0", f->tubelet_depth);
  const int D = f->tubelet_depth > 0 ? f->tubelet_depth : 1;     // video: tubelets of D frames; image: one frame
  if (f->tubelet_depth > 0) {
    const int g = f->patch_size > 0 ? f->image_size / f->patch_size : 0;
    PB_CHECK_ARG(f->n_frames >= D && f->n_patches == g * g * (f->n_frames / D),
                 "pb_vit_forward: n_patches %d != (S/P)^2 * (n_frames %d / tubelet_depth %d)", f->n_patches, f->n_frames, D);
  }
  const int CPP = f->n_channels * D * f->patch_size * f->patch_size;   // patch GEMM K
  const Chain c = chain_init(B, T, d, f->n_heads, f->d_head, f->d_mlp, f->dtype, f->gemm_impl, f->act, f->eps, f->attn_scale,
                             f->lo_scratch);
  PbGemm g;

  // ---- patch (or tubelet) embedding: im2col + GEMM (+bias) -> hook_embed; cls/pos assembly -> hook_full_embed
  if (f->tubelet_depth > 0)
    PB_TRY(pb_im2col_tubelets(f->images, f->patches, B, f->n_channels, f->n_frames, f->image_size, f->patch_size, D, f->dtype, stream));
  else
    PB_TRY(pb_im2col_patches(f->images, f->patches, B, f->n_channels, f->image_size, f->patch_size, f->dtype, stream));
  gemm_init(&g, c, B * f->n_patches, d, CPP);
  g.A = f->patches; g.B = f->patch_w; g.bias = f->patch_b; g.out0 = f->embed;
  if (c.x3 && f->patch_w_lo) {
    PB_TRY(pb_split_tf32((const float*)f->patches, c.lo_a, (int64_t)B * f->n_patches * CPP, stream));
    g.A_lo = c.lo_a; g.B_lo = f->patch_w_lo;
  }
  PB_TRY(pb_gemm(&g, stream));
  PB_TRY(pb_embed_assemble(f->embed, f->cls, f->pos, f->full_embed, B, f->n_patches, d, f->use_cls, f->dtype, stream));

  const void* resid = f->full_embed;
  if (f->layer_norm_pre) {
    PB_CHECK_ARG(f->lnpre_out, "pb_vit_forward: lnpre_out missing");
    PB_TRY(layernorm_rows(c, resid, f->lnpre_w, f->lnpre_b, f->lnpre_scale, f->lnpre_norm_f32, f->lnpre_out, nullptr, stream));
    resid = f->lnpre_out;
  }

  PB_TRY(run_blocks(c, f->layers_host, f->spills_host, f->n_layers_run, &resid, "pb_vit_forward", stream));
  if (!f->run_head) return PB_OK;

  // ---- ln_final -> pool -> head -> normalise
  PB_CHECK_ARG(f->lnf_out && f->pre_normalize && f->out, "pb_vit_forward: head stage pointers missing");
  PB_TRY(layernorm_rows(c, resid, f->lnf_w, f->lnf_b, f->lnf_scale, f->lnf_norm_f32, f->lnf_out, nullptr, stream));

  // pooling: cls token = row b*T of the ln_final output (a strided view, lda = T*d); gaap = token mean
  const void* pooled = f->lnf_out;
  int64_t pooled_ld = (int64_t)T * d;
  if (f->pool_gaap) {
    PB_CHECK_ARG(f->pooled, "pb_vit_forward: pooled buffer missing for gaap");
    PB_TRY(pb_mean_tokens(f->lnf_out, f->pooled, B, T, d, f->dtype, stream));
    pooled = f->pooled;
    pooled_ld = d;
  }
  return run_head(c, pooled, pooled_ld, f->head_proj, f->n_classes, f->head_w, f->head_b, f->normalize_output, f->pre_normalize,
                  f->out, "pb_vit_forward", stream);
}

extern "C" int pb_text_forward(const PbTextForward* f, pb_stream_t stream) {
  PB_CHECK_ARG(f, "pb_text_forward: null descriptor");
  PB_CHECK_ARG(f->dtype == PB_F32 || f->dtype == PB_BF16, "pb_text_forward: unknown dtype %d", f->dtype);
  PB_CHECK_ARG(f->batch >= 0 && f->n_tokens > 0 && f->vocab > 0 && f->d_model > 0 && f->n_heads > 0 && f->d_head > 0,
               "pb_text_forward: bad geometry");
  PB_CHECK_ARG(f->ids && f->token_w && f->pos && f->embed && f->full_embed, "pb_text_forward: embed stage pointers missing");
  PB_CHECK_ARG(f->n_layers == 0 || (f->layers_host && f->spills_host), "pb_text_forward: layer tables missing");
  PB_CHECK_ARG(f->lnf_out && f->pooled && f->pre_normalize && f->out, "pb_text_forward: head stage pointers missing");
  if (f->batch == 0) return PB_OK;
  const int B = f->batch, T = f->n_tokens, d = f->d_model;
  PB_CHECK_ARG((int64_t)B * T < (1ll << 31), "pb_text_forward: batch*tokens overflows int32");
  Chain c = chain_init(B, T, d, f->n_heads, f->d_head, f->d_mlp, f->dtype, f->gemm_impl, f->act, f->eps, f->attn_scale, f->lo_scratch);
  c.causal = f->causal;

  // ---- token embedding -> hook_embed; + pos_embed[:T] -> hook_full_embed (ln_pre exists but is never applied)
  PB_TRY(pb_embed_tokens(f->ids, f->token_w, f->pos, f->embed, f->full_embed, B, T, d, f->vocab, f->dtype, stream));
  const void* resid = f->full_embed;
  PB_TRY(run_blocks(c, f->layers_host, f->spills_host, f->n_layers, &resid, "pb_text_forward", stream));

  // ---- ln_final over every token (a cache key) -> end-of-text pooling -> head -> normalise
  PB_TRY(layernorm_rows(c, resid, f->lnf_w, f->lnf_b, f->lnf_scale, f->lnf_norm_f32, f->lnf_out, nullptr, stream));
  PB_TRY(pb_gather_argmax_rows(f->ids, f->lnf_out, f->pooled, B, T, d, f->dtype, stream));
  return run_head(c, f->pooled, d, f->head_proj, f->n_classes, f->head_w, f->head_b, f->normalize_output, f->pre_normalize, f->out,
                  "pb_text_forward", stream);
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
    case 10: return (int)sizeof(PbTextForward);
    default: return pb_abi_sizeof_sae(which);
  }
}
