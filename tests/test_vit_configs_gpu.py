"""HookedViT at every config branch the fused chain and the hooked route take, at tensor-core sizes, against the float64 oracle.

The real-size ViT tests elsewhere run one config, the CLIP shape (LN, ln_pre, cls pooling, class_logits, normalize_output,
gelu).  Every other branch the engine accepts ran only in the tiny golden configs, where every GEMM and every attention
takes the FFMA kernels.  Here a table of two-layer models at real widths covers, on both routes and both dtypes:
normalization LN / LNPre, ln_pre on / off, cls pooling with and without a cls token, gaap, class_logits / pre_logits with
and without normalize_output, all six element-wise activations inside a tensor-core MLP-in epilogue, every store branch of
that epilogue (16-byte row vectors with and without a partial last 32-column chunk, column pairs, single columns -- the
last two also writing the tf32 residual plane in fp32), d_head 64 at up to 64, 65-128 and more tokens, d_head 80 and 32,
a QKV split whose blocks are not whole 32-column chunks, every LayerNorm register-kernel width and the generic kernel,
scalar and vector im2col / embedding assembly, and unscaled attention scores.

Bars.  fp32: every cache key and the output within 1e-4 (max-norm relative) of the oracle run in float64 on the same
weights and input, on both routes.  The one exception is measured and named at ``UNSCALED_FP32_FUSED_BAR``: three attention
key families of the fused route with unscaled scores.  bf16: every key within ``_bar`` (tests/test_vit_gpu.py) of the
oracle's bf16 run, which rounds where the reference does (where that run is itself more than the bar from the truth --
unscaled scores, where one bf16 ulp of a score of 50 is a 28 % change of its exp -- the truth rule below implies all this
comparison can say, 2.25x the oracle's distance + 1e-3).  Every key whose bar is above 1e-2, and the output, must be no
less accurate than the oracle's bf16 run against the float64 truth on the bf16-rounded weights: 1.25x over the whole
tensor (RMS, + 1e-4), and at the worst element 1.25x + one bf16 ulp of the tensor's largest value (4e-3 to 8e-3 relative).
The ulp replaces the 1e-3 of test_clip_b32_bf16_matches_oracle because a single element rounding the other way exceeds
that; measured on the H100 below, these keys needed more than 1.25x + 1e-3 (ours / oracle distance, excess over 1.25x):
clip_b16 blocks.0.hook_resid_post 9.99e-3 / 7.06e-3 (1.2e-3), blocks.1.ln1.hook_normalized 1.01e-2 / 6.41e-3 (2.1e-3),
blocks.1.hook_resid_mid 1.07e-2 / 7.69e-3 (1.1e-3), all with an RMS ratio of 0.93; vith14 hook_full_embed 6.50e-3 / 4.04e-3
(1.5e-3, inherits hook_embed); l14_lnpre blocks.0.attn.hook_pattern 1.11e-2 / 7.98e-3 (1.1e-3, RMS 0.99); odd202
blocks.1.attn.hook_pattern 1.68e-2 / 1.05e-2 (3.7e-3, RMS 1.06); the use_attn_result toggle blocks.1.hook_attn_out 9.88e-3 / 6.92e-3
(1.2e-3, RMS 1.0) and blocks.1.ln2.hook_normalized 9.82e-3 / 6.52e-3 (1.7e-3, RMS 0.95), on both routes where both run.
hook_embed gets 2x where the patch GEMM's epilogue rounds the product and then the bias sum (every branch but the
16-byte-row one) while the reference's Conv2d rounds once: measured 1.99x max-norm and 1.41x RMS (vith14, patch 14 on
FFMA), 1.85x / 1.41x (l14_lnpre), 1.43x RMS (odd202, single-column tensor-core epilogue).

Premises.  ``_branches`` restates the dispatch rules (csrc/gemm.cu's AUTO rule and pb_gemm_tc_eligible in csrc/gemm_tc.cu,
pb_make_epi in csrc/gemm_epi.cuh, pb_attention in csrc/attention.cu, launch_ln in csrc/layernorm.cu, launch_im2col and
pb_embed_assemble in csrc/elementwise.cu) for the fused route; every case asserts the branches it is in the table for, and
``test_config_table_reaches_every_branch`` (CPU) checks that the table as a whole reaches each of them on each dtype.  The
fused route's buffers are all 256-byte aligned arena / scratch slots or parameters, so pointer alignment only enters
through the tf32 residual plane ``lo_b``, which starts B*T*d floats into the residual scratch.

Also here: the head GEMM at batch 96 (bf16 on the tensor cores through each epilogue branch, with cls pooling reading the
strided ln_final rows; fp32 on FFMA by design), the hooked route's cfg.use_* toggles (per-head GEMMs on strided views), and
the arena plan: any names_filter / stop_at_layer gives bit-identical values to the unfiltered run.

Measured on an H100 80GB HBM3 (700 W power limit).  fp32, worst key family against float64 outside the unscaled-score
exception: attn.hook_z 9.6e-5, attn.hook_pattern 9.2e-5 (p8_gaap, unscaled scores over 144 tokens), up to 8.9e-5 on the
keys after the attention of b32_lnpre's second block (resid_mid .. the output), everything else below 6e-5 (the FFMA
hooked route stays near 2e-6).
The file runs in about 45 s; the test process peaks at 6.5 GB resident host memory, CUDA context included.
"""
import functools
import math

import pytest
import torch

from oracle.vit_oracle import recipe_state_dict, vit_forward_with_cache
from tests.test_vit_gpu import _bar
from tests.util import rel_err

ACTS = ("relu", "gelu", "silu", "gelu_new", "gelu_fast", "quick_gelu")
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}


def _vit(d, H, dh, dm, P, S, *, norm="LN", ln_pre=False, cls_tok=True, pool="cls", head="class_logits", n_classes=1000,
         normalize=False, act="gelu", scale=True, n_layers=2):
    return dict(n_layers=n_layers, d_model=d, d_head=dh, n_heads=H, d_mlp=dm, patch_size=P, image_size=S, n_channels=3,
                n_classes=n_classes, eps=1e-5, activation_name=act, normalization_type=norm, use_cls_token=cls_tok,
                layer_norm_pre=ln_pre, normalize_output=normalize, return_type=head, classification_type=pool,
                use_attn_scale=scale)


# name: (config, the branches the config is in the table for; a {dname: value} entry differs per dtype)
CONFIGS = {
    # OpenAI CLIP B/16 tower: quick_gelu, 197 tokens (64-key-chunk attention)
    "clip_b16": (_vit(768, 12, 64, 3072, 16, 224, ln_pre=True, n_classes=512, normalize=True, act="quick_gelu"),
                 dict(ln=6, attn="long", mlp_epi="vec16", qkv_epi="vec16", patch="vec")),
    # timm ViT-S/16: LN, no ln_pre, cls, 1000 classes, no normalisation
    "timm_s16": (_vit(384, 6, 64, 1536, 16, 224), dict(ln=4, attn="long", mlp_epi="vec16")),
    # DINO-like: gaap pooling of pre_logits, 65 tokens, d_mlp 1000 (partial last chunk)
    "dino_s8": (_vit(256, 4, 64, 1000, 8, 64, pool="gaap", head="pre_logits", act="gelu_new"),
                dict(ln=2, attn="mma", attn_T="65-128", mlp_epi="vec16_partial")),
    # ViT-H/14-like: d_head 80 (FFMA attention), P = 14 (scalar im2col), d_mlp 1022 (single-column epilogue)
    "vith14": (_vit(1280, 16, 80, 1022, 14, 112, ln_pre=True, n_classes=1024, normalize=True, act="gelu_fast"),
               dict(ln=12, attn="ffma", mlp_epi="scalar", qkv_epi="vec16", patch="scalar")),
    # ViT-L/14-like with LayerNormPre everywhere, 50 tokens; d_mlp 1020: column pairs in bf16, 16-byte rows + tail in fp32
    "l14_lnpre": (_vit(1024, 16, 64, 1020, 14, 98, norm="LNPre", ln_pre=True, head="pre_logits", normalize=True, act="silu"),
                  dict(ln=8, attn="mma", attn_T="<=64", mlp_epi={"fp32": "vec16_partial", "bf16": "pair"}, patch="scalar")),
    # cls pooling without a cls token (row 0 is a patch), 100 tokens, unscaled scores
    "nocls_b16": (_vit(768, 12, 64, 3072, 16, 160, cls_tok=False, n_classes=100, act="relu", scale=False),
                  dict(ln=6, attn="mma", attn_T="65-128", mlp_epi="vec16")),
    # d_model 202: generic LayerNorm, scalar embedding assembly, FFMA QKV / MLP-in; d_head 32
    "odd202": (_vit(202, 2, 32, 808, 32, 192, norm="LNPre", pool="gaap", n_classes=37, normalize=True),
               dict(ln="generic", attn="ffma", assemble="scalar", gemm_qkv="ffma", gemm_mlp_in="ffma")),
    # 3 heads of 80: the QKV split blocks (240 columns) are not whole 32-column chunks
    "split240": (_vit(256, 3, 80, 1536, 32, 224, norm="LNPre", pool="gaap", normalize=True, act="quick_gelu"),
                 dict(ln=2, attn="ffma", qkv_epi="pair", mlp_epi="vec16")),
    # B/32 with LayerNormPre and ln_pre, 50 tokens, unscaled scores
    "b32_lnpre": (_vit(768, 12, 64, 3072, 32, 224, norm="LNPre", ln_pre=True, act="gelu_new", scale=False),
                  dict(ln=6, attn="mma", attn_T="<=64", mlp_epi="vec16")),
    # SigLIP-like: no cls token, gaap, 196 tokens
    "siglip_s16": (_vit(384, 6, 64, 1536, 16, 224, cls_tok=False, pool="gaap", n_classes=768, normalize=True, act="gelu_new"),
                   dict(ln=4, attn="long", mlp_epi="vec16")),
    # 12 heads of 32 at 65 tokens
    "dh32_s16": (_vit(384, 12, 32, 1536, 16, 128, ln_pre=True, act="gelu_fast"), dict(ln=4, attn="ffma", mlp_epi="vec16")),
    # patch 8, 144 tokens without a cls token, gaap of normalised pre_logits, unscaled scores
    "p8_gaap": (_vit(512, 8, 64, 2048, 8, 96, ln_pre=True, cls_tok=False, pool="gaap", head="pre_logits", normalize=True,
                     act="silu", scale=False),
                dict(ln=4, attn="long", mlp_epi="vec16")),
}
BATCH = 2


# ------------------------------------------------------------------------------------------------ restated dispatch rules
def _gemm_route(dname, M, N, K, lda, ldb, lo=True):
    """pb_gemm's AUTO rule: pb_gemm_tc_eligible (16-byte operand rows, K >= one 128-byte slab, fp32 needs both tf32 residual
    planes, 16-byte aligned) and M >= 64, N >= 64."""
    es = 2 if dname == "bf16" else 4
    ok = M >= 1 and N >= 16 and K >= 128 // es and lda * es % 16 == 0 and ldb * es % 16 == 0 and (dname == "bf16" or lo)
    return "tc" if ok and M >= 64 and N >= 64 else "ffma"


def _epi(dname, N, lds, split_n=None, aligned=True):
    """Which store branch of the tensor-core epilogue the chunks of an N-column product take (pb_make_epi + k_gemm_tc):
    16-byte row vectors when vec16_ok, the column-pair walk for a partial last chunk or when only vec_ok, else single columns."""
    e16 = 8 if dname == "bf16" else 4
    vec = aligned and N % 4 == 0 and all(ld % 4 == 0 for ld in lds) and (split_n is None or split_n % 4 == 0)
    vec16 = vec and all(ld % e16 == 0 for ld in lds) and (split_n is None or split_n % 32 == 0)
    if vec16:
        return "vec16_partial" if N % 32 else "vec16"
    return "pair" if vec else "scalar"


def _ln_kernel(d):
    """launch_ln: the register kernel with CHUNKS float4 per lane when every pointer is 16-byte aligned and d % 4 == 0."""
    if d % 4 == 0:
        for chunks in (1, 2, 4, 6, 8, 12):
            if d <= 128 * chunks:
                return chunks
    return "generic"


def _attention(dh, T):
    """pb_attention: d_head 64 with aligned q / k / v / z on the tensor cores (whole rows up to 128 tokens, 64-key chunks
    beyond), the FFMA kernel otherwise."""
    return ("mma" if T <= 128 else "long") if dh == 64 else "ffma"


def _tokens(cfg):
    return (cfg["image_size"] // cfg["patch_size"]) ** 2 + (1 if cfg["use_cls_token"] else 0)


def _branches(cfg, dname, B=BATCH):
    """The fused route's branch on every axis of the table for this config, dtype and batch."""
    d, H, dh, dm, P, S = cfg["d_model"], cfg["n_heads"], cfg["d_head"], cfg["d_mlp"], cfg["patch_size"], cfg["image_size"]
    T, NP, HD = _tokens(cfg), (S // P) ** 2, H * dh
    M, Kp = B * T, 3 * P * P
    lo_b_aligned = dname == "bf16" or B * T * d % 4 == 0      # lo_b = lo_a + B*T*d floats: A_lo of O / MLP-out, out1_lo of MLP-in
    g = {"gemm_patch": _gemm_route(dname, B * NP, d, Kp, Kp, Kp),
         "gemm_qkv": _gemm_route(dname, M, 3 * HD, d, d, d),
         "gemm_o": _gemm_route(dname, M, d, HD, HD, HD, lo=lo_b_aligned),
         "gemm_mlp_in": _gemm_route(dname, M, dm, d, d, d),
         "gemm_mlp_out": _gemm_route(dname, M, d, dm, dm, dm, lo=lo_b_aligned)}
    out = dict(g)
    out["qkv_epi"] = _epi(dname, 3 * HD, (HD, 3 * HD, 3 * HD), split_n=HD) if g["gemm_qkv"] == "tc" else "ffma"
    out["patch_epi"] = _epi(dname, d, (d, d, d)) if g["gemm_patch"] == "tc" else "ffma"
    out["mlp_epi"] = _epi(dname, dm, (dm, dm, dm), aligned=lo_b_aligned) if g["gemm_mlp_in"] == "tc" else "ffma"
    out["tc_act"] = cfg["activation_name"] if g["gemm_mlp_in"] == "tc" else None
    out["attn"] = _attention(dh, T)
    out["attn_T"] = "<=64" if T <= 64 else "65-128" if T <= 128 else ">128"
    out["dh"] = dh
    out["ln"] = _ln_kernel(d)
    # LayerNormPre (w == NULL) writing the tf32 residual plane of the QKV / MLP-in A operand: fp32 blocks with 3xTF32 GEMMs
    out["lnpre_lo"] = cfg["normalization_type"] == "LNPre" and dname == "fp32" and g["gemm_qkv"] == "tc"
    out["patch"] = "vec" if P % 4 == 0 and S % 4 == 0 else "scalar"
    out["assemble"] = "vec" if d % 4 == 0 else "scalar"
    out["norm"] = cfg["normalization_type"]
    out["ln_pre"] = cfg["layer_norm_pre"]
    out["pool"] = cfg["classification_type"] if cfg["use_cls_token"] or cfg["classification_type"] == "gaap" else "cls_notok"
    out["head"] = cfg["return_type"]
    out["normalize"] = cfg["normalize_output"]
    out["attn_scale"] = cfg["use_attn_scale"]
    return out


def _head_branch(cfg, dname, B):
    """run_head: fp32 heads are forced onto FFMA; bf16 takes the AUTO rule with A = the cls rows of ln_final (lda = T*d) or the
    gaap mean (lda = d)."""
    if cfg["return_type"] == "pre_logits":
        return "gather"
    d, N = cfg["d_model"], cfg["n_classes"]
    lda = _tokens(cfg) * d if cfg["classification_type"] == "cls" else d
    if dname == "fp32" or _gemm_route(dname, B, N, d, lda, d) == "ffma":
        return "ffma"
    return "tc_" + _epi(dname, N, (N, N, N))


# every value each axis must reach on each dtype
REQUIRED = {
    "norm": {"LN", "LNPre"}, "ln_pre": {True, False}, "pool": {"cls", "cls_notok", "gaap"}, "head": {"class_logits", "pre_logits"},
    "normalize": {True, False}, "tc_act": set(ACTS), "attn": {"mma", "long", "ffma"}, "attn_T": {"<=64", "65-128", ">128"},
    "dh": {64, 80, 32}, "qkv_epi": {"vec16", "pair"}, "ln": {2, 4, 6, 8, 12, "generic"}, "patch": {"vec", "scalar"},
    "assemble": {"vec", "scalar"}, "attn_scale": {True, False}, "gemm_qkv": {"tc", "ffma"}, "gemm_mlp_in": {"tc", "ffma"},
}
REQUIRED_BY_DTYPE = {"fp32": dict(REQUIRED, mlp_epi={"vec16", "vec16_partial", "scalar"}, lnpre_lo={True}),
                     "bf16": dict(REQUIRED, mlp_epi={"vec16", "vec16_partial", "pair", "scalar"})}


def _declared(name, dname):
    return {k: (v[dname] if isinstance(v, dict) else v) for k, v in CONFIGS[name][1].items()}


def test_config_table_reaches_every_branch():
    """CPU: the restated dispatch rules, walked over the table, reach every branch on each dtype, and every config takes the
    branches it is listed for."""
    for dname, required in REQUIRED_BY_DTYPE.items():
        seen = {}
        for name, (cfg, _) in CONFIGS.items():
            br = _branches(cfg, dname)
            for axis, want in _declared(name, dname).items():
                assert br[axis] == want, (name, dname, axis, br[axis], want)
            for axis, v in br.items():
                seen.setdefault(axis, set()).add(v)
        for axis, values in required.items():
            assert values <= seen[axis], (dname, axis, values - seen[axis])
    heads = {_head_branch(_head_cfg(pool, n), "bf16", HEAD_BATCH) for pool in ("cls", "gaap") for n in HEAD_CLASSES}
    assert heads == {"tc_vec16_partial", "tc_pair", "tc_scalar"}
    assert _head_branch(_head_cfg("cls", 1000), "fp32", HEAD_BATCH) == "ffma"
    for dname in DTYPES:
        assert _branches(TOGGLE_CFG, dname)["attn"] == "mma" and _tokens(PLAN_CFG) > 1


# ------------------------------------------------------------------------------------------------ helpers
def _images(batch, cfg, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(batch, cfg["n_channels"], cfg["image_size"], cfg["image_size"], generator=g)


def _model(cfg, dtype, seed=1234):
    from vit_prisma.configs.HookedViTConfig import HookedViTConfig
    from vit_prisma.models.base_vit import HookedViT
    model = HookedViT(HookedViTConfig(**cfg, dtype=dtype))
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    sd = recipe_state_dict(shapes, seed)
    model.load_state_dict(sd)
    return model.to("cuda", dtype).eval(), sd


@functools.lru_cache(maxsize=2)
def _oracle(cfg_items, dname, batch, seed):
    """(x, runs) for a config: fp32 -> {"f64": float64 run on the fp32 weights}; bf16 -> {"ref": the oracle's bf16 run,
    "truth": float64 on the bf16-rounded weights and input}.  Cached so both routes share one CPU run."""
    cfg = dict(cfg_items)
    from vit_prisma.configs.HookedViTConfig import HookedViTConfig
    from vit_prisma.models.base_vit import HookedViT
    shapes = {k: tuple(v.shape) for k, v in HookedViT(HookedViTConfig(**cfg)).state_dict().items()}
    sd = recipe_state_dict(shapes, 1234)
    x = _images(batch, cfg, seed)
    if dname == "fp32":
        runs = {"f64": vit_forward_with_cache({k: v.double() for k, v in sd.items()}, dict(cfg, dtype=torch.float64), x.double())}
    else:
        sd16 = {k: v.to(torch.bfloat16) for k, v in sd.items()}
        x16 = x.to(torch.bfloat16)
        runs = {"ref": vit_forward_with_cache(sd16, dict(cfg, dtype=torch.bfloat16), x16),
                "truth": vit_forward_with_cache({k: v.double() for k, v in sd16.items()}, dict(cfg, dtype=torch.float64), x16.double())}
    return x, runs


def _family(k):
    parts = k.split(".")
    return ".".join(parts[2:]) if parts[0] == "blocks" else k


def _rms(got, ref):
    got, ref = got.detach().to("cpu", torch.float64), ref.detach().to("cpu", torch.float64)
    return ((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt().clamp_min(1e-30)).item()


def _ulp(t):
    """One bf16 ulp at the largest magnitude of ``t``, relative to that magnitude (the granularity of a max-norm error)."""
    m = t.detach().abs().max().item()
    return 2.0 ** (math.floor(math.log2(m)) - 7) / m if m > 0 else 0.0


# FINDING: with unscaled scores (use_attn_scale=False, |score| ~ 50 at d_model 768) the fused fp32 route misses 1e-4 on the
# attention keys.  The 3xTF32 QKV product carries ~1.4e-5 relative error into q and k (the FFMA hooked route: ~1e-6), and an
# unscaled score turns that into an absolute score error of ~1e-4 -- the truncating wgmma fp32 accumulator of
# tests/test_sae_dense_steps_gpu.py.  Measured on an H100 80GB HBM3 (700 W), against the oracle's own fp32 run in brackets:
#   nocls_b16  blocks.1  attn.hook_pattern 1.6e-4 (2.0e-5), attn.hook_z 1.5e-4 (1.9e-5), hook_attn_out 7.1e-5;
#   b32_lnpre  blocks.0  attn.hook_pattern 1.1e-4 (1.3e-5), attn.hook_z 9.2e-5;
#              blocks.1  attn.hook_pattern 3.2e-4 (3.6e-5), attn.hook_z 2.7e-4 (3.0e-5), hook_attn_out 1.4e-4 (1.8e-5).
# Every other key of these cases, the residual stream behind hook_attn_out included, stays below 9e-5 and is held to 1e-4.
# Only these three key families, only on the fused fp32 route and only with unscaled scores, get the bars below.
UNSCALED_FP32_FUSED_BAR = {"attn.hook_pattern": 4e-4, "attn.hook_z": 4e-4, "hook_attn_out": 2e-4}


def _fp32_bar(k, route, cfg):
    if route == "fused" and not cfg["use_attn_scale"]:
        return UNSCALED_FP32_FUSED_BAR.get(_family(k), 1e-4)
    return 1e-4


def _compare(cache, out, dname, x_runs, cfg, route, extra_ok=()):
    """Every oracle key (and the output) against the bars; returns {key family: worst fp32 error vs float64 | worst bf16
    max-norm truth ratio}."""
    _, runs = x_runs
    H = cfg["n_heads"]
    # the patch GEMM's epilogue rounds the product and then the bias sum everywhere but in the 16-byte-row branch
    embed_two_roundings = _branches(cfg, dname, out.shape[0])["patch_epi"] != "vec16"
    if dname == "fp32":
        ref_out, ref_cache = runs["f64"]
    else:
        ref_out, ref_cache = runs["ref"]
        true_out, true_cache = runs["truth"]
    assert [k for k in cache if k in ref_cache] == list(ref_cache), "cache key order differs from the oracle"
    assert set(cache) - set(ref_cache) <= set(extra_ok), set(cache) - set(ref_cache)
    stats = {}
    for k, ref in list(ref_cache.items()) + [("__out", ref_out)]:
        got = out if k == "__out" else cache[k]
        t = None if dname == "fp32" else true_out if k == "__out" else true_cache[k]
        if tuple(got.shape) != tuple(ref.shape):
            # ln1 on the [B, T, H, d] split / attn_in input of the hooked route: the oracle's value repeated over heads
            assert got.dim() == ref.dim() + 1 and got.shape[2] == H, (k, tuple(got.shape), tuple(ref.shape))
            ref = ref.unsqueeze(2).expand(*got.shape)
            t = None if t is None else t.unsqueeze(2).expand(*got.shape)
        assert got.dtype == (torch.float32 if dname == "fp32" and ref.dtype == torch.float64 else ref.dtype), (k, got.dtype, ref.dtype)
        got = got.detach().cpu()
        fam = _family(k)
        if dname == "fp32":
            e, bar = rel_err(got, ref), _fp32_bar(k, route, cfg)
            assert e <= bar, f"{k}: {e:.2e} from float64 > {bar:.0e}"
            stats[fam] = max(stats.get(fam, 0.0), e)
        else:
            bar = _bar("hook_post_head_pre_normalize" if k == "__out" else k, "bf16")
            e, ref_t = rel_err(got, ref), rel_err(ref, t)
            # within the bar of the oracle's bf16 run; where that run is itself far from the truth (patterns of unscaled
            # scores: one bf16 ulp of a score of 50 is 0.25, a 28 % change of its exp), the truth rule below implies
            # |ours - oracle| <= 2.25x its distance + 1e-3, and that is all this comparison can say
            assert e <= max(bar, 2.25 * ref_t + 1e-3), f"{k}: {e:.2e} from the oracle's bf16 run > {bar:.0e} (oracle vs truth {ref_t:.2e})"
            if bar > 1e-2 or k == "__out":
                # no less accurate than the oracle's bf16 run: 1.25x over the whole tensor (RMS), 1.25x + one bf16 ulp of
                # the tensor's largest value at the worst element (see "Bars" in the module docstring for the keys that
                # needed the ulp).  hook_embed gets 2x where the patch GEMM rounds twice: the reference's Conv2d adds
                # the bias before its one rounding.
                f = 2.0 if k == "hook_embed" and embed_two_roundings else 1.25
                mine_t, mine_r, ref_r = rel_err(got, t), _rms(got, t), _rms(ref, t)
                assert mine_t <= f * ref_t + _ulp(t), f"{k}: {mine_t:.2e} from the float64 truth, the oracle's bf16 run {ref_t:.2e}"
                assert mine_r <= f * ref_r + 1e-4, f"{k}: RMS {mine_r:.2e} from the float64 truth, the oracle's bf16 run {ref_r:.2e}"
                stats[fam] = max(stats.get(fam, 0.0), mine_t / max(ref_t, 1e-9))
                stats["RMS ratio"] = max(stats.get("RMS ratio", 0.0), mine_r / max(ref_r, 1e-9))
    return stats


def _check(cfg, dtype, route, batch, seed, monkeypatch, extra_ok=()):
    """Build the model from the oracle's recipe, run run_with_cache on ``route``, compare every key and the output."""
    dname = "fp32" if dtype == torch.float32 else "bf16"
    x_runs = _oracle(tuple(sorted(cfg.items())), dname, batch, seed)
    model, _ = _model(cfg, dtype)
    if route == "hooked":
        monkeypatch.setenv("PRISMA_B200_ROUTE", "hooked")
    out, cache = model.run_with_cache(x_runs[0].to("cuda", dtype))
    torch.cuda.synchronize()
    assert model.last_route.startswith(route), model.last_route
    stats = _compare(cache, out, dname, x_runs, cfg, route, extra_ok)
    worst = max(stats.items(), key=lambda t: t[1])
    print(f"[{dname} {route}] worst {'rel err vs float64' if dname == 'fp32' else 'truth ratio'}: {worst[0]} {worst[1]:.3g}; "
          + " ".join(f"{f}={v:.2g}" for f, v in sorted(stats.items())))
    return model, cache, out, stats


# ------------------------------------------------------------------------------------------------ the config table
CASES = [(n, dn, r) for n in CONFIGS for dn in DTYPES for r in ("fused", "hooked")]


@pytest.mark.gpu
@pytest.mark.parametrize("name,dname,route", CASES, ids=[f"{n}-{dn}-{r}" for n, dn, r in CASES])
def test_config_matches_oracle(name, dname, route, monkeypatch):
    cfg = CONFIGS[name][0]
    br = _branches(cfg, dname)
    for axis, want in _declared(name, dname).items():
        assert br[axis] == want, (axis, br[axis], want)
    _check(cfg, DTYPES[dname], route, BATCH, 0, monkeypatch)


# ------------------------------------------------------------------------------------------------ head at batch >= 64
HEAD_BATCH = 96
HEAD_CLASSES = (1000, 100, 101)      # bf16 head GEMM epilogue: 16-byte rows + partial tail, column pairs, single columns


def _head_cfg(pool, n_classes):
    # image 32, patch 8: 16 patches + cls = 17 tokens
    return _vit(256, 4, 64, 1024, 8, 32, pool=pool, n_classes=n_classes, normalize=pool == "cls", act="gelu")


HEAD_CASES = [("bf16", pool, n) for pool in ("cls", "gaap") for n in HEAD_CLASSES] + [("fp32", "cls", 1000)]


@pytest.mark.gpu
@pytest.mark.parametrize("dname,pool,n_classes", HEAD_CASES, ids=[f"{d}-{p}-{n}" for d, p, n in HEAD_CASES])
@pytest.mark.parametrize("route", ["fused", "hooked"])
def test_head_at_batch_96(dname, pool, n_classes, route, monkeypatch):
    cfg = _head_cfg(pool, n_classes)
    expect = "ffma" if dname == "fp32" else {1000: "tc_vec16_partial", 100: "tc_pair", 101: "tc_scalar"}[n_classes]
    assert _head_branch(cfg, dname, HEAD_BATCH) == expect
    _check(cfg, DTYPES[dname], route, HEAD_BATCH, 3, monkeypatch)


# ------------------------------------------------------------------------------------------------ hooked-route toggles
TOGGLES = ("use_split_qkv_input", "use_attn_in", "use_hook_mlp_in", "use_attn_result")
TOGGLE_CFG = _vit(256, 4, 64, 1024, 16, 128, ln_pre=True, n_classes=512, normalize=True)   # 65 tokens
TOGGLE_KEYS = {"use_split_qkv_input": ("hook_q_input", "hook_k_input", "hook_v_input"), "use_attn_in": ("hook_attn_in",),
               "use_hook_mlp_in": ("hook_mlp_in",), "use_attn_result": ("attn.hook_result",)}
TOGGLE_SETS = [(t,) for t in TOGGLES] + [TOGGLES]


@pytest.mark.gpu
@pytest.mark.parametrize("toggles", TOGGLE_SETS, ids=["+".join(t) if len(t) == 1 else "all" for t in TOGGLE_SETS])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_hooked_toggles(toggles, dname, monkeypatch):
    cfg = dict(TOGGLE_CFG, **{t: True for t in toggles})
    B, T, d, H, dh = BATCH, _tokens(cfg), cfg["d_model"], cfg["n_heads"], cfg["d_head"]
    # premise: in bf16 the per-head GEMMs run on the tensor cores, reading (and writing) column slices of larger matrices
    # (the hooked route passes no tf32 residual planes, so its fp32 GEMMs run on FFMA)
    per_head_qkv = _gemm_route(dname, B * T, dh, d, H * d, d, lo=False)            # x[:, :, h, :] (lda H*d) @ W_Q[h]
    per_head_result = _gemm_route(dname, B * T, d, dh, H * dh, H * dh, lo=False)   # z[:, :, h, :] @ W_O[:, h*dh:(h+1)*dh]
    assert (per_head_qkv, per_head_result) == (("tc", "tc") if dname == "bf16" else ("ffma", "ffma"))
    extra = {f"blocks.{l}.{k}" for l in range(cfg["n_layers"]) for t in toggles for k in TOGGLE_KEYS[t]}
    model, cache, _, _ = _check(cfg, DTYPES[dname], "hooked", BATCH, 5, monkeypatch, extra_ok=extra)
    assert extra <= set(cache)
    bar = 1e-4 if dname == "fp32" else _bar("blocks.0.hook_attn_out", "bf16")
    for l in range(cfg["n_layers"]):
        p = f"blocks.{l}."
        rep = cache[p + "hook_resid_pre"].unsqueeze(2).expand(-1, -1, H, -1)
        for k in ("hook_attn_in", "hook_q_input", "hook_k_input", "hook_v_input"):
            if p + k in cache:
                assert torch.equal(cache[p + k], rep), p + k
        if p + "hook_mlp_in" in cache:
            assert torch.equal(cache[p + "hook_mlp_in"], cache[p + "hook_resid_mid"])
        if p + "attn.hook_result" in cache:
            summed = cache[p + "attn.hook_result"].double().sum(2) + model.blocks[l].attn.b_O.double()
            e = rel_err(summed, cache[p + "hook_attn_out"])
            assert e <= bar, f"{p}: sum of hook_result + b_O is {e:.2e} from hook_attn_out"


# ------------------------------------------------------------------------------------------------ arena plan
PLAN_CFG = _vit(256, 4, 64, 1024, 16, 128, ln_pre=True, n_classes=512, normalize=True, n_layers=4)


@functools.lru_cache(maxsize=1)
def _plan_full(dname):
    model, sd = _model(PLAN_CFG, DTYPES[dname])
    x = _images(BATCH, PLAN_CFG, 7)
    out, cache = model.run_with_cache(x.to("cuda", DTYPES[dname]))
    assert model.last_route == "fused"
    sd = {k: v.to(DTYPES[dname]) for k, v in sd.items()}
    return model, sd, x.to(DTYPES[dname]), out, cache


def _plan_case(dname, names, stop):
    model, sd, x, out_full, full = _plan_full(dname)
    flt = None if names is None else (lambda n: n in names)
    out, cache = model.run_with_cache(x.cuda(), names_filter=None if names is None else list(names), stop_at_layer=stop)
    assert model.last_route == "fused"
    _, ref_cache = vit_forward_with_cache(sd, dict(PLAN_CFG, dtype=DTYPES[dname]), x, names_filter=flt, stop_at_layer=stop)
    assert list(cache.keys()) == list(ref_cache.keys()), (names, stop)
    for k, v in cache.items():
        assert torch.equal(v, full[k]), f"{k} differs from the unfiltered run (filter {names}, stop {stop})"
    if stop is None:
        assert torch.equal(out, out_full)
    else:
        n = len(range(PLAN_CFG["n_layers"])[:stop])
        assert torch.equal(out, full[f"blocks.{n - 1}.hook_resid_post"] if n else full["hook_ln_pre"]), stop
    return len(cache)


@pytest.mark.gpu
@pytest.mark.parametrize("dname", list(DTYPES))
def test_plan_single_key_filters(dname):
    _, _, _, _, full = _plan_full(dname)
    for k in full:
        assert _plan_case(dname, (k,), None) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("dname", list(DTYPES))
@pytest.mark.parametrize("names,stop", [
    (("blocks.1.hook_resid_pre",), None),                                  # kept without blocks.0.hook_resid_post
    (("blocks.1.hook_resid_pre", "blocks.2.attn.hook_q", "hook_ln_final"), None),
    (("blocks.1.hook_resid_pre", "blocks.3.hook_resid_pre"), 3),
    (None, 0), (None, 1), (None, -1), (None, 4),
], ids=["resid_pre1", "resid_pre1_q2_lnf", "resid_pre13_stop3", "stop0", "stop1", "stop-1", "stop4"])
def test_plan_filters_and_stops(dname, names, stop):
    assert PLAN_CFG["n_layers"] == 4
    _plan_case(dname, names, stop)
