"""Generate the golden fixtures by running the UNMODIFIED reference (/root/reference) on CPU.

    python tests/golden/make_golden.py [vit] [sae]

Runs only in the build container (the GPU box has no /root/reference); the fixtures it writes are
committed and are what tests/ and smoke() compare against.  Inputs and weights come from seeded
recipes (oracle/vit_oracle.recipe_state_dict) because no pretrained checkpoint can be downloaded here.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import _ref_shims  # noqa: E402

_ref_shims.install()

from oracle.vit_oracle import CLIP_B32, digest, recipe_state_dict  # noqa: E402

TINY_A = dict(n_layers=2, d_model=32, d_head=8, n_heads=4, d_mlp=64, patch_size=16, image_size=32, n_channels=3,
              n_classes=10, eps=1e-5, activation_name="gelu", normalization_type="LN", use_cls_token=True,
              layer_norm_pre=True, normalize_output=True, return_type="class_logits", classification_type="cls")
TINY_B = dict(n_layers=2, d_model=24, d_head=8, n_heads=2, d_mlp=40, patch_size=8, image_size=32, n_channels=3,
              n_classes=7, eps=1e-6, activation_name="quick_gelu", normalization_type="LNPre", use_cls_token=False,
              layer_norm_pre=False, normalize_output=False, return_type="pre_logits", classification_type="gaap")
# c: LayerNormPre in front of the blocks, cls pooling without a cls token (fp32: unscaled attention scores, which in
#    bf16 are ~0.25 per ulp and put the reference's own bf16 run beyond any flat bar);
# d: gaap pooling with a cls token and a normalised pre_logits output.  The activation differs per fixture.
TINY_C = dict(n_layers=2, d_model=32, d_head=8, n_heads=4, d_mlp=48, patch_size=8, image_size=32, n_channels=3,
              n_classes=9, eps=1e-5, normalization_type="LNPre", use_cls_token=False, layer_norm_pre=True,
              normalize_output=True, return_type="class_logits", classification_type="cls")
TINY_D = dict(n_layers=2, d_model=24, d_head=8, n_heads=3, d_mlp=56, patch_size=16, image_size=48, n_channels=3,
              n_classes=5, eps=1e-6, normalization_type="LN", use_cls_token=True, layer_norm_pre=False,
              normalize_output=True, return_type="pre_logits", classification_type="gaap")
TINY_OVERRIDE = {("c", "fp32"): dict(activation_name="gelu_new", use_attn_scale=False), ("c", "bf16"): dict(activation_name="gelu_fast"),
                 ("d", "fp32"): dict(activation_name="silu"), ("d", "bf16"): dict(activation_name="relu")}


def ref_model(cfg: dict, dtype=torch.float32):
    from vit_prisma.configs.HookedViTConfig import HookedViTConfig
    from vit_prisma.models.base_vit import HookedViT
    model = HookedViT(HookedViTConfig(**cfg, dtype=dtype))
    model = model.to(dtype)
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    sd = recipe_state_dict(shapes, seed=1234, dtype=dtype)
    model.load_state_dict(sd)
    model.eval()
    return model, shapes


def images(batch, cfg, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(batch, cfg["n_channels"], cfg["image_size"], cfg["image_size"], generator=g)


def make_vit():
    for tag, base in (("a", TINY_A), ("b", TINY_B), ("c", TINY_C), ("d", TINY_D)):
        for dtype, dname in ((torch.float32, "fp32"), (torch.bfloat16, "bf16")):
            cfg = dict(base, **TINY_OVERRIDE.get((tag, dname), {}))
            model, shapes = ref_model(cfg, dtype)
            x = images(3, cfg).to(dtype)
            with torch.no_grad():
                out, cache = model.run_with_cache(x, return_cache_object=False)
                stop_out, stop_cache = model.run_with_cache(
                    x, names_filter=["blocks.0.hook_resid_post", "blocks.1.ln1.hook_normalized"], stop_at_layer=1,
                    return_cache_object=False)
            path = os.path.join(HERE, f"vit_tiny_{tag}_{dname}.pt")
            torch.save({"cfg": cfg, "dtype": dname, "shapes": shapes, "weights_seed": 1234, "images_seed": 0, "batch": 3,
                        "keys": list(cache.keys()), "cache": {k: v.clone() for k, v in cache.items()}, "out": out.clone(),
                        "stop_keys": list(stop_cache.keys()), "stop_out": stop_out.clone()}, path)
            print("wrote", path, len(cache), "keys", os.path.getsize(path), "bytes")

    model, shapes = ref_model(CLIP_B32)
    x = images(4, CLIP_B32)
    with torch.no_grad():
        out, cache = model.run_with_cache(x, return_cache_object=False)
    path = os.path.join(HERE, "vit_b32_fp32_digest.pt")
    torch.save({"cfg": CLIP_B32, "weights_seed": 1234, "images_seed": 0, "batch": 4, "keys": list(cache.keys()),
                "digests": {k: digest(v) for k, v in cache.items()}, "out": out.clone(),
                "bytes_materialised": sum(v.numel() * v.element_size() for v in cache.values())}, path)
    print("wrote", path, len(cache), "keys", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    what = sys.argv[1:] or ["vit", "sae"]
    if "vit" in what:
        make_vit()
    if "sae" in what:
        from make_golden_sae import make_sae
        make_sae()
