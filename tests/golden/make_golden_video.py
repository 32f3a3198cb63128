"""Generate the video (tubelet) golden fixtures by running the UNMODIFIED reference on CPU.

    python tests/golden/make_golden_video.py

Like make_golden.py this needs the reference sources and runs only where they are; the fixtures it writes are committed.
Weights come from tests/video_oracle.video_recipe_state_dict and the clips from tests/video_oracle.videos (seeded).

  vit_video_c_{fp32,bf16}.pt  tiny video model, image 32, patch 8, 7 frames in tubelets of 2 (the 7th frame is dropped):
                              3 x 16 tubelets + cls = 49 tokens, batch 2, 2 heads of 16.  Every cache key, full tensors,
                              plus a names_filter + stop_at_layer call as the activation store makes it.
  vit_video_d_fp32.pt         d_head 64 past the 608 tokens of the FFMA attention kernel: image 64, patch 8, 20 frames in
                              tubelets of 2 -> 640 + 1 = 641 tokens.  Per-key digests, the output and the full
                              blocks.1.hook_resid_post.

Every file stays well under 1 MB: the [B,H,T,T] scores / pattern tensors dominate, so the tiny model keeps B*H small.
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

from oracle.vit_oracle import digest  # noqa: E402
from tests.video_oracle import video_recipe_state_dict, videos  # noqa: E402

VIDEO_C = dict(n_layers=2, d_model=32, d_head=16, n_heads=2, d_mlp=64, patch_size=8, image_size=32, n_channels=3,
               n_classes=10, eps=1e-5, activation_name="gelu", normalization_type="LN", use_cls_token=True,
               layer_norm_pre=True, normalize_output=True, return_type="class_logits", classification_type="cls",
               is_video_transformer=True, video_tubelet_depth=2, video_num_frames=7)
VIDEO_D = dict(n_layers=2, d_model=128, d_head=64, n_heads=2, d_mlp=256, patch_size=8, image_size=64, n_channels=3,
               n_classes=16, eps=1e-5, activation_name="gelu", normalization_type="LN", use_cls_token=True,
               layer_norm_pre=True, normalize_output=True, return_type="class_logits", classification_type="cls",
               is_video_transformer=True, video_tubelet_depth=2, video_num_frames=20)
STOP_FILTER = ["blocks.0.hook_resid_post", "blocks.1.ln1.hook_normalized"]


def ref_model(cfg: dict, dtype=torch.float32):
    from vit_prisma.configs.HookedViTConfig import HookedViTConfig
    from vit_prisma.models.base_vit import HookedViT
    model = HookedViT(HookedViTConfig(**cfg, dtype=dtype)).to(dtype)
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict(video_recipe_state_dict(shapes, seed=1234, dtype=dtype))
    model.eval()
    return model, shapes


def make_video():
    for dtype, dname in ((torch.float32, "fp32"), (torch.bfloat16, "bf16")):
        model, shapes = ref_model(VIDEO_C, dtype)
        x = videos(2, VIDEO_C, seed=0).to(dtype)
        with torch.no_grad():
            out, cache = model.run_with_cache(x, return_cache_object=False)
            stop_out, stop_cache = model.run_with_cache(x, names_filter=STOP_FILTER, stop_at_layer=1, return_cache_object=False)
        assert cache["hook_embed"].shape == (2, 48, VIDEO_C["d_model"]), cache["hook_embed"].shape
        path = os.path.join(HERE, f"vit_video_c_{dname}.pt")
        torch.save({"cfg": VIDEO_C, "dtype": dname, "shapes": shapes, "weights_seed": 1234, "images_seed": 0, "batch": 2,
                    "keys": list(cache.keys()), "cache": {k: v.clone() for k, v in cache.items()}, "out": out.clone(),
                    "stop_keys": list(stop_cache.keys()), "stop_out": stop_out.clone()}, path)
        print("wrote", path, len(cache), "keys", os.path.getsize(path), "bytes")

    model, shapes = ref_model(VIDEO_D)
    x = videos(2, VIDEO_D, seed=0)
    with torch.no_grad():
        out, cache = model.run_with_cache(x, return_cache_object=False)
    assert cache["blocks.0.attn.hook_pattern"].shape[-1] == 641
    path = os.path.join(HERE, "vit_video_d_fp32.pt")
    torch.save({"cfg": VIDEO_D, "dtype": "fp32", "shapes": shapes, "weights_seed": 1234, "images_seed": 0, "batch": 2,
                "keys": list(cache.keys()), "digests": {k: digest(v) for k, v in cache.items()}, "out": out.clone(),
                "resid_post_1": cache["blocks.1.hook_resid_post"].clone()}, path)
    print("wrote", path, len(cache), "keys", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    make_video()
