"""Pin the video checker (tests/video_oracle.py) to fixtures made by the unmodified reference (tests/golden/make_golden_video.py).

CPU-only: the GPU routes are then held to these fixtures and to the checker in test_vit_video_gpu.py."""
import pytest
import torch
import torch.nn.functional as F

from oracle.vit_oracle import digest
from tests.util import assert_close, load_golden
from tests.video_oracle import (tubelets_as_image, video_forward_with_cache, video_recipe_state_dict, video_state_dict_shapes,
                                videos)

TOL = {"fp32": 2e-5, "bf16": 1.6e-2}


@pytest.mark.parametrize("dname", ["fp32", "bf16"])
def test_video_oracle_matches_reference_tiny(dname):
    gold = load_golden(f"vit_video_c_{dname}.pt")
    cfg = dict(gold["cfg"])
    dtype = torch.float32 if dname == "fp32" else torch.bfloat16
    assert video_state_dict_shapes(cfg) == gold["shapes"], "state-dict layout drifted from the reference"
    assert gold["shapes"]["embed.proj.weight"] == (cfg["d_model"], 3, 2, 8, 8) and gold["shapes"]["pos_embed.W_pos"][0] == 49
    sd = video_recipe_state_dict(gold["shapes"], gold["weights_seed"], dtype)
    x = videos(gold["batch"], cfg, gold["images_seed"]).to(dtype)
    out, cache = video_forward_with_cache(sd, dict(cfg, dtype=dtype), x)
    assert list(cache.keys()) == gold["keys"], "cache key order differs from the reference"
    for k in gold["keys"]:
        assert_close(cache[k], gold["cache"][k], TOL[dname], k)
    assert_close(out, gold["out"], TOL[dname], "model output")
    flt = ["blocks.0.hook_resid_post", "blocks.1.ln1.hook_normalized"]
    stop_out, stop_cache = video_forward_with_cache(sd, dict(cfg, dtype=dtype), x, names_filter=lambda n: n in flt, stop_at_layer=1)
    assert list(stop_cache.keys()) == gold["stop_keys"]
    assert_close(stop_out, gold["stop_out"], TOL[dname], "stop_at_layer output")


def test_video_oracle_matches_reference_641_tokens():
    gold = load_golden("vit_video_d_fp32.pt")
    cfg = dict(gold["cfg"])
    assert video_state_dict_shapes(cfg) == gold["shapes"]
    sd = video_recipe_state_dict(gold["shapes"], gold["weights_seed"])
    out, cache = video_forward_with_cache(sd, cfg, videos(gold["batch"], cfg, gold["images_seed"]))
    assert list(cache.keys()) == gold["keys"]
    assert cache["blocks.0.attn.hook_pattern"].shape == (2, 2, 641, 641)
    for k, dg in gold["digests"].items():
        mine = digest(cache[k])
        assert mine["shape"] == dg["shape"] and mine["dtype"] == dg["dtype"], k
        assert (mine["samples"] - dg["samples"]).abs().max().item() / max(dg["max_abs"], 1e-30) < 2e-5, k
        assert abs(mine["sum"] - dg["sum"]) <= 2e-5 * max(dg["abs_sum"], 1e-30), k
    assert_close(cache["blocks.1.hook_resid_post"], gold["resid_post_1"], 2e-5, "blocks.1.hook_resid_post")
    assert_close(out, gold["out"], 2e-5, "model output")


def test_tubelet_rearrangement_is_conv3d():
    """The checker's Conv2d over stacked tubelet slabs equals Conv3d(kernel=stride=(D,P,P)) + "b c t h w -> b (t h w) c",
    including the dropped trailing frame."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 3, 7, 16, 16, generator=g, dtype=torch.float64)
    w = torch.randn(5, 3, 2, 4, 4, generator=g, dtype=torch.float64)
    ref = F.conv3d(x, w, stride=(2, 4, 4)).flatten(2).transpose(1, 2)
    got = F.conv2d(tubelets_as_image(x, 2), w.reshape(5, 6, 4, 4), stride=4).flatten(2).transpose(1, 2)
    assert ref.shape == got.shape == (2, 3 * 16, 5)
    assert torch.allclose(ref, got, rtol=0, atol=1e-12)


def test_video_oracle_rejects_other_tubelet_counts():
    gold = load_golden("vit_video_c_fp32.pt")
    cfg = dict(gold["cfg"])
    sd = video_recipe_state_dict(gold["shapes"], gold["weights_seed"])
    with pytest.raises(RuntimeError):
        video_forward_with_cache(sd, cfg, videos(1, cfg, n_frames=9))      # 4 tubelets against W_pos for 3


def test_video_config_counts_tubelets():
    from vit_prisma.configs.HookedViTConfig import HookedViTConfig
    c = HookedViTConfig(2, 32, 8, 64, n_heads=4, patch_size=8, image_size=32, is_video_transformer=True, video_tubelet_depth=2,
                        video_num_frames=7)
    assert c.n_patches == 48 and c.n_tokens == 49
    vivit_b = HookedViTConfig(12, 768, 64, 3072, n_heads=12, patch_size=16, image_size=224, is_video_transformer=True,
                              video_tubelet_depth=2, video_num_frames=16)
    assert vivit_b.n_tokens == 1569
    assert HookedViTConfig(2, 32, 8, 64, patch_size=8, image_size=32).n_patches == 16
