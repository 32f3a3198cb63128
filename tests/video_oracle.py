"""CPU checker for video (tubelet) HookedViTs, built on the image oracle (oracle/vit_oracle.py).

A tubelet embedding is ``Conv3d(C, d, kernel=stride=(D, P, P))`` over ``[B, C, F, S, S]`` followed by
``rearrange("b c t h w -> b (t h w) c")`` (reference models/layers/patch_embedding.py:36-62).  With stride == kernel it is
the same linear map as a ``Conv2d(C*D, d, kernel=stride=P)`` over the ``nt = F // D`` tubelet slabs stacked along the
image height: channel ``c*D + dt`` of row block ``t`` holds frame ``t*D + dt`` of channel ``c``, and the 2-D weight is the
5-D one viewed as ``[d, C*D, P, P]``.  The 2-D output flattens to tokens ordered ``(t, h, w)`` with t slowest, exactly
the reference's order, so everything after the embedding is the image oracle unchanged.

Only tests and the fixture generator import this module, and only as the checker.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, Optional

import torch

from oracle.vit_oracle import recipe_state_dict, state_dict_shapes, vit_forward_with_cache


def video_state_dict_shapes(cfg: dict) -> Dict[str, tuple]:
    """Parameter shapes of a video HookedViT: ``embed.proj.weight [d, C, D, P, P]`` and ``W_pos`` with
    ``(S/P)^2 * (video_num_frames // D) (+1)`` rows (reference position_embedding.py:25-27)."""
    shapes = state_dict_shapes(cfg)
    d, C, P, D = cfg["d_model"], cfg.get("n_channels", 3), cfg["patch_size"], cfg["video_tubelet_depth"]
    n = (cfg["image_size"] // P) ** 2 * (cfg["video_num_frames"] // D)
    shapes["embed.proj.weight"] = (d, C, D, P, P)
    shapes["pos_embed.W_pos"] = (n + (1 if cfg.get("use_cls_token", True) else 0), d)
    return shapes


def video_recipe_state_dict(shapes: Dict[str, tuple], seed: int = 1234, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """The image recipe (same generator stream, same draws) with the conv weight scaled by 1 / sqrt(C*D*P*P), its fan-in,
    so the embedding stays O(1) as it does for images."""
    sd = recipe_state_dict(shapes, seed, torch.float32)
    w = sd["embed.proj.weight"]
    sd["embed.proj.weight"] = w / math.sqrt(w.shape[-1])       # recipe: 1 / sqrt(C*D*P); fan-in is C*D*P*P
    return {k: v.to(dtype) for k, v in sd.items()}


def tubelets_as_image(videos: torch.Tensor, depth: int) -> torch.Tensor:
    """[B, C, F, S, S] -> [B, C*D, nt*S, S]: image[b, c*D + dt, t*S + y, x] = videos[b, c, t*D + dt, y, x]; frames past nt*D dropped."""
    B, C, F, S, S2 = videos.shape
    nt = F // depth
    v = videos[:, :, :nt * depth].reshape(B, C, nt, depth, S, S2)     # [B, C, t, dt, y, x]
    return v.permute(0, 1, 3, 2, 4, 5).reshape(B, C * depth, nt * S, S2)


def video_forward_with_cache(sd: Dict[str, torch.Tensor], cfg: dict, videos: torch.Tensor,
                             names_filter: Optional[Callable[[str], bool]] = None, stop_at_layer: Optional[int] = None):
    """``HookedViT.run_with_cache(videos, ...)`` of a video config, as ``oracle.vit_oracle.vit_forward_with_cache`` does it for
    images.  Raises when ``F // D`` differs from ``video_num_frames // D``, as the reference's position add does."""
    D = cfg["video_tubelet_depth"]
    w = sd["embed.proj.weight"]
    sd2 = dict(sd)
    sd2["embed.proj.weight"] = w.reshape(w.shape[0], w.shape[1] * w.shape[2], w.shape[3], w.shape[4])
    return vit_forward_with_cache(sd2, cfg, tubelets_as_image(videos, D), names_filter=names_filter, stop_at_layer=stop_at_layer)


def videos(batch: int, cfg: dict, seed: int = 0, n_frames: Optional[int] = None) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    F = n_frames if n_frames is not None else cfg["video_num_frames"]
    return torch.randn(batch, cfg.get("n_channels", 3), F, cfg["image_size"], cfg["image_size"], generator=g)
