"""Patch embedding (reference models/layers/patch_embedding.py:8-62).

The reference runs ``nn.Conv2d(C, d, kernel=P, stride=P)``; with stride == kernel that is a GEMM over
non-overlapping patches: im2col kernel -> [B*n_patches, C*P*P] @ proj.weight.view(d, C*P*P)^T + bias.
``self.proj`` stays an ``nn.Conv2d`` purely as the parameter container so the state-dict keys and
shapes (``embed.proj.weight [d, C, P, P]``, ``embed.proj.bias [d]``) are unchanged.
"""
from __future__ import annotations

import torch

from vit_prisma.b200.staging import host_staged
import torch.nn as nn

from vit_prisma.b200 import ops


class PatchEmbedding(nn.Module):
    def __init__(self, config, logger=None):
        super().__init__()
        self.logger = logger
        self.config = config
        self.proj = nn.Conv2d(config.n_channels, config.d_model, kernel_size=config.patch_size,
                              stride=config.patch_size, bias=True)

    def _log(self, stage: str, tensor: torch.Tensor) -> None:
        if self.logger:
            self.logger.info(f"{stage} size: {tensor.shape}")

    @host_staged
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        self._log("PatchEmbedding input", x)
        B = x.shape[0]
        P, d = self.config.patch_size, self.config.d_model
        w = self.proj.weight
        x = ops.cast(x, w.dtype) if x.is_cuda else x.to(w.dtype)
        patches = ops.im2col_patches(x, P)                       # [B*np, C*P*P]
        out, _ = ops.gemm(patches, w.detach().reshape(d, -1), self.proj.bias)
        out = out.view(B, -1, d)                                 # [B, n_patches, d_model]
        self._log("PatchEmbedding output", out)
        return out


class TubeletEmbedding(nn.Module):
    """Video tubelet embedding (reference :36-62): ``nn.Conv3d(C, d, kernel=stride=(D, P, P))`` over ``[B, C, F, S, S]``.
    With stride == kernel it is the same GEMM as the 2-D case: tubelet im2col -> [B*n_tubelets, C*D*P*P] @
    proj.weight.view(d, C*D*P*P)^T + bias, tokens ordered (t, h, w) with t slowest.  Frames past (F // D) * D are
    dropped, as Conv3d drops them.  ``self.proj`` stays an ``nn.Conv3d`` as the parameter container
    (``embed.proj.weight [d, C, D, P, P]``)."""

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        size = [cfg.video_tubelet_depth, cfg.patch_size, cfg.patch_size]
        self.proj = nn.Conv3d(cfg.n_channels, cfg.d_model, kernel_size=size, stride=size, bias=True)

    @host_staged
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        B = x.shape[0]
        D, P, d = self.cfg.video_tubelet_depth, self.cfg.patch_size, self.cfg.d_model
        w = self.proj.weight
        x = ops.cast(x, w.dtype) if x.is_cuda else x.to(w.dtype)
        patches = ops.im2col_tubelets(x, P, D)                   # [B*n_tubelets, C*D*P*P]
        out, _ = ops.gemm(patches, w.detach().reshape(d, -1), self.proj.bias)
        return out.view(B, -1, d)                                # [B, n_tubelets, d_model]
