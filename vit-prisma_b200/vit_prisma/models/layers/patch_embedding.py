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
    """Video tubelet embedding (reference :36-62).  Parameter container only: the H100 hot path covers
    image towers; calling it raises instead of silently running somewhere else."""

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        size = [cfg.video_tubelet_depth, cfg.patch_size, cfg.patch_size]
        self.proj = nn.Conv3d(cfg.n_channels, cfg.d_model, kernel_size=size, stride=size, bias=True)

    @host_staged
    def forward(self, x):
        raise NotImplementedError("TubeletEmbedding (video) is outside the H100 hot-path scope (SURVEY #6)")
