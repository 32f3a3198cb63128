"""Hooked multi-head attention (reference models/layers/attention.py:23-281).

Parameter names / shapes are the reference's (``W_Q/K/V [H, d_model, d_head]``, ``W_O [H, d_head,
d_model]``, biases) so state dicts load unchanged; the kernels read K-major packs cached per
parameter version (vit_prisma/b200/packing.py).

This module is the *hooked, op-by-op* route used whenever user hooks are present:
  q/k/v GEMMs -> hook_q/k/v -> scores kernel -> hook_attn_scores -> softmax kernel (NaN->0) ->
  hook_pattern -> PV kernel -> hook_z -> O GEMM (or per-head ``hook_result`` when cfg.use_attn_result).
Between any two hook points user code may replace the tensor, so nothing is fused across them here.
The fused route (one QKV launch, one attention kernel) lives in vit_prisma/b200/vit_engine.py.
"""
from __future__ import annotations

from typing import Dict, Optional, Union

import numpy as np
import torch

from vit_prisma.b200.staging import host_staged
import torch.nn as nn

from vit_prisma.b200 import ops
from vit_prisma.b200.packing import PackCache, pack_heads_nk, pack_out_nk, with_lo
from vit_prisma.configs.HookedViTConfig import HookedViTConfig
from vit_prisma.prisma_tools.factored_matrix import FactoredMatrix
from vit_prisma.prisma_tools.hook_point import HookPoint


class Attention(nn.Module):
    def __init__(self, cfg: Union[Dict, HookedViTConfig], layer_id: Optional[int] = None):
        super().__init__()
        if isinstance(cfg, Dict):
            cfg = HookedViTConfig.from_dict(cfg)
        self.cfg = cfg
        H, d, dh, dt = cfg.n_heads, cfg.d_model, cfg.d_head, cfg.dtype
        for name in ("W_Q", "W_K", "W_V"):
            setattr(self, name, nn.Parameter(torch.empty(H, d, dh, dtype=dt)))
        self.W_O = nn.Parameter(torch.empty(H, dh, d, dtype=dt))
        for name in ("b_Q", "b_K", "b_V"):
            setattr(self, name, nn.Parameter(torch.zeros(H, dh, dtype=dt)))
        self.b_O = nn.Parameter(torch.zeros(d, dtype=dt))

        self.hook_k = HookPoint()            # [batch, pos, head_index, d_head]
        self.hook_q = HookPoint()            # [batch, pos, head_index, d_head]
        self.hook_v = HookPoint()            # [batch, pos, head_index, d_head]
        self.hook_z = HookPoint()            # [batch, pos, head_index, d_head]
        self.hook_attn_scores = HookPoint()  # [batch, head_index, query_pos, key_pos]
        self.hook_pattern = HookPoint()      # [batch, head_index, query_pos, key_pos]
        self.hook_result = HookPoint()       # [batch, pos, head_index, d_model]

        self.layer_id = layer_id
        self.attn_scale = np.sqrt(cfg.d_head) if cfg.use_attn_scale else 1.0
        self._packs = PackCache()

    # --------------------------------------------------------------- circuits
    @property
    def OV(self) -> FactoredMatrix:
        return FactoredMatrix(self.W_V, self.W_O)

    @property
    def QK(self) -> FactoredMatrix:
        return FactoredMatrix(self.W_Q, self.W_K.transpose(-2, -1))

    # ------------------------------------------------------------------ packs
    def packed_qkv(self):
        """([3*H*dh, d] weights, lo | None, [3*H*dh] bias) with q rows first, then k, then v."""
        def build():
            w = torch.cat([pack_heads_nk(self.W_Q), pack_heads_nk(self.W_K), pack_heads_nk(self.W_V)], dim=0)
            b = torch.cat([self.b_Q.detach().reshape(-1), self.b_K.detach().reshape(-1), self.b_V.detach().reshape(-1)])
            w, lo = with_lo(w)
            return w, lo, b.contiguous()
        return self._packs.get("qkv", (self.W_Q, self.W_K, self.W_V, self.b_Q, self.b_K, self.b_V), build)

    def packed_o(self):
        """([d, H*dh] weights, lo | None)."""
        return self._packs.get("o", (self.W_O,), lambda: with_lo(pack_out_nk(self.W_O)))

    # ---------------------------------------------------------------- forward
    def _project(self, x: torch.Tensor, which: int) -> torch.Tensor:
        """x: [B,T,d] or per-head [B,T,H,d] -> [B,T,H,dh] (+bias)."""
        H, dh = self.cfg.n_heads, self.cfg.d_head
        w_all, _, b_all = self.packed_qkv()
        w = w_all[which * H * dh:(which + 1) * H * dh]
        b = b_all[which * H * dh:(which + 1) * H * dh]
        if x.dim() == 3:
            out, _ = ops.gemm(x, w, b)
            return out.view(*x.shape[:2], H, dh)
        B, T = x.shape[:2]
        x = x.contiguous()
        out = torch.empty((B, T, H, dh), dtype=x.dtype, device=x.device)
        for h in range(H):   # split-input mode: every head reads its own copy of the residual
            ops.gemm(x[:, :, h, :], w[h * dh:(h + 1) * dh], b[h * dh:(h + 1) * dh], out0=out[:, :, h, :])
        return out

    def calculate_qkv_matrices(self, query_input, key_input, value_input):
        q = self.hook_q(self._project(query_input, 0))
        k = self.hook_k(self._project(key_input, 1))
        v = self.hook_v(self._project(value_input, 2))
        return q, k, v

    def calculate_attn_scores(self, q, k, attention_mask=None):
        scores = ops.attn_scores(q, k, float(self.attn_scale))
        if attention_mask is not None:
            mask = attention_mask.to(scores.dtype)
            # [T, T] (the text towers' causal mask) broadcasts over batch and head as in the reference's
            # ``scores + mask``; [B, T, T] gets a head axis
            scores = ops.add(scores, (mask if mask.dim() == 2 else mask.unsqueeze(1)).expand_as(scores))
        return scores

    def calculate_z_scores(self, v, pattern):
        return self.hook_z(ops.attn_pv(pattern, v))

    @host_staged
    def forward(self, query_input, key_input, value_input, attention_mask=None) -> torch.Tensor:
        q, k, v = self.calculate_qkv_matrices(query_input, key_input, value_input)
        scores = self.hook_attn_scores(self.calculate_attn_scores(q, k, attention_mask))
        pattern = self.hook_pattern(ops.softmax_rows(scores))     # softmax + NaN->0 in one kernel
        pattern = ops.cast(pattern, self.cfg.dtype)
        z = self.calculate_z_scores(v, pattern)

        H, dh, d = self.cfg.n_heads, self.cfg.d_head, self.cfg.d_model
        wo, _ = self.packed_o()
        B, T = z.shape[:2]
        if not self.cfg.use_attn_result:
            out, _ = ops.gemm(z.reshape(B, T, H * dh), wo, self.b_O)
            return out
        # per-head results exposed to hook_result, then summed over heads (+ b_O)
        z = z.contiguous()
        result = torch.empty((B, T, H, d), dtype=z.dtype, device=z.device)
        for h in range(H):
            ops.gemm(z[:, :, h, :], wo[:, h * dh:(h + 1) * dh], None, out0=result[:, :, h, :])
        result = self.hook_result(result)
        out = result[:, :, 0, :].contiguous()
        for h in range(1, H):
            out = ops.add(out, result[:, :, h, :])
        return ops.add(out, self.b_O.expand_as(out))
