"""ActivationCache -- dictionary facade over the activations of one forward pass.

Container semantics from reference src/vit_prisma/prisma_tools/activation_cache.py:29-158
(``cache[name]``, shorthand ``cache["q", 3]`` via ``get_act_name``, negative layer
indices, ``keys/values/items``, iteration, ``remove_batch_dim``).  A handful of the
residual-stream analysis helpers (``accumulated_resid``, ``decompose_resid``,
``stack_activation``, ``apply_ln_to_stack``; reference :160-735) are provided as plain
PyTorch post-processing -- they run on whatever device the cached tensors live on and are
not kernel targets.

On the fused H100 path the values are *views into one cache arena* written by the CUDA
chain (see vit_prisma/b200/vit_engine.py); the views own the arena, so it lives exactly
as long as any cached tensor does.
"""
from __future__ import annotations

import logging
from typing import Dict, Iterator, List, Optional, Tuple, Union

import torch

from vit_prisma.utils.prisma_utils import Slice, SliceInput, get_act_name


class ActivationCache:
    def __init__(self, cache_dict: Dict[str, torch.Tensor], model, has_batch_dim: bool = True):
        self.cache_dict = cache_dict
        self.model = model
        self.has_batch_dim = has_batch_dim
        self.has_embed = "hook_embed" in cache_dict
        self.has_pos_embed = "hook_pos_embed" in cache_dict

    # ------------------------------------------------------------- container
    def _resolve(self, key) -> str:
        if type(key) == str:
            return get_act_name(key)
        if len(key) > 1 and key[1] is not None and key[1] < 0:
            key = (key[0], self.model.cfg.n_layers + key[1], *key[2:])
        return get_act_name(*key)

    def __getitem__(self, key) -> torch.Tensor:
        if key in self.cache_dict:
            return self.cache_dict[key]
        return self.cache_dict[self._resolve(key)]

    def __len__(self) -> int:
        return len(self.cache_dict)

    def __iter__(self) -> Iterator[str]:
        return iter(self.cache_dict)

    def __contains__(self, key) -> bool:
        return key in self.cache_dict

    def keys(self):
        return self.cache_dict.keys()

    def values(self):
        return self.cache_dict.values()

    def items(self):
        return self.cache_dict.items()

    def __repr__(self) -> str:
        return f"ActivationCache with keys {list(self.cache_dict.keys())}"

    def remove_batch_dim(self) -> "ActivationCache":
        if not self.has_batch_dim:
            logging.warning("Tried removing batch dimension after already having removed it.")
            return self
        for key, value in self.cache_dict.items():
            assert value.size(0) == 1, (
                f"Cannot remove batch dimension from cache with batch size > 1, "
                f"for key {key} with shape {value.shape}"
            )
            self.cache_dict[key] = value[0]
        self.has_batch_dim = False
        return self

    def to(self, device, move_model: bool = False) -> "ActivationCache":
        self.cache_dict = {k: v.to(device) for k, v in self.cache_dict.items()}
        if move_model:
            self.model.to(device)
        return self

    # ------------------------------------------------- residual-stream helpers
    def accumulated_resid(self, layer: Optional[int] = None, incl_mid: bool = False,
                          apply_ln: bool = False, pos_slice: Union[Slice, SliceInput] = None,
                          mlp_input: bool = False, return_labels: bool = False):
        """Residual stream at the input of every layer up to ``layer`` (reference :160-292)."""
        n_layers = self.model.cfg.n_layers
        pos_slice = pos_slice if isinstance(pos_slice, Slice) else Slice(pos_slice)
        if layer is None or layer == -1:
            layer = n_layers
        parts, labels = [], []
        for l in range(layer + 1):
            if l == n_layers:
                parts.append(self[("resid_post", n_layers - 1)])
                labels.append("final_post")
                continue
            parts.append(self[("resid_pre", l)])
            labels.append(f"{l}_pre")
            if (incl_mid and l < layer) or (mlp_input and l == layer):
                parts.append(self[("resid_mid", l)])
                labels.append(f"{l}_mid")
        stack = torch.stack([pos_slice.apply(p, dim=-2) for p in parts], dim=0)
        if apply_ln:
            stack = self.apply_ln_to_stack(stack, layer, pos_slice=pos_slice, mlp_input=mlp_input)
        return (stack, labels) if return_labels else stack

    def decompose_resid(self, layer: Optional[int] = None, mlp_input: bool = False,
                        mode: str = "all", apply_ln: bool = False,
                        pos_slice: Union[Slice, SliceInput] = None, incl_embeds: bool = True,
                        return_labels: bool = False):
        """Per-component contributions (embed, pos_embed, each attn_out / mlp_out) up to
        ``layer`` (reference :294-386)."""
        n_layers = self.model.cfg.n_layers
        pos_slice = pos_slice if isinstance(pos_slice, Slice) else Slice(pos_slice)
        if layer is None or layer == -1:
            layer = n_layers
        want_attn = mode in ("all", "attn")
        want_mlp = mode in ("all", "mlp") and not self.model.cfg.attn_only
        parts, labels = [], []
        if incl_embeds:
            if self.has_embed:
                embed = self["hook_embed"]
                if self.model.cfg.use_cls_token and "hook_full_embed" in self.cache_dict:
                    # hook_embed holds patches only; align to the token axis via full - pos
                    embed = self["hook_full_embed"] - self["hook_pos_embed"]
                parts.append(embed)
                labels.append("embed")
            if self.has_pos_embed:
                parts.append(self["hook_pos_embed"])
                labels.append("pos_embed")
        for l in range(layer):
            if want_attn:
                parts.append(self[("attn_out", l)])
                labels.append(f"{l}_attn_out")
            if want_mlp:
                parts.append(self[("mlp_out", l)])
                labels.append(f"{l}_mlp_out")
        if mlp_input and want_attn:
            parts.append(self[("attn_out", layer)])
            labels.append(f"{layer}_attn_out")
        stack = torch.stack([pos_slice.apply(p, dim=-2) for p in parts], dim=0)
        if apply_ln:
            stack = self.apply_ln_to_stack(stack, layer, pos_slice=pos_slice, mlp_input=mlp_input)
        return (stack, labels) if return_labels else stack

    def stack_activation(self, activation_name: str, layer: int = -1,
                         sublayer_type: Optional[str] = None) -> torch.Tensor:
        """Stack one activation over layers ``[0, layer)`` (reference :492-521)."""
        if layer is None or layer == -1:
            layer = self.model.cfg.n_layers
        return torch.stack([self[(activation_name, l, sublayer_type)] for l in range(layer)], dim=0)

    def apply_ln_to_stack(self, residual_stack: torch.Tensor, layer: Optional[int] = None,
                          mlp_input: bool = False, pos_slice: Union[Slice, SliceInput] = None,
                          batch_slice: Union[Slice, SliceInput] = None,
                          has_batch_dim: bool = True) -> torch.Tensor:
        """Centre + divide a stack by the *cached* LN scale that the model applied at
        ``layer`` (ln1, or ln2 with ``mlp_input``; ln_final when layer == n_layers)
        (reference :656-735)."""
        n_layers = self.model.cfg.n_layers
        if self.model.cfg.normalization_type not in ("LN", "LNPre"):
            return residual_stack
        pos_slice = pos_slice if isinstance(pos_slice, Slice) else Slice(pos_slice)
        batch_slice = batch_slice if isinstance(batch_slice, Slice) else Slice(batch_slice)
        if layer is None or layer == -1:
            layer = n_layers
        if has_batch_dim:
            residual_stack = batch_slice.apply(residual_stack, dim=1)
        residual_stack = residual_stack - residual_stack.mean(dim=-1, keepdim=True)
        if layer == n_layers:
            scale = self["ln_final.hook_scale"]
        else:
            scale = self[f"blocks.{layer}.ln{2 if mlp_input else 1}.hook_scale"]
        scale = pos_slice.apply(scale, dim=-2)
        if self.has_batch_dim:
            scale = batch_slice.apply(scale)
        return residual_stack / scale
