"""HookedTextTransformer -- the hooked CLIP text tower, H100-native (reference models/base_text_transformer.py).

The ViT block stack behind a token embedding, with an additive causal mask on the attention scores and pooling at each
row's end-of-text position (the largest id, ``x[arange(B), ids.argmax(-1)]``).  Two routes produce the same numbers from
the same kernels, chosen exactly as HookedViT chooses (``_TwoRouteModel`` in base_vit.py):

* **fused** (vit_prisma/b200/vit_engine.py ``TextEngine`` -> csrc/vit_chain.cu ``pb_text_forward``): every HookPoint inert,
  no torch hooks, no ``cfg.use_*`` toggle, a CUDA integer ``[B, context_length]`` input (or shorter without the causal
  mask).  The causal mask is a flag of the attention kernels.
* **hooked** (this file + models/layers/*): module by module, every HookPoint fired in the reference's order; the blocks get
  the ``[T, T]`` mask buffer and add it to the scores as the reference does.

Quirks of the reference kept on purpose: ``ln_pre`` exists but is never applied (``hook_ln_pre`` never fires); the
``attn_mask`` argument of ``forward`` is ignored; an input shorter than the context raises ``RuntimeError`` under the causal
mask; ``cls_token=True`` constructs but every forward raises ``RuntimeError``.  ``hook_pos_embed`` is ``pos_embed[:T]``,
``[T, d]`` without a batch axis.
"""
from __future__ import annotations

from typing import Dict, Optional, Union

import torch
import torch.nn as nn

from vit_prisma.b200 import ops
from vit_prisma.b200.vit_engine import TextEngine, text_fusable_reason
from vit_prisma.configs.HookedTextTransformerConfig import HookedTextTransformerConfig
from vit_prisma.models.base_vit import _TwoRouteModel, init_he
from vit_prisma.models.layers.head import Head
from vit_prisma.models.layers.layer_norm import LayerNorm, LayerNormPre
from vit_prisma.models.layers.transformer_block import TransformerBlock
from vit_prisma.prisma_tools.hook_point import HookPoint


def check_token_ids(ids: torch.Tensor, vocab_size: int) -> torch.Tensor:
    """int64 ids (int32 is cast once); ``IndexError`` for an id outside ``[0, vocab_size)``, as ``nn.Embedding`` raises."""
    if ids.dtype not in (torch.int32, torch.int64):
        raise TypeError(f"token ids must be int32 or int64, got {ids.dtype}")
    if ids.dtype == torch.int32:
        ids = ids.to(torch.int64)
    if ids.numel():
        lo, hi = torch.aminmax(ids)
        lo, hi = int(lo), int(hi)
        if lo < 0 or hi >= vocab_size:
            raise IndexError(f"index out of range in self: token ids span [{lo}, {hi}], vocabulary is [0, {vocab_size})")
    return ids


class HookedTextTransformer(_TwoRouteModel):
    """Token ids may be int32 or int64.  Every forward checks that they lie in ``[0, vocab_size)`` before any launch and
    raises ``IndexError`` otherwise, as ``nn.Embedding`` does; the check reads the ids' minimum and maximum back to the
    host, which costs one device synchronisation per call."""

    def __init__(self, cfg: Union[HookedTextTransformerConfig, Dict], no_causal_mask: bool = False, proj_type: str = "linear",
                 cls_token: bool = False):
        super().__init__()
        if isinstance(cfg, Dict):
            cfg = HookedTextTransformerConfig(**cfg)
        elif isinstance(cfg, str):
            raise ValueError(
                "Please pass in a config dictionary or HookedTextTransformerConfig"
                " object. If you want to load a pretrained model, use "
                "HookedTextTransformer.from_pretrained() instead."
            )
        self.cfg = cfg
        self.num_pos = self.context_length = cfg.context_length

        self.token_embed = nn.Embedding(cfg.vocab_size, cfg.d_model)
        self.hook_embed = HookPoint()
        self.pad_id = 0
        self.pos_embed = nn.Parameter(torch.empty(self.num_pos, cfg.d_model))
        self.hook_pos_embed = HookPoint()
        if cls_token:
            self.cls_emb = nn.Parameter(torch.empty(cfg.d_model))
            self.num_pos += 1
        else:
            self.cls_emb = None
        self.hook_full_embed = HookPoint()

        if cfg.normalization_type != "LN":
            raise ValueError(f"Invalid normalization type: {cfg.normalization_type}")
        self.ln_pre = LayerNorm(cfg)                   # never applied (reference :65-71)
        self.hook_ln_pre = HookPoint()
        self.blocks = nn.ModuleList([TransformerBlock(cfg, i) for i in range(cfg.n_layers)])
        self.ln_final = LayerNorm(cfg) if cfg.normalization_type == "LN" else LayerNormPre(cfg)
        self.hook_ln_final = HookPoint()
        if no_causal_mask:
            self.attn_mask = None
        else:
            self.register_buffer("attn_mask", self.build_causal_mask(), persistent=False)
        self.head = Head(cfg)
        self.hook_post_head_pre_normalize = HookPoint()

        self.init_weights()
        self.setup()
        self._engine = TextEngine(self)
        self.last_route: Optional[str] = None   # "fused" | "hooked: <why>" -- introspection for tests/bench

    def _probe(self) -> torch.Tensor:
        return self.token_embed.weight

    def _fusable_reason(self, x) -> Optional[str]:
        return text_fusable_reason(self, x)

    # ------------------------------------------------------------------ masks
    def build_cls_mask(self, text, cast_dtype: torch.dtype):
        cls_mask = (text != self.pad_id).unsqueeze(1)
        cls_mask = nn.functional.pad(cls_mask, (1, 0, cls_mask.shape[2], 0), value=True)
        additive_mask = torch.empty(cls_mask.shape, dtype=cast_dtype, device=cls_mask.device)
        additive_mask.fill_(0)
        additive_mask.masked_fill_(~cls_mask, float("-inf"))
        return torch.repeat_interleave(additive_mask, self.cfg.n_heads, 0)

    def build_causal_mask(self):
        """[num_pos, num_pos]: 0 on and below the diagonal, -inf above it (additive, as PyTorch attention masks are)."""
        mask = torch.empty(self.num_pos, self.num_pos)
        mask.fill_(float("-inf"))
        mask.triu_(1)
        return mask

    # ----------------------------------------------------------------- forward
    def forward(self, input: torch.Tensor, attn_mask: Optional[torch.Tensor] = None):
        """``attn_mask`` is accepted and ignored: the model's own mask buffer is used, as in the reference."""
        if self.cls_emb is not None:
            bool(self.cls_emb)          # the reference's ``if self.cls_emb:`` -- RuntimeError for a d_model-vector
        if isinstance(input, torch.Tensor) and self._host_resident():
            with self._staged_on_gpu():
                return self.forward(input.to("cuda")).to(input.device)
        if isinstance(input, torch.Tensor) and not input.is_cuda:
            input = input.to(self._probe().device)                 # device-resident model, host input: one H2D copy
        why = self._fused_blocker(input)
        if why is None:
            self.last_route = "fused"
            out, _ = self._engine.run(check_token_ids(input, self.cfg.vocab_size), lambda name: False)
            return out
        self.last_route = f"hooked: {why}"
        return self._forward_hooked(check_token_ids(input, self.cfg.vocab_size))

    def _forward_hooked(self, ids: torch.Tensor):
        cfg = self.cfg
        T = ids.shape[1]
        if T > self.pos_embed.shape[0]:
            raise RuntimeError(f"The size of tensor a ({T}) must match the size of tensor b ({self.pos_embed.shape[0]}) at "
                               "non-singleton dimension 1")   # token_embed + pos_embed[:T] in the reference
        embed, _ = ops.embed_tokens(ids, self.token_embed.weight, self.pos_embed)
        embed = self.hook_embed(embed)
        pos = self.hook_pos_embed(self.pos_embed[:T])
        x = ops.add(embed, pos.expand_as(embed))
        self.hook_full_embed(x)                             # observer: return value discarded (:143)
        for block in self.blocks:
            x = block(x, attn_mask=self.attn_mask)
        x = self.ln_final(x)
        self.hook_ln_final(x)                               # observer
        x = ops.gather_argmax_rows(ids, x)
        x = x if cfg.return_type == "pre_logits" else self.head(x)
        self.hook_post_head_pre_normalize(x)                # observer
        if cfg.normalize_output:
            x = ops.l2_normalize_rows(x)
        return x

    def _run_with_cache_impl(self, *model_args, **kwargs):
        if self.cls_emb is not None:
            bool(self.cls_emb)
        if model_args and isinstance(model_args[0], torch.Tensor):
            model_args = (check_token_ids(model_args[0], self.cfg.vocab_size),) + tuple(model_args[1:])
        return super()._run_with_cache_impl(*model_args, **kwargs)

    # -------------------------------------------------------------------- init
    def init_weights(self) -> None:
        if self.cls_emb is not None:
            nn.init.normal_(self.cls_emb, std=self.cfg.cls_std)
        nn.init.normal_(self.token_embed.weight, std=0.02)
        nn.init.normal_(self.pos_embed, std=0.01)
        if self.cfg.weight_type == "he":
            init_he(self)
