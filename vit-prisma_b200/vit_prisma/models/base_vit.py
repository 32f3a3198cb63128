"""HookedViT -- the hooked vision transformer, H100-native (reference models/base_vit.py:60-824).

Two execution routes produce the same numbers from the same kernels:

* **fused** (vit_prisma/b200/vit_engine.py -> csrc/vit_chain.cu): taken by ``forward`` /
  ``run_with_cache`` whenever no user code can observe or alter an intermediate -- i.e. every
  HookPoint is inert, no module-level torch hooks are registered, and no ``cfg.use_*`` toggle is on.
  The cache is written by kernel epilogues straight into one arena; ``names_filter`` prunes the
  writes, ``stop_at_layer`` prunes the launches.
* **hooked** (this file + models/layers/*): the module-by-module forward of the reference, every
  arithmetic step one C-ABI op, every HookPoint fired in the reference's order -- used as soon as a
  user hook (``run_with_hooks``, ``add_hook``, perma hooks, ``hooks()`` contexts) is present.

Module tree, parameter names and shapes equal the reference's, so ``load_state_dict`` from a
reference ``HookedViT`` works unchanged (state-dict layout: SURVEY section 8b).
"""
from __future__ import annotations

import contextlib

import logging
import os
from contextlib import contextmanager
from typing import Dict, List, Optional, Tuple, Union

import torch
import torch.nn as nn

from vit_prisma.b200 import ops
from vit_prisma.b200._lib import PrismaB200Error  # noqa: F401
from vit_prisma.b200.staging import _move, host_staged, staged_on_gpu
from vit_prisma.b200.vit_engine import VitEngine, fusable_reason
from vit_prisma.configs.HookedViTConfig import HookedViTConfig
from vit_prisma.models.layers.attention import Attention
from vit_prisma.models.layers.head import Head
from vit_prisma.models.layers.layer_norm import LayerNorm, LayerNormPre
from vit_prisma.models.layers.mlp import MLP
from vit_prisma.models.layers.patch_embedding import PatchEmbedding, TubeletEmbedding
from vit_prisma.models.layers.position_embedding import PosEmbedding
from vit_prisma.models.layers.transformer_block import BertBlock, TransformerBlock
from vit_prisma.prisma_tools.activation_cache import ActivationCache
from vit_prisma.prisma_tools.hook_point import HookPoint, _global_module_hooks_present
from vit_prisma.prisma_tools.hooked_root_module import HookedRootModule, normalise_names_filter

DTYPE_FROM_STRING = {
    "float32": torch.float32, "fp32": torch.float32,
    "float16": torch.float16, "fp16": torch.float16,
    "bfloat16": torch.bfloat16, "bf16": torch.bfloat16,
}


def _make_norm(cfg):
    if cfg.normalization_type == "LN":
        return LayerNorm(cfg)
    if cfg.normalization_type == "LNPre":
        return LayerNormPre(cfg)
    if cfg.normalization_type is None:
        return nn.Identity()
    raise ValueError(f"Invalid normalization type: {cfg.normalization_type}")


def init_he(model: nn.Module) -> None:
    """The reference's ``weight_type == "he"`` initialisation of every submodule (base_vit.py, base_text_transformer.py)."""
    cfg = model.cfg
    for m in model.modules():
        if isinstance(m, PosEmbedding):
            nn.init.normal_(m.W_pos, std=cfg.pos_std)
        elif isinstance(m, Attention):
            for w in (m.W_Q, m.W_K, m.W_V, m.W_O):
                nn.init.xavier_uniform_(w)
        elif isinstance(m, MLP):
            nn.init.kaiming_normal_(m.W_in, nonlinearity="relu")
            nn.init.kaiming_normal_(m.W_out, nonlinearity="relu")
            nn.init.zeros_(m.b_out)
            nn.init.zeros_(m.b_in)
        elif isinstance(m, Head):
            nn.init.kaiming_normal_(m.W_H, nonlinearity="relu")
            nn.init.zeros_(m.b_H)
        elif isinstance(m, (nn.Linear, nn.Conv2d)):
            nn.init.kaiming_normal_(m.weight, nonlinearity="relu")
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)


class _TwoRouteModel(HookedRootModule):
    """Route choice, host staging, ``run_with_cache`` and device moves shared by the hooked towers.

    A subclass provides ``_probe()`` (the parameter whose device and dtype stand for the model's), ``_fusable_reason(x)``
    (None when its fused engine can serve ``x``) and ``self._engine`` (whose ``run(x, want, stop_at_layer)`` returns
    ``(out, cache)``)."""

    def _probe(self) -> torch.Tensor:
        raise NotImplementedError

    def _fusable_reason(self, x) -> Optional[str]:
        raise NotImplementedError

    # ------------------------------------------------------------ route choice
    def _fused_blocker(self, x) -> Optional[str]:
        """Why the fused chain cannot serve this call (None = it can)."""
        if os.environ.get("PRISMA_B200_ROUTE") == "hooked":
            return "forced by PRISMA_B200_ROUTE"
        why = self._fusable_reason(x)
        if why:
            return why
        if _global_module_hooks_present():
            return "global torch module hooks registered"
        for mod in self.modules():
            if mod._forward_hooks or mod._forward_pre_hooks or mod._backward_hooks or mod._backward_pre_hooks:
                return f"torch hook registered on {getattr(mod, 'name', type(mod).__name__)}"
        return None

    # ----------------------------------------------------------------- host-resident models
    # Device policy: vit_prisma/b200/staging.py.  A model whose parameters live in host memory (the reference's default
    # ``HookedViTConfig.device = "cpu"``) is staged on the GPU for the duration of a call; nothing ever computes on the CPU.
    def _host_resident(self) -> bool:
        return not self._probe().is_cuda

    def _staged_on_gpu(self):
        return staged_on_gpu(self)

    @staticmethod
    def _to_like(obj, device):
        return _move(obj, device)

    # ----------------------------------------------------------------- caching
    def run_with_cache(self, *model_args, return_cache_object: bool = True, remove_batch_dim: bool = False, **kwargs
                       ) -> Tuple[torch.Tensor, Union[ActivationCache, Dict[str, torch.Tensor]]]:
        """``(model_out, cache)``; cache is an ActivationCache unless ``return_cache_object=False``.

        Accepts every keyword of the reference (names_filter, device, incl_bwd, reset_hooks_end,
        clear_contexts, fwd_hooks, bwd_hooks, stop_at_layer, ...).  The fused route is used when the
        only thing attached to the model would have been the internal save-hook."""
        out, cache_dict = self._run_with_cache_impl(*model_args, remove_batch_dim=remove_batch_dim, **kwargs)
        if return_cache_object:
            return out, ActivationCache(cache_dict, self, has_batch_dim=not remove_batch_dim)
        return out, cache_dict

    def _run_with_cache_impl(self, *model_args, names_filter=None, device=None, remove_batch_dim=False,
                             incl_bwd=False, reset_hooks_end=True, clear_contexts=False, fwd_hooks=[],
                             bwd_hooks=[], **model_kwargs):
        if model_args and isinstance(model_args[0], torch.Tensor) and self._host_resident():
            home = model_args[0].device                              # host-resident model: stage, run on the GPU, bring results home
            with self._staged_on_gpu():
                out, cache = self._run_with_cache_impl(model_args[0].to("cuda"), *model_args[1:], names_filter=names_filter,
                                                       device=device if device is not None else home, remove_batch_dim=remove_batch_dim,
                                                       incl_bwd=incl_bwd, reset_hooks_end=reset_hooks_end, clear_contexts=clear_contexts,
                                                       fwd_hooks=fwd_hooks, bwd_hooks=bwd_hooks, **model_kwargs)
            return self._to_like(out, home), cache
        if model_args and isinstance(model_args[0], torch.Tensor) and not model_args[0].is_cuda:
            model_args = (model_args[0].to(self._probe().device),) + tuple(model_args[1:])
        plain = (len(model_args) == 1 and not incl_bwd and not fwd_hooks and not bwd_hooks
                 and set(model_kwargs) <= {"stop_at_layer"})
        why = self._fused_blocker(model_args[0]) if plain else "user hooks / backward requested"
        if why is None:
            self.last_route = "fused"
            want = normalise_names_filter(names_filter)
            known = self.hook_dict
            out, cache = self._engine.run(model_args[0], lambda n: n in known and want(n), model_kwargs.get("stop_at_layer"))
            if device is not None or remove_batch_dim:
                for key, val in cache.items():
                    val = val.to(device) if device is not None else val
                    cache[key] = val[0] if remove_batch_dim else val
            # mirror the reference's side effects of a caching run
            self.is_caching = False
            return out, cache
        self.last_route = f"hooked: {why}"
        return super().run_with_cache(*model_args, names_filter=names_filter, device=device,
                                      remove_batch_dim=remove_batch_dim, incl_bwd=incl_bwd,
                                      reset_hooks_end=reset_hooks_end, clear_contexts=clear_contexts,
                                      fwd_hooks=fwd_hooks, bwd_hooks=bwd_hooks, **model_kwargs)

    # ------------------------------------------------------- device / dtype moves
    def to(self, *args, **kwargs):
        """``nn.Module.to`` that also keeps ``cfg.device`` / ``cfg.dtype`` truthful -- the kernels pick
        their arithmetic type from ``cfg.dtype`` (the reference's LayerNorm does the same, layer_norm.py:82)."""
        out = super().to(*args, **kwargs)
        probe = self._probe()
        self.cfg.device = str(probe.device)
        if probe.dtype != self.cfg.dtype and probe.dtype.is_floating_point:
            self.cfg.dtype = probe.dtype
        return out

    def cuda(self, device=None):
        return self.to("cuda" if device is None else device)

    def cpu(self):
        return self.to("cpu")


class HookedViT(_TwoRouteModel):
    def __init__(self, cfg: Union[HookedViTConfig, Dict]):
        super().__init__()
        if isinstance(cfg, Dict):
            cfg = HookedViTConfig(**cfg)
        elif isinstance(cfg, str):
            raise ValueError(
                "Please pass in a config dictionary or HookedViT object. If you want to load a "
                "pretrained model, use HookedViT.from_pretrained() instead."
            )
        self.cfg = cfg

        self.cls_token = nn.Parameter(torch.randn(1, 1, cfg.d_model))
        self.embed = TubeletEmbedding(cfg) if cfg.is_video_transformer else PatchEmbedding(cfg)
        self.hook_embed = HookPoint()
        self.pos_embed = PosEmbedding(cfg)
        self.hook_pos_embed = HookPoint()
        self.hook_full_embed = HookPoint()

        if cfg.layer_norm_pre:
            self.ln_pre = _make_norm(cfg)
            self.hook_ln_pre = HookPoint()
        else:
            print("ln_pre not set")

        block_cls = BertBlock if cfg.use_bert_block else TransformerBlock
        self.blocks = nn.ModuleList([block_cls(cfg, i) for i in range(cfg.n_layers)])
        self.ln_final = _make_norm(cfg)
        self.hook_ln_final = HookPoint()
        self.head = Head(cfg)
        self.hook_post_head_pre_normalize = HookPoint()

        self.init_weights()
        self.setup()
        self._engine = VitEngine(self)
        self.last_route: Optional[str] = None   # "fused" | "hooked: <why>" -- introspection for tests/bench

    def _probe(self) -> torch.Tensor:
        return self.cls_token

    def _fusable_reason(self, x) -> Optional[str]:
        return fusable_reason(self, x)

    # ----------------------------------------------------------------- forward
    def forward(self, input: torch.Tensor, stop_at_layer: Optional[int] = None):
        """``stop_at_layer`` (exclusive, negative allowed) returns the residual stream after that many blocks."""
        if isinstance(input, torch.Tensor) and self._host_resident():
            with self._staged_on_gpu():
                return self.forward(input.to("cuda"), stop_at_layer).to(input.device)
        if isinstance(input, torch.Tensor) and not input.is_cuda:
            input = input.to(self.cls_token.device)                 # device-resident model, host input: one H2D copy
        why = self._fused_blocker(input)
        if why is None:
            self.last_route = "fused"
            out, _ = self._engine.run(input, lambda name: False, stop_at_layer)
            return out
        self.last_route = f"hooked: {why}"
        return self._forward_hooked(input, stop_at_layer)

    def _forward_hooked(self, input: torch.Tensor, stop_at_layer: Optional[int] = None):
        cfg = self.cfg
        batch = input.shape[0]
        embed = self.hook_embed(self.embed(input))
        if cfg.use_cls_token:
            embed = torch.cat((self.cls_token.to(embed.dtype).expand(batch, -1, -1), embed), dim=1)   # data movement only
        pos = self.hook_pos_embed(self.pos_embed(input))
        residual = ops.add(embed, pos)
        self.hook_full_embed(residual)                     # observer: return value discarded (base_vit.py:181)
        if cfg.layer_norm_pre:
            residual = self.hook_ln_pre(self.ln_pre(residual))
        for block in self.blocks[:stop_at_layer]:
            residual = block(residual)
        if stop_at_layer is not None:
            return residual

        x = self.ln_final(residual)
        self.hook_ln_final(x)                              # observer
        if cfg.classification_type == "gaap":
            x = ops.mean_tokens(x)
        elif cfg.classification_type == "cls":
            cls_tok = x[:, 0]
            if "dino-vitb" in cfg.model_name:
                pooled = ops.mean_tokens(x[:, 1:].contiguous())
                x = torch.cat((cls_tok.unsqueeze(-1), pooled.unsqueeze(-1)), dim=-1)
            else:
                x = cls_tok
        x = x if cfg.return_type == "pre_logits" else self.head(x)
        self.hook_post_head_pre_normalize(x)               # observer
        if cfg.normalize_output:
            x = ops.l2_normalize_rows(x)
        return x

    # -------------------------------------------------------------------- init
    def init_weights(self) -> None:
        cfg = self.cfg
        if cfg.use_cls_token:
            nn.init.normal_(self.cls_token, std=cfg.cls_std)
        if cfg.weight_type == "he":
            init_he(self)

    # --------------------------------------------------------- toggles / checks
    def set_use_attn_result(self, use_attn_result: bool):
        self.cfg.use_attn_result = use_attn_result

    def set_use_split_qkv_input(self, use_split_qkv_input: bool):
        self.cfg.use_split_qkv_input = use_split_qkv_input

    def set_use_hook_mlp_in(self, use_hook_mlp_in: bool):
        assert not self.cfg.attn_only, "Can't use hook_mlp_in with attn_only model"
        self.cfg.use_hook_mlp_in = use_hook_mlp_in

    def set_use_attn_in(self, use_attn_in: bool):
        self.cfg.use_attn_in = use_attn_in

    def check_hooks_to_add(self, hook_point, hook_point_name, hook, dir="fwd", is_permanent=False, prepend=False) -> None:
        gates = (
            (("attn.hook_result",), self.cfg.use_attn_result, "use_attn_result_hook"),
            (("hook_q_input", "hook_k_input", "hook_v_input"), self.cfg.use_split_qkv_input, "use_split_qkv_input"),
            (("mlp_in",), self.cfg.use_hook_mlp_in, "use_hook_mlp_in"),
            (("attn_in",), self.cfg.use_attn_in, "use_attn_in"),
        )
        for suffixes, enabled, flag in gates:
            if hook_point_name.endswith(suffixes):
                assert enabled, f"Cannot add hook {hook_point_name} if {flag} is False"

    # ---------------------------------------------------------------- analysis
    def tokens_to_residual_directions(self, labels: torch.Tensor) -> torch.Tensor:
        return self.head.W_H[:, labels].movedim(0, -1)

    def accumulated_bias(self, layer: int, mlp_input: bool = False, include_mlp_biases: bool = True) -> torch.Tensor:
        total = torch.zeros(self.cfg.d_model, device=self.cls_token.device)
        for i in range(layer):
            total += self.blocks[i].attn.b_O
            if include_mlp_biases:
                total += self.blocks[i].mlp.b_out
        if mlp_input:
            assert layer < self.cfg.n_layers, "Cannot include attn_bias from beyond the final layer"
            total += self.blocks[layer].attn.b_O
        return total

    @classmethod
    def from_local(cls, model_config, checkpoint_path: str):
        model = cls(model_config)
        if not os.path.exists(checkpoint_path):
            raise Exception(f"Attempting to load a Prisma ViT but no file was found at {checkpoint_path}")
        ckpt = torch.load(checkpoint_path, map_location=torch.device(model_config.device), weights_only=False)
        model.load_state_dict(ckpt["model_state_dict"])
        return model

    # ------------------------------------------------------ stacked weight views
    def _stack(self, getter) -> torch.Tensor:
        return torch.stack([getter(block) for block in self.blocks], dim=0)

    W_E = property(lambda self: self.embed.proj.weight)
    b_E = property(lambda self: self.embed.proj.bias)
    W_pos = property(lambda self: self.pos_embed.W_pos)
    W_K = property(lambda self: self._stack(lambda b: b.attn.W_K))
    b_K = property(lambda self: self._stack(lambda b: b.attn.b_K))
    W_Q = property(lambda self: self._stack(lambda b: b.attn.W_Q))
    b_Q = property(lambda self: self._stack(lambda b: b.attn.b_Q))
    W_V = property(lambda self: self._stack(lambda b: b.attn.W_V))
    b_V = property(lambda self: self._stack(lambda b: b.attn.b_V))
    W_O = property(lambda self: self._stack(lambda b: b.attn.W_O))
    b_O = property(lambda self: self._stack(lambda b: b.attn.b_O))
    W_in = property(lambda self: self._stack(lambda b: b.mlp.W_in))
    b_in = property(lambda self: self._stack(lambda b: b.mlp.b_in))
    W_out = property(lambda self: self._stack(lambda b: b.mlp.W_out))
    b_out = property(lambda self: self._stack(lambda b: b.mlp.b_out))
    W_H = property(lambda self: self.head.W_H)
    b_H = property(lambda self: self.head.b_H)


# ------------------------------------------------------------------------------------------------ SAE splice
def _walk_to_parent(root, dotted: str):
    """('blocks.3.hook_resid_post') -> (module blocks[3], 'hook_resid_post'); numeric parts index containers."""
    parts = dotted.split(".")
    obj = root
    for part in parts[:-1]:
        obj = obj[int(part)] if part.isdigit() else getattr(obj, part)
    return obj, parts[-1]


class HookedSAEViT(HookedViT):
    """HookedViT with sparse autoencoders spliced in at hook points (reference models/base_vit.py:827-1086).

    ``add_sae`` puts the SAE module in the place of the HookPoint named ``sae.cfg.hook_point``: the block calls it where it
    called the hook, the SAE (``cfg.return_out_only = True``) hands back its reconstruction, and its own hook points appear in
    ``hook_dict`` / caches as ``<hook_point>.hook_sae_in`` ... ``.hook_sae_out``.  While any SAE is attached the model runs its
    module-by-module route (every op still a C-ABI kernel; the SAE forward is the fused encode -> TopK -> decode engine).
    The reference reads ``sae.cfg.hook_name`` in ``saes()`` but ``sae.cfg.hook_point`` in ``add_sae`` (:857 vs :1078); the config
    only defines ``hook_point``, which is what both use here."""

    def __init__(self, *model_args, **model_kwargs):
        super().__init__(*model_args, **model_kwargs)
        self.acts_to_saes: Dict[str, torch.nn.Module] = {}

    def _fused_blocker(self, x):
        if self.acts_to_saes:
            return f"SAE spliced in at {', '.join(self.acts_to_saes)}"
        return super()._fused_blocker(x)

    def add_sae(self, sae, use_error_term: Optional[bool] = None):
        act_name = sae.cfg.hook_point
        if act_name not in self.acts_to_saes and act_name not in self.hook_dict:
            logging.warning(f"No hook found for {act_name}. Skipping. Check model.hook_dict for available hooks.")
            return
        if use_error_term is not None:
            if not hasattr(sae, "_original_use_error_term"):
                sae._original_use_error_term = getattr(sae, "use_error_term", False)
            sae.use_error_term = use_error_term
        sae.cfg.return_out_only = True
        self.acts_to_saes[act_name] = sae
        parent, leaf = _walk_to_parent(self, act_name)
        setattr(parent, leaf, sae)
        self.setup()

    def _reset_sae(self, act_name: str, prev_sae=None):
        if act_name not in self.acts_to_saes:
            logging.warning(f"No SAE is attached to {act_name}. There's nothing to reset.")
            return
        current = self.acts_to_saes[act_name]
        if hasattr(current, "_original_use_error_term"):
            current.use_error_term = current._original_use_error_term
            delattr(current, "_original_use_error_term")
        parent, leaf = _walk_to_parent(self, act_name)
        if prev_sae:
            setattr(parent, leaf, prev_sae)
            self.acts_to_saes[act_name] = prev_sae
        else:
            setattr(parent, leaf, HookPoint())
            del self.acts_to_saes[act_name]

    def reset_saes(self, act_names: Optional[Union[str, List[str]]] = None, prev_saes: Optional[list] = None):
        if isinstance(act_names, str):
            act_names = [act_names]
        elif act_names is None:
            act_names = list(self.acts_to_saes.keys())
        if prev_saes:
            if len(act_names) != len(prev_saes):
                raise ValueError("act_names and prev_saes must have the same length")
        else:
            prev_saes = [None] * len(act_names)
        for act_name, prev in zip(act_names, prev_saes):
            self._reset_sae(act_name, prev)
        self.setup()

    @contextmanager
    def saes(self, saes=(), reset_saes_end: bool = True, use_error_term: Optional[bool] = None):
        """Temporarily attach ``saes``; previously attached SAEs at the same hook points come back on exit."""
        if isinstance(saes, torch.nn.Module):
            saes = [saes]
        names, previous = [], []
        try:
            for sae in saes:
                names.append(sae.cfg.hook_point)
                previous.append(self.acts_to_saes.get(sae.cfg.hook_point))
                self.add_sae(sae, use_error_term=use_error_term)
            yield self
        finally:
            if reset_saes_end:
                self.reset_saes(names, previous)

    def run_with_saes(self, *model_args, saes=(), reset_saes_end: bool = True, use_error_term: Optional[bool] = None, **model_kwargs):
        with self.saes(saes=saes, reset_saes_end=reset_saes_end, use_error_term=use_error_term):
            return self(*model_args, **model_kwargs)

    def run_with_cache_with_saes(self, *model_args, saes=(), reset_saes_end: bool = True, use_error_term: Optional[bool] = None,
                                 return_cache_object: bool = True, remove_batch_dim: bool = False, **kwargs):
        with self.saes(saes=saes, reset_saes_end=reset_saes_end, use_error_term=use_error_term):
            return self.run_with_cache(*model_args, return_cache_object=return_cache_object, remove_batch_dim=remove_batch_dim, **kwargs)

    def run_with_hooks_with_saes(self, *model_args, saes=(), reset_saes_end: bool = True, fwd_hooks=(), bwd_hooks=(),
                                 reset_hooks_end: bool = True, clear_contexts: bool = False, **model_kwargs):
        with self.saes(saes=saes, reset_saes_end=reset_saes_end):
            return self.run_with_hooks(*model_args, fwd_hooks=list(fwd_hooks), bwd_hooks=list(bwd_hooks), reset_hooks_end=reset_hooks_end,
                                       clear_contexts=clear_contexts, **model_kwargs)
