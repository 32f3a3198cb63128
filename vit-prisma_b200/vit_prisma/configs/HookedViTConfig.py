"""HookedViTConfig -- hyper-parameter record for the hooked ViT.

The constructor signature is API: the reference's callers (and its tests) build the config positionally,
``HookedViTConfig(n_layers, d_model, d_head, d_mlp, ...)``, and by keyword with every name below
(reference: src/vit_prisma/configs/HookedViTConfig.py:8-123).  The record is generated from one table so that the order,
the names and the defaults live in a single place; what the H100 engine does with each group:

  geometry      -> sizes baked into kernel launch descriptors (PbVitForward)
  graph toggles -> select the fused chain vs. the module-by-module hooked route
  inert         -> accepted and stored for drop-in compatibility, never read by the hot path
"""
from __future__ import annotations

from dataclasses import field, make_dataclass
from typing import Any, Dict, List, Optional

import torch

# (name, type, default) in constructor order
_FIELDS = [
    # positional quartet (order is load-bearing)
    ("n_layers", int, None),
    ("d_model", int, None),
    ("d_head", int, None),
    ("d_mlp", int, None),
    # geometry
    ("model_name", str, "custom"),
    ("use_cls_token", bool, True),
    ("n_heads", int, 4),
    ("activation_name", str, "gelu"),
    ("d_vocab", int, -1),
    ("eps", float, 1e-6),
    # graph toggles (mutated at run time by HookedViT.set_use_*)
    ("use_attn_result", bool, False),
    ("use_attn_scale", bool, True),
    ("use_split_qkv_input", bool, False),
    ("use_hook_mlp_in", bool, False),
    ("use_attn_in", bool, False),
    ("use_local_attn", bool, False),
    # inert: provenance / tokenizer leftovers
    ("original_architecture", Optional[str], None),
    ("from_checkpoint", bool, False),
    ("checkpoint_index", Optional[int], None),
    ("checkpoint_label_type", Optional[str], None),
    ("checkpoint_value", Optional[int], None),
    ("tokenizer_name", Optional[str], None),
    ("window_size", Optional[int], None),
    ("attn_types", Optional[List], None),
    ("init_mode", str, "gpt2"),
    ("normalization_type", Optional[str], "LN"),
    ("normalize_output", bool, False),
    ("device", Optional[str], "cpu"),
    ("n_devices", int, 1),
    ("attention_dir", str, "bidirectional"),
    ("attn_only", bool, False),
    ("seed", Optional[int], None),
    ("initializer_range", float, -1.0),
    ("init_weights", bool, True),
    ("scale_attn_by_inverse_layer_idx", bool, False),
    ("positional_embedding_type", str, "standard"),
    ("final_rms", bool, False),
    ("d_vocab_out", int, -1),
    ("parallel_attn_mlp", bool, False),
    ("rotary_dim", Optional[int], None),
    ("n_params", Optional[int], None),
    ("use_hook_tokens", bool, False),
    ("gated_mlp", bool, False),
    ("default_prepend_bos", bool, True),
    ("dtype", torch.dtype, torch.float32),
    ("tokenizer_prepends_bos", Optional[bool], None),
    ("n_key_value_heads", Optional[int], None),
    ("post_embedding_ln", bool, False),
    ("rotary_base", int, 10000),
    ("trust_remote_code", bool, False),
    ("rotary_adjacent_pairs", bool, False),
    # LayerNorm in front of the block stack (CLIP-style towers)
    ("layer_norm_pre", bool, False),
    ("use_bert_block", bool, False),
    # parameter initialisation
    ("weight_type", str, "he"),
    ("cls_std", float, 1e-6),
    ("pos_std", float, 0.02),
    # image geometry
    ("n_channels", int, 3),
    ("patch_size", int, 32),
    ("image_size", int, 224),
    # head
    ("classification_type", str, "cls"),
    ("n_classes", int, 10),
    ("return_type", str, "pre_logits"),
    # inert: logging
    ("log_dir", str, "logs"),
    ("use_wandb", bool, True),
    ("wandb_team_name", str, "perceptual-alignment"),
    ("wandb_project_name", str, None),
    ("log_frequency", int, 1),
    ("print_every", int, 0),
    # inert: supervised-training knobs of the toy trainer
    ("optimizer_name", str, "AdamW"),
    ("lr", float, 3e-4),
    ("weight_decay", float, 0.01),
    ("loss_fn_name", str, "CrossEntropy"),
    ("batch_size", int, 512),
    ("warmup_steps", int, 10),
    ("scheduler_step", int, 200),
    ("scheduler_gamma", float, 0.8),
    ("scheduler_type", str, "WarmupThenStep"),
    ("early_stopping", bool, False),
    ("early_stopping_patience", int, 2),
    ("num_epochs", int, 50),
    ("attn_dropout_rate", float, 0.0),
    ("mlp_dropout_rate", float, 0.0),
    # inert: checkpoint paths
    ("parent_dir", str, ""),
    ("save_dir", str, "Checkpoints"),
    ("save_checkpoints", bool, True),
    ("save_cp_frequency", int, 5),
    # video (tubelet) towers: input [B, C, video_num_frames, S, S], tubelets of video_tubelet_depth frames x P x P
    ("is_video_transformer", bool, False),
    ("video_tubelet_depth", Optional[int], None),
    ("video_num_frames", Optional[int], None),
]


def _from_dict(cls, config_dict: Dict[str, Any]):
    return cls(**config_dict)


def _n_patches(self) -> int:
    n = (self.image_size // self.patch_size) ** 2
    if self.is_video_transformer:
        n *= self.video_num_frames // self.video_tubelet_depth
    return n


def _n_tokens(self) -> int:
    return self.n_patches + (1 if self.use_cls_token else 0)


HookedViTConfig = make_dataclass(
    "HookedViTConfig",
    [(name, typ, field(default=default)) for name, typ, default in _FIELDS],
    namespace={
        "__doc__": "Hyper-parameters of a HookedViT (see the module docstring for the field groups).",
        "max_grad_norm": 1.0,                      # plain class attribute in the reference as well (no annotation -> not a field)
        "from_dict": classmethod(_from_dict),
        # helpers used by the engine (not part of the reference surface)
        "n_patches": property(_n_patches),
        "n_tokens": property(_n_tokens),
    },
)
HookedViTConfig.__module__ = __name__
