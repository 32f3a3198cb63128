"""CPU checker for HookedTextTransformer (reference models/base_text_transformer.py), built on the image oracle's pieces.

The text tower is the ViT block stack behind a token embedding, with an additive ``[T, T]`` mask on the attention scores
(``-inf`` above the diagonal, ``build_causal_mask``, :188-194) and pooling at each row's end-of-text position
(``x[arange(B), ids.argmax(-1)]``, :151).  ``ln_pre`` exists in the module but is never applied.  The LayerNorm and the
activations are ``oracle.vit_oracle``'s; the block loop below is the oracle's loop with the mask added after the scale, as
the reference's ``calculate_attn_scores`` adds it (layers/attention.py:262-264).

Only tests and the fixture generator import this module, and only as the checker.
"""
from __future__ import annotations

import math
from collections import OrderedDict
from typing import Callable, Dict, Optional

import torch
import torch.nn.functional as F

from oracle.vit_oracle import _act, _layer_norm, recipe_state_dict, state_dict_shapes


def text_state_dict_shapes(cfg: dict) -> Dict[str, tuple]:
    """Parameter names and shapes of a HookedTextTransformer: the ViT's blocks, ``ln_pre``, ``ln_final`` and head, with
    ``token_embed.weight [vocab, d]`` and a bare ``pos_embed [context_length, d]`` in place of the patch and position modules."""
    shapes = state_dict_shapes(dict(cfg, layer_norm_pre=True, patch_size=1, image_size=1))
    for k in ("cls_token", "embed.proj.weight", "embed.proj.bias", "pos_embed.W_pos"):
        del shapes[k]
    shapes["token_embed.weight"] = (cfg["vocab_size"], cfg["d_model"])
    shapes["pos_embed"] = (cfg["context_length"], cfg["d_model"])
    return shapes


def text_recipe_state_dict(shapes: Dict[str, tuple], seed: int = 1234, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """The image recipe for the blocks, ln and head; unit-variance token embeddings and 0.1-scale positions from a second
    seeded stream, so the residual entering block 0 is O(1)."""
    emb = {"token_embed.weight", "pos_embed"}
    sd = recipe_state_dict({k: v for k, v in shapes.items() if k not in emb}, seed, torch.float32)
    g = torch.Generator().manual_seed(seed + 1)
    sd["token_embed.weight"] = torch.randn(shapes["token_embed.weight"], generator=g)
    sd["pos_embed"] = 0.1 * torch.randn(shapes["pos_embed"], generator=g)
    return {k: v.to(dtype) for k, v in sd.items()}


def token_batch(batch: int, n_tokens: int, vocab: int, seed: int = 0) -> torch.Tensor:
    """int64 ids in [1, vocab - 1) with the end-of-text id ``vocab - 1`` (the largest) placed at position 0 in row 0, at
    position T-1 in row 1, twice in row 2 (a tie: the first one pools), and at a seeded position in every further row."""
    assert batch >= 3 and n_tokens >= 4
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, vocab - 1, (batch, n_tokens), generator=g)
    eot = vocab - 1
    ids[0, 0] = eot
    ids[1, n_tokens - 1] = eot
    ids[2, 2] = eot
    ids[2, n_tokens - 2] = eot
    for b in range(3, batch):
        ids[b, int(torch.randint(0, n_tokens, (1,), generator=g))] = eot
    return ids


def causal_mask(context_length: int, dtype=torch.float32) -> torch.Tensor:
    """build_causal_mask (:188-194): 0 on and below the diagonal, -inf above it."""
    return torch.full((context_length, context_length), float("-inf")).triu_(1).to(dtype)


def text_forward_with_cache(sd: Dict[str, torch.Tensor], cfg: dict, ids: torch.Tensor, causal: bool = True,
                            names_filter: Optional[Callable[[str], bool]] = None,
                            hooks: Optional[Dict[str, Callable[[torch.Tensor], torch.Tensor]]] = None):
    """``HookedTextTransformer(cfg, no_causal_mask=not causal).run_with_cache(ids, return_cache_object=False)``.

    With ``causal`` the ``[context_length, context_length]`` mask is added to ``[B, H, T, T]`` scores, so a shorter input
    raises ``RuntimeError`` exactly as the reference's does.  ``hooks`` maps a hook name to a function whose result replaces
    the activation at that point, as a forward hook's return value does."""
    dtype = cfg.get("dtype", torch.float32)
    want = names_filter or (lambda name: True)
    cache: "OrderedDict[str, torch.Tensor]" = OrderedDict()

    def emit(name: str, t: torch.Tensor):
        if hooks and name in hooks:
            t = hooks[name](t)
        if want(name):
            cache[name] = t.detach()
        return t

    L, H, dh, eps = cfg["n_layers"], cfg["n_heads"], cfg["d_head"], cfg["eps"]
    B, T = ids.shape
    embed = emit("hook_embed", sd["token_embed.weight"][ids])            # :125
    pos = emit("hook_pos_embed", sd["pos_embed"][:T])                     # :139
    resid = emit("hook_full_embed", embed + pos)                          # :141-143
    mask = causal_mask(cfg["context_length"], dtype) if causal else None

    attn_scale = math.sqrt(dh) if cfg.get("use_attn_scale", True) else 1.0
    for l in range(L):
        p = f"blocks.{l}."
        emit(p + "hook_resid_pre", resid)
        n1 = _layer_norm(resid, sd[p + "ln1.w"], sd[p + "ln1.b"], eps, dtype, emit, p + "ln1.")
        q = emit(p + "attn.hook_q", torch.einsum("bpd,hde->bphe", n1, sd[p + "attn.W_Q"]) + sd[p + "attn.b_Q"])
        k = emit(p + "attn.hook_k", torch.einsum("bpd,hde->bphe", n1, sd[p + "attn.W_K"]) + sd[p + "attn.b_K"])
        v = emit(p + "attn.hook_v", torch.einsum("bpd,hde->bphe", n1, sd[p + "attn.W_V"]) + sd[p + "attn.b_V"])
        scores = torch.einsum("bqhe,bkhe->bhqk", q, k) / attn_scale
        if mask is not None:
            scores = scores + mask                                        # layers/attention.py:263-264
        scores = emit(p + "attn.hook_attn_scores", scores)
        pattern = F.softmax(scores, dim=-1)
        pattern = torch.where(torch.isnan(pattern), torch.zeros_like(pattern), pattern)
        pattern = emit(p + "attn.hook_pattern", pattern)
        z = emit(p + "attn.hook_z", torch.einsum("bkhe,bhqk->bqhe", v, pattern.to(dtype)))
        attn_out = emit(p + "hook_attn_out", torch.einsum("bqhe,hed->bqd", z, sd[p + "attn.W_O"]) + sd[p + "attn.b_O"])
        resid_mid = emit(p + "hook_resid_mid", resid + attn_out)
        n2 = _layer_norm(resid_mid, sd[p + "ln2.w"], sd[p + "ln2.b"], eps, dtype, emit, p + "ln2.")
        pre = emit(p + "mlp.hook_pre", n2 @ sd[p + "mlp.W_in"] + sd[p + "mlp.b_in"])
        post = emit(p + "mlp.hook_post", _act(cfg["activation_name"], pre))
        mlp_out = emit(p + "hook_mlp_out", post @ sd[p + "mlp.W_out"] + sd[p + "mlp.b_out"])
        resid = emit(p + "hook_resid_post", resid_mid + mlp_out)

    xf = _layer_norm(resid, sd["ln_final.w"], sd["ln_final.b"], eps, dtype, emit, "ln_final.")   # :148
    emit("hook_ln_final", xf)
    pooled = xf[torch.arange(B), ids.argmax(dim=-1)]                      # :151
    if cfg.get("return_type", "pre_logits") != "pre_logits":
        pooled = pooled @ sd["head.W_H"] + sd["head.b_H"]
    emit("hook_post_head_pre_normalize", pooled)
    if cfg.get("normalize_output", False):
        pooled = F.normalize(pooled, dim=-1)
    return pooled, cache


# CLIP ViT-B/32 text tower geometry (open_clip "ViT-B-32": width 512, 8 heads, 12 layers, context 77, vocab 49408, embed 512)
CLIP_B32_TEXT = dict(n_layers=12, d_model=512, d_head=64, n_heads=8, d_mlp=2048, context_length=77, vocab_size=49408,
                     n_classes=512, eps=1e-5, activation_name="quick_gelu", normalization_type="LN", normalize_output=True,
                     return_type="class_logits")
