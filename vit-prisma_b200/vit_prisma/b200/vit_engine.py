"""Fused HookedViT forward: plan the cache arena, fill the C descriptors, one ``pb_vit_forward`` call.

What the reference does with 262 Python hook dispatches per forward
(prisma_tools/hooked_root_module.py:289-332 ``_save_hook`` + models/base_vit.py:152-217) happens here as:

  1. decide, per hook name, whether it is wanted (``names_filter``) -- pure Python, no tensors;
  2. carve ONE arena allocation into per-key views with the reference's shapes and dtypes
     (wanted keys) and a per-call scratch allocation for operands nobody asked to keep;
  3. hand raw pointers to the native chain (csrc/vit_chain.cu), which writes every wanted
     activation from a GEMM / LayerNorm / attention epilogue directly into its view;
  4. return ``{name: view}`` in the reference's first-fire key order.

Aliases are preserved, not copied: ``blocks.l.hook_resid_pre`` is the same tensor as
``blocks.l-1.hook_resid_post`` (or ``hook_ln_pre`` / ``hook_full_embed`` for l = 0), ``hook_ln_final``
is ``ln_final``'s output, ``hook_pos_embed`` is a stride-0 view of ``W_pos`` -- exactly the
object identity the reference cache has, because its HookPoints are identities on live tensors.
The views own the arena; nothing is recycled while a returned cache is alive.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Dict, List, Optional, Tuple

import torch

from . import _lib as L
from .ops import dtype_code, _need_cuda
from .packing import PackCache, pack_t, with_lo
from vit_prisma.models import activation_fns

_ALIGN = 256


class _Arena:
    """Two-pass bump allocator: ``reserve`` during planning, ``view`` after ``commit``."""

    def __init__(self, device):
        self.device = device
        self.size = 0
        self.buf: Optional[torch.Tensor] = None

    def reserve(self, shape, dtype) -> Tuple[int, tuple, torch.dtype]:
        n = 1
        for s in shape:
            n *= s
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        off = self.size
        self.size = (off + nbytes + _ALIGN - 1) // _ALIGN * _ALIGN
        return off, tuple(shape), dtype

    def commit(self) -> None:
        self.buf = torch.empty(max(self.size, 1), dtype=torch.uint8, device=self.device)

    def view(self, slot) -> torch.Tensor:
        off, shape, dtype = slot
        n = 1
        for s in shape:
            n *= s
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        return self.buf[off:off + nbytes].view(dtype).view(shape)


class _Plan:
    """One call's cache arena (wanted keys) and scratch (operands nobody asked to keep), and the slot of every buffer."""

    def __init__(self, device, want: Callable[[str], bool]):
        self.want = want
        self.arena, self.scratch = _Arena(device), _Arena(device)
        self.slots: Dict[str, tuple] = {}          # wanted key -> arena slot
        self.tmp: Dict[str, tuple] = {}            # internal name -> scratch slot

    def place(self, key: str, shape, dtype, required: bool, share: Optional[str] = None, force: bool = False):
        """Arena slot if the key is wanted (or ``force``), scratch if only compute needs it, else None.
        ``share`` names a scratch buffer reused by every layer: on one in-order stream layer l-1's
        unkept operands are dead by the time layer l produces its own."""
        if force or self.want(key):
            self.slots[key] = self.arena.reserve(shape, dtype)
            return ("a", key)
        if required:
            skey = share or key
            if skey not in self.tmp:
                self.tmp[skey] = self.scratch.reserve(shape, dtype)
            return ("s", skey)
        return None

    def place_either(self, key: str, shape, dtype, wanted_any: bool):
        """A required buffer kept under ``key`` when any of the names it serves is wanted, else scratch."""
        if wanted_any:
            self.slots[key] = self.arena.reserve(shape, dtype)
            return ("a", key)
        self.tmp[key] = self.scratch.reserve(shape, dtype)
        return ("s", key)

    def commit(self) -> None:
        self.arena.commit()
        self.scratch.commit()

    def get(self, ref) -> torch.Tensor:
        kind, key = ref
        return self.arena.view(self.slots[key]) if kind == "a" else self.scratch.view(self.tmp[key])

    def ptr(self, ref) -> Optional[int]:
        return None if ref is None else self.get(ref).data_ptr()


_SPILL_NAMES = ("ln1_scale", "ln1_norm_f32", "ln1_out", "q", "k", "v", "scores", "pattern", "z", "attn_out",
                "resid_mid", "ln2_scale", "ln2_norm_f32", "ln2_out", "pre", "post", "mlp_out", "resid_post")


def _layer_weights(blocks, affine: bool):
    """The PbVitLayerW table of ``blocks`` and the packed tensors it points into."""
    keep: List[torch.Tensor] = []
    layers = (L.PbVitLayerW * len(blocks))()
    for l, blk in enumerate(blocks):
        wqkv, wqkv_lo, bqkv = blk.attn.packed_qkv()
        wo, wo_lo = blk.attn.packed_o()
        win, win_lo = blk.mlp.packed_in()
        wout, wout_lo = blk.mlp.packed_out()
        keep += [wqkv, wqkv_lo, bqkv, wo, wo_lo, win, win_lo, wout, wout_lo]
        W = layers[l]
        if affine:
            W.ln1_w, W.ln1_b = blk.ln1.w.data_ptr(), blk.ln1.b.data_ptr()
            W.ln2_w, W.ln2_b = blk.ln2.w.data_ptr(), blk.ln2.b.data_ptr()
        W.wqkv, W.bqkv = wqkv.data_ptr(), bqkv.data_ptr()
        W.wo, W.bo = wo.data_ptr(), blk.attn.b_O.data_ptr()
        W.win, W.bin = win.data_ptr(), blk.mlp.b_in.data_ptr()
        W.wout, W.bout = wout.data_ptr(), blk.mlp.b_out.data_ptr()
        if wqkv_lo is not None:
            W.wqkv_lo, W.wo_lo = wqkv_lo.data_ptr(), wo_lo.data_ptr()
            W.win_lo, W.wout_lo = win_lo.data_ptr(), wout_lo.data_ptr()
    return layers, keep


def _plan_blocks(pl: _Plan, cfg, B: int, T: int, n_run: int, run_head: bool) -> list:
    """Slots of every block's buffers; resid_post(l) is kept when it doubles as a wanted resid_pre(l+1)."""
    d, H, dh, dm, dt = cfg.d_model, cfg.n_heads, cfg.d_head, cfg.d_mlp, cfg.dtype
    fp32, want, place = dt == torch.float32, pl.want, pl.place
    layer_plans = []
    for l in range(n_run):
        p = f"blocks.{l}."
        lp = {}
        for ln_name in ("ln1", "ln2"):
            lp[f"{ln_name}_scale"] = place(p + f"{ln_name}.hook_scale", (B, T, 1), torch.float32, False)
            if fp32:
                lp[f"{ln_name}_norm_f32"] = None
                lp[f"{ln_name}_out"] = place(p + f"{ln_name}.hook_normalized", (B, T, d), dt, True, share=f"L.{ln_name}")
            else:
                lp[f"{ln_name}_norm_f32"] = place(p + f"{ln_name}.hook_normalized", (B, T, d), torch.float32, False)
                if f"L.{ln_name}" not in pl.tmp:
                    pl.tmp[f"L.{ln_name}"] = pl.scratch.reserve((B, T, d), dt)
                lp[f"{ln_name}_out"] = ("s", f"L.{ln_name}")
        for nm in ("q", "k", "v", "z"):
            lp[nm] = place(p + f"attn.hook_{nm}", (B, T, H, dh), dt, True, share=f"L.{nm}")
        lp["scores"] = place(p + "attn.hook_attn_scores", (B, H, T, T), dt, False)
        lp["pattern"] = place(p + "attn.hook_pattern", (B, H, T, T), dt, False)
        lp["attn_out"] = place(p + "hook_attn_out", (B, T, d), dt, False)
        lp["resid_mid"] = place(p + "hook_resid_mid", (B, T, d), dt, True, share="L.resid_mid")
        lp["pre"] = place(p + "mlp.hook_pre", (B, T, dm), dt, False)
        lp["post"] = place(p + "mlp.hook_post", (B, T, dm), dt, True, share="L.post")
        lp["mlp_out"] = place(p + "hook_mlp_out", (B, T, d), dt, False)
        # resid_post doubles as the next block's resid_pre (same tensor in the reference cache);
        # unkept ones ping-pong between two scratch buffers
        keep = (l + 1 < cfg.n_layers and want(f"blocks.{l + 1}.hook_resid_pre")) or (l == n_run - 1 and not run_head)
        lp["resid_post"] = place(p + "hook_resid_post", (B, T, d), dt, True, share=f"L.resid_post{l % 2}", force=keep)
        layer_plans.append(lp)
    return layer_plans


def _spill_table(pl: _Plan, layer_plans: list):
    spills = (L.PbVitLayerSpill * max(len(layer_plans), 1))()
    for l, lp in enumerate(layer_plans):
        for name in _SPILL_NAMES:
            setattr(spills[l], name, pl.ptr(lp[name]))
    return spills


def _emit_blocks(emit, get, layer_plans: list, fp32: bool, resid_ref):
    """Cache entries of every block in the reference's first-fire order; returns the last residual's slot."""
    for l, lp in enumerate(layer_plans):
        p = f"blocks.{l}."
        emit(p + "hook_resid_pre", lambda r=resid_ref: get(r))
        emit(p + "ln1.hook_scale", lambda: get(lp["ln1_scale"]))
        emit(p + "ln1.hook_normalized", lambda: get(lp["ln1_out"] if fp32 else lp["ln1_norm_f32"]))
        emit(p + "attn.hook_q", lambda: get(lp["q"]))
        emit(p + "attn.hook_k", lambda: get(lp["k"]))
        emit(p + "attn.hook_v", lambda: get(lp["v"]))
        emit(p + "attn.hook_attn_scores", lambda: get(lp["scores"]))
        emit(p + "attn.hook_pattern", lambda: get(lp["pattern"]))
        emit(p + "attn.hook_z", lambda: get(lp["z"]))
        emit(p + "hook_attn_out", lambda: get(lp["attn_out"]))
        emit(p + "hook_resid_mid", lambda: get(lp["resid_mid"]))
        emit(p + "ln2.hook_scale", lambda: get(lp["ln2_scale"]))
        emit(p + "ln2.hook_normalized", lambda: get(lp["ln2_out"] if fp32 else lp["ln2_norm_f32"]))
        emit(p + "mlp.hook_pre", lambda: get(lp["pre"]))
        emit(p + "mlp.hook_post", lambda: get(lp["post"]))
        emit(p + "hook_mlp_out", lambda: get(lp["mlp_out"]))
        emit(p + "hook_resid_post", lambda: get(lp["resid_post"]))
        resid_ref = lp["resid_post"]
    return resid_ref


def _plan_ln_final(pl: _Plan, plan: dict, B: int, T: int, d: int, dt) -> None:
    plan["lnf_scale"] = pl.place("ln_final.hook_scale", (B, T, 1), torch.float32, False)
    if dt == torch.float32:
        # one tensor serves ln_final.hook_normalized and hook_ln_final
        wanted_any = pl.want("ln_final.hook_normalized") or pl.want("hook_ln_final")
        plan["lnf_out"] = pl.place_either("ln_final.hook_normalized", (B, T, d), dt, wanted_any)
        plan["lnf_norm_f32"] = None
    else:
        plan["lnf_norm_f32"] = pl.place("ln_final.hook_normalized", (B, T, d), torch.float32, False)
        plan["lnf_out"] = pl.place("hook_ln_final", (B, T, d), dt, True)


def _emit_tail(emit, pl: _Plan, plan: dict, fp32: bool, normalize_output: bool):
    """ln_final .. hook_post_head_pre_normalize cache entries; returns the model output."""
    emit("ln_final.hook_scale", lambda: pl.get(plan["lnf_scale"]))
    emit("ln_final.hook_normalized", lambda: pl.get(plan["lnf_out"] if fp32 else plan["lnf_norm_f32"]))
    emit("hook_ln_final", lambda: pl.get(plan["lnf_out"]))
    pre_norm = pl.arena.view(pl.slots["__pre_normalize"])
    emit("hook_post_head_pre_normalize", lambda: pre_norm)
    return pl.arena.view(pl.slots["__out"]) if normalize_output else pre_norm


def fusable_reason(model, x: torch.Tensor) -> Optional[str]:
    """None when the fused chain can serve ``model(x)``; else a human-readable reason."""
    cfg = model.cfg
    video = cfg.is_video_transformer
    if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dim() == (5 if video else 4)):
        return "input is not a CUDA [B,C,F,H,W] tensor" if video else "input is not a CUDA [B,C,H,W] tensor"
    if cfg.dtype not in (torch.float32, torch.bfloat16):
        return f"dtype {cfg.dtype}"
    if cfg.use_bert_block or cfg.attn_only:
        return "bert / attn-only architecture"
    if cfg.normalization_type not in ("LN", "LNPre"):
        return "normalization_type is not LN/LNPre"
    if cfg.activation_name not in activation_fns.ELEMENTWISE:
        return f"activation {cfg.activation_name} is not element-wise"
    if cfg.use_attn_result or cfg.use_split_qkv_input or cfg.use_attn_in or cfg.use_hook_mlp_in:
        return "a cfg.use_* toggle adds conditional hook points"
    if cfg.classification_type not in ("cls", "gaap") or "dino-vitb" in cfg.model_name:
        return "pooling variant"
    if cfg.classification_type == "cls" and not cfg.use_cls_token:
        pass  # x[:, 0] is still well defined
    if model.training and (cfg.attn_dropout_rate > 0 or cfg.mlp_dropout_rate > 0):
        return "dropout active"
    if x.shape[1] != cfg.n_channels or x.shape[-2] != cfg.image_size or x.shape[-1] != cfg.image_size:
        return "image geometry differs from cfg"
    if video and x.shape[2] // cfg.video_tubelet_depth != cfg.video_num_frames // cfg.video_tubelet_depth:
        return "number of tubelets differs from cfg (W_pos would not match)"
    if model.cls_token.device != x.device:
        return "model and input on different devices"
    if torch.is_grad_enabled() and any(p.requires_grad for p in (model.cls_token,)) and x.requires_grad:
        return "autograd through the input requested"
    return None


class VitEngine:
    """Per-model helper owning the packed-weight cache and the descriptor builders."""

    def __init__(self, model):
        self.model = model
        self._packs = PackCache()
        self._wtable = None
        self._wtable_stamp = None

    # ------------------------------------------------------------------ weights
    def _weight_table(self):
        m, cfg = self.model, self.model.cfg
        params = [p for p in m.parameters()]
        stamp = tuple((p.data_ptr(), p._version) for p in params)
        if self._wtable is not None and self._wtable_stamp == stamp:
            return self._wtable
        layers, keep = _layer_weights(m.blocks, cfg.normalization_type == "LN")   # keep: tensors the table points into
        head_w, head_w_lo = m.head.packed()
        pw = m.embed.proj.weight.detach().reshape(cfg.d_model, -1)
        patch_w, patch_w_lo = self._packs.get("patch", (m.embed.proj.weight,), lambda: with_lo(pw.contiguous()))
        keep += [head_w, head_w_lo, patch_w, patch_w_lo]
        self._wtable = (layers, keep, head_w, head_w_lo, patch_w, patch_w_lo)
        self._wtable_stamp = stamp
        return self._wtable

    # --------------------------------------------------------------------- run
    @torch.no_grad()
    def run(self, x: torch.Tensor, want: Callable[[str], bool], stop_at_layer: Optional[int],
            gemm_impl: int = L.GEMM_AUTO):
        """Returns (model_out, cache_dict) -- cache_dict ordered like the reference's first-fire order."""
        m, cfg = self.model, self.model.cfg
        _need_cuda(x)
        dev, dt = x.device, cfg.dtype
        fp32 = dt == torch.float32
        B, T, NP = x.shape[0], cfg.n_tokens, cfg.n_patches
        d, H, dh, dm = cfg.d_model, cfg.n_heads, cfg.d_head, cfg.d_mlp
        HD = H * dh
        n_run = len(range(cfg.n_layers)[:stop_at_layer]) if stop_at_layer is not None else cfg.n_layers
        run_head = stop_at_layer is None
        affine = cfg.normalization_type == "LN"
        head_proj = cfg.return_type != "pre_logits"
        out_cols = cfg.n_classes if head_proj else d

        x = x.contiguous()
        if x.dtype != dt:
            from . import ops
            x = ops.cast(x, dt)

        pl = _Plan(dev, want)
        place, tmp, scratch = pl.place, pl.tmp, pl.scratch
        plan: Dict[str, object] = {}
        depth = cfg.video_tubelet_depth if cfg.is_video_transformer else 1
        K_patch = cfg.n_channels * depth * cfg.patch_size ** 2          # patch GEMM K: C*D*P*P (D = 1 for images)
        plan["patches"] = ("s", "patches")
        tmp["patches"] = scratch.reserve((B * NP, K_patch), dt)
        plan["embed"] = place("hook_embed", (B, NP, d), dt, True)
        plan["full_embed"] = place("hook_full_embed", (B, T, d), dt, True)
        if cfg.layer_norm_pre:
            plan["lnpre_scale"] = place("ln_pre.hook_scale", (B, T, 1), torch.float32, False)
            if fp32:
                # one tensor serves ln_pre.hook_normalized, hook_ln_pre and blocks.0.hook_resid_pre
                wanted_any = want("ln_pre.hook_normalized") or want("hook_ln_pre") or want("blocks.0.hook_resid_pre")
                plan["lnpre_out"] = pl.place_either("ln_pre.hook_normalized", (B, T, d), dt, wanted_any)
                plan["lnpre_norm_f32"] = None
            else:
                plan["lnpre_norm_f32"] = place("ln_pre.hook_normalized", (B, T, d), torch.float32, False)
                wanted_any = want("hook_ln_pre") or want("blocks.0.hook_resid_pre")
                plan["lnpre_out"] = pl.place_either("hook_ln_pre", (B, T, d), dt, wanted_any)

        layer_plans = _plan_blocks(pl, cfg, B, T, n_run, run_head)

        if run_head:
            _plan_ln_final(pl, plan, B, T, d, dt)
            if cfg.classification_type == "gaap":
                tmp["pooled"] = scratch.reserve((B, d), dt)
            pl.slots["__pre_normalize"] = pl.arena.reserve((B, out_cols), dt)
            if cfg.normalize_output:
                pl.slots["__out"] = pl.arena.reserve((B, out_cols), dt)

        x3 = fp32 and gemm_impl != L.GEMM_SIMT
        if x3:
            lo_elems = max(B * T * (d + max(dm, HD)), B * NP * K_patch)
            tmp["lo"] = scratch.reserve((lo_elems,), torch.float32)

        pl.commit()
        ptr = pl.ptr

        layers, _keep, head_w, head_w_lo, patch_w, patch_w_lo = self._weight_table()
        f = L.PbVitForward()
        f.batch, f.n_channels, f.image_size, f.patch_size = B, cfg.n_channels, cfg.image_size, cfg.patch_size
        f.n_patches, f.n_tokens, f.d_model, f.n_heads, f.d_head, f.d_mlp = NP, T, d, H, dh, dm
        f.n_classes, f.n_layers_run, f.run_head = cfg.n_classes, n_run, int(run_head)
        f.use_cls, f.layer_norm_pre = int(cfg.use_cls_token), int(cfg.layer_norm_pre)
        f.normalize_output, f.head_proj = int(cfg.normalize_output), int(head_proj)
        f.pool_gaap = int(cfg.classification_type == "gaap")
        f.act, f.dtype, f.gemm_impl = L.ACT[cfg.activation_name], dtype_code(dt), gemm_impl
        f.eps = float(cfg.eps)
        f.attn_scale = float(m.blocks[0].attn.attn_scale) if cfg.n_layers else 1.0
        f.images = x.data_ptr()
        if cfg.is_video_transformer:
            f.n_frames, f.tubelet_depth = x.shape[2], depth
        f.patch_w, f.patch_b = patch_w.data_ptr(), m.embed.proj.bias.data_ptr()
        f.patch_w_lo = patch_w_lo.data_ptr() if patch_w_lo is not None else None
        f.cls, f.pos = m.cls_token.data_ptr(), m.pos_embed.W_pos.data_ptr()
        if cfg.layer_norm_pre and affine:
            f.lnpre_w, f.lnpre_b = m.ln_pre.w.data_ptr(), m.ln_pre.b.data_ptr()
        if affine:
            f.lnf_w, f.lnf_b = m.ln_final.w.data_ptr(), m.ln_final.b.data_ptr()
        f.head_w, f.head_b = head_w.data_ptr(), m.head.b_H.data_ptr()
        f.head_w_lo = head_w_lo.data_ptr() if head_w_lo is not None else None
        f.layers_host = C.cast(layers, C.POINTER(L.PbVitLayerW))
        f.patches, f.embed, f.full_embed = ptr(plan["patches"]), ptr(plan["embed"]), ptr(plan["full_embed"])
        if cfg.layer_norm_pre:
            f.lnpre_scale, f.lnpre_norm_f32, f.lnpre_out = ptr(plan["lnpre_scale"]), ptr(plan["lnpre_norm_f32"]), ptr(plan["lnpre_out"])
        spills = _spill_table(pl, layer_plans)
        f.spills_host = C.cast(spills, C.POINTER(L.PbVitLayerSpill))
        if run_head:
            f.lnf_scale, f.lnf_norm_f32, f.lnf_out = ptr(plan["lnf_scale"]), ptr(plan["lnf_norm_f32"]), ptr(plan["lnf_out"])
            if "pooled" in tmp:
                f.pooled = scratch.view(tmp["pooled"]).data_ptr()
            f.pre_normalize = pl.arena.view(pl.slots["__pre_normalize"]).data_ptr()
            f.out = pl.arena.view(pl.slots["__out"] if cfg.normalize_output else pl.slots["__pre_normalize"]).data_ptr()
        if x3:
            f.lo_scratch = scratch.view(tmp["lo"]).data_ptr()

        L.check(L.get_lib().pb_vit_forward(C.byref(f), torch.cuda.current_stream().cuda_stream), "pb_vit_forward")

        # ------------------------------------------------------------ cache dict
        get = pl.get
        cache: Dict[str, torch.Tensor] = {}

        def emit(key: str, tensor_fn):
            if want(key):
                cache[key] = tensor_fn()

        emit("hook_embed", lambda: get(plan["embed"]))
        emit("hook_pos_embed", lambda: m.pos_embed.W_pos.detach().unsqueeze(0).expand(B, -1, -1))
        emit("hook_full_embed", lambda: get(plan["full_embed"]))
        resid_ref = plan["full_embed"]
        if cfg.layer_norm_pre:
            emit("ln_pre.hook_scale", lambda: get(plan["lnpre_scale"]))
            emit("ln_pre.hook_normalized", lambda: get(plan["lnpre_out"] if fp32 else plan["lnpre_norm_f32"]))
            emit("hook_ln_pre", lambda: get(plan["lnpre_out"]))
            resid_ref = plan["lnpre_out"]
        resid_ref = _emit_blocks(emit, get, layer_plans, fp32, resid_ref)
        if not run_head:
            return get(resid_ref), cache
        return _emit_tail(emit, pl, plan, fp32, cfg.normalize_output), cache


def text_fusable_reason(model, ids: torch.Tensor) -> Optional[str]:
    """None when the fused text chain can serve ``model(ids)``; else a human-readable reason."""
    cfg = model.cfg
    if not (isinstance(ids, torch.Tensor) and ids.is_cuda and ids.dim() == 2 and ids.dtype in (torch.int32, torch.int64)):
        return "input is not a CUDA integer [B, T] tensor"
    if model.cls_emb is not None:
        return "cls token"
    T = ids.shape[1]
    if model.attn_mask is not None and T != model.attn_mask.shape[-1]:
        return f"{T} tokens against a causal mask of {model.attn_mask.shape[-1]}"
    if T > cfg.context_length:
        return f"{T} tokens exceed the context of {cfg.context_length}"
    if cfg.dtype not in (torch.float32, torch.bfloat16):
        return f"dtype {cfg.dtype}"
    if cfg.activation_name not in activation_fns.ELEMENTWISE:
        return f"activation {cfg.activation_name} is not element-wise"
    if cfg.use_attn_result or cfg.use_split_qkv_input or cfg.use_attn_in or cfg.use_hook_mlp_in:
        return "a cfg.use_* toggle adds conditional hook points"
    if model.training and (cfg.attn_dropout_rate > 0 or cfg.mlp_dropout_rate > 0):
        return "dropout active"
    if model.token_embed.weight.device != ids.device:
        return "model and input on different devices"
    return None


class TextEngine:
    """The fused HookedTextTransformer forward: the arena plan of ``VitEngine.run`` around ``pb_text_forward``."""

    def __init__(self, model):
        self.model = model
        self._wtable = None
        self._wtable_stamp = None

    def _weight_table(self):
        m = self.model
        stamp = tuple((p.data_ptr(), p._version) for p in m.parameters())
        if self._wtable is None or self._wtable_stamp != stamp:
            layers, keep = _layer_weights(m.blocks, True)
            head_w, head_w_lo = m.head.packed()
            self._wtable = (layers, keep + [head_w, head_w_lo], head_w, head_w_lo)
            self._wtable_stamp = stamp
        return self._wtable

    @torch.no_grad()
    def run(self, ids: torch.Tensor, want: Callable[[str], bool], stop_at_layer: Optional[int] = None,
            gemm_impl: int = L.GEMM_AUTO):
        """``ids``: int64 CUDA [B, T], already range-checked.  Returns (model_out, cache_dict) in the reference's key order."""
        if stop_at_layer is not None:
            raise TypeError("HookedTextTransformer.forward() got an unexpected keyword argument 'stop_at_layer'")
        m, cfg = self.model, self.model.cfg
        _need_cuda(ids)
        ids = ids.contiguous()
        dev, dt = ids.device, cfg.dtype
        fp32 = dt == torch.float32
        B, T = ids.shape
        d, H, dh, dm = cfg.d_model, cfg.n_heads, cfg.d_head, cfg.d_mlp
        head_proj = cfg.return_type != "pre_logits"
        out_cols = cfg.n_classes if head_proj else d

        pl = _Plan(dev, want)
        plan: Dict[str, object] = {}
        plan["embed"] = pl.place("hook_embed", (B, T, d), dt, True)
        plan["full_embed"] = pl.place("hook_full_embed", (B, T, d), dt, True)
        layer_plans = _plan_blocks(pl, cfg, B, T, cfg.n_layers, True)
        _plan_ln_final(pl, plan, B, T, d, dt)
        pl.tmp["pooled"] = pl.scratch.reserve((B, d), dt)
        pl.slots["__pre_normalize"] = pl.arena.reserve((B, out_cols), dt)
        if cfg.normalize_output:
            pl.slots["__out"] = pl.arena.reserve((B, out_cols), dt)
        x3 = fp32 and gemm_impl != L.GEMM_SIMT
        if x3:
            pl.tmp["lo"] = pl.scratch.reserve((B * T * (d + max(dm, H * dh)),), torch.float32)
        pl.commit()
        ptr = pl.ptr

        layers, _keep, head_w, head_w_lo = self._weight_table()
        f = L.PbTextForward()
        f.batch, f.n_tokens, f.vocab, f.d_model, f.n_heads, f.d_head, f.d_mlp = B, T, cfg.vocab_size, d, H, dh, dm
        f.n_classes, f.n_layers, f.causal = cfg.n_classes, cfg.n_layers, int(m.attn_mask is not None)
        f.normalize_output, f.head_proj = int(cfg.normalize_output), int(head_proj)
        f.act, f.dtype, f.gemm_impl = L.ACT[cfg.activation_name], dtype_code(dt), gemm_impl
        f.eps = float(cfg.eps)
        f.attn_scale = float(m.blocks[0].attn.attn_scale) if cfg.n_layers else 1.0
        f.ids = ids.data_ptr()
        f.token_w, f.pos = m.token_embed.weight.data_ptr(), m.pos_embed.data_ptr()
        f.lnf_w, f.lnf_b = m.ln_final.w.data_ptr(), m.ln_final.b.data_ptr()
        f.head_w, f.head_b = head_w.data_ptr(), m.head.b_H.data_ptr()
        f.head_w_lo = head_w_lo.data_ptr() if head_w_lo is not None else None
        f.layers_host = C.cast(layers, C.POINTER(L.PbVitLayerW))
        f.embed, f.full_embed = ptr(plan["embed"]), ptr(plan["full_embed"])
        spills = _spill_table(pl, layer_plans)
        f.spills_host = C.cast(spills, C.POINTER(L.PbVitLayerSpill))
        f.lnf_scale, f.lnf_norm_f32, f.lnf_out = ptr(plan["lnf_scale"]), ptr(plan["lnf_norm_f32"]), ptr(plan["lnf_out"])
        f.pooled = pl.scratch.view(pl.tmp["pooled"]).data_ptr()
        f.pre_normalize = pl.arena.view(pl.slots["__pre_normalize"]).data_ptr()
        f.out = pl.arena.view(pl.slots["__out"] if cfg.normalize_output else pl.slots["__pre_normalize"]).data_ptr()
        if x3:
            f.lo_scratch = pl.scratch.view(pl.tmp["lo"]).data_ptr()

        L.check(L.get_lib().pb_text_forward(C.byref(f), torch.cuda.current_stream().cuda_stream), "pb_text_forward")

        cache: Dict[str, torch.Tensor] = {}

        def emit(key: str, tensor_fn):
            if want(key):
                cache[key] = tensor_fn()

        emit("hook_embed", lambda: pl.get(plan["embed"]))
        emit("hook_pos_embed", lambda: m.pos_embed.detach()[:T])        # a view of pos_embed, as the reference caches it
        emit("hook_full_embed", lambda: pl.get(plan["full_embed"]))
        _emit_blocks(emit, pl.get, layer_plans, fp32, plan["full_embed"])
        return _emit_tail(emit, pl, plan, fp32, cfg.normalize_output), cache
