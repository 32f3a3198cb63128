"""ORACLE (test infrastructure, not product code): CPU restatement of the SAE forward and training step
(TopK and dense ReLU + L1 activations, optional ghost-grad auxiliary loss).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may import this, and only
as the checker.  Restates, with explicit gradient formulas instead of autograd (so the hand-written CUDA backward is
checked against an independent derivation that is itself pinned to the reference's autograd):

  StandardSparseAutoencoder.encode/decode/forward      sae/sae.py:557-645
  run-time input normalisation ("layer_norm")           sae/sae.py:78-90
  _compute_mse_loss                                     sae/sae.py:144-149
  TopK activation                                       sae/sae.py:795-808
  ReLU activation + L1 sparsity term                    sae/sae.py:617-626, 810-839
  ghost-grad residual loss on dead features             sae/sae.py:151-179, train_sae.py:330-332
  set_decoder_norm_to_unit_norm / remove_gradient_...   sae/sae.py:275-297
  VisionSAETrainer.train_step ordering, clipping, Adam  sae/train_sae.py:278-411 (torch.optim.Adam defaults)
  cosineannealingwarmup schedule                        sae/training/get_scheduler.py:42-53, train_sae.py:235
  GatedSparseAutoencoder forward / training step        sae/sae.py:648-792
  Transcoder forward / training step on (input, target) sae/transcoder.py:6-116, train_sae.py:299-301

Pinning: tests/test_oracle_golden.py compares against tests/golden/{sae_tiny_*, sae_gated_*, transcoder_*, sae_bf16_v}.pt, produced by running the
UNMODIFIED reference modules + torch autograd + torch.optim.Adam in the build container
(tests/golden/make_golden_sae.py).  The reference has no numeric test of this path (SURVEY section 4), so the
reference itself, run here, is the anchor.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch


def normalise_in(x: torch.Tensor, mode: str, eps: float = 1e-5):
    if mode == "layer_norm":                           # sae.py:78-87
        mu = x.mean(dim=-1, keepdim=True)
        xc = x - mu
        std = xc.std(dim=-1, keepdim=True)             # unbiased
        return xc / (std + eps), mu, std
    if mode == "constant_norm_rescale":                # sae.py:60-72
        coeff = (x.shape[-1] ** 0.5) / x.norm(dim=-1, keepdim=True)
        return x * coeff, torch.zeros_like(coeff), 1.0 / coeff
    return x, torch.zeros_like(x[..., :1]), torch.ones_like(x[..., :1])


def sae_forward(p: Dict[str, torch.Tensor], x: torch.Tensor, k: int, mode: str = "layer_norm", xbar: Optional[torch.Tensor] = None,
                global_rows: Optional[int] = None, act: str = "topk", l1_coefficient: float = 0.0,
                dead_mask: Optional[torch.Tensor] = None, topk_idx: Optional[torch.Tensor] = None,
                topk_val: Optional[torch.Tensor] = None, relu_mask: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """p: W_enc [d,F], W_dec [F,d], b_enc [F], b_dec [d].
    ``xbar`` / ``global_rows``: data-parallel shard view -- batch mean and token count of the GLOBAL batch, so that the
    shard's loss share and gradients sum over shards to the single-process values.
    ``act``: "topk" | "relu".  ``dead_mask`` [F] bool (not None <=> cfg.use_ghost_grads in training mode): ghost term.
    ``topk_idx`` [rows, k] (and ``topk_val``): take this TopK selection (and these pre-activation values) instead of
    torch.topk's, so that the rest of the step can be checked on the same support as an implementation whose fp32
    selection legitimately differs in a near-tie row.
    ``relu_mask`` [rows, F] bool (act="relu"): take this support instead of hidden_pre > 0 (feature_acts = hidden_pre * mask,
    the gradient masked by it), so that a pre-activation within round-off of zero that an implementation puts on the other side
    of the ReLU does not hide the rest of the step.  ``active`` in the result is the support the gradient and the counters use."""
    xn, mu, std = normalise_in(x, mode)
    sae_in = xn - p["b_dec"]                            # sae.py:564-566
    hidden_pre = sae_in @ p["W_enc"] + p["b_enc"]      # :568-574
    if act == "topk":
        if topk_idx is None:
            top = torch.topk(hidden_pre, k=k, dim=-1)   # :803-805
            idx, raw_val = top.indices, top.values
        else:
            idx = topk_idx.to(hidden_pre.device).long()
            raw_val = hidden_pre.gather(-1, idx) if topk_val is None else topk_val.to(hidden_pre)
        feature_acts = torch.zeros_like(hidden_pre).scatter_(-1, idx, torch.relu(raw_val))   # :806-808
    elif act == "relu":
        if relu_mask is None:
            feature_acts = torch.relu(hidden_pre)       # :810-839 get_activation_fn("relu")
        else:
            feature_acts = hidden_pre * relu_mask.to(hidden_pre.device, torch.bool)
        idx = raw_val = None
    else:
        raise ValueError(act)
    out_n = feature_acts @ p["W_dec"] + p["b_dec"]     # :584-592
    sae_out = out_n * std + mu if mode == "layer_norm" else (out_n * std if mode == "constant_norm_rescale" else out_n)
    x_centred = x - (x.mean(dim=0, keepdim=True) if xbar is None else xbar)   # :145
    nf = torch.norm(x_centred, p=2, dim=-1, keepdim=True)
    rows = global_rows or x.shape[0]
    mse = (((sae_out - x) ** 2) / nf).sum() / (rows * x.shape[1])   # :146-148 (.mean())
    l1 = None
    if act != "topk":                                   # :617-626 (lp_norm = 1)
        l1 = l1_coefficient * feature_acts.abs().sum(dim=1).sum() / rows
    active = feature_acts > 0 if relu_mask is None else relu_mask.to(hidden_pre.device, torch.bool)
    out = dict(sae_in=sae_in, hidden_pre=hidden_pre, idx=idx, raw_val=raw_val, feature_acts=feature_acts, active=active,
               sae_out=sae_out, mse=mse, nf=nf, std=std, mu=mu, l1=l1, ghost=torch.zeros(()))
    if dead_mask is not None:                           # :151-179 _compute_ghost_residual_loss (single-process form)
        r = x - sae_out
        rcn = (r - r.mean(dim=0, keepdim=True)).pow(2).sum(dim=-1, keepdim=True).sqrt()
        l2r = torch.norm(r, dim=-1)
        E = torch.exp(hidden_pre[:, dead_mask])
        G0 = E @ p["W_dec"][dead_mask, :]
        scale = l2r / (1e-6 + torch.norm(G0, dim=-1) * 2)
        G = G0 * scale[:, None]
        Lel = (G - r).pow(2) / rcn
        c = mse / (Lel + 1e-6)
        out.update(ghost=(c * Lel).mean(), ghost_E=E, ghost_dG0=(c * 2.0 * (G - r) / rcn / Lel.numel()) * scale[:, None])
    out["loss"] = mse + (l1 if l1 is not None else 0.0) + out["ghost"]
    return out


def sae_grads(p: Dict[str, torch.Tensor], x: torch.Tensor, fwd: Dict[str, torch.Tensor], mode: str = "layer_norm",
              global_rows: Optional[int] = None, l1_coefficient: float = 0.0, dead_mask: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """Gradients of the loss wrt the four parameters, closed form (matches loss.backward() of the reference graph)."""
    Bt, d = x.shape
    Bt = global_rows or Bt
    std = fwd["std"] if mode != "none" else torch.ones_like(fwd["nf"])
    g = 2.0 * (fwd["sae_out"] - x) * std / (fwd["nf"] * Bt * d)          # dL/d out_n
    acts = fwd["feature_acts"]
    gW_dec = acts.t() @ g
    d_acts = g @ p["W_dec"].t()
    if fwd["l1"] is not None:
        d_acts = d_acts + l1_coefficient / Bt                             # d(l1)/d(acts) where acts > 0 (|a| = a)
    d_pre = d_acts * fwd["active"]                                        # ReLU mask (AND the TopK support)
    if dead_mask is not None:                                             # ghost path: only G depends on the parameters
        E, dG0 = fwd["ghost_E"], fwd["ghost_dG0"]
        gW_dec[dead_mask] += E.t() @ dG0
        d_pre = d_pre.clone()
        d_pre[:, dead_mask] += (dG0 @ p["W_dec"][dead_mask, :].t()) * E
    gW_enc = fwd["sae_in"].t() @ d_pre
    gb_enc = d_pre.sum(0)
    d_sae_in = d_pre @ p["W_enc"].t()
    gb_dec = g.sum(0) - d_sae_in.sum(0)                                   # decoder bias + (sae_in = xn - b_dec)
    return dict(W_enc=gW_enc, W_dec=gW_dec, b_enc=gb_enc, b_dec=gb_dec)


def lr_multiplier(step: int, warm_up_steps: int, training_steps: int, lr_end: float) -> float:
    """get_warmup_cosine_lambda (get_scheduler.py:42-53); note lr_end is used as a *multiplier* (train_sae.py:235 passes lr/10)."""
    if step < warm_up_steps:
        return (step + 1) / warm_up_steps
    progress = (step - warm_up_steps) / (training_steps - warm_up_steps)
    return lr_end + 0.5 * (1 - lr_end) * (1 + math.cos(math.pi * progress))


def new_adam_state(p: Dict[str, torch.Tensor]) -> Dict[str, Dict[str, torch.Tensor]]:
    return {k: dict(m=torch.zeros_like(v), v=torch.zeros_like(v)) for k, v in p.items()}


def sae_train_step(p: Dict[str, torch.Tensor], state, x: torch.Tensor, k: int, lr: float, t: int, mode: str = "layer_norm",
                   max_grad_norm: Optional[float] = 1.0, betas=(0.9, 0.999), eps: float = 1e-8,
                   since_fired: Optional[torch.Tensor] = None, act_freq: Optional[torch.Tensor] = None, act: str = "topk",
                   l1_coefficient: float = 0.0, use_ghost_grads: bool = False, dead_feature_window: int = 5000,
                   topk_idx: Optional[torch.Tensor] = None, topk_val: Optional[torch.Tensor] = None,
                   relu_mask: Optional[torch.Tensor] = None):
    """One reference train_step (train_sae.py:278-411), in place on p / state.  t = 1-based optimizer step.
    ``topk_idx`` / ``topk_val`` / ``relu_mask``: see sae_forward."""
    p["W_dec"] /= torch.norm(p["W_dec"], dim=1, keepdim=True)             # :307 set_decoder_norm_to_unit_norm
    dead_mask = (since_fired > dead_feature_window) if (use_ghost_grads and since_fired is not None) else None   # train_sae.py:330-332
    fwd = sae_forward(p, x, k, mode, act=act, l1_coefficient=l1_coefficient, dead_mask=dead_mask, topk_idx=topk_idx, topk_val=topk_val,
                      relu_mask=relu_mask)
    grads = sae_grads(p, x, fwd, mode, l1_coefficient=l1_coefficient, dead_mask=dead_mask)
    raw_grads = {n: g.clone() for n, g in grads.items()}
    active = fwd["active"]                                                # acts > 0 (acts >= 0: also acts.abs() > 0)
    if since_fired is not None:                                           # :356-361
        did_fire = active.float().sum(-2) > 0
        since_fired += 1
        since_fired[did_fire] = 0
    if act_freq is not None:
        act_freq += active.float().sum(0)
    l0 = active.float().sum(-1).mean()
    total_norm = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).float()
    clip = 1.0
    if max_grad_norm:                                                     # :394-397 clip_grad_norm_
        clip = min(1.0, max_grad_norm / (total_norm.item() + 1e-6))
        for g in grads.values():
            g *= clip
    par = (grads["W_dec"] * p["W_dec"]).sum(1, keepdim=True)              # :399 / sae.py:279-297
    grads["W_dec"] = grads["W_dec"] - par * p["W_dec"]
    b1, b2 = betas
    for name in p:                                                        # torch.optim.Adam (no amsgrad, no weight decay)
        st, g = state[name], grads[name]
        st["m"].mul_(b1).add_(g, alpha=1 - b1)
        st["v"].mul_(b2).addcmul_(g, g, value=1 - b2)
        denom = st["v"].sqrt() / math.sqrt(1 - b2 ** t) + eps
        p[name] -= (lr / (1 - b1 ** t)) * st["m"] / denom
    return dict(loss=fwd["loss"], l1=fwd["l1"], ghost=fwd["ghost"], n_dead=(0 if dead_mask is None else int(dead_mask.sum())),
                mse=fwd["mse"], l0=l0, grad_norm=total_norm, clip=clip, idx=fwd["idx"], fwd=fwd, grads=grads, raw_grads=raw_grads)


# ------------------------------------------------------------------------------------------------ Gated SAE (sae/sae.py:648-792)
GATED_PARAMS = ("W_enc", "b_gate", "r_mag", "b_mag", "W_dec", "b_dec")     # b_enc exists in the module but never enters the graph


def gated_forward_grads(p: Dict[str, torch.Tensor], x: torch.Tensor, mode: str, l1_coefficient: float,
                        gate_mask: Optional[torch.Tensor] = None, mag_mask: Optional[torch.Tensor] = None):
    """GatedSparseAutoencoder.forward (ReLU activation) and the closed-form gradients of loss = mse + l1 + aux.
    The magnitude path shares the encoder: sae_in @ (W_enc * exp(r_mag)) + b_mag = (pi - b_gate) * exp(r_mag) + b_mag.
    ``gate_mask`` / ``mag_mask`` [rows, F] bool: take these supports instead of pi > 0 / mag_pre > 0 (relu(pi) becomes
    pi * gate_mask, relu(mag_pre) mag_pre * mag_mask), as ``relu_mask`` in sae_forward."""
    Bt, d = x.shape
    xn, mu, std = normalise_in(x, mode)
    sae_in = xn - p["b_dec"]                                              # :698
    u = sae_in @ p["W_enc"]
    pi = u + p["b_gate"]                                                  # :701 gating pre-activation
    gate = pi > 0 if gate_mask is None else gate_mask.to(pi.device, torch.bool)   # :702 (no gradient); x * gate == x * float(gate)
    er = p["r_mag"].exp()
    mag_pre = u * er + p["b_mag"]                                         # :705
    mag = mag_pre > 0 if mag_mask is None else mag_mask.to(pi.device, torch.bool)
    acts = (torch.relu(mag_pre) if mag_mask is None else mag_pre * mag) * gate   # :707-709
    out_n = acts @ p["W_dec"] + p["b_dec"]                                # :713-722
    sae_out = out_n * std + mu if mode == "layer_norm" else (out_n * std if mode == "constant_norm_rescale" else out_n)
    nf = torch.norm(x - x.mean(dim=0, keepdim=True), p=2, dim=-1, keepdim=True)
    mse = (((sae_out - x) ** 2) / nf).mean()                              # :144-149
    pi_act = torch.relu(pi) if gate_mask is None else pi * gate           # :769-774
    wnorm = p["W_dec"].norm(dim=1)
    l1 = l1_coefficient * (pi_act * wnorm).sum(-1).mean()                 # :776-781
    via = pi_act @ p["W_dec"] + p["b_dec"]                                # :786-787
    aux = ((via - sae_in) ** 2).sum(-1).mean()                            # :788
    # ---- backward
    sd = std if mode != "none" else torch.ones_like(nf)
    g = 2.0 * (sae_out - x) * sd / (nf * Bt * d)                          # d mse / d out_n
    ga = 2.0 * (via - sae_in) / Bt                                        # d aux / d via  (= - d aux / d sae_in)
    gW_dec = acts.t() @ g + pi_act.t() @ ga + (l1_coefficient / Bt) * pi_act.sum(0)[:, None] * p["W_dec"] / wnorm[:, None]
    del pi_act
    # [rows, F] products in place where that computes the same values: the float64 step at 4,096 x 16,384 holds 512 MB per array
    d_mag = (g @ p["W_dec"].t()).mul_(gate).mul_(mag)
    d_pi = (ga @ p["W_dec"].t()).add_((l1_coefficient / Bt) * wnorm).mul_(gate)
    D = (d_mag * er).add_(d_pi)                                           # d loss / d (sae_in @ W_enc)
    grads = dict(W_enc=sae_in.t() @ D, b_gate=d_pi.sum(0), b_mag=d_mag.sum(0), r_mag=(d_mag * u).mul_(er).sum(0), W_dec=gW_dec,
                 b_dec=g.sum(0) + 2.0 * ga.sum(0) - (D @ p["W_enc"].t()).sum(0))
    del d_mag, d_pi, D, u
    return dict(sae_out=sae_out, feature_acts=acts, active=gate & mag, pi=pi, mag_pre=mag_pre, mse=mse, l1=l1, aux=aux, loss=mse + l1 + aux, grads=grads)


def gated_train_step(p: Dict[str, torch.Tensor], state, x: torch.Tensor, lr: float, t: int, mode: str, l1_coefficient: float,
                     max_grad_norm: Optional[float] = 1.0, betas=(0.9, 0.999), eps: float = 1e-8,
                     since_fired: Optional[torch.Tensor] = None, act_freq: Optional[torch.Tensor] = None,
                     gate_mask: Optional[torch.Tensor] = None, mag_mask: Optional[torch.Tensor] = None):
    """One reference train_step with architecture="gated" (train_sae.py:278-411), in place on p / state (keys GATED_PARAMS).
    ``gate_mask`` / ``mag_mask``: see gated_forward_grads."""
    p["W_dec"] /= torch.norm(p["W_dec"], dim=1, keepdim=True)
    out = gated_forward_grads(p, x, mode, l1_coefficient, gate_mask=gate_mask, mag_mask=mag_mask)
    grads = out["grads"]
    raw = {n: g.clone() for n, g in grads.items()}
    active = out["active"]                                                # acts > 0 (acts >= 0: also acts.abs() > 0)
    if since_fired is not None:
        did_fire = active.float().sum(-2) > 0
        since_fired += 1
        since_fired[did_fire] = 0
    if act_freq is not None:
        act_freq += active.float().sum(0)
    total_norm = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).float()
    clip = 1.0
    if max_grad_norm:
        clip = min(1.0, max_grad_norm / (total_norm.item() + 1e-6))
        for g in grads.values():
            g *= clip
    grads["W_dec"] = grads["W_dec"] - (grads["W_dec"] * p["W_dec"]).sum(1, keepdim=True) * p["W_dec"]
    b1, b2 = betas
    for name in GATED_PARAMS:
        st, g = state[name], grads[name]
        st["m"].mul_(b1).add_(g, alpha=1 - b1)
        st["v"].mul_(b2).addcmul_(g, g, value=1 - b2)
        p[name] -= (lr / (1 - b1 ** t)) * st["m"] / (st["v"].sqrt() / math.sqrt(1 - b2 ** t) + eps)
    out.update(raw_grads=raw, grad_norm=total_norm, clip=clip, l0=active.float().sum(-1).mean())
    return out


# ------------------------------------------------------------------------------------------------ Transcoder (sae/transcoder.py:6-116)
def transcoder_forward_grads(p: Dict[str, torch.Tensor], x: torch.Tensor, y: torch.Tensor, mode: str, act: str, k: int, l1_coefficient: float,
                             topk_idx: Optional[torch.Tensor] = None, relu_mask: Optional[torch.Tensor] = None):
    """Forward, loss and closed-form gradients of the reference Transcoder: the encoder reads the INPUT activation ``x``
    (normalised, minus ``b_dec``), the decoder reconstructs the TARGET activation ``y`` with its own bias ``b_dec_out`` and an
    optional linear skip ``x @ W_skip^T`` (added before the output de-normalisation, which uses the INPUT's row mean / std,
    transcoder.py:75-78); the loss is ``_compute_mse_loss(y, out)`` (sae.py:144-149) plus the L1 term for dense activations.
    p: W_enc [d,F], W_dec [F,d_out], b_enc [F], b_dec [d], b_dec_out [d_out], optional W_skip [d_out, d].
    ``topk_idx`` [rows, k] (act="topk") / ``relu_mask`` [rows, F] bool (act="relu"): take this support, as in sae_forward."""
    Bt, d_out = y.shape
    xn, mu, std = normalise_in(x, mode)
    sae_in = xn - p["b_dec"]                                            # transcoder.py:33-37
    hidden_pre = sae_in @ p["W_enc"] + p["b_enc"]                      # :39-46
    if act == "topk":
        if topk_idx is None:
            top = torch.topk(hidden_pre, k=k, dim=-1)
            idx, val = top.indices, top.values
        else:
            idx = topk_idx.to(hidden_pre.device).long()
            val = hidden_pre.gather(-1, idx)
        acts = torch.zeros_like(hidden_pre).scatter_(-1, idx, torch.relu(val))
        active = acts > 0
    elif relu_mask is None:
        acts = torch.relu(hidden_pre)
        active = acts > 0
    else:
        active = relu_mask.to(hidden_pre.device, torch.bool)
        acts = hidden_pre * active
    out_n = acts @ p["W_dec"] + p["b_dec_out"]                         # :56-64
    if "W_skip" in p:
        out_n = out_n + x @ p["W_skip"].t()                             # :75-76 (the raw input, not the normalised one)
    out = out_n * std + mu if mode == "layer_norm" else (out_n * std if mode == "constant_norm_rescale" else out_n)   # :78
    nf = torch.norm(y - y.mean(dim=0, keepdim=True), p=2, dim=-1, keepdim=True)
    mse = (((out - y) ** 2) / nf).sum() / (Bt * d_out)                 # :80
    l1 = None if act == "topk" else l1_coefficient * acts.abs().sum(dim=1).sum() / Bt   # :89-97
    loss = mse + (l1 if l1 is not None else 0.0)
    scale = std if mode != "none" else torch.ones_like(nf)
    g = 2.0 * (out - y) * scale / (nf * Bt * d_out)                    # dL/d out_n
    grads = {"W_dec": acts.t() @ g, "b_dec_out": g.sum(0)}
    if "W_skip" in p:
        grads["W_skip"] = g.t() @ x
    d_acts = g @ p["W_dec"].t()
    if l1 is not None:
        d_acts = d_acts + l1_coefficient / Bt
    d_pre = d_acts * active
    grads["W_enc"] = sae_in.t() @ d_pre
    grads["b_enc"] = d_pre.sum(0)
    grads["b_dec"] = -(d_pre @ p["W_enc"].t()).sum(0)                   # b_dec only enters through sae_in = xn - b_dec
    return dict(sae_out=out, hidden_pre=hidden_pre, feature_acts=acts, active=active, loss=loss, mse=mse, l1=l1, grads=grads)


def transcoder_train_step(p: Dict[str, torch.Tensor], state, x: torch.Tensor, y: torch.Tensor, lr: float, t: int, mode: str, act: str, k: int,
                          l1_coefficient: float, max_grad_norm: Optional[float] = 1.0, betas=(0.9, 0.999), eps: float = 1e-8,
                          since_fired: Optional[torch.Tensor] = None, act_freq: Optional[torch.Tensor] = None,
                          topk_idx: Optional[torch.Tensor] = None, relu_mask: Optional[torch.Tensor] = None):
    """One reference train_step on an (input, target) pair (train_sae.py:299-301, 335-344, 392-401), in place on p / state.
    ``topk_idx`` / ``relu_mask``: see transcoder_forward_grads."""
    p["W_dec"] /= torch.norm(p["W_dec"], dim=1, keepdim=True)           # :306-307
    out = transcoder_forward_grads(p, x, y, mode, act, k, l1_coefficient, topk_idx=topk_idx, relu_mask=relu_mask)
    grads = out["grads"]
    raw = {n: g.clone() for n, g in grads.items()}
    acts, active = out["feature_acts"], out["active"]                    # active: acts > 0 (acts >= 0: also acts.abs() > 0)
    if since_fired is not None:
        did_fire = active.float().sum(-2) > 0
        since_fired += 1
        since_fired[did_fire] = 0
    if act_freq is not None:
        act_freq += active.float().sum(0)
    total_norm = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).float()
    if max_grad_norm:
        clip = min(1.0, max_grad_norm / (total_norm.item() + 1e-6))
        for g in grads.values():
            g *= clip
    par = (grads["W_dec"] * p["W_dec"]).sum(1, keepdim=True)
    grads["W_dec"] = grads["W_dec"] - par * p["W_dec"]
    b1, b2 = betas
    for name in p:
        st, g = state[name], grads[name]
        st["m"].mul_(b1).add_(g, alpha=1 - b1)
        st["v"].mul_(b2).addcmul_(g, g, value=1 - b2)
        p[name] -= (lr / (1 - b1 ** t)) * st["m"] / (st["v"].sqrt() / math.sqrt(1 - b2 ** t) + eps)
    return dict(loss=out["loss"], mse=out["mse"], l1=out["l1"], l0=active.float().sum(-1).mean(), grad_norm=total_norm,
                sae_out=out["sae_out"], hidden_pre=out["hidden_pre"], feature_acts=acts, active=active, raw_grads=raw)
