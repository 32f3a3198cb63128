"""Transcoder on the H100 path (reference sae/transcoder.py:6-116): a sparse coder whose decoder reconstructs a DIFFERENT
activation (``cfg.out_hook_point``, e.g. the MLP output) from the one it encodes, optionally with a linear skip connection.

Same surface as the reference class -- parameters ``W_skip [d_in, d_in] | None``, ``W_dec [d_sae, d_out]``, ``W_enc [d_in, d_sae]``,
``b_enc``, ``b_dec``, ``b_dec_out``; ``encode`` / ``decode`` / ``forward(x, y, dead_neuron_mask)`` -> 7-tuple -- on top of
``vit_prisma/b200/sae_transcoder.py`` (dense 3xTF32 wgmma products + the shared Adam kernels).  ``forward`` builds no autograd graph;
``VisionSAETrainer`` trains through the engine's hand-written backward.  Ghost grads are not built for this class."""
from __future__ import annotations

import torch
from torch import nn

from vit_prisma.b200 import _lib as L
from vit_prisma.b200 import ops
from vit_prisma.sae.sae import SparseAutoencoder


class Transcoder(SparseAutoencoder):
    def initialize_sae_weights(self):                                     # reference :8-29, same order of random draws
        cfg = self.cfg
        if getattr(cfg, "d_out", self.d_in) != self.d_in:
            raise NotImplementedError("H100 Transcoder: d_out must equal d_in (the reference default)")
        self.W_skip = nn.Parameter(self.initialize_weights(self.d_in, self.d_in)) if cfg.transcoder_with_skip_connection else None
        self.W_dec = nn.Parameter(self.initialize_weights(self.d_sae, cfg.d_out))
        enc = self.initialize_weights(self.d_in, self.d_sae)                # [d_in, d_sae], rows unit-norm
        self.W_enc = nn.Parameter(enc.t().contiguous().t())                 # feature-major storage behind the reference shape
        z = lambda n: nn.Parameter(torch.zeros(n, dtype=self.dtype, device=self.device))  # noqa: E731
        self.b_enc, self.b_dec, self.b_dec_out = z(self.d_sae), z(self.d_in), z(cfg.d_out)

    # ------------------------------------------------------------------ engine plumbing
    def _canonical_params(self):
        if not self.W_enc.data.t().is_contiguous():
            self.W_enc.data = self.W_enc.data.t().contiguous().t()
        for p in (self.W_dec, self.W_skip):
            if p is not None and not p.data.is_contiguous():
                p.data = p.data.contiguous()
        return (self.W_enc.data.t(), self.W_dec.data, self.b_enc.data, self.b_dec.data, self.b_dec_out.data,
                None if self.W_skip is None else self.W_skip.data)

    def step_engine(self, gemm_impl: int = L.GEMM_AUTO):
        from vit_prisma.b200.sae_transcoder import SaeTranscoderStepEngine
        if self.cfg.use_ghost_grads:
            raise NotImplementedError("H100 Transcoder: ghost grads are not built")
        if self.dtype != torch.float32:
            raise NotImplementedError("H100 Transcoder runs in float32")
        params = self._canonical_params()
        key = tuple(0 if t is None else t.data_ptr() for t in params) + (gemm_impl,)
        eng = self._engine
        if eng is None or eng._key != key:
            wt, wd, be, bd, bo, ws = params
            act = self.cfg.activation_fn_str
            eng = SaeTranscoderStepEngine(wt, wd, be, bd, bo, ws, k=self.cfg.activation_fn_kwargs.get("k", 1) if act == "topk" else 1,
                                          activation=act, l1_coefficient=self.cfg.l1_coefficient, normalize_activations=self._norm_mode,
                                          max_grad_norm=self.cfg.max_grad_norm, gemm_impl=gemm_impl)
            eng._key = key
            eng._enc_version = self.W_enc._version
            self._engine = eng
        return eng

    def _fresh_engine(self):
        eng = self.step_engine()
        if eng._enc_version != self.W_enc._version:
            eng.refresh_lo()
            eng._enc_version = self.W_enc._version
        return eng

    # ------------------------------------------------------------------ module-by-module route (hooks fire, reference :32-71)
    def encode(self, x: torch.Tensor, return_hidden_pre: bool = False):
        from vit_prisma.b200.sae_engine import sae_prep
        x = ops.cast(x, self.dtype) if x.dtype != self.dtype else x
        lead = x.shape[:-1]
        wt, _wd, be, bd, _bo, _ws = self._canonical_params()
        sae_in2, mu, sd = sae_prep(x.reshape(-1, self.d_in).contiguous(), bd, self._norm_mode)
        self.ln_mu, self.ln_std = mu.view(*lead, 1), sd.view(*lead, 1)
        sae_in = self.hook_sae_in(sae_in2.view(*lead, self.d_in))
        hidden_pre, _ = ops.gemm(sae_in, wt, be)
        hidden_pre = self.hook_hidden_pre(hidden_pre)
        feature_acts = self.hook_hidden_post(self.activation_fn(hidden_pre))
        return (sae_in, feature_acts, hidden_pre) if return_hidden_pre else (sae_in, feature_acts)

    def decode(self, features: torch.Tensor):
        _wt, wd, _be, _bd, bo, _ws = self._canonical_params()
        out, _ = ops.gemm(features, wd.t().contiguous(), bo)                # features @ W_dec + b_dec_out  (:58-68; no norm_out here)
        return self.hook_sae_out(out)

    # ------------------------------------------------------------------ forward (reference :73-116)
    @torch.no_grad()
    def forward(self, x: torch.Tensor, y: torch.Tensor = None, dead_neuron_mask: torch.Tensor = None, *args, **kwargs):
        lead = x.shape[:-1]
        x2 = (ops.cast(x, self.dtype) if x.dtype != self.dtype else x).reshape(-1, self.d_in).contiguous()
        y2 = None if y is None else (ops.cast(y, self.dtype) if y.dtype != self.dtype else y).reshape(-1, self.d_in).contiguous()
        eng = self._fresh_engine()
        acts = eng.forward_losses(x2, y2, want_out=True)
        self.ln_mu, self.ln_std = eng.mu.clone().view(*lead, 1), eng.sd.clone().view(*lead, 1)
        for hook, t in ((self.hook_sae_in, eng.sae_in), (self.hook_hidden_pre, eng.hidden_pre), (self.hook_hidden_post, acts)):
            hook(t.view(*lead, -1))                                          # observers on the fused route
        sae_out = self.hook_sae_out(eng.sae_out.clone().view(*lead, self.d_in))
        if getattr(self.cfg, "return_out_only", False):
            return sae_out
        if y2 is None:
            raise ValueError("Transcoder.forward needs the target activation y to compute its loss (reference transcoder.py:83)")
        rows = x2.shape[0]
        mse_loss = eng.scalars[3].clone()
        l1_loss = None if self.cfg.activation_fn_str == "topk" else eng.aux[0] * (self.l1_coefficient / rows)
        loss = mse_loss + (l1_loss if l1_loss is not None else 0)
        return (sae_out, acts.view(*lead, self.d_sae), loss, mse_loss, l1_loss, self.zero_loss.to(sae_out.device), torch.tensor(0.0))
