"""Gated SAE training step (``GatedSparseAutoencoder``, reference sae/sae.py:648-792 under ``VisionSAETrainer.train_step``).

    pi = sae_in @ W_enc + b_gate                      gate path              (:701)
    mag_pre = sae_in @ (W_enc * exp(r_mag)) + b_mag   magnitude path         (:705)   = (pi - b_gate) * exp(r_mag) + b_mag
    acts = [pi > 0] * relu(mag_pre)                                          (:707-709)
    loss = mse(decode(acts)) + l1 * mean_b sum_f relu(pi) ||W_dec[f]|| + mean_b ||relu(pi) @ W_dec + b_dec - sae_in||^2   (:726-744)

Because the magnitude path shares the encoder matrix, ONE encoder GEMM feeds both paths and one GEMM carries both paths'
gradient back to it (D = d_pi + d_mag * exp(r_mag)); the reference executes three encoder products forward.  The dense
products (encoder, two decoder products, their four transposed products) run on ``pb_gemm`` (3xTF32); the element-wise
pieces are ``pb_gated_*`` in csrc/sae_dense.cu; ``pb_sae_adam`` (W_dec projection + renorm, W_enc, b_gate in the b_enc slot,
b_dec, dead-feature counters) and ``pb_adam_vec`` (r_mag, b_mag) finish the step.  ``b_enc`` exists in the reference module but
never enters its graph (gradient ``None``, untouched by Adam): it is not an engine parameter.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib as L
from . import ops
from .sae_dense import SaeDenseStepEngine, _dense_loss, colsum, transpose
from .sae_engine import _need_cuda, _stream

i32, f32, vp = C.c_int32, C.c_float, C.c_void_p

L.register_signatures({
    "pb_gated_fwd": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, vp]),
    "pb_gated_aux": (i32, [vp, vp, vp, vp, i32, i32, vp]),
    "pb_gated_bwd": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, f32, vp, vp, vp, vp, i32, i32, vp]),
    "pb_row_norms": (i32, [vp, vp, i32, i32, vp]),
    "pb_gated_l1_rows": (i32, [vp, vp, vp, vp, f32, vp, i32, i32, vp]),
})


class SaeGatedStepEngine(SaeDenseStepEngine):
    """Parameters: W_encT [F,d] (feature-major view of W_enc), W_dec [F,d], b_gate, r_mag, b_mag [F], b_dec [d].
    aux = [sum_f colsum(pi_act) ||W_dec[f]||, sum (via - sae_in)^2, -, -]."""

    def __init__(self, W_encT: torch.Tensor, W_dec: torch.Tensor, b_gate: torch.Tensor, r_mag: torch.Tensor, b_mag: torch.Tensor,
                 b_dec: torch.Tensor, l1_coefficient: float, **kw):
        # b_gate rides in the b_enc slot of pb_sae_adam
        super().__init__(W_encT, W_dec, b_gate, b_dec, k=1, l1_coefficient=l1_coefficient, **kw)
        _need_cuda(r_mag, b_mag)
        self.b_gate, self.r_mag, self.b_mag = b_gate, r_mag, b_mag
        z = lambda n: torch.zeros(n, device=W_dec.device)  # noqa: E731
        self.m_r, self.v_r, self.m_bm, self.v_bm = z(self.F), z(self.F), z(self.F), z(self.F)
        self.gr_mag, self.gb_mag, self.dsum, self.piact_colsum, self.wnorm = z(self.F), z(self.F), z(self.F), z(self.F), z(self.F)

    # ------------------------------------------------------------------ forward pieces (shared by training and inference)
    def _forward(self, x: torch.Tensor, want_out: bool, training: bool):
        lib, st = L.get_lib(), _stream()
        rows, d, F = x.shape[0], self.d, self.F
        self._prep(x)
        self.piact_colsum.zero_()
        self.gemm32(self.sae_in, self.sae_in_lo, self.W_encT, self.W_encT_lo, self.b_gate, out0=self.hidden_pre)   # pi
        dev = x.device
        acts, pi_act = torch.empty(rows, F, device=dev), torch.empty(rows, F, device=dev)
        acts_lo, pi_act_lo = torch.empty(rows, F, device=dev), torch.empty(rows, F, device=dev)
        L.check(lib.pb_gated_fwd(self.hidden_pre.data_ptr(), self.b_gate.data_ptr(), self.r_mag.data_ptr(), self.b_mag.data_ptr(),
                                 acts.data_ptr(), acts_lo.data_ptr(), pi_act.data_ptr(), pi_act_lo.data_ptr(), self.fired.data_ptr(),
                                 self.piact_colsum.data_ptr(), self.scalars.data_ptr(), rows, F, st), "pb_gated_fwd")
        WdT, WdT_lo = transpose(self.W_dec)                           # [d, F]: K-major B operand of both decoder products
        out_n, _ = self.gemm32(acts, acts_lo, WdT, WdT_lo, self.b_dec)
        via, _ = self.gemm32(pi_act, pi_act_lo, WdT, WdT_lo, self.b_dec)   # via-gate reconstruction (:786-787)
        _dense_loss(x, out_n, self.xsum, self.mu, self.sd, self.norm_mode, sae_out=self.sae_out if want_out else None,
                    g=self.g if training else None, scalars=self.scalars)
        ga = torch.empty(rows, d, device=dev)
        L.check(lib.pb_gated_aux(via.data_ptr(), self.sae_in.data_ptr(), ga.data_ptr(), self.aux[1:].data_ptr(), rows, d, st), "pb_gated_aux")
        L.check(lib.pb_row_norms(self.W_dec.data_ptr(), self.wnorm.data_ptr(), F, d, st), "pb_row_norms")
        self.last_acts = acts
        return acts, pi_act, ga

    @torch.no_grad()
    def forward_losses(self, x: torch.Tensor, want_out: bool = True) -> torch.Tensor:
        """Inference / logging: fills sae_out, scalars (loss_sum, pos_count) and aux; returns feature_acts [rows, F]."""
        _need_cuda(x)
        x = x.contiguous().float()
        lib, st = L.get_lib(), _stream()
        acts, _, _ = self._forward(x, want_out, training=False)
        # l1 value without touching any gradient buffer: sum_f colsum(pi_act)[f] * ||W_dec[f]||
        scratch = torch.zeros(self.F, self.d, device=x.device) if not hasattr(self, "_l1_scratch") else self._l1_scratch
        self._l1_scratch = scratch
        L.check(lib.pb_gated_l1_rows(scratch.data_ptr(), self.W_dec.data_ptr(), self.piact_colsum.data_ptr(), self.wnorm.data_ptr(), 0.0,
                                     self.aux.data_ptr(), self.F, self.d, st), "pb_gated_l1_rows")
        L.check(lib.pb_sae_clip_finish(self.scalars.data_ptr(), 0.0, x.shape[0], self.d, st), "pb_sae_clip_finish")
        return acts

    # ------------------------------------------------------------------ one optimizer step
    def train_step_gated(self, x: torch.Tensor, lr: float, since_fired: Optional[torch.Tensor] = None, act_freq=None,
                         want_out: bool = False) -> torch.Tensor:
        _need_cuda(x)
        x = x.contiguous().float()
        lib, st = L.get_lib(), _stream()
        rows, d, F = x.shape[0], self.d, self.F
        self.step_count += 1
        acts, pi_act, ga = self._forward(x, want_out, training=True)
        l1_grad = self.l1_coefficient / rows
        Wd_lo = ops.split_tf32(self.W_dec)
        D, _ = self.gemm32(self.g, None, self.W_dec, Wd_lo)          # d_acts = g @ W_dec^T, becomes D in place
        d_pia, _ = self.gemm32(ga, None, self.W_dec, Wd_lo)
        # no tf32 plane of D: the transpose for gW_encT makes the one its product reads
        L.check(lib.pb_gated_bwd(D.data_ptr(), None, d_pia.data_ptr(), self.hidden_pre.data_ptr(), self.b_gate.data_ptr(),
                                 self.r_mag.data_ptr(), self.b_mag.data_ptr(), self.wnorm.data_ptr(), l1_grad, self.gb_enc.data_ptr(),
                                 self.gb_mag.data_ptr(), self.gr_mag.data_ptr(), self.dsum.data_ptr(), rows, F, st), "pb_gated_bwd")
        del d_pia
        # gW_dec = acts^T @ g + pi_act^T @ ga (+ L1 rows); the second product accumulates through the residual epilogue
        self._at_b(pi_act, ga, out=self.gW_dec, residual=self._at_b(acts, self.g))
        L.check(lib.pb_gated_l1_rows(self.gW_dec.data_ptr(), self.W_dec.data_ptr(), self.piact_colsum.data_ptr(), self.wnorm.data_ptr(),
                                     l1_grad, self.aux.data_ptr(), F, d, st), "pb_gated_l1_rows")
        self._at_b(D, self.sae_in, out=self.gW_encT)                 # gW_enc^T = D^T @ sae_in
        # gb_dec = colsum(g) + 2 colsum(ga) - colsum(D) @ W_enc^T      (decoder bias twice, sae_in = xn - b_dec in the aux target and the encoder)
        colsum(self.g, out=self.gb_dec)
        self._add_gb_dec(colsum(ga), 2.0)
        self._gb_dec_through_sae_in(self.dsum, self.W_encT)
        # global norm over the six trained tensors -> clip coefficient -> Adam
        self._clip_and_adam(x, float(lr), since_fired, act_freq,
                            (self.gW_dec, self.gW_encT, self.gb_enc, self.gb_dec, self.gr_mag, self.gb_mag),
                            ((self.r_mag, self.gr_mag, self.m_r, self.v_r), (self.b_mag, self.gb_mag, self.m_bm, self.v_bm)))
        return self.scalars

    def loss_terms(self, rows: int) -> dict:
        """Host read (synchronises): mse, l1, aux reconstruction loss and their sum."""
        sc, aux = self.scalars.tolist(), self.aux.tolist()
        out = dict(mse=sc[3], l0=sc[4], grad_norm=sc[6], clip_coef=sc[2], l1=self.l1_coefficient * aux[0] / rows, aux=aux[1] / rows)
        out["loss"] = out["mse"] + out["l1"] + out["aux"]
        return out
