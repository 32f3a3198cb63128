"""Transcoder training step and forward on the C-ABI kernels (reference sae/transcoder.py:6-116, trained by train_sae.py:278-411
with ``layer_acts[:, 0]`` as the input activation and ``layer_acts[:, 1]`` as the target).

    sae_in      = norm_in(x) - b_dec                                          (transcoder.py:33-39)
    hidden_pre  = sae_in @ W_enc + b_enc ; acts = relu(.) | TopK(.)           (:41-51)
    out_n       = acts @ W_dec + b_dec_out  [+ x @ W_skip^T]                   (:58-79: the skip term uses the RAW x)
    sae_out     = norm_out(out_n)   with the INPUT's row statistics           (:81)
    loss        = mean((sae_out - y)^2 / ||y - mean_batch(y)||) + l1           (:83, 93-103; l1 only for dense activations)

The dense products run on ``pb_gemm`` (3xTF32 wgmma) exactly as in ``SaeDenseStepEngine``; this module adds the target-vs-input
split of the loss, the skip matrix (one more forward product through the residual epilogue, one more gradient product) and the
second decoder bias.  ``pb_sae_adam`` updates W_dec (clip, decoder-parallel-gradient removal, Adam, row renorm), W_enc, b_enc and
b_dec; ``pb_adam_vec`` updates W_skip and b_dec_out with the same clip coefficient.  Requires d_out == d_in (the reference default).
"""
from __future__ import annotations

from typing import Optional

import torch

from . import _lib as L
from .sae_dense import SaeDenseStepEngine, colsum, transpose
from .sae_engine import _need_cuda, _stream


class SaeTranscoderStepEngine(SaeDenseStepEngine):
    """Parameters: W_encT [F, d] (feature-major view of W_enc), W_dec [F, d_out = d], b_enc [F], b_dec [d], b_dec_out [d],
    W_skip [d, d] or None."""

    def __init__(self, W_encT, W_dec, b_enc, b_dec, b_dec_out: torch.Tensor, W_skip: Optional[torch.Tensor], k: int, activation: str,
                 l1_coefficient: float = 0.0, **kw):
        super().__init__(W_encT, W_dec, b_enc, b_dec, k=max(int(k), 1), l1_coefficient=l1_coefficient, **kw)
        if W_dec.shape[1] != self.d:
            raise L.PrismaB200Error("H100 transcoder step: d_out must equal d_in")
        if activation not in ("relu", "topk"):
            raise NotImplementedError(f"H100 transcoder step: activation {activation!r} is not built (relu and topk are)")
        _need_cuda(b_dec_out, W_skip)
        self.activation, self.b_dec_out, self.W_skip = activation, b_dec_out, W_skip
        dev, d = W_dec.device, self.d
        z = lambda *s: torch.zeros(*s, device=dev)  # noqa: E731
        self.gb_dec_out, self.m_bo, self.v_bo = z(d), z(d), z(d)
        if W_skip is not None:
            self.gW_skip, self.m_sk, self.v_sk = z(d, d), z(d, d), z(d, d)
        self.ysum = z(d)

    # ------------------------------------------------------------------ forward pieces
    def _forward(self, x: torch.Tensor, y: Optional[torch.Tensor], want_out: bool, training: bool):
        if y is not None:                                     # loss against the TARGET activation, centred on its batch mean
            colsum(y, out=self.ysum)
        return self._dense_forward(x, y, self.ysum, self.b_dec_out, want_out, training, topk=self.activation == "topk", skip=self.W_skip)

    @torch.no_grad()
    def forward_losses(self, x: torch.Tensor, y: Optional[torch.Tensor], want_out: bool = True) -> torch.Tensor:
        """Inference / logging: fills sae_out and (with a target) scalars.mse / l0 and aux[0] = sum |acts|; returns feature_acts."""
        _need_cuda(x, y)
        x = x.contiguous().float()
        y = None if y is None else y.contiguous().float()
        acts = self._forward(x, y, want_out, training=False)
        L.check(L.get_lib().pb_sae_clip_finish(self.scalars.data_ptr(), 0.0, x.shape[0], self.d, _stream()), "pb_sae_clip_finish")
        return acts

    # ------------------------------------------------------------------ one optimizer step
    @torch.no_grad()
    def train_step_transcoder(self, x: torch.Tensor, y: torch.Tensor, lr: float, since_fired: Optional[torch.Tensor] = None,
                              act_freq: Optional[torch.Tensor] = None, want_out: bool = False) -> torch.Tensor:
        _need_cuda(x, y)
        x, y = x.contiguous().float(), y.contiguous().float()
        self.step_count += 1
        acts = self._forward(x, y, want_out, training=True)
        l1_grad = (self.l1_coefficient / x.shape[0]) if self.activation != "topk" else 0.0   # TopK: no sparsity term (transcoder.py:96-100)
        gT = transpose(self.g)                                               # [d, rows]: gW_dec's operand, and gW_skip's
        self._dense_backward(acts, l1_grad, gT)
        colsum(self.g, out=self.gb_dec_out)                                   # b_dec_out enters the output only
        self.gb_dec.zero_()
        self._gb_dec_through_sae_in(self.gb_enc, self.W_encT)                 # b_dec enters through sae_in = norm(x) - b_dec only
        grads = [self.gW_dec, self.gW_encT, self.gb_enc, self.gb_dec, self.gb_dec_out]
        extra = [(self.b_dec_out, self.gb_dec_out, self.m_bo, self.v_bo)]
        if self.W_skip is not None:
            self._at_b(gT, x, out=self.gW_skip)                              # gW_skip = g^T @ x   ([d_out, d_in], out += x @ W_skip^T)
            grads.append(self.gW_skip)
            extra.append((self.W_skip, self.gW_skip, self.m_sk, self.v_sk))
        self._clip_and_adam(x, float(lr), since_fired, act_freq, grads, extra)
        return self.scalars

    def loss_terms(self, rows: int) -> dict:
        sc, aux = self.scalars.tolist(), self.aux.tolist()
        l1 = self.l1_coefficient * aux[0] / rows if self.activation != "topk" else 0.0
        return dict(mse=sc[3], l0=sc[4], grad_norm=sc[6], clip_coef=sc[2], l1=l1, loss=sc[3] + l1)
