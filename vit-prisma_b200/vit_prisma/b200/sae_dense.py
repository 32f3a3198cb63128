"""Dense-activation SAE training step (ReLU + L1) and the ghost-grad auxiliary loss, on the C-ABI kernels.

Stands in for ``StandardSparseAutoencoder.forward`` + ``VisionSAETrainer.train_step`` when ``activation_fn_str == "relu"``
(the reference's default; sae/sae.py:557-645, 810-839) and for ``_compute_ghost_residual_loss`` (sae/sae.py:151-179) with
either activation.  The six dense products of the reference graph run on ``pb_gemm`` (wgmma, 3xTF32, K-major operands:
``pb_transpose`` supplies the transposed views autograd uses); ``csrc/sae_dense.cu`` holds the glue; clip / projection /
Adam / renorm / dead-feature counters are ``pb_sae_adam``, shared with the TopK pipeline.  ``SaeDenseStepEngine`` also holds
the pieces the Gated and Transcoder engines share with it: the GEMM route, the products over tokens, prep, the b_dec path.

Per step (tokens Bt, d = d_in, F = d_sae):
  prep -> hidden_pre, acts = relu(.) [GEMM + epilogue] -> stats -> out_n = acts @ W_dec + b_dec [GEMM] -> loss, g
  d_acts = g @ W_dec^T [GEMM] -> d_hid = (d_acts + l1/Bt) * [acts > 0]
  gW_dec = acts^T @ g [GEMM], gW_encT = d_hid^T @ sae_in [GEMM], gb_enc = colsum(d_hid), gb_dec = colsum(g) - gb_enc @ W_enc^T
  (+ ghost blocks on the dead features) -> grad norm / clip -> pb_sae_adam
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib as L
from . import ops
from .sae_engine import SaeStepEngine, _need_cuda, _stream, topk_dense

i32, i64, f32, vp = C.c_int32, C.c_int64, C.c_float, C.c_void_p

L.register_signatures({
    "pb_transpose": (i32, [vp, vp, vp, i32, i32, vp]),
    "pb_colsum": (i32, [vp, vp, i32, i32, i32, vp]),
    "pb_gemv_rows": (i32, [vp, vp, vp, i32, i32, i32, vp]),
    "pb_sae_dense_stats": (i32, [vp, i32, i32, vp, vp, vp, vp]),
    "pb_sae_dense_loss": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "pb_sae_dense_dhid": (i32, [vp, vp, vp, f32, i64, vp]),
    "pb_sae_ghost_gather": (i32, [vp, vp, i32, i32, i32, vp, i32, vp]),
    "pb_gather_rows": (i32, [vp, vp, i32, i32, i32, vp, vp]),
    "pb_scatter_add_rows": (i32, [vp, vp, i32, i32, vp, f32, vp]),
    "pb_mul_inplace": (i32, [vp, vp, i64, vp]),
    "pb_sae_ghost_rows": (i32, [vp, vp, vp, vp, vp, i32, i32, vp]),
})


def _p(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def transpose(x: torch.Tensor, want_lo: bool = True):
    """[rows, cols] fp32 -> ([cols, rows], its tf32 residual | None)."""
    _need_cuda(x)
    assert x.dim() == 2 and x.dtype == torch.float32 and x.is_contiguous()
    rows, cols = x.shape
    out = torch.empty(cols, rows, device=x.device)
    lo = torch.empty(cols, rows, device=x.device) if want_lo else None
    L.check(L.get_lib().pb_transpose(x.data_ptr(), out.data_ptr(), _p(lo), rows, cols, _stream()), "pb_transpose")
    return out, lo


def colsum(x: torch.Tensor, out: Optional[torch.Tensor] = None, accumulate: bool = False) -> torch.Tensor:
    rows, cols = x.shape
    out = torch.empty(cols, device=x.device) if out is None else out
    L.check(L.get_lib().pb_colsum(x.data_ptr(), out.data_ptr(), rows, cols, int(accumulate), _stream()), "pb_colsum")
    return out


def gemv_rows(W: torch.Tensor, v: torch.Tensor, out: Optional[torch.Tensor] = None, accumulate: bool = False) -> torch.Tensor:
    F, d = W.shape
    out = torch.empty(d, device=W.device) if out is None else out
    L.check(L.get_lib().pb_gemv_rows(W.data_ptr(), v.data_ptr(), out.data_ptr(), F, d, int(accumulate), _stream()), "pb_gemv_rows")
    return out


def _dense_loss(x, out_n, xsum, mu=None, sd=None, norm_mode: int = 0, *, sae_out=None, g=None, resid=None, scalars=None) -> None:
    """pb_sae_dense_loss on [rows, d]: sae_out = norm_out(out_n), g = dL/d out_n, resid = x - sae_out (each optional), loss sum into
    ``scalars``.  Without ``scalars`` only the per-element outputs are wanted: the loss sum goes to scratch that nothing reads."""
    scalars = torch.empty(8, device=x.device) if scalars is None else scalars
    L.check(L.get_lib().pb_sae_dense_loss(x.data_ptr(), out_n.data_ptr(), _p(mu), _p(sd), xsum.data_ptr(), _p(sae_out), _p(g), _p(resid),
                                          scalars.data_ptr(), x.shape[0], 0, x.shape[1], norm_mode, _stream()), "pb_sae_dense_loss")


def _residual(x: torch.Tensor, sae_out: torch.Tensor, xsum: torch.Tensor) -> torch.Tensor:
    """x - sae_out for an output in x's units; ``xsum`` = column sums of x."""
    resid = torch.empty_like(x)
    _dense_loss(x, sae_out, xsum, resid=resid)
    return resid


def _ghost_block(hidden_pre, W_dec, dead_idx, resid, scalars, ghost_sum):
    """The ghost loss (sae.py:157-178) of the dead features ``dead_idx`` (int32, sorted, distinct): E = exp(hidden_pre[:, dead])
    [rows, ndp], W_dec[dead] [ndp, d] and G0 = E @ W_dec[dead] [rows, d]; pb_sae_ghost_rows adds the loss sum into ``ghost_sum``
    (the mse is ``scalars.loss_sum`` / (rows * d)) and overwrites G0 with dL_ghost/dG0.  ``resid = x - sae_out``.
    Returns (E, W_dec[dead], dL_ghost/dG0)."""
    lib, st = L.get_lib(), _stream()
    (rows, F), d, dev = hidden_pre.shape, W_dec.shape[1], resid.device
    nd = int(dead_idx.numel())
    ndp = max(32, (nd + 31) // 32 * 32)                         # zero-padded block width (TMA-legal K / N)
    E = torch.empty(rows, ndp, device=dev)
    L.check(lib.pb_sae_ghost_gather(hidden_pre.data_ptr(), _p(dead_idx), nd, rows, F, E.data_ptr(), ndp, st), "pb_sae_ghost_gather")
    WdD = torch.empty(ndp, d, device=dev)
    L.check(lib.pb_gather_rows(W_dec.data_ptr(), _p(dead_idx), nd, ndp, d, WdD.data_ptr(), st), "pb_gather_rows")
    WdDT, _ = transpose(WdD, want_lo=False)
    # [rows, d] = exp(h_dead) @ W_dec[dead] (sae.py:165) on the exact-fp32 FFMA kernel: the ghost loss divides by
    # (G - r)^2 / rcn + 1e-6 element-wise, which amplifies round-off in G by ~1e3 (fp32 torch vs fp64: 6e-4 on the
    # gradients; with the 3xTF32 product here: 4e-2).  Every later ghost product is linear in dL/dG0 and stays on the tensor cores.
    G0, _ = ops.gemm(E, WdDT, None, impl=L.GEMM_SIMT)
    L.check(lib.pb_sae_ghost_rows(resid.data_ptr(), colsum(resid).data_ptr(), G0.data_ptr(), scalars.data_ptr(), ghost_sum.data_ptr(),
                                  rows, d, st), "pb_sae_ghost_rows")
    return E, WdD, G0


def ghost_loss_value(hidden_pre: torch.Tensor, W_dec: torch.Tensor, x2: torch.Tensor, sae_out2: torch.Tensor, mse: torch.Tensor,
                     dead_mask: torch.Tensor) -> torch.Tensor:
    """``_compute_ghost_residual_loss`` (sae/sae.py:151-179) as a 0-dim device tensor, for ``forward()``'s 7-tuple.
    hidden_pre [rows, F], x2 / sae_out2 [rows, d] fp32 contiguous; ``mse`` 0-dim device tensor; ``dead_mask`` [F] bool."""
    _need_cuda(hidden_pre, W_dec, x2, sae_out2)
    rows, d = x2.shape
    dead_idx = torch.nonzero(dead_mask).flatten().to(torch.int32)
    sc = torch.zeros(8, device=x2.device)
    sc[0] = mse * float(rows * d)                                    # the row kernel reads mse as loss_sum / (rows * d)
    out = torch.zeros(1, device=x2.device)
    _ghost_block(hidden_pre, W_dec, dead_idx, _residual(x2, sae_out2, colsum(x2)), sc, out)
    return out[0] / float(rows * d)


class SaeDenseStepEngine(SaeStepEngine):
    """``SaeStepEngine`` plus the dense (ReLU + L1) step and the ghost-grad terms.  ``k`` is unused on the dense path."""

    def __init__(self, *a, l1_coefficient: float = 0.0, **kw):
        kw["encoder"] = "dense"               # the dense / ghost terms read hidden_pre
        super().__init__(*a, **kw)
        self.l1_coefficient = float(l1_coefficient)
        self.aux = torch.zeros(4, device=self.W_dec.device)          # [l1_sum, ghost_sum, -, -]
        self._zero_idx = torch.zeros(1, dtype=torch.int32, device=self.W_dec.device)
        self.last_n_dead = 0

    # ------------------------------------------------------------------ pieces of every dense-product step
    def gemm32(self, a: torch.Tensor, a_lo: Optional[torch.Tensor], b_nk: torch.Tensor, b_lo: Optional[torch.Tensor], bias=None, act=None,
               out0=None, out1=None, residual=None, want_pre=True):
        """fp32-grade ``a @ b_nk.T`` (``+ residual`` into the second output) on the engine's route: GEMM_SIMT = the exact FFMA
        kernel (cross-check route); otherwise pb_gemm's AUTO rule with both residual planes supplied (split here when missing):
        the 3xTF32 tensor-core GEMM when the shape is TMA-legal, the exact FFMA kernel otherwise."""
        if self.gemm_impl == L.GEMM_SIMT:
            impl, a_lo, b_lo = L.GEMM_SIMT, None, None
        else:
            impl = L.GEMM_AUTO
            a_lo = ops.split_tf32(a) if a_lo is None else a_lo
            b_lo = ops.split_tf32(b_nk) if b_lo is None else b_lo
        return ops.gemm(a, b_nk, bias, act=act, residual=residual, a_lo=a_lo, w_lo=b_lo, out0=out0, out1=out1, want_pre=want_pre,
                        want_post=out1 is not None, impl=impl)

    def _at_b(self, a, b, out=None, residual=None) -> torch.Tensor:
        """``a^T @ b`` over the tokens ([rows, m], [rows, n] -> [m, n], ``+ residual``): pb_gemm takes K-major operands, so both
        are transposed first with their tf32 planes.  An operand given as a (transposed, tf32 plane) pair is used as it is."""
        aT, aT_lo = a if isinstance(a, tuple) else transpose(a)
        bT, bT_lo = b if isinstance(b, tuple) else transpose(b)
        if residual is None:
            return self.gemm32(aT, aT_lo, bT, bT_lo, out0=out)[0]
        return self.gemm32(aT, aT_lo, bT, bT_lo, residual=residual, out1=out, want_pre=False)[1]

    def _add_gb_dec(self, v: torch.Tensor, scale: float) -> None:
        """gb_dec += scale * v ([d]), as a one-row pb_scatter_add_rows through the index 0."""
        L.check(L.get_lib().pb_scatter_add_rows(self.gb_dec.data_ptr(), self._zero_idx.data_ptr(), 1, self.d, v.data_ptr(), scale,
                                                _stream()), "pb_scatter_add_rows")

    def _gb_dec_through_sae_in(self, v: torch.Tensor, W_rows: torch.Tensor) -> None:
        """gb_dec -= v @ W_rows: b_dec's gradient through sae_in = norm(x) - b_dec, where ``v`` [F'] is the token sum of the
        gradient at sae_in @ W_rows^T for rows ``W_rows`` [F', d] of W_enc^T."""
        self._add_gb_dec(gemv_rows(W_rows, v), -1.0)

    def _prep(self, x: torch.Tensor) -> None:
        """sae_in = norm(x) - b_dec (+ its tf32 plane), mu, sd, xsum; zeroes the step's scalars, aux and fired."""
        rows = x.shape[0]
        self._ensure_rows(rows)
        L.check(L.get_lib().pb_sae_prep(x.data_ptr(), self.b_dec.data_ptr(), self.sae_in.data_ptr(), self.sae_in_lo.data_ptr(),
                                        self.mu.data_ptr(), self.sd.data_ptr(), self.xsum.data_ptr(), rows, self.d, self.norm_mode,
                                        _stream()), "pb_sae_prep")
        self.scalars.zero_(); self.aux.zero_(); self.fired.zero_()

    def _dense_forward(self, x, y, ysum, b_out, want_out: bool, training: bool, resid=None, topk: bool = False, skip=None) -> torch.Tensor:
        """prep -> hidden_pre, acts = relu | TopK [encoder GEMM] -> stats -> out_n = acts @ W_dec + b_out [+ x @ skip^T through the
        residual epilogue] -> sae_out, loss against the target ``y`` (column sums ``ysum``), g when training, resid = y - sae_out
        on request.  ``y`` None: inference without a target, sae_out only.  Returns acts."""
        rows = x.shape[0]
        self._prep(x)
        if topk:
            self.gemm32(self.sae_in, self.sae_in_lo, self.W_encT, self.W_encT_lo, self.b_enc, out0=self.hidden_pre)
            acts = topk_dense(self.hidden_pre, self.k)                       # zeros.scatter_(topk idx, relu(topk values))
        else:
            acts = torch.empty(rows, self.F, device=x.device)
            self.gemm32(self.sae_in, self.sae_in_lo, self.W_encT, self.W_encT_lo, self.b_enc, act="relu", out0=self.hidden_pre, out1=acts)
        L.check(L.get_lib().pb_sae_dense_stats(acts.data_ptr(), rows, self.F, self.fired.data_ptr(), self.aux.data_ptr(),
                                               self.scalars.data_ptr(), _stream()), "pb_sae_dense_stats")
        WdT, WdT_lo = transpose(self.W_dec)                          # [d, F]: K-major B operand of the decoder product
        out_n, _ = self.gemm32(acts, None, WdT, WdT_lo, b_out)
        if skip is not None:                                         # skip [d_out, d_in] is already K-major
            _, out_n = self.gemm32(x, None, skip, None, residual=out_n, want_pre=False)
        if y is not None:
            _dense_loss(y, out_n, ysum, self.mu, self.sd, self.norm_mode, sae_out=self.sae_out if want_out else None,
                        g=self.g if training else None, resid=resid, scalars=self.scalars)
        elif want_out:
            _dense_loss(x, out_n, self.xsum, self.mu, self.sd, self.norm_mode, sae_out=self.sae_out)
        self.last_acts = acts
        return acts

    def _dense_backward(self, acts: torch.Tensor, l1_grad: float, gT=None) -> None:
        """d_hid = (g @ W_dec^T + l1_grad) * [acts > 0] -> gW_dec = acts^T @ g, gW_encT = d_hid^T @ sae_in, gb_enc = colsum(d_hid).
        ``gT``: the caller's (g^T, tf32 plane), when it needs g^T again."""
        d_hid, _ = self.gemm32(self.g, None, self.W_dec, None)            # d_acts [rows, F] = g @ W_dec^T
        # in place, without a tf32 plane: the transpose for gW_encT makes the one its product reads
        L.check(L.get_lib().pb_sae_dense_dhid(d_hid.data_ptr(), acts.data_ptr(), None, l1_grad, d_hid.numel(), _stream()),
                "pb_sae_dense_dhid")
        self._at_b(acts, self.g if gT is None else gT, out=self.gW_dec)
        self._at_b(d_hid, self.sae_in, out=self.gW_encT)
        colsum(d_hid, out=self.gb_enc)

    # ------------------------------------------------------------------ ghost grads (either activation)
    def _ghost_terms(self, x: torch.Tensor, resid: torch.Tensor, dead_idx: torch.Tensor) -> None:
        """Adds d(ghost loss)/d(params) for the dead features ``dead_idx`` (int32, sorted, distinct) into the gradient arrays
        and the loss value into ``aux[1]``.  Needs hidden_pre, sae_in, scalars.loss_sum of this step; ``resid = x - sae_out``."""
        lib, st = L.get_lib(), _stream()
        nd, d = int(dead_idx.numel()), self.d
        self.last_n_dead = nd
        E, WdD, dG0 = _ghost_block(self.hidden_pre, self.W_dec, dead_idx, resid, self.scalars, self.aux[1:])
        if nd == 0:
            return                                                    # loss value only: no parameter depends on it
        dE, _ = self.gemm32(dG0, None, WdD, None)                    # [rows, ndp]
        L.check(lib.pb_mul_inplace(dE.data_ptr(), E.data_ptr(), dE.numel(), st), "pb_mul_inplace")    # d h_dead = dE * exp(h)
        gWd_D = self._at_b(E, dG0)                                   # [ndp, d] = E^T @ dG0
        gWe_D = self._at_b(dE, self.sae_in)                          # [ndp, d] = d h_dead^T @ sae_in
        gbe_D = colsum(dE)                                           # [ndp]
        WeD = torch.empty_like(WdD)
        L.check(lib.pb_gather_rows(self.W_encT.data_ptr(), _p(dead_idx), nd, WdD.shape[0], d, WeD.data_ptr(), st), "pb_gather_rows")
        sc = lib.pb_scatter_add_rows
        L.check(sc(self.gW_dec.data_ptr(), _p(dead_idx), nd, d, gWd_D.data_ptr(), 1.0, st), "pb_scatter_add_rows")
        L.check(sc(self.gW_encT.data_ptr(), _p(dead_idx), nd, d, gWe_D.data_ptr(), 1.0, st), "pb_scatter_add_rows")
        L.check(sc(self.gb_enc.data_ptr(), _p(dead_idx), nd, 1, gbe_D.data_ptr(), 1.0, st), "pb_scatter_add_rows")
        self._gb_dec_through_sae_in(gbe_D, WeD)                      # sum over tokens of d h_dead @ W_enc[:, dead]^T

    # ------------------------------------------------------------------ TopK + ghost grads
    def train_step_topk_ghost(self, x: torch.Tensor, lr: float, since_fired: torch.Tensor, act_freq, dead_feature_window: int) -> torch.Tensor:
        """TopK step with ``cfg.use_ghost_grads`` (train_sae.py:330-354): the sparse pipeline computes the main gradients, the
        ghost blocks are added before the norm / clip."""
        _need_cuda(x)
        x = x.contiguous().float()
        lib, st = L.get_lib(), _stream()
        dead_idx = torch.nonzero(since_fired > dead_feature_window).flatten().to(torch.int32)   # host sync, as the reference's mask indexing
        self.encode_topk(x)
        self.scalars.zero_(); self.aux.zero_()
        self.step_count += 1
        s = self._desc(x, training=True, lr=float(lr), since_fired=since_fired, act_freq=act_freq, want_out=True)
        s.dist = 1                                                    # local gradients only; norm / clip after the ghost blocks
        L.check(lib.pb_sae_decode(C.byref(s), st), "pb_sae_decode")
        L.check(lib.pb_sae_backward(C.byref(s), st), "pb_sae_backward")
        self._ghost_terms(x, _residual(x, self.sae_out, self.xsum), dead_idx)
        self._clip_and_adam(x, float(lr), since_fired, act_freq, (self.gW_dec, self.gW_encT, self.gb_enc, self.gb_dec), ())
        return self.scalars

    # ------------------------------------------------------------------ dense ReLU + L1 (+ ghost grads)
    def train_step_dense(self, x: torch.Tensor, lr: float, since_fired: Optional[torch.Tensor] = None, act_freq=None,
                         use_ghost_grads: bool = False, dead_feature_window: int = 5000, want_out: bool = False) -> torch.Tensor:
        """One optimizer step with ``feature_acts = relu(hidden_pre)`` and ``loss = mse + l1_coefficient * mean_b ||acts||_1``."""
        _need_cuda(x)
        x = x.contiguous().float()
        dead_idx = torch.nonzero(since_fired > dead_feature_window).flatten().to(torch.int32) if use_ghost_grads else None
        self.step_count += 1
        resid = torch.empty_like(x) if use_ghost_grads else None
        acts = self._dense_forward(x, x, self.xsum, self.b_dec, want_out, training=True, resid=resid)
        self._dense_backward(acts, self.l1_coefficient / x.shape[0])
        colsum(self.g, out=self.gb_dec)
        self._gb_dec_through_sae_in(self.gb_enc, self.W_encT)       # sum_b d_sae_in = gb_enc @ W_enc^T
        if use_ghost_grads:
            self._ghost_terms(x, resid, dead_idx)
        self._clip_and_adam(x, float(lr), since_fired, act_freq, (self.gW_dec, self.gW_encT, self.gb_enc, self.gb_dec), ())
        return self.scalars

    def loss_terms(self, rows: int) -> dict:
        """Host read (synchronises): mse, l1, ghost and their sum for logging / tests."""
        sc, aux = self.scalars.tolist(), self.aux.tolist()
        out = dict(mse=sc[3], l0=sc[4], grad_norm=sc[6], clip_coef=sc[2], l1=self.l1_coefficient * aux[0] / rows,
                   ghost=aux[1] / (rows * self.d))
        out["loss"] = out["mse"] + out["l1"] + out["ghost"]
        return out
