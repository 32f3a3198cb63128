"""Sparse autoencoders on the H100 path (reference sae/sae.py:29-839).

``StandardSparseAutoencoder`` keeps the reference surface -- ``encode`` / ``decode`` / ``forward`` (7-tuple),
``set_decoder_norm_to_unit_norm``, ``initialize_b_dec*``, ``save_model`` / ``load_from_pretrained``, the four
HookPoints, state-dict keys ``W_enc [d_in,d_sae]``, ``W_dec [d_sae,d_in]``, ``b_enc``, ``b_dec`` -- with two routes:

* **sparse** (TopK, no hooks attached): vit_prisma/b200/sae_engine.py -- prep -> tensor-core encoder GEMM -> exact
  TopK -> sparse decode + normalised MSE.  The dense ``feature_acts`` the API returns is scattered from the
  ``[rows, k]`` support only because the signature promises a dense tensor.
* **dense / hooked** (``encode`` / ``decode`` called directly, ReLU activations, or any hook attached): op by op through
  the same kernels, every HookPoint fired in the reference order with replace-on-return semantics.

The encoder weight lives feature-major in memory (``W_enc`` is a transposed view of a contiguous ``[d_sae, d_in]``
buffer): that is the K-major operand the encoder GEMM wants and gives the optimizer one contiguous row per feature,
while ``state_dict()['W_enc']`` keeps the reference shape.

Training happens in ``VisionSAETrainer`` through the fused step engine (hand-written backward); this module's
``forward`` does not build an autograd graph.
"""
from __future__ import annotations

import gzip
import logging
import math
import os
import pickle
from abc import ABC, abstractmethod
from typing import Any, Callable, Optional

import torch
from torch import nn

from vit_prisma.b200 import _lib as L
from vit_prisma.b200 import ops
from vit_prisma.prisma_tools.hook_point import HookPoint
from vit_prisma.prisma_tools.hooked_root_module import HookedRootModule
from vit_prisma.sae.config import VisionModelSAERunnerConfig
from vit_prisma.sae.training.geometric_median import compute_geometric_median


class TopK(nn.Module):
    """``zeros.scatter_(topk(x, k).indices, postact(topk values))`` (reference :795-808)."""

    def __init__(self, k: int, postact_fn: Callable[[torch.Tensor], torch.Tensor] = nn.ReLU()):
        super().__init__()
        self.k = k
        self.postact_fn = postact_fn

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        from vit_prisma.b200.sae_engine import topk_dense
        if not isinstance(self.postact_fn, nn.ReLU):
            raise NotImplementedError("TopK on the H100 path supports the default ReLU post-activation")
        return topk_dense(x, self.k)


def get_activation_fn(activation_fn: str, **kwargs: Any) -> Callable[[torch.Tensor], torch.Tensor]:
    logging.info(f"get_activation_fn received: activation_fn={activation_fn}, kwargs={kwargs}")
    if activation_fn == "relu":
        return lambda x: ops.activation(x, "relu")
    if activation_fn == "tanh-relu":
        return lambda x: ops.activation(x, "tanh-relu")
    if activation_fn == "topk":
        assert "k" in kwargs, "TopK activation function requires a k value."
        return TopK(kwargs.get("k", 64), kwargs.get("postact_fn", nn.ReLU()))
    raise ValueError(f"Unknown activation function: {activation_fn}")


class SparseAutoencoder(HookedRootModule, ABC):
    def __init__(self, cfg: VisionModelSAERunnerConfig):
        super().__init__()
        self.cfg = cfg
        self.d_in = cfg.d_in
        if not isinstance(self.d_in, int):
            raise ValueError(f"d_in must be an int but was {self.d_in}; {type(self.d_in)}")
        assert cfg.d_sae is not None
        self.d_sae = cfg.d_sae
        self.l1_coefficient = cfg.l1_coefficient
        self.lp_norm = cfg.lp_norm
        self.dtype = cfg.dtype
        self.device = cfg.device
        self.initialization_method = cfg.initialization_method
        self.zero_loss = torch.tensor(0.0, dtype=self.dtype, device=self.device)
        self.initialize_sae_weights()
        self.hook_sae_in = HookPoint()
        self.hook_hidden_pre = HookPoint()
        self.hook_hidden_post = HookPoint()
        self.hook_sae_out = HookPoint()
        if cfg.normalize_activations not in ("layer_norm", "constant_norm_rescale"):
            self._norm_mode = "none"
        else:
            self._norm_mode = cfg.normalize_activations
        self.activation_fn = get_activation_fn(cfg.activation_fn_str, **cfg.activation_fn_kwargs)
        self._engine = None
        self._masters, self._masters_ver = None, None      # fp32 master parameters of reduced-precision configs (StandardSparseAutoencoder)
        self.setup()

    # ------------------------------------------------------------------ init helpers
    def initialize_weights(self, out_features: int, in_features: int) -> torch.Tensor:
        """Kaiming-uniform(a=sqrt 5) then unit-norm rows (reference :104-130)."""
        weight = torch.empty(out_features, in_features, dtype=self.dtype, device=self.device)
        nn.init.kaiming_uniform_(weight, a=math.sqrt(5))
        with torch.no_grad():
            weight /= torch.norm(weight, dim=1, keepdim=True)      # one-off init on whatever device cfg names
        return weight

    @abstractmethod
    def encode(self, x: torch.Tensor): ...

    @abstractmethod
    def decode(self, features: torch.Tensor): ...

    @abstractmethod
    def initialize_sae_weights(self): ...

    @abstractmethod
    def forward(self, x: torch.Tensor, dead_neuron_mask: torch.Tensor = None): ...

    # ------------------------------------------------------------------ b_dec initialisation (reference :181-242)
    @torch.no_grad()
    def initialize_b_dec_with_precalculated(self, origin: torch.Tensor, transcoder_dec_b: torch.Tensor = None):
        self.b_dec.data = origin.clone().detach().to(dtype=self.dtype, device=self.b_dec.device)

    @torch.no_grad()
    def initialize_b_dec(self, all_activations: torch.Tensor):
        method = self.cfg.b_dec_init_method
        if method == "geometric_median":
            self.initialize_b_dec_with_geometric_median(all_activations)
        elif method == "mean":
            self.initialize_b_dec_with_mean(all_activations)
        elif method != "zeros":
            raise ValueError(f"Unexpected b_dec_init_method: {method}")

    @torch.no_grad()
    def initialize_b_dec_with_geometric_median(self, all_activations: torch.Tensor):
        out = compute_geometric_median(all_activations, maxiter=100).median
        logging.info("Reinitializing b_dec with geometric median of activations")
        self.b_dec.data = out.to(dtype=self.dtype, device=self.b_dec.device)

    @torch.no_grad()
    def initialize_b_dec_with_mean(self, all_activations: torch.Tensor):
        logging.info("Reinitializing b_dec with mean of activations")
        self.b_dec.data = all_activations.mean(dim=0).to(self.dtype).to(self.b_dec.device)

    # ------------------------------------------------------------------ decoder geometry (reference :275-297)
    @torch.no_grad()
    def set_decoder_norm_to_unit_norm(self):
        if self.W_dec.is_cuda and self.W_dec.dtype == torch.float32 and self.W_dec.is_contiguous():
            from vit_prisma.b200.sae_engine import unit_norm_rows_
            unit_norm_rows_(self.W_dec.data)
        else:
            self.W_dec.data /= torch.norm(self.W_dec.data, dim=1, keepdim=True)

    @torch.no_grad()
    def remove_gradient_parallel_to_decoder_directions(self):
        """Kept for API compatibility with hand-rolled training loops that populated ``W_dec.grad`` themselves;
        VisionSAETrainer fuses this projection into the optimizer kernel."""
        par = (self.W_dec.grad * self.W_dec.data).sum(dim=1, keepdim=True)
        self.W_dec.grad -= par * self.W_dec.data

    # ------------------------------------------------------------------ persistence (reference :299-528)
    def save_model(self, path: str):
        folder = os.path.dirname(path)
        if folder:
            os.makedirs(folder, exist_ok=True)
        payload = {"cfg": self.cfg, "state_dict": {k: v.contiguous() for k, v in self.state_dict().items()}}
        if path.endswith(".pt"):
            torch.save(payload, path)
        elif path.endswith("pkl.gz"):
            with gzip.open(path, "wb") as f:
                pickle.dump(payload, f)
        else:
            raise ValueError(f"Unexpected file extension: {path}, supported extensions are .pt and .pkl.gz")
        print(f"Saved SAE to {path}")

    @staticmethod
    def _read_checkpoint(weights_path: str):
        readers = ((".pt", lambda p: torch.load(p, map_location="cpu", weights_only=False)),
                   (".pkl.gz", lambda p: pickle.load(gzip.open(p, "rb"))),
                   (".pkl", lambda p: pickle.load(open(p, "rb"))))
        for suffix, read in readers:
            if weights_path.endswith(suffix):
                try:
                    return read(weights_path)
                except Exception as e:
                    raise IOError(f"Error loading the state dictionary from {suffix} file: {e}")
        raise ValueError(f"Unexpected file extension: {weights_path}, supported extensions are .pt, .pkl, and .pkl.gz")

    @classmethod
    def load_from_pretrained(cls, weights_path: str, current_cfg=None, config_path: Optional[str] = None):
        """Reference sae/sae.py:409-523.  Accepts (a) a combined ``{"cfg", "state_dict"}`` checkpoint (what ``save_model`` writes),
        (b) a weights-only file with ``config.json`` next to it (or ``config_path``).  ``current_cfg`` is a mapping of overrides
        applied to fields the loaded config already has.  The class is chosen from the loaded config's ``architecture`` /
        ``is_transcoder``, so the canonical call ``SparseAutoencoder.load_from_pretrained(path)`` works on the abstract base."""
        if not os.path.isfile(weights_path):
            raise FileNotFoundError(f"No weights file found at: {weights_path}")
        payload = cls._read_checkpoint(weights_path)
        combined = isinstance(payload, dict) and "cfg" in payload and "state_dict" in payload
        if combined and config_path is None:
            loaded_cfg, weights = payload["cfg"], payload["state_dict"]
        else:
            cfg_file = config_path or os.path.join(os.path.dirname(weights_path), "config.json")
            if not os.path.isfile(cfg_file):
                raise FileNotFoundError(f"No config file found at {cfg_file} and no legacy format detected")
            loaded_cfg = VisionModelSAERunnerConfig.load_config(cfg_file)
            weights = payload["state_dict"] if combined else payload
        if not hasattr(loaded_cfg, "activation_fn_kwargs"):                # checkpoints older than the TopK option
            loaded_cfg.activation_fn_kwargs = ({"negative_slope": 0.01} if getattr(loaded_cfg, "activation_fn_str", "relu") == "leaky_relu"
                                               else {})
        if current_cfg is not None:
            items = current_cfg.items() if hasattr(current_cfg, "items") else vars(current_cfg).items()
            for key, value in items:
                if hasattr(loaded_cfg, key):
                    try:
                        setattr(loaded_cfg, key, value)
                    except AttributeError:       # read-only derived property on the config
                        pass
        if getattr(loaded_cfg, "is_transcoder", False):
            from vit_prisma.sae.transcoder import Transcoder
            model_cls = Transcoder
        elif loaded_cfg.architecture in ("standard", "vanilla"):
            model_cls = StandardSparseAutoencoder
        elif loaded_cfg.architecture == "gated":
            model_cls = GatedSparseAutoencoder
        else:
            raise ValueError(f"Unsupported architecture type: {loaded_cfg.architecture}")
        instance = model_cls(loaded_cfg)
        instance.load_state_dict(weights)
        return instance

    def get_name(self) -> str:
        return f"sparse_autoencoder_{self.cfg.model_name}_{self.cfg.hook_point}_{self.cfg.d_sae}"


class StandardSparseAutoencoder(SparseAutoencoder):
    def initialize_sae_weights(self):
        self.W_dec = nn.Parameter(self.initialize_weights(self.d_sae, self.d_in))
        if self.initialization_method == "independent":
            enc = self.initialize_weights(self.d_in, self.d_sae)          # [d_in, d_sae], rows unit-norm (reference :541)
            enc_t = enc.t().contiguous()                                   # feature-major storage
        elif self.initialization_method == "encoder_transpose_decoder":
            enc_t = self.W_dec.data.clone()
        else:
            raise ValueError(f"Unknown initialization method: {self.initialization_method}")
        self.W_enc = nn.Parameter(enc_t.t())                               # [d_in, d_sae] view, strides (1, d_in)
        self.b_enc = nn.Parameter(torch.zeros(self.d_sae, dtype=self.dtype, device=self.device))
        self.b_dec = nn.Parameter(torch.zeros(self.d_in, dtype=self.dtype, device=self.device))

    # ------------------------------------------------------------------ engine plumbing
    def _canonical_params(self):
        """(W_encT [F,d] contiguous view, W_dec, b_enc, b_dec) -- re-lays W_enc out feature-major if something
        (load_state_dict into a fresh tensor, user assignment) made it row-major."""
        if not self.W_enc.data.t().is_contiguous():
            self.W_enc.data = self.W_enc.data.t().contiguous().t()
        if not self.W_dec.data.is_contiguous():
            self.W_dec.data = self.W_dec.data.contiguous()
        return self.W_enc.data.t(), self.W_dec.data, self.b_enc.data, self.b_dec.data

    # ------------------------------------------------------------------ reduced-precision configs (cfg.dtype = bfloat16)
    @property
    def low_precision(self) -> bool:
        return self.dtype != torch.float32

    def _param_versions(self):
        return tuple((p.data_ptr(), p._version) for p in (self.W_enc, self.W_dec, self.b_enc, self.b_dec))

    def _engine_params(self):
        """The fp32 tensors the step engine trains.  float32 configs: the parameters' own storage.  Reduced-precision configs
        (cfg #5, ``dtype="bfloat16"``): fp32 MASTER copies -- the reference would run Adam on bf16 parameters with bf16 moments
        (torch.optim.Adam keeps state in the parameter dtype); here the optimizer math, the moments and the accumulated
        parameters are fp32 and the module's bf16 nn.Parameters (what state_dict / save_model / forward see) are the masters
        rounded once per step (``export_masters``).  Masters are rebuilt when someone writes the parameters (load_state_dict)."""
        if not self.low_precision:
            return self._canonical_params()
        wt, wd, be, bd = self._canonical_params()
        if self._masters is None or self._masters_ver != self._param_versions():
            self._masters = tuple(ops.cast(t.contiguous(), torch.float32) for t in (wt, wd, be, bd))
            self._masters_ver = self._param_versions()
        return self._masters

    @torch.no_grad()
    def export_masters(self):
        """Round the fp32 masters into the module's reduced-precision parameter storage (no-op for float32 configs)."""
        if not self.low_precision or self._masters is None:
            return
        eng = self._engine
        if eng is not None and getattr(eng, "is_data_parallel", False):
            eng.wait_parameters()                      # the deferred W_dec all-gather lands on a side stream
        for src, dst in zip(self._masters, self._canonical_params()):
            ops.cast_into(src, dst)

    @torch.no_grad()
    def set_decoder_norm_to_unit_norm(self):
        if self.low_precision and self.W_dec.is_cuda:
            from vit_prisma.b200.sae_engine import unit_norm_rows_
            masters = self._engine_params()
            unit_norm_rows_(masters[1])                 # normalise the fp32 master, then round: ||row|| = 1 to bf16 precision
            ops.cast_into(masters[1], self._canonical_params()[1])
            return
        super().set_decoder_norm_to_unit_norm()

    def step_engine(self, gemm_impl: int = L.GEMM_AUTO):
        """The step engine bound to this module's parameter storage (rebuilt if the storage moved): the fused sparse TopK
        pipeline, or ``SaeDenseStepEngine`` for ``activation_fn_str == "relu"`` (dense products + L1) and for
        ``cfg.use_ghost_grads`` with either activation (vit_prisma/b200/sae_dense.py)."""
        from vit_prisma.b200.sae_engine import SaeStepEngine
        act = self.cfg.activation_fn_str
        if act not in ("topk", "relu"):
            raise NotImplementedError(f"H100 training step: activation_fn_str {act!r} is not built (topk and relu are)")
        if act == "relu" and getattr(self.cfg, "lp_norm", 1) != 1:
            raise NotImplementedError("H100 dense training step: only lp_norm == 1 (the reference default) is built")
        dense = act == "relu" or bool(self.cfg.use_ghost_grads)
        wt, wd, be, bd = self._engine_params()
        eng = self._engine
        if eng is not None and getattr(eng, "is_data_parallel", False) and eng._key[:4] == self._engine_key(gemm_impl, dense)[:4]:
            return eng                       # the peer-memory engine owns the parameter storage: never rebuilt behind the trainer's back
        key = self._engine_key(gemm_impl, dense)
        if eng is None or eng._key != key:
            k = self.cfg.activation_fn_kwargs["k"] if act == "topk" else 1
            kw = dict(k=k, normalize_activations=self._norm_mode, max_grad_norm=self.cfg.max_grad_norm, gemm_impl=gemm_impl)
            if dense:
                from vit_prisma.b200.sae_dense import SaeDenseStepEngine
                eng = SaeDenseStepEngine(wt, wd, be, bd, l1_coefficient=self.cfg.l1_coefficient, **kw)
            else:
                eng = SaeStepEngine(wt, wd, be, bd, **kw)
            eng._key = key
            eng._enc_version = self.W_enc._version
            self._engine = eng
        return eng

    def _engine_key(self, gemm_impl: int, dense: bool):
        """Identity of the storage a step engine is bound to (+ the options that change which engine class serves it)."""
        wt, wd, be, bd = self._engine_params()
        return (wt.data_ptr(), wd.data_ptr(), be.data_ptr(), bd.data_ptr(), gemm_impl, dense)

    def enable_data_parallel(self, group, gemm_impl: int = L.GEMM_AUTO):
        """Move the parameters into NVLink peer-visible buffers and make ``step_engine()`` return the data-parallel engine
        (vit_prisma/b200/p2p.py): every rank then feeds its own token shard to ``train_step`` and all ranks hold identical
        parameters after each step.  ``group`` is a ``P2PGroup`` (one process per GPU)."""
        from vit_prisma.b200.p2p import SaeDPEngine
        if self.cfg.activation_fn_str != "topk":
            raise NotImplementedError("the fused step engine covers activation_fn_str == 'topk'")
        wt, wd, be, bd = self._engine_params()
        eng = SaeDPEngine(group, wt.contiguous(), wd, be, bd, k=self.cfg.activation_fn_kwargs["k"], normalize_activations=self._norm_mode,
                          max_grad_norm=self.cfg.max_grad_norm, gemm_impl=gemm_impl)
        if self.low_precision:
            # the peer-visible fp32 buffers become the masters; the bf16 nn.Parameters keep their storage and are refreshed per step
            self._masters = (eng.W_encT, eng.W_dec, eng.b_enc, eng.b_dec)
        else:
            # the nn.Parameters become views of the shared buffers, so state_dict()/save_model() see what the kernels update
            self.W_enc.data, self.W_dec.data, self.b_enc.data, self.b_dec.data = eng.W_encT.t(), eng.W_dec, eng.b_enc, eng.b_dec
        eng._key = self._engine_key(gemm_impl, False)
        eng._enc_version = self.W_enc._version
        self._engine = eng
        return eng

    def _hooks_attached(self) -> bool:
        return not all(hp.is_inert for hp in self.hook_points())

    # ------------------------------------------------------------------ dense / hooked route
    def _norm_in(self, x2: torch.Tensor):
        """run_time_activation_norm_fn_in: returns (x_normalised - 0, mu, std) using the prep kernel with a zero bias."""
        from vit_prisma.b200.sae_engine import sae_prep
        return sae_prep(x2, torch.zeros_like(self.b_dec.data), self._norm_mode)

    def _fire(self, hook: HookPoint, t: torch.Tensor) -> torch.Tensor:
        """Fire a HookPoint.  Reduced-precision configs compute in fp32 on the master parameters; the hook sees (and may replace)
        the tensor rounded to cfg.dtype -- the reference's own rounding points -- and the computation continues from what it returns."""
        if not self.low_precision:
            return hook(t)
        return ops.cast(hook(ops.cast(t, self.dtype)), torch.float32)

    def _compute_params(self):
        """fp32 tensors the module-by-module route multiplies with: the parameters (float32 configs) or their masters."""
        if self.low_precision and self.W_dec.is_cuda:
            return self._engine_params()
        return self._canonical_params()

    def _out(self, t: torch.Tensor) -> torch.Tensor:
        return ops.cast(t, self.dtype) if t.dtype != self.dtype else t

    def encode(self, x: torch.Tensor, return_hidden_pre: bool = False):
        from vit_prisma.b200.sae_engine import sae_prep
        x = ops.cast(x.contiguous(), torch.float32)
        lead = x.shape[:-1]
        x2 = x.reshape(-1, self.d_in).contiguous()
        wt, wd, be, bd = self._compute_params()
        sae_in2, mu, sd = sae_prep(x2, bd, self._norm_mode)               # norm_in(x) - b_dec  (reference :560-566)
        self.ln_mu, self.ln_std = mu.view(*lead, 1), sd.view(*lead, 1)
        sae_in = self._fire(self.hook_sae_in, sae_in2.view(*lead, self.d_in))
        hidden_pre, _ = ops.gemm(sae_in, wt, be)                           # sae_in @ W_enc + b_enc  (:568-574)
        hidden_pre = self._fire(self.hook_hidden_pre, hidden_pre)
        feature_acts = self._fire(self.hook_hidden_post, self.activation_fn(hidden_pre))
        if return_hidden_pre:
            return self._out(sae_in), self._out(feature_acts), self._out(hidden_pre)
        return self._out(sae_in), self._out(feature_acts)

    def decode(self, features: torch.Tensor):
        wt, wd, be, bd = self._compute_params()
        features = ops.cast(features.contiguous(), torch.float32)
        wd_nk = wd.t().contiguous()                                        # [d_in, d_sae]: K-major operand of features @ W_dec
        out, _ = ops.gemm(features, wd_nk, bd)                             # (:584-592)
        out = self._fire(self.hook_sae_out, out)
        if self._norm_mode == "layer_norm":                                 # x * std + mu  (:89-90)
            out = ops.add(ops.mul(out, self.ln_std.expand_as(out)), self.ln_mu.expand_as(out))
        elif self._norm_mode == "constant_norm_rescale":
            out = ops.mul(out, self.ln_std.expand_as(out))
        return self._out(out)

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, x: torch.Tensor, dead_neuron_mask: torch.Tensor = None, *args, **kwargs):
        from vit_prisma.b200.sae_engine import sae_mse
        want_ghost = bool(self.cfg.use_ghost_grads) and self.training and dead_neuron_mask is not None   # (:609-614)
        lead = x.shape[:-1]
        x32 = ops.cast(x.contiguous(), torch.float32)             # reduced-precision configs: fp32 arithmetic on the master parameters
        x2 = x32.reshape(-1, self.d_in).contiguous()
        sparse_ok = self.cfg.activation_fn_str == "topk" and not self._hooks_attached()
        if sparse_ok:
            eng = self.step_engine()
            if eng._enc_version != self.W_enc._version:                    # parameters written outside the engine
                eng.refresh_lo()
                eng._enc_version = self.W_enc._version
            sae_out2, _idx, _val = eng.forward(x2)
            sae_out = self._out(sae_out2.clone().view(*lead, self.d_in))
            mse_loss = self._out(eng.scalars[3].clone())
            if getattr(self.cfg, "return_out_only", False):      # spliced into HookedSAEViT (reference :636-640)
                # use_error_term: sae_out + (x - sae_out).detach() == x -- the clean activation flows on, the SAE's hooks still fired
                return x if getattr(self, "use_error_term", False) else sae_out
            feature_acts = self._out(eng.dense_feature_acts().view(*lead, self.d_sae))
            hidden_pre2 = eng.hidden_pre       # None on the fused encoder route (no dense pre-activations exist)
            if hidden_pre2 is None and want_ghost:
                hidden_pre2, _ = ops.gemm(eng.sae_in, self._compute_params()[0], self._compute_params()[2])
        else:
            _, feature_acts, _hidden_pre = self.encode(x32, return_hidden_pre=True)
            sae_out = self.decode(feature_acts)
            if getattr(self.cfg, "return_out_only", False):      # spliced into HookedSAEViT (reference :636-640)
                # use_error_term: sae_out + (x - sae_out).detach() == x -- the clean activation flows on, the SAE's hooks still fired
                return x if getattr(self, "use_error_term", False) else sae_out
            mse_loss = self._out(sae_mse(x2, ops.cast(sae_out.reshape(-1, self.d_in).contiguous(), torch.float32)))
            hidden_pre2 = _hidden_pre.reshape(-1, self.d_sae)
        ghost_loss = self.zero_loss.to(sae_out.device)
        if want_ghost:
            from vit_prisma.b200.sae_dense import ghost_loss_value
            ghost_loss = ghost_loss_value(hidden_pre2.float().contiguous(), self._compute_params()[1], x2.float(),
                                          sae_out.reshape(-1, self.d_in).float().contiguous(), mse_loss.float(), dead_neuron_mask)
        if self.cfg.activation_fn_str != "topk":
            # sparsity = ||feature_acts||_p over dim 1, mean over dim 0 (reference :617; tiny reduction, host-side glue)
            sparsity = feature_acts.norm(p=self.lp_norm, dim=1).mean(dim=(0,))
            l1_loss = self.l1_coefficient * sparsity
            loss = mse_loss + l1_loss + ghost_loss
        else:
            l1_loss = None
            loss = mse_loss + ghost_loss
        return (sae_out, feature_acts, loss, mse_loss, l1_loss, ghost_loss, torch.tensor(0.0))


class GatedSparseAutoencoder(SparseAutoencoder):
    """Gated SAE (reference sae/sae.py:648-792): gate path ``[sae_in @ W_enc + b_gate > 0]``, magnitude path
    ``relu(sae_in @ (W_enc * exp(r_mag)) + b_mag)`` with the shared encoder, L1 on ``relu(pi) * ||W_dec||`` and the via-gate
    auxiliary reconstruction loss.  Forward and training step run on ``vit_prisma/b200/sae_gated.py`` (one encoder GEMM for
    both paths).  HookPoints fire as observers; a hook that *replaces* an activation is refused (the module-by-module route the
    Standard SAE has is not built for this variant)."""

    def __init__(self, cfg):
        super().__init__(cfg)
        assert self.cfg.use_ghost_grads == False, "Gated SAE does not support ghost grads"   # noqa: E712  (reference :655-657)
        if cfg.activation_fn_str != "relu":
            raise NotImplementedError("H100 Gated SAE: activation_fn_str must be 'relu' (the reference default)")
        if self.dtype != torch.float32:
            raise NotImplementedError("H100 Gated SAE runs in float32")

    def initialize_sae_weights(self):                                     # reference :659-693 (plain kaiming_uniform_, no row norm)
        enc = torch.nn.init.kaiming_uniform_(torch.empty(self.cfg.d_in, self.cfg.d_sae, dtype=self.dtype, device=self.device))
        self.W_enc = nn.Parameter(enc.t().contiguous().t())               # [d_in, d_sae] view of feature-major storage
        z = lambda n: nn.Parameter(torch.zeros(n, dtype=self.dtype, device=self.device))  # noqa: E731
        self.b_gate, self.r_mag, self.b_mag = z(self.cfg.d_sae), z(self.cfg.d_sae), z(self.cfg.d_sae)
        self.W_dec = nn.Parameter(torch.nn.init.kaiming_uniform_(torch.empty(self.cfg.d_sae, self.cfg.d_in, dtype=self.dtype, device=self.device)))
        self.b_enc = z(self.d_sae)                                        # exists in the reference, never used by its graph
        self.b_dec = z(self.d_in)

    def _canonical_params(self):
        if not self.W_enc.data.t().is_contiguous():
            self.W_enc.data = self.W_enc.data.t().contiguous().t()
        if not self.W_dec.data.is_contiguous():
            self.W_dec.data = self.W_dec.data.contiguous()
        return self.W_enc.data.t(), self.W_dec.data, self.b_gate.data, self.r_mag.data, self.b_mag.data, self.b_dec.data

    def step_engine(self, gemm_impl: int = L.GEMM_AUTO):
        from vit_prisma.b200.sae_gated import SaeGatedStepEngine
        params = self._canonical_params()
        key = tuple(t.data_ptr() for t in params) + (gemm_impl,)
        eng = self._engine
        if eng is None or eng._key != key:
            wt, wd, bg, rm, bm, bd = params
            eng = SaeGatedStepEngine(wt, wd, bg, rm, bm, bd, l1_coefficient=self.cfg.l1_coefficient, normalize_activations=self._norm_mode,
                                     max_grad_norm=self.cfg.max_grad_norm, gemm_impl=gemm_impl)
            eng._key = key
            eng._enc_version = self.W_enc._version
            self._engine = eng
        return eng

    def _fire(self, hook: HookPoint, t: torch.Tensor) -> torch.Tensor:
        out = hook(t)
        if out is not t and out.data_ptr() != t.data_ptr():
            raise NotImplementedError("H100 Gated SAE: hooks may observe activations but not replace them")
        return t

    def _run(self, x: torch.Tensor):
        x32 = ops.cast(x, self.dtype) if x.dtype != self.dtype else x
        lead = x32.shape[:-1]
        x2 = x32.reshape(-1, self.d_in).contiguous()
        eng = self.step_engine()
        if eng._enc_version != self.W_enc._version:
            eng.refresh_lo()
            eng._enc_version = self.W_enc._version
        acts = eng.forward_losses(x2, want_out=True)
        self.ln_mu, self.ln_std = eng.mu.clone().view(*lead, 1), eng.sd.clone().view(*lead, 1)
        sae_in = self._fire(self.hook_sae_in, eng.sae_in.clone().view(*lead, self.d_in))
        feature_acts = self._fire(self.hook_hidden_post, acts.view(*lead, self.d_sae))
        sae_out = self._fire(self.hook_sae_out, eng.sae_out.clone().view(*lead, self.d_in))
        return eng, x2.shape[0], sae_in, feature_acts, sae_out

    @torch.no_grad()
    def encode(self, x: torch.Tensor):
        _, _, sae_in, feature_acts, _ = self._run(x)
        return sae_in, feature_acts

    @torch.no_grad()
    def decode(self, features: torch.Tensor):
        wd, bd = self.W_dec.data, self.b_dec.data
        out, _ = ops.gemm(features, wd.t().contiguous(), bd)               # (:711-722)
        out = self.hook_sae_out(out)
        if self._norm_mode == "layer_norm":
            out = ops.add(ops.mul(out, self.ln_std.expand_as(out)), self.ln_mu.expand_as(out))
        elif self._norm_mode == "constant_norm_rescale":
            out = ops.mul(out, self.ln_std.expand_as(out))
        return out

    @torch.no_grad()
    def forward(self, x: torch.Tensor, *args, **kwargs):
        eng, rows, _sae_in, feature_acts, sae_out = self._run(x)
        if getattr(self.cfg, "return_out_only", False):
            return sae_out
        mse_loss = eng.scalars[3].clone()
        l1_loss = eng.aux[0] * (self.l1_coefficient / rows)
        aux_reconstruction_loss = eng.aux[1] / rows
        loss = mse_loss + l1_loss + aux_reconstruction_loss
        return (sae_out, feature_acts, loss, mse_loss, l1_loss, self.zero_loss.to(sae_out.device), aux_reconstruction_loss)
