"""VisionSAETrainer -- SAE training entry point on the H100 path (reference sae/train_sae.py:61-861).

Same constructor, ``run()`` / ``train_step(...)`` / ``checkpoint(...)`` surface and the same order of operations per
step (train_sae.py:278-411):

    decoder rows to unit norm -> forward -> dead-feature statistics -> backward -> global-norm clip ->
    remove decoder-parallel gradient -> Adam -> LR schedule

but the whole step is six kernel launches' worth of native code (vit_prisma/b200/sae_engine.py, csrc/sae.cu) with a
hand-written sparse backward instead of autograd over dense ``[batch, d_sae]`` tensors, and it never synchronises with
the host: the reference's per-step ``loss.item()`` for the progress bar (train_sae.py:846-848) becomes a read every
``cfg.wandb_log_frequency`` steps.

Notes on fidelity
  * the unit-norm renormalisation of ``W_dec`` that the reference performs at the *start* of step t+1 is folded into the
    end of step t (same numbers seen by every forward/backward; parameters compare equal after applying
    ``set_decoder_norm_to_unit_norm()`` on the reference side);
  * ``optimizer`` / ``scheduler`` returned by ``initialize_training_variables`` are light handles (``param_groups[0]["lr"]``,
    ``step()``, ``get_last_lr()``) -- the optimizer state lives in the engine's device buffers;
  * transcoders (``cfg.is_transcoder``) train through ``vit_prisma/b200/sae_transcoder.py``: ``layer_acts[:, 0]`` is the input, ``[:, 1]`` the target.
"""
from __future__ import annotations

import os
import uuid
from typing import Optional

import torch

from vit_prisma.sae.config import VisionModelSAERunnerConfig
from vit_prisma.sae.sae import GatedSparseAutoencoder, StandardSparseAutoencoder
from vit_prisma.sae.training.activations_store import CacheVisionActivationStore, VisionActivationsStore
from vit_prisma.sae.training.geometric_median import compute_geometric_median
from vit_prisma.sae.training.get_scheduler import lr_multiplier_fn


class FusedAdamHandle:
    """What callers of the reference loop touch on a torch optimizer: ``param_groups[0]['lr']`` and ``zero_grad``."""

    def __init__(self, lr: float):
        self.param_groups = [{"lr": lr, "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 0}]

    def zero_grad(self, set_to_none: bool = True):
        pass

    def step(self):
        pass


class FusedSchedule:
    def __init__(self, handle: FusedAdamHandle, base_lr: float, multiplier):
        self.handle, self.base_lr, self.multiplier = handle, base_lr, multiplier
        self.last_epoch = 0
        handle.param_groups[0]["lr"] = base_lr * multiplier(0)

    def step(self):
        self.last_epoch += 1
        self.handle.param_groups[0]["lr"] = self.base_lr * self.multiplier(self.last_epoch)

    def get_last_lr(self):
        return [self.handle.param_groups[0]["lr"]]


class VisionSAETrainer:
    def __init__(self, cfg: VisionModelSAERunnerConfig, model, dataset, eval_dataset=None, activations_store=None, p2p_group=None):
        self.cfg = cfg
        self.p2p_group = p2p_group       # vit_prisma.b200.p2p.P2PGroup: data-parallel training, one process per GPU
        self.is_transcoder = cfg.is_transcoder
        for attr in ("min_l0", "min_explained_variance"):          # older configs may lack these
            if not hasattr(cfg, attr):
                setattr(cfg, attr, None)
        self.bad_run_check = bool(cfg.min_l0 and cfg.min_explained_variance)
        self.model = model
        if self.is_transcoder:                                       # train_sae.py:73-75
            from vit_prisma.sae.transcoder import Transcoder
            self.sparse_coder = Transcoder(cfg)
        elif cfg.architecture == "gated":
            self.sparse_coder = GatedSparseAutoencoder(cfg)
        elif cfg.architecture in ("standard", "vanilla"):
            self.sparse_coder = StandardSparseAutoencoder(cfg)
        else:
            raise ValueError(f"Loading of {cfg.architecture} not supported")
        self.dataset, self.eval_dataset = dataset, eval_dataset
        self.activations_store = activations_store if activations_store is not None else self.initialize_activations_store(dataset, eval_dataset)
        if not cfg.wandb_project:
            cfg.wandb_project = (cfg.model_name.replace("/", "-") + "-expansion-" + str(cfg.expansion_factor) + "-layer-"
                                 + str(cfg.hook_point_layer))
        cfg.unique_hash = uuid.uuid4().hex[:8]
        cfg.run_name = cfg.unique_hash + "-" + cfg.wandb_project
        self.checkpoint_thresholds = self.get_checkpoint_thresholds()
        self.setup_checkpoint_path()
        self._wandb = None
        if cfg.verbose:
            cfg.pretty_print()

    # ------------------------------------------------------------------ setup
    def setup_checkpoint_path(self):
        if self.cfg.n_checkpoints:
            self.cfg.checkpoint_path = f"{self.cfg.checkpoint_path}/{self.cfg.run_name}"
            os.makedirs(self.cfg.checkpoint_path, exist_ok=True)
        else:
            print("Not saving checkpoints so skipping creating checkpoint directory")

    def initialize_activations_store(self, dataset, eval_dataset):
        if self.cfg.use_cached_activations:
            return CacheVisionActivationStore(self.cfg)
        return VisionActivationsStore(self.cfg, self.model, dataset, eval_dataset=eval_dataset, num_workers=self.cfg.num_workers)

    def get_checkpoint_thresholds(self):
        if self.cfg.n_checkpoints > 0:
            total = self.cfg.total_training_tokens
            return list(range(0, total, total // self.cfg.n_checkpoints))[1:]
        return []

    def initialize_training_variables(self):
        dev = self.sparse_coder.W_dec.device
        act_freq_scores = torch.zeros(int(self.cfg.d_sae), device=dev)
        n_forward_passes_since_fired = torch.zeros(int(self.cfg.d_sae), device=dev)
        optimizer = FusedAdamHandle(self.cfg.lr)
        scheduler = FusedSchedule(optimizer, self.cfg.lr, lr_multiplier_fn(
            self.cfg.lr_scheduler_name, warm_up_steps=self.cfg.lr_warm_up_steps, training_steps=self.cfg.total_training_steps,
            lr_end=self.cfg.lr / 10))
        return act_freq_scores, n_forward_passes_since_fired, 0, optimizer, scheduler

    def initialize_geometric_medians(self):
        cfg = self.sparse_coder.cfg
        layers = cfg.hook_point_layer if isinstance(cfg.hook_point_layer, list) else [cfg.hook_point_layer]
        layer_id = layers.index(cfg.hook_point_layer) if not isinstance(cfg.hook_point_layer, list) else 0
        medians = {}
        if cfg.b_dec_init_method == "geometric_median":
            acts = self.activations_store.storage_buffer.detach()[:, layer_id, :]
            medians[layer_id] = compute_geometric_median(acts.float(), maxiter=200).median
            self.sparse_coder.initialize_b_dec_with_precalculated(medians[layer_id])
        elif cfg.b_dec_init_method == "mean":
            acts = self.activations_store.storage_buffer.detach()[:, layer_id, :]
            self.sparse_coder.initialize_b_dec_with_mean(acts)
        self.sparse_coder.train()
        return medians

    def _canonical_param_storages(self):
        """Contiguous tensors behind the four parameters (W_enc is a transposed view of a [d_sae, d_in] buffer)."""
        wt, wd, be, bd = self.sparse_coder._canonical_params()
        return [wt, wd, be, bd]

    def enable_data_parallel_if_requested(self):
        """With a P2PGroup: rank 0's b_dec initialisation is broadcast (every rank must start from identical parameters),
        then the parameters move into NVLink peer-visible buffers (sae.enable_data_parallel)."""
        if self.p2p_group is None or self.p2p_group.world == 1:
            return
        cfg = self.cfg
        if self.is_transcoder or cfg.architecture == "gated" or cfg.activation_fn_str != "topk" or cfg.use_ghost_grads:
            raise NotImplementedError("data-parallel SAE training over NVLink peer memory covers the TopK step (standard architecture, "
                                      "no ghost grads); the dense / ghost / gated steps run single-GPU")
        import torch.distributed as dist
        for prm in self._canonical_param_storages():
            dist.broadcast(prm, src=0)
        self.sparse_coder.enable_data_parallel(self.p2p_group)

    # ------------------------------------------------------------------ one step
    def train_step(self, sparse_autoencoder, optimizer, scheduler, act_freq_scores, n_forward_passes_since_fired,
                   n_frac_active_tokens, layer_acts, n_training_steps, n_training_tokens):
        cfg = sparse_autoencoder.cfg
        layers = cfg.hook_point_layer if isinstance(cfg.hook_point_layer, list) else [cfg.hook_point_layer]
        layer_id = 0 if isinstance(cfg.hook_point_layer, list) else layers.index(cfg.hook_point_layer)
        target_activation = None
        if self.is_transcoder:                                       # train_sae.py:299-301: input and target ride in one tensor
            sae_in, target_activation = layer_acts[:, 0, :], layer_acts[:, 1, :]
        else:
            sae_in = layer_acts[:, layer_id, :]
        sparse_autoencoder.train()
        engine = sparse_autoencoder.step_engine()
        if engine.step_count == 0:
            sparse_autoencoder.set_decoder_norm_to_unit_norm()      # later steps leave the rows normalised themselves
            engine.refresh_lo()

        if (n_training_steps + 1) % self.cfg.feature_sampling_window == 0:   # train_sae.py:309-326
            feature_sparsity = act_freq_scores / n_frac_active_tokens
            if self.cfg.log_to_wandb:
                self._log({"metrics/mean_log10_feature_sparsity": torch.log10(feature_sparsity + 1e-10).mean().item(),
                           "sparsity/below_1e-5": (feature_sparsity < 1e-5).float().mean().item(),
                           "sparsity/below_1e-6": (feature_sparsity < 1e-6).float().mean().item()}, n_training_steps)
            act_freq_scores.zero_()
            n_frac_active_tokens = 0

        lr = optimizer.param_groups[0]["lr"]
        l1_loss = None
        gated = cfg.architecture == "gated" and not self.is_transcoder
        if self.is_transcoder:                                       # dense products + skip matrix + second decoder bias, sae_transcoder.py
            scalars = engine.train_step_transcoder(sae_in, target_activation, lr, since_fired=n_forward_passes_since_fired,
                                                   act_freq=act_freq_scores)
        elif gated:                                                    # one encoder GEMM for gate + magnitude paths, sae_gated.py
            scalars = engine.train_step_gated(sae_in, lr, since_fired=n_forward_passes_since_fired, act_freq=act_freq_scores)
        elif cfg.activation_fn_str == "relu":                        # dense products + L1 (+ ghost grads), sae_dense.py
            scalars = engine.train_step_dense(sae_in, lr, since_fired=n_forward_passes_since_fired, act_freq=act_freq_scores,
                                              use_ghost_grads=bool(cfg.use_ghost_grads), dead_feature_window=cfg.dead_feature_window)
        elif cfg.use_ghost_grads:                                    # sparse TopK gradients + ghost blocks on the dead features
            scalars = engine.train_step_topk_ghost(sae_in, lr, n_forward_passes_since_fired, act_freq_scores, cfg.dead_feature_window)
        else:
            scalars = engine.train_step(sae_in, lr, since_fired=n_forward_passes_since_fired, act_freq=act_freq_scores)
        if getattr(sparse_autoencoder, "low_precision", False):
            sparse_autoencoder.export_masters()      # bf16 configs: the engine trained fp32 masters; refresh the module's parameters
        n_frac_active_tokens += sae_in.shape[0]
        # the engine's scalars buffer is rewritten by the next step: hand out copies (device-side, no host sync)
        mse_loss = scalars[3].clone()
        loss = mse_loss            # TopK: loss == mse (no L1 term, train_sae.py:617-626)
        ghost_loss = aux_loss = None
        if gated:                                                    # loss = mse + l1 + aux reconstruction (sae.py:744)
            l1_loss = engine.aux[0] * (engine.l1_coefficient / sae_in.shape[0])
            aux_loss = engine.aux[1] / float(sae_in.shape[0])
            loss = loss + l1_loss + aux_loss
        elif self.is_transcoder:                                     # loss = mse (+ l1 for dense activations), transcoder.py:93-103
            if cfg.activation_fn_str != "topk":
                l1_loss = engine.aux[0] * (engine.l1_coefficient / sae_in.shape[0])
                loss = loss + l1_loss
        elif hasattr(engine, "aux"):                                 # device-side: loss = mse + l1 + ghost (sae.py:628)
            ghost_loss = engine.aux[1] / float(sae_in.shape[0] * engine.d)
            if cfg.activation_fn_str != "topk":
                l1_loss = engine.aux[0] * (engine.l1_coefficient / sae_in.shape[0])
                loss = loss + l1_loss
            loss = loss + ghost_loss
        l0 = scalars[4].clone()
        if self.cfg.log_to_wandb and (n_training_steps + 1) % self.cfg.wandb_log_frequency == 0:
            vals = engine.scalars_dict()
            metrics = {"losses/mse_loss": vals["mse"], "losses/overall_loss": float(loss), "metrics/l0": vals["l0"],
                       "metrics/grad_norm": vals["grad_norm"], "details/current_learning_rate": lr,
                       "details/n_training_tokens": n_training_tokens,
                       "metrics/mean_passes_since_fired": n_forward_passes_since_fired.mean().item(),
                       "sparsity/dead_features": (n_forward_passes_since_fired > cfg.dead_feature_window).sum().item()}
            if l1_loss is not None:
                metrics["losses/l1_loss"] = float(l1_loss)
            if ghost_loss is not None:
                metrics["losses/ghost_grad_loss"] = float(ghost_loss)
            if aux_loss is not None:
                metrics["losses/aux_reconstruction_loss"] = float(aux_loss)
            self._log(metrics, n_training_steps)
        scheduler.step()
        return loss, mse_loss, l1_loss, l0, act_freq_scores, n_forward_passes_since_fired, n_frac_active_tokens

    # ------------------------------------------------------------------ logging / checkpoints
    def initalize_wandb(self):
        try:
            import wandb
            wandb.init(project=self.cfg.wandb_project, entity=self.cfg.wandb_entity, name=self.cfg.run_name, mode=os.environ.get("WANDB_MODE", "offline"))
            self._wandb = wandb
        except Exception as e:  # wandb is optional plumbing, never a reason to stop training
            print(f"wandb unavailable ({e}); metrics will not be logged")
            self._wandb = None

    def _log(self, metrics: dict, step: int) -> None:
        if self._wandb is not None:
            self._wandb.log(metrics, step=step)

    def checkpoint(self, sae, n_training_tokens, act_freq_scores, n_frac_active_tokens):
        self.cfg.save_config(f"{self.cfg.checkpoint_path}/config.json")
        n_images = n_training_tokens // self.cfg.context_size
        path = self.cfg.checkpoint_path + f"/n_images_{n_images}.pt"
        sae.set_decoder_norm_to_unit_norm()
        sae.save_model(path)
        sparsity_path = self.cfg.checkpoint_path + f"/n_images_{n_images}_log_feature_sparsity.pt"
        feature_sparsity = act_freq_scores / max(n_frac_active_tokens, 1)
        torch.save(torch.log10(feature_sparsity + 1e-10).detach().cpu(), sparsity_path)
        self._log({"details/checkpoint_path": path}, n_training_tokens // self.cfg.train_batch_size)
        return path

    # ------------------------------------------------------------------ loop
    def run(self, progress_every: Optional[int] = None):
        from tqdm import tqdm
        if self.cfg.log_to_wandb:
            self.initalize_wandb()
        act_freq_scores, since_fired, n_frac_active_tokens, optimizer, scheduler = self.initialize_training_variables()
        self.initialize_geometric_medians()
        self.enable_data_parallel_if_requested()
        n_steps, n_tokens = 0, 0
        world = self.p2p_group.world if self.p2p_group is not None else 1
        progress_every = progress_every or max(self.cfg.wandb_log_frequency, 1)
        pbar = tqdm(total=self.cfg.total_training_tokens, desc="Training SAE", mininterval=20)
        while n_tokens < self.cfg.total_training_tokens:
            layer_acts = self.activations_store.next_batch()
            if world > 1 and layer_acts.shape[0] != self.cfg.train_batch_size:
                continue          # data parallel: every rank must bring the same row count to the peer barriers (short tail batches are dropped)
            loss, mse_loss, l1_loss, l0, act_freq_scores, since_fired, n_frac_active_tokens = self.train_step(
                sparse_autoencoder=self.sparse_coder, optimizer=optimizer, scheduler=scheduler, layer_acts=layer_acts,
                n_training_steps=n_steps, n_training_tokens=n_tokens, act_freq_scores=act_freq_scores,
                n_forward_passes_since_fired=since_fired, n_frac_active_tokens=n_frac_active_tokens)
            n_steps += 1
            n_tokens += self.cfg.train_batch_size * world        # tokens of the GLOBAL step (each rank's store feeds its own shard)
            if self.checkpoint_thresholds and n_tokens > self.checkpoint_thresholds[0]:
                self.checkpoint(self.sparse_coder, n_tokens, act_freq_scores, n_frac_active_tokens)
                self.checkpoint_thresholds.pop(0)
            pbar.update(self.cfg.train_batch_size * world)
            if n_steps % progress_every == 0:                       # one host read per N steps, not per step
                pbar.set_description(f"Training SAE: Loss: {loss.item():.4f}, MSE Loss: {mse_loss.item():.4f}, L0: {l0.item():.4f}", refresh=False)
        if self.cfg.n_checkpoints:
            self.checkpoint(self.sparse_coder, n_tokens, act_freq_scores, n_frac_active_tokens)
        pbar.close()
        return self.sparse_coder
