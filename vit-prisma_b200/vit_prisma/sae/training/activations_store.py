"""Activation supply for SAE training (reference sae/training/activations_store.py:21-574).

``VisionActivationsStore`` keeps the reference's interface and mixing semantics -- a storage half-buffer, refills of
``n_batches_in_buffer // 2`` image batches through ``model.run_with_cache(names_filter=[hook], stop_at_layer=layer+1)``,
concatenate + ``randperm`` shuffle, keep half, serve half -- with two H100-minded changes:

* refills hit the fused ViT chain with a one-key ``names_filter`` (nothing but the requested hook point is spilled,
  blocks after the hook layer are never launched);
* the serving side is a device-resident tensor walked through a ``randperm`` index: ``next_batch`` is one gather, not the
  reference's ``DataLoader(tensor, shuffle=True)`` whose default collate stacks 4096 single-row tensors in Python
  (activations_store.py:486-490).

``SyntheticActivationsStore`` serves seeded random activations of the same shape contract (bench / tests / no dataset).
"""
from __future__ import annotations

import os
from typing import Any, Iterator, Optional

import torch
from torch.utils.data import DataLoader


def collate_fn(data):
    return torch.stack([d[0] for d in data], dim=0)


def collate_fn_eval(data):
    return torch.stack([d[0] for d in data], dim=0), torch.tensor([d[1] for d in data])


class _ShuffledServer:
    """Serve ``[n, ...]`` rows in a fresh random order, ``batch`` at a time (drops nothing: last batch may be short)."""

    def __init__(self, data: torch.Tensor, batch: int):
        self.data, self.batch = data, batch
        self.perm = torch.randperm(data.shape[0], device=data.device)
        self.pos = 0

    def __iter__(self):
        return self

    def __next__(self) -> torch.Tensor:
        if self.pos >= self.data.shape[0]:
            raise StopIteration
        sel = self.perm[self.pos:self.pos + self.batch]
        self.pos += self.batch
        return self.data.index_select(0, sel)


class VisionActivationsStore:
    def __init__(self, cfg, model, dataset, create_dataloader: bool = True, eval_dataset=None, num_workers: int = 0):
        self.cfg = cfg
        self.model = model.to(cfg.device)
        self.dataset = dataset
        self.image_dataloader = DataLoader(dataset, shuffle=True, num_workers=num_workers, batch_size=cfg.store_batch_size,
                                           collate_fn=collate_fn, drop_last=True)
        if eval_dataset is not None:
            self.image_dataloader_eval = DataLoader(eval_dataset, shuffle=True, num_workers=num_workers,
                                                    batch_size=cfg.store_batch_size, collate_fn=collate_fn_eval, drop_last=True)
            self.image_dataloader_eval_iter = self._eval_batch_stream(self.image_dataloader_eval, cfg.device)
        self.image_dataloader_iter = self._batch_stream(self.image_dataloader, cfg.device)
        if create_dataloader:
            if cfg.is_transcoder:                                 # (input, target) activation pairs, reference :216-222
                self.storage_buffer, self.storage_buffer_out = self.get_buffer(cfg.n_batches_in_buffer // 2)
            else:
                self.storage_buffer = self.get_buffer(cfg.n_batches_in_buffer)
            self.dataloader = self.get_data_loader()

    @staticmethod
    def _batch_stream(dataloader: DataLoader, device) -> Iterator[torch.Tensor]:
        while True:
            for batch in dataloader:
                batch.requires_grad_(False)
                yield batch.to(device, non_blocking=True)

    @staticmethod
    def _eval_batch_stream(dataloader: DataLoader, device):
        while True:
            for images, labels in dataloader:
                yield images.to(device), labels.to(device)

    def _layers(self):
        hp = self.cfg.hook_point_layer
        return hp if isinstance(hp, list) else [hp]

    def _out_layers(self):
        hp = self.cfg.out_hook_point_layer
        return hp if isinstance(hp, list) else [hp]

    def _pick(self, cache, names):
        per_layer = []
        for name in names:
            acts = cache[name]
            if self.cfg.hook_point_head_index is not None:
                acts = acts[:, :, self.cfg.hook_point_head_index]
            if self.cfg.cls_token_only:
                acts = acts[:, 0:1]
            per_layer.append(acts)
        return torch.stack(per_layer, dim=2)

    @torch.no_grad()
    def get_activations(self, batch_images: torch.Tensor):
        """[b, T', n_layers, d_in] for the configured hook point(s) (reference :252-296); for a transcoder the pair
        (input activations, target activations at ``cfg.out_hook_point``) from ONE run_with_cache call."""
        layers = self._layers()
        names = [self.cfg.hook_point.format(layer=layer) for layer in layers]
        if not self.cfg.is_transcoder:
            _, cache = self.model.run_with_cache(batch_images, names_filter=names, stop_at_layer=max(layers) + 1)
            return self._pick(cache, names)
        out_layers = self._out_layers()
        out_names = [self.cfg.out_hook_point.format(layer=layer) for layer in out_layers]
        _, cache = self.model.run_with_cache(batch_images, names_filter=names + out_names, stop_at_layer=max(max(layers), max(out_layers)) + 1)
        return self._pick(cache, names), self._pick(cache, out_names)

    def get_buffer(self, n_batches_in_buffer: int):
        cfg = self.cfg
        if cfg.use_cached_activations:
            assert not cfg.is_transcoder, "Transcoder not supported with cached activations"       # reference :322
            return self._load_cached_activations(cfg.store_batch_size * n_batches_in_buffer, cfg.context_size, len(self._layers()), cfg.d_in)
        chunks, chunks_out = [], []
        for _ in range(n_batches_in_buffer):
            acts = self.get_activations(next(self.image_dataloader_iter))
            acts, acts_out = acts if cfg.is_transcoder else (acts, None)
            if cfg.use_patches_only:
                acts = acts[:, 1:, :, :]
                acts_out = None if acts_out is None else acts_out[:, 1:, :, :]
            chunks.append(acts.reshape(-1, acts.shape[2], cfg.d_in).to(cfg.dtype))
            if acts_out is not None:
                chunks_out.append(acts_out.reshape(-1, acts_out.shape[2], cfg.d_out).to(cfg.dtype))
        buf = torch.cat(chunks, dim=0)
        perm = torch.randperm(buf.shape[0], device=buf.device)
        if cfg.is_transcoder:
            return buf[perm], torch.cat(chunks_out, dim=0)[perm]                 # the same permutation keeps the pairs together
        return buf[perm]

    def _load_cached_activations(self, total_size, context_size, num_layers, d_in) -> torch.Tensor:
        """fp16/fp32 ``{idx}.pt`` shards of ``[tokens, n_layers, d_in]`` (reference :371-415)."""
        want = total_size * context_size
        parts, have, idx = [], 0, 0
        while have < want:
            path = f"{self.cfg.cached_activations_path}/{idx}.pt"
            if not os.path.exists(path):
                break
            acts = torch.load(path, map_location=self.cfg.device, weights_only=True)[: want - have]
            parts.append(acts.to(self.cfg.dtype))
            have += acts.shape[0]
            idx += 1
        if not parts:
            return torch.zeros((0, num_layers, d_in), dtype=self.cfg.dtype, device=self.cfg.device)
        return torch.cat(parts, dim=0)

    def generate_cached_activations_from_dataset(self, tokens_per_file: int = 1_000_000, shuffle_data: bool = False) -> int:
        """Write the dataset's activations as the reference's disk cache (reference :505-574): fp16 ``{idx}.pt`` files of
        ``[tokens, n_layers, d_in]``, ``tokens_per_file`` tokens each (the last one holds the remainder), readable by
        ``_load_cached_activations`` / ``CacheVisionActivationStore`` here and in the reference.  Returns the number of files."""
        cfg = self.cfg
        os.makedirs(cfg.cached_activations_path, exist_ok=True)
        loader = DataLoader(self.dataset, batch_size=cfg.store_batch_size, shuffle=shuffle_data, num_workers=getattr(cfg, "num_workers", 0),
                            drop_last=False)
        n_layers = len(self._layers())
        shard = _ShardWriter(cfg.cached_activations_path, tokens_per_file)
        for batch in loader:
            images = batch[0] if isinstance(batch, (tuple, list)) else batch
            acts = self.get_activations(images.to(cfg.device))              # [b, T, n_layers, d_in]
            if getattr(cfg, "use_patches_only", False):
                acts = acts[:, 1:, :, :]
            shard.add(acts.reshape(-1, n_layers, cfg.d_in).to(torch.float16))
        return shard.close()

    def get_data_loader(self) -> Iterator[Any]:
        half = self.cfg.n_batches_in_buffer // 2
        if self.cfg.is_transcoder:                                   # reference :450-477: both halves shuffled with one permutation
            new_in, new_out = self.get_buffer(half)
            mix_in = torch.cat([new_in, self.storage_buffer], dim=0)
            mix_out = torch.cat([new_out, self.storage_buffer_out], dim=0)
            perm = torch.randperm(mix_in.shape[0], device=mix_in.device)
            mix_in, mix_out = mix_in[perm], mix_out[perm]
            keep = mix_in.shape[0] // 2
            self.storage_buffer, self.storage_buffer_out = mix_in[:keep], mix_out[:keep]
            return _ShuffledServer(torch.cat([mix_in[keep:], mix_out[keep:]], dim=1), self.cfg.train_batch_size)   # [tokens, 2, d]
        mixing = torch.cat([self.get_buffer(half), self.storage_buffer], dim=0)
        mixing = mixing[torch.randperm(mixing.shape[0], device=mixing.device)]
        keep = mixing.shape[0] // 2
        self.storage_buffer = mixing[:keep]
        return _ShuffledServer(mixing[keep:], self.cfg.train_batch_size)

    def next_batch(self) -> torch.Tensor:
        try:
            return next(self.dataloader)
        except StopIteration:
            self.dataloader = self.get_data_loader()
            return next(self.dataloader)


class _ShardWriter:
    """Cuts a stream of ``[tokens, n_layers, d_in]`` blocks into ``{idx}.pt`` files of exactly ``tokens_per_file`` tokens."""

    def __init__(self, directory: str, tokens_per_file: int):
        self.dir, self.per_file = directory, int(tokens_per_file)
        self.pending: list = []
        self.n_pending = 0
        self.n_files = 0

    def _flush(self, n: int) -> None:
        block = torch.cat(self.pending, dim=0)
        torch.save(block[:n].cpu().contiguous(), os.path.join(self.dir, f"{self.n_files}.pt"))
        self.n_files += 1
        rest = block[n:]
        self.pending, self.n_pending = ([rest], rest.shape[0]) if rest.shape[0] else ([], 0)

    def add(self, block: torch.Tensor) -> None:
        self.pending.append(block)
        self.n_pending += block.shape[0]
        while self.n_pending >= self.per_file:
            self._flush(self.per_file)

    def close(self) -> int:
        if self.n_pending:
            self._flush(self.n_pending)
        return self.n_files


class SyntheticActivationsStore:
    """``next_batch()`` -> ``[train_batch_size, 1, d_in]`` seeded synthetic residual-stream-like activations
    (randn * 2 + per-feature offset: non-zero mean so b_dec init, layer-norm and batch centring all matter, SURVEY 8d).
    Keeps a device-resident pool and serves shuffled windows of it."""

    def __init__(self, cfg, pool_tokens: int = 1 << 18, seed: int = 0, device=None):
        self.cfg = cfg
        dev = torch.device(device) if device is not None else cfg.device
        g = torch.Generator(device="cpu").manual_seed(seed)
        offset = torch.randn(cfg.d_in, generator=g)
        pool = torch.randn(pool_tokens, cfg.d_in, generator=g) * 2.0 + offset
        self.storage_buffer = pool.to(dev).unsqueeze(1)          # [tokens, n_layers=1, d_in]
        self.dataloader = _ShuffledServer(self.storage_buffer, cfg.train_batch_size)

    def next_batch(self) -> torch.Tensor:
        try:
            batch = next(self.dataloader)
        except StopIteration:
            self.dataloader = _ShuffledServer(self.storage_buffer, self.cfg.train_batch_size)
            batch = next(self.dataloader)
        if batch.shape[0] < self.cfg.train_batch_size:            # keep the step shape fixed
            self.dataloader = _ShuffledServer(self.storage_buffer, self.cfg.train_batch_size)
            batch = next(self.dataloader)
        return batch


class CacheVisionActivationStore:
    """Serve pre-computed activation shards from ``cfg.cached_activations_path`` with the reference's half-buffer mixing
    (reference :21-152): ``storage_buffer`` holds half a buffer, every refill concatenates a fresh half-buffer read from disk,
    shuffles, keeps one half and serves the other.  One deliberate difference: the reference restarts at ``0.pt`` on every
    refill (its file cursor is a local variable, :54), so it re-serves the first ``buffer`` tokens forever; here the cursor
    (file index + offset inside the file) persists, walking all shards round-robin."""

    def __init__(self, cfg: Any):
        self.cfg = cfg
        if not cfg.use_cached_activations:
            raise ValueError("CacheVisionActivationStore cannot be initialized with cfg.use_cached_activations = False ")
        self._file_idx, self._file_off, self._file = 0, 0, None
        half = cfg.n_batches_in_buffer // 2
        self.storage_buffer = self.get_buffer(half)
        self.dataloader = self.get_data_loader()

    def _num_layers(self) -> int:
        hp = self.cfg.hook_point_layer
        return len(hp) if isinstance(hp, list) else 1

    def _open(self, idx: int) -> torch.Tensor:
        path = f"{self.cfg.cached_activations_path}/{idx}.pt"
        if not os.path.exists(path):
            if idx == 0:
                raise FileNotFoundError(path)
            return None
        return torch.load(path, map_location=self.cfg.device, weights_only=True)

    def _load_cached_activations(self, total_size, context_size, num_layers, d_in) -> torch.Tensor:
        want = total_size * context_size
        parts, have, gained_since_wrap = [], 0, True
        while have < want:
            if self._file is None:
                self._file = self._open(self._file_idx)
                if self._file is None:                      # past the last shard: start over (a cache smaller than the buffer repeats)
                    if not gained_since_wrap:
                        break
                    self._file_idx, self._file_off, gained_since_wrap = 0, 0, False
                    continue
            take = self._file[self._file_off: self._file_off + (want - have)]
            parts.append(take.to(self.cfg.dtype))
            have += take.shape[0]
            gained_since_wrap = gained_since_wrap or take.shape[0] > 0
            self._file_off += take.shape[0]
            if self._file_off >= self._file.shape[0]:
                self._file, self._file_idx, self._file_off = None, self._file_idx + 1, 0
        if not parts:
            return torch.zeros((0, num_layers, d_in), dtype=self.cfg.dtype, device=self.cfg.device)
        return torch.cat(parts, dim=0)

    def get_buffer(self, n_batches_in_buffer: int) -> torch.Tensor:
        cfg = self.cfg
        return self._load_cached_activations(cfg.store_batch_size * n_batches_in_buffer, cfg.context_size, self._num_layers(), cfg.d_in)

    def get_data_loader(self) -> Iterator[Any]:
        half = self.cfg.n_batches_in_buffer // 2
        mixing = torch.cat([self.get_buffer(half), self.storage_buffer], dim=0)
        mixing = mixing[torch.randperm(mixing.shape[0], device=mixing.device)]
        keep = mixing.shape[0] // 2
        self.storage_buffer = mixing[:keep]
        return _ShuffledServer(mixing[keep:], self.cfg.train_batch_size)

    def next_batch(self) -> torch.Tensor:
        try:
            return next(self.dataloader)
        except StopIteration:
            self.dataloader = self.get_data_loader()
            return next(self.dataloader)
