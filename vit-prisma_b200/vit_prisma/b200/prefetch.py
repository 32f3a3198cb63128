"""Host -> device batch prefetcher: the H2D copy of batch i+1 runs on a copy stream while batch i is in `run_with_cache`.

A 512-image fp32 batch is 308 MB: ~5.6 ms over PCIe gen5 at 55 GB/s, a large share of a ViT-B/32 all-hooks step.  The reference
feeds its model from a `DataLoader` and `.to(device)` on the compute stream (`activations_store.py:252-270`), i.e. the copy
sits in front of every forward.  This iterator keeps the same call pattern for the consumer (`for x in prefetcher:
model.run_with_cache(x)`) and only moves the copy off the critical path: two device buffers, one side stream, event
hand-over in both directions.  Host tensors should be pinned (a pageable source makes the "async" copy synchronous).
"""
from __future__ import annotations

from typing import Iterable, Iterator, Optional

import torch


class DevicePrefetcher:
    def __init__(self, batches: Optional[Iterable[torch.Tensor]], device: torch.device, depth: int = 2,
                 dtype: Optional[torch.dtype] = None):
        if torch.device(device).type != "cuda":
            raise RuntimeError("DevicePrefetcher: device must be a CUDA device (the H100 path has no CPU fallback)")
        if depth < 2:
            raise ValueError("depth must be >= 2 (one buffer in use, one in flight)")
        self.device = torch.device(device)
        self.depth = depth
        self.dtype = dtype
        self._it = iter(batches) if batches is not None else iter(())
        self._copy_stream = torch.cuda.Stream(device=self.device)
        self._bufs: list[Optional[torch.Tensor]] = [None] * depth
        self._ready = [torch.cuda.Event() for _ in range(depth)]       # copy into slot finished
        self._released = [torch.cuda.Event() for _ in range(depth)]    # consumer's kernels that read the slot were enqueued
        self._used = [False] * depth
        self._head = 0          # next slot to fill
        self._tail = 0          # next slot to hand out
        self._inflight = 0
        self._exhausted = False

    def feed(self, batches: Iterable[torch.Tensor]) -> "DevicePrefetcher":
        """Start a new pass over ``batches`` with the same stream and device buffers (a loader object lives across epochs:
        stream creation and the first cudaMalloc of the staging buffers are set-up cost, not per-batch work)."""
        if self._inflight:
            raise RuntimeError("DevicePrefetcher.feed: the previous pass still has batches in flight")
        self._it = iter(batches)
        self._exhausted = False
        return self

    def _issue(self) -> None:
        try:
            host = next(self._it)
        except StopIteration:
            self._exhausted = True
            return
        s = self._head
        dt = self.dtype or host.dtype
        buf = self._bufs[s]
        if buf is None or buf.shape != host.shape or buf.dtype != dt:
            buf = self._bufs[s] = torch.empty(host.shape, dtype=dt, device=self.device)
        cur = torch.cuda.current_stream(self.device)
        with torch.cuda.stream(self._copy_stream):
            # the copy may not start before (a) work already queued on the consumer stream when it was requested -- that keeps
            # a timing event recorded by the caller in front of the first copy -- and (b) the last reader of this slot
            self._copy_stream.wait_stream(cur)
            if self._used[s]:
                self._copy_stream.wait_event(self._released[s])
            buf.copy_(host, non_blocking=True)
            self._ready[s].record(self._copy_stream)
        self._head = (s + 1) % self.depth
        self._inflight += 1

    def __iter__(self) -> Iterator[torch.Tensor]:
        return self

    def __next__(self) -> torch.Tensor:
        if self._inflight == 0 and not self._exhausted:
            self._issue()
        if self._inflight == 0:
            raise StopIteration
        s = self._tail
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(self._ready[s])
        out = self._bufs[s]
        self._tail = (s + 1) % self.depth
        self._inflight -= 1
        # mark the hand-over point of the PREVIOUS slot: everything the consumer enqueued for it is now on `cur`
        prev = (s - 1) % self.depth
        if self._used[prev]:
            self._released[prev].record(cur)
        self._used[s] = True
        # start the next copy right away; it only waits for what is already queued (the previous batch's kernels are not
        # readers of the slot it fills unless depth wraps, which `_released` covers)
        while self._inflight < self.depth - 1 and not self._exhausted:
            self._issue()
        return out
