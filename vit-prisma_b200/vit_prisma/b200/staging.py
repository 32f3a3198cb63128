"""Host-resident modules on a GPU-only compute path.

Device policy of this package: every arithmetic operation runs in the sm_90a kernels; there is no CPU compute path.  The reference's
default ``HookedViTConfig.device`` is ``"cpu"`` and its own offline tests build host-resident models / layers and feed host tensors.
Such a module is *staged*: for the duration of one call its parameters and buffers point at cached device copies (refreshed when a
parameter's version counter or storage changes), tensor arguments are copied host -> device, the same CUDA kernels run, and tensor
results are copied back to the caller's device.  Hook functions see device tensors.  Two memcpys around the GPU path -- data
movement, not a fallback: without a CUDA device the call raises ``PrismaB200Error``.
"""
from __future__ import annotations

import contextlib
import functools

import torch

from ._lib import PrismaB200Error


def _move(obj, device):
    if isinstance(obj, torch.Tensor):
        return obj.to(device)
    if isinstance(obj, tuple):
        return tuple(_move(o, device) for o in obj)
    if isinstance(obj, list):
        return [_move(o, device) for o in obj]
    if isinstance(obj, dict):
        return {k: _move(v, device) for k, v in obj.items()}
    return obj


@contextlib.contextmanager
def staged_on_gpu(module: torch.nn.Module):
    """Point every host parameter / buffer of ``module`` at a cached device copy for the duration of the block."""
    if not torch.cuda.is_available():
        raise PrismaB200Error("prisma_b200: this module lives in host memory and no CUDA device is visible -- the hot path is "
                              "hand-written sm_90a CUDA and has no CPU fallback")
    cache = module.__dict__.setdefault("_stage_cache", {})
    swapped = []
    for name, t in list(module.named_parameters()) + list(module.named_buffers()):
        if t.is_cuda:
            continue
        key = (t.data_ptr(), t._version, tuple(t.shape), t.dtype)
        hit = cache.get(name)
        if hit is None or hit[0] != key:
            hit = (key, t.data.to("cuda"))
            cache[name] = hit
        swapped.append((t, t.data))
        t.data = hit[1]
    cfg = getattr(module, "cfg", None)
    prev = getattr(cfg, "device", None)
    if cfg is not None and prev is not None:
        try:
            cfg.device = "cuda"
        except Exception:
            prev = None
    try:
        yield
    finally:
        for t, host in swapped:
            t.data = host
        if cfg is not None and prev is not None:
            cfg.device = prev


def host_resident(module: torch.nn.Module) -> bool:
    p = next(module.parameters(), None)
    if p is None:
        p = next(module.buffers(), None)
    return p is not None and not p.is_cuda


def host_staged(forward):
    """Decorator for ``nn.Module.forward``: host tensor arguments make the call run staged (see the module docstring); calls with
    device tensors -- every call made from inside an already staged parent -- go straight through."""

    @functools.wraps(forward)
    def wrapper(self, *args, **kwargs):
        first = next((a for a in list(args) + list(kwargs.values()) if isinstance(a, torch.Tensor)), None)
        if first is None or first.is_cuda:
            return forward(self, *args, **kwargs)
        if not host_resident(self):                         # device-resident module, host input: one H2D copy, result stays on the device
            dev = next(self.parameters()).device if next(self.parameters(), None) is not None else "cuda"
            return forward(self, *_move(args, dev), **_move(kwargs, dev))
        with staged_on_gpu(self):
            out = forward(self, *_move(args, "cuda"), **_move(kwargs, "cuda"))
        return _move(out, first.device)

    return wrapper
