"""HookPoint -- the identity module every cached activation flows through.

Behavioural contract taken from reference src/vit_prisma/prisma_tools/hook_point.py:16-112:

* identity on its input; forward hooks are called as ``hook(tensor, hook=self)``
  and a non-``None`` return value *replaces* the activation for downstream code;
* ``fwd_hooks`` / ``bwd_hooks`` are public lists of ``LensHandle``;
* ``add_hook(hook, dir, is_permanent, level, prepend)``, ``add_perma_hook``,
  ``remove_hooks(dir, including_permanent, level)``, ``clear_context``, ``layer()``.

H100 notes.  On the fused fast path (``HookedViT.run_with_cache`` with nothing
but the internal save-hook attached) HookPoints are never *called*: the CUDA
chain writes every requested activation straight into the cache arena and the
Python side only builds the key -> view dictionary.  On the per-op hooked path
they are called ~260x per forward, so ``__call__`` short-circuits past
``nn.Module._call_impl`` when nothing is registered (``is_inert``).
``is_inert`` is also what the fast-path eligibility check reads.
"""
from __future__ import annotations

from typing import Callable, List

import torch.nn as nn
from torch.nn.modules import module as _torch_module

from vit_prisma.prisma_tools.lens_handle import LensHandle


def _global_module_hooks_present() -> bool:
    m = _torch_module
    return bool(
        m._global_forward_hooks
        or m._global_forward_pre_hooks
        or m._global_backward_hooks
        or m._global_backward_pre_hooks
    )


class HookPoint(nn.Module):
    def __init__(self):
        super().__init__()
        self.fwd_hooks: List[LensHandle] = []
        self.bwd_hooks: List[LensHandle] = []
        self.ctx = {}
        # filled in by HookedRootModule.setup()
        self.name = None

    # ------------------------------------------------------------------ state
    @property
    def is_inert(self) -> bool:
        """True when calling this module cannot run any user code."""
        return not (
            self._forward_hooks
            or self._forward_pre_hooks
            or self._backward_hooks
            or self._backward_pre_hooks
        )

    def __call__(self, x):
        if self.is_inert and not _global_module_hooks_present():
            return x
        return super().__call__(x)

    def forward(self, x):
        return x

    # ------------------------------------------------------------- attachment
    def add_perma_hook(self, hook: Callable, dir: str = "fwd") -> None:
        self.add_hook(hook, dir=dir, is_permanent=True)

    def add_hook(self, hook: Callable, dir: str = "fwd", is_permanent: bool = False,
                 level=None, prepend: bool = False) -> None:
        """Attach ``hook``; with ``prepend`` it runs before every hook already present."""
        point = self
        if dir == "fwd":
            def adapter(_module, _inputs, output):
                return hook(output, hook=point)
            registry, records = self._forward_hooks, self.fwd_hooks
            torch_handle = self.register_forward_hook(adapter)
        elif dir == "bwd":
            def adapter(_module, _grad_in, grad_out):
                return hook(grad_out[0], hook=point)
            registry, records = self._backward_hooks, self.bwd_hooks
            torch_handle = self.register_full_backward_hook(adapter)
        else:
            raise ValueError(f"Invalid dir {dir}. dir must be 'fwd' or 'bwd'")
        adapter.__name__ = repr(hook)

        record = LensHandle(torch_handle, is_permanent, level)
        if prepend:
            registry.move_to_end(torch_handle.id, last=False)
            records.insert(0, record)
        else:
            records.append(record)

    # -------------------------------------------------------------- detachment
    def remove_hooks(self, dir: str = "fwd", including_permanent: bool = False, level=None) -> None:
        if dir not in ("fwd", "bwd", "both"):
            raise ValueError(f"Invalid direction {dir}. dir must be 'fwd', 'bwd', or 'both'")

        def sweep(records: List[LensHandle]) -> List[LensHandle]:
            survivors = []
            for rec in records:
                doomed = including_permanent or (
                    not rec.is_permanent and (level is None or rec.context_level == level)
                )
                if doomed:
                    rec.hook.remove()
                else:
                    survivors.append(rec)
            return survivors

        # NB: the reference's ``dir == "both"`` only ever sweeps the forward list
        # (hook_point.py:92-95, an if/elif); backward hooks are swept here as well
        # since leaving them attached is never what a caller of "both" wants.
        if dir in ("fwd", "both"):
            self.fwd_hooks = sweep(self.fwd_hooks)
        if dir in ("bwd", "both"):
            self.bwd_hooks = sweep(self.bwd_hooks)

    def clear_context(self) -> None:
        self.ctx = {}

    def layer(self) -> int:
        """Block index for names shaped like ``blocks.{layer}.<...>``."""
        return int(self.name.split(".")[1])
