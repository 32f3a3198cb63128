"""K-major weight packs for the GEMM engines, cached per parameter version.

The reference stores attention weights head-major (``W_Q [H, d_model, d_head]``,
``W_O [H, d_head, d_model]``; models/layers/attention.py:37-80) and MLP/head weights input-major
(``W_in [d_model, d_mlp]``; mlp.py:25-36, head.py:19-24).  wgmma wants both operands K-major, so
each weight gets a packed ``[N, K]`` shadow copy (plus the tf32 residual ``lo`` in fp32 mode).
Packs are rebuilt when a parameter's ``_version`` or storage changes (optimizer step,
``load_state_dict``, ``.to()``), so the nn.Parameters stay the single source of truth.
Re-layout is data movement (permute/contiguous); the tf32 split runs through pb_split_tf32.
"""
from __future__ import annotations

from typing import Callable, Dict, Tuple

import torch

from . import ops


def _stamp(*params: torch.Tensor) -> Tuple:
    return tuple((p.data_ptr(), p._version, p.dtype, p.device) for p in params)


class PackCache:
    """Attach one to a module; ``get(name, params, builder)`` memoises ``builder()`` on the params' stamps."""

    def __init__(self):
        self._store: Dict[str, Tuple[Tuple, object]] = {}

    def get(self, name: str, params, builder: Callable[[], object]):
        stamp = _stamp(*params)
        hit = self._store.get(name)
        if hit is not None and hit[0] == stamp:
            return hit[1]
        with torch.no_grad():
            value = builder()
        self._store[name] = (stamp, value)
        return value

    def clear(self) -> None:
        self._store.clear()


def with_lo(w: torch.Tensor):
    """(w, lo) where lo is the tf32 residual for fp32 weights on CUDA, else (w, None)."""
    if w.dtype == torch.float32 and w.is_cuda:
        return w, ops.split_tf32(w)
    return w, None


def pack_heads_nk(w_hde: torch.Tensor) -> torch.Tensor:
    """[H, d_model, d_head] -> [H*d_head, d_model] (row h*dh+e holds W[h, :, e])."""
    H, d, dh = w_hde.shape
    return w_hde.detach().permute(0, 2, 1).reshape(H * dh, d).contiguous()


def pack_out_nk(w_o: torch.Tensor) -> torch.Tensor:
    """W_O [H, d_head, d_model] -> [d_model, H*d_head]."""
    H, dh, d = w_o.shape
    return w_o.detach().reshape(H * dh, d).t().contiguous()


def pack_t(w_kn: torch.Tensor) -> torch.Tensor:
    """[K, N] -> [N, K]."""
    return w_kn.detach().t().contiguous()
