"""Activation names understood by the H100 ops (reference models/activation_fns.py:19-57, mlp.py:41-62).

The closed forms are evaluated inside the CUDA kernels (csrc/common.cuh ``apply_act``); this module
only maps ``HookedViTConfig.activation_name`` to the kernel's activation code and implements
``solu`` (x * softmax(x)), which is a row op rather than an element-wise one.
"""
from __future__ import annotations

import torch

from vit_prisma.b200 import ops

ELEMENTWISE = ("relu", "gelu", "silu", "gelu_new", "gelu_fast", "quick_gelu")


def _unary(name):
    def fn(x: torch.Tensor) -> torch.Tensor:
        return ops.activation(x, name)
    fn.__name__ = name
    return fn


relu, gelu, silu = _unary("relu"), _unary("gelu"), _unary("silu")
gelu_new, gelu_fast, quick_gelu = _unary("gelu_new"), _unary("gelu_fast"), _unary("quick_gelu")


def solu(x: torch.Tensor) -> torch.Tensor:
    return ops.mul(x, ops.softmax_rows(x))


BY_NAME = {"relu": relu, "gelu": gelu, "silu": silu, "gelu_new": gelu_new, "gelu_fast": gelu_fast,
           "quick_gelu": quick_gelu, "solu_ln": solu}
