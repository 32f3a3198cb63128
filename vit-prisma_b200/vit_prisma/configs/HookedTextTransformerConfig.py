"""HookedTextTransformerConfig -- HookedViTConfig plus the text tower's context length and vocabulary
(reference: src/vit_prisma/configs/HookedTextTransformerConfig.py).  The two fields follow every HookedViTConfig field, as
the reference's dataclass subclass appends them."""
from __future__ import annotations

from dataclasses import field, make_dataclass

from vit_prisma.configs.HookedViTConfig import HookedViTConfig


def _n_tokens(self) -> int:
    return self.context_length


HookedTextTransformerConfig = make_dataclass(
    "HookedTextTransformerConfig",
    [("context_length", int, field(default=77)), ("vocab_size", int, field(default=10_000))],
    bases=(HookedViTConfig,),
    namespace={
        "__doc__": "Hyper-parameters of a HookedTextTransformer: a HookedViTConfig with context_length and vocab_size.",
        "n_tokens": property(_n_tokens),
    },
)
HookedTextTransformerConfig.__module__ = __name__
