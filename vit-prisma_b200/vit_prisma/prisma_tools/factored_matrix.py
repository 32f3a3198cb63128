"""FactoredMatrix -- low-rank product ``A @ B`` kept in factored form.

Analysis-side utility (reference src/vit_prisma/prisma_tools/factored_matrix.py:22-245,
out of the H100 hot-path scope, SURVEY #22); provided so ``Attention.OV`` /
``Attention.QK`` and ``HookedViT.fold_value_biases``-style post-processing keep
working.  Plain PyTorch -- it never touches the activation path.
"""
from __future__ import annotations

from functools import cached_property
from typing import Union

import torch


class FactoredMatrix:
    def __init__(self, A: torch.Tensor, B: torch.Tensor):
        if A.size(-1) != B.size(-2):
            raise ValueError(f"inner dims differ: {tuple(A.shape)} @ {tuple(B.shape)}")
        self.A, self.B = A, B
        self.ldim, self.mdim, self.rdim = A.size(-2), A.size(-1), B.size(-1)
        self.has_leading_dims = A.ndim > 2 or B.ndim > 2
        self.shape = torch.broadcast_shapes(A.shape[:-2], B.shape[:-2]) + (self.ldim, self.rdim)
        self.A = A.broadcast_to(self.shape[:-2] + (self.ldim, self.mdim))
        self.B = B.broadcast_to(self.shape[:-2] + (self.mdim, self.rdim))

    # -- products ------------------------------------------------------------
    def __matmul__(self, other: Union[torch.Tensor, "FactoredMatrix"]):
        if isinstance(other, FactoredMatrix):
            return (self @ other.A) @ other.B
        if other.ndim < 2:  # vector on the right
            return (self.A @ (self.B @ other.unsqueeze(-1))).squeeze(-1)
        if self.rdim > self.mdim:
            return FactoredMatrix(self.A, self.B @ other)
        return FactoredMatrix(self.AB, other)

    def __rmatmul__(self, other: Union[torch.Tensor, "FactoredMatrix"]):
        if isinstance(other, FactoredMatrix):
            return other.A @ (other.B @ self)
        if other.ndim < 2:  # vector on the left
            return ((other.unsqueeze(-2) @ self.A) @ self.B).squeeze(-2)
        if self.ldim > self.mdim:
            return FactoredMatrix(other @ self.A, self.B)
        return FactoredMatrix(other, self.AB)

    def __mul__(self, scalar):
        return FactoredMatrix(self.A * scalar, self.B)

    __rmul__ = __mul__

    @property
    def AB(self) -> torch.Tensor:
        return self.A @ self.B

    @property
    def BA(self) -> torch.Tensor:
        assert self.ldim == self.rdim, "BA needs a square product"
        return self.B @ self.A

    @property
    def T(self) -> "FactoredMatrix":
        return FactoredMatrix(self.B.transpose(-2, -1), self.A.transpose(-2, -1))

    # -- spectra -------------------------------------------------------------
    @cached_property
    def _svd(self):
        Ua, Sa, Vha = torch.linalg.svd(self.A, full_matrices=False)
        Ub, Sb, Vhb = torch.linalg.svd(self.B, full_matrices=False)
        mid = Sa[..., :, None] * (Vha @ Ub) * Sb[..., None, :]
        Um, Sm, Vhm = torch.linalg.svd(mid, full_matrices=False)
        return Ua @ Um, Sm, (Vhm @ Vhb).transpose(-2, -1)

    def svd(self):
        """(U, S, Vh) with ``U @ diag(S) @ Vh.T == AB``; Vh is returned un-transposed like the reference."""
        return self._svd

    @property
    def U(self):
        return self._svd[0]

    @property
    def S(self):
        return self._svd[1]

    @property
    def Vh(self):
        return self._svd[2]

    @property
    def eigenvalues(self):
        return torch.linalg.eig(self.BA).eigenvalues

    # -- misc ----------------------------------------------------------------
    def __getitem__(self, idx):
        idx = idx if isinstance(idx, tuple) else (idx,)
        lead = len(self.shape) - 2
        if len(idx) <= lead:
            return FactoredMatrix(self.A[idx], self.B[idx])
        if len(idx) == lead + 1:
            return FactoredMatrix(self.A[idx], self.B[idx[:-1]])
        a_idx = idx[:-1]
        b_idx = idx[:-2] + (slice(None), idx[-1])
        return FactoredMatrix(self.A[a_idx], self.B[b_idx])

    def norm(self) -> torch.Tensor:
        return self.S.pow(2).sum(-1).sqrt()

    def __repr__(self):
        return f"FactoredMatrix: Shape({self.shape}), Hidden Dim({self.mdim})"

    def make_even(self) -> "FactoredMatrix":
        U, S, Vh = self.svd()
        root = S.sqrt()
        return FactoredMatrix(U * root[..., None, :], root[..., :, None] * Vh.transpose(-2, -1))

    def get_corner(self, k=3):
        return self.A[..., :k, :] @ self.B[..., :, :k]

    @property
    def ndim(self) -> int:
        return len(self.shape)

    def collapse_l(self):
        return self.S[..., :, None] * self.Vh.transpose(-2, -1)

    def collapse_r(self):
        return self.U * self.S[..., None, :]

    def unsqueeze(self, k: int) -> "FactoredMatrix":
        return FactoredMatrix(self.A.unsqueeze(k), self.B.unsqueeze(k))

    @property
    def pair(self):
        return self.A, self.B
