"""Regularisers (drop-in for ``nets/drop.py``): stochastic depth per graph and irrep-wise dropout.

Kept so that the reference's constructors and training mode work unchanged.  ``GraphDropPath`` also hands its per-node
factor to the planar transformer blocks (``TransBlock.forward_planar``) and, given the number of graphs, draws without
a host synchronisation.  (``alpha_drop`` is drawn in ``GraphAttention`` and applied inside the fused attention kernel.)
"""
from __future__ import annotations

import torch
from torch import nn

from ..o3 import Irreps


def drop_path(x, drop_prob: float = 0.0, training: bool = False):
    if drop_prob == 0.0 or not training:
        return x
    keep = 1.0 - drop_prob
    mask = torch.rand((x.shape[0],) + (1,) * (x.ndim - 1), dtype=x.dtype, device=x.device).add_(keep).floor_()
    return x.div(keep) * mask


class DropPath(nn.Module):
    def __init__(self, drop_prob=None):
        super().__init__()
        self.drop_prob = drop_prob

    def forward(self, x):
        return drop_path(x, self.drop_prob, self.training)

    def extra_repr(self) -> str:
        return f"drop_prob={self.drop_prob}"


class GraphDropPath(nn.Module):
    """One keep/drop decision per graph of the batch, broadcast to its nodes."""

    def __init__(self, drop_prob=None):
        super().__init__()
        self.drop_prob = drop_prob

    def forward(self, x, batch, n_graphs=None):
        return x * self.node_scale(x, batch, n_graphs)

    def node_scale(self, x, batch, n_graphs=None):
        """The per-node factor (0 or 1/(1-p), 1 outside training) shaped to broadcast against ``x``.  ``n_graphs`` (the
        number of graphs in the batch) avoids reading ``batch.max()`` on the host, so the draw can be captured in a CUDA
        graph; it makes the same draws."""
        if n_graphs is None:
            n_graphs = int(batch.max()) + 1
        ones = torch.ones((n_graphs,) + (1,) * (x.ndim - 1), dtype=x.dtype, device=x.device)
        return drop_path(ones, self.drop_prob, self.training)[batch]

    def extra_repr(self) -> str:
        return f"drop_prob={self.drop_prob}"


class EquivariantDropout(nn.Module):
    """Drop whole irrep channels (one Bernoulli per channel, shared by its 2l+1 components)."""

    def __init__(self, irreps, drop_prob):
        super().__init__()
        self.irreps = Irreps(irreps)
        self.num_irreps = self.irreps.num_irreps
        self.drop_prob = drop_prob
        self.drop = nn.Dropout(drop_prob, True)

    def forward(self, x):
        if not self.training or self.drop_prob == 0.0:
            return x
        mask = self.drop(torch.ones((x.shape[0], self.num_irreps), dtype=x.dtype, device=x.device))
        pieces, off, moff = [], 0, 0
        for mul, ir in self.irreps:
            blk = x.narrow(-1, off, mul * ir.dim).reshape(-1, mul, ir.dim)
            pieces.append((blk * mask.narrow(-1, moff, mul).unsqueeze(-1)).reshape(-1, mul * ir.dim))
            off += mul * ir.dim
            moff += mul
        return torch.cat(pieces, dim=-1)


class EquivariantScalarsDropout(nn.Module):
    def __init__(self, irreps, drop_prob):
        super().__init__()
        self.irreps = Irreps(irreps)
        self.drop_prob = drop_prob

    def forward(self, x):
        if not self.training or self.drop_prob == 0.0:
            return x
        pieces, off = [], 0
        for mul, ir in self.irreps:
            chunk = x.narrow(-1, off, mul * ir.dim)
            off += mul * ir.dim
            if ir.is_scalar():
                chunk = nn.functional.dropout(chunk, p=self.drop_prob, training=self.training)
            pieces.append(chunk)
        return torch.cat(pieces, dim=-1)

    def extra_repr(self) -> str:
        return f"irreps={self.irreps}, drop_prob={self.drop_prob}"
