"""Per-graph equivariant normalisation (drop-in for ``EquivariantGraphNorm``, ``nets/graph_norm.py:9-134``).

Per irreps entry ``[N, mul, 2l+1]`` and graph of the batch: 0e entries subtract the graph's channel mean times the
learned ``mean_shift``; every entry is scaled by ``(mean over the graph's nodes of the component-mean square (or
squared norm, ``normalization='norm'``) + eps)^-1/2`` times ``affine_weight``; 0e entries add ``affine_bias``.
``reduce='max'`` takes the largest square instead of the mean.  ``state_dict`` keys ``mean_shift`` / ``affine_weight``
/ ``affine_bias``.

The affine 'mean' norm of at most 8 entries runs on the kernels of ``libeqf_b200_norm.so`` (``ops.SegmentNorm``) for
CUDA fp32 inputs, in the e3nn layout and on the planar blocks the transformer blocks keep; everything else runs the
torch statement ``ops.segment_norm_torch``.
"""
from __future__ import annotations

import torch
from torch import nn

from .. import ops
from ..norm_kernels import SegNormLayout
from ..o3 import Irreps


class EquivariantGraphNorm(nn.Module):
    _mean_shift = True

    def __init__(self, irreps, eps=1e-5, affine=True, reduce="mean", normalization="component"):
        super().__init__()
        self.irreps = Irreps(irreps)
        self.eps = eps
        self.affine = affine
        num_scalar = sum(mul for mul, ir in self.irreps if ir.l == 0 and ir.p == 1)
        if self._mean_shift:
            self.mean_shift = nn.Parameter(torch.ones(num_scalar))
        if affine:
            self.affine_weight = nn.Parameter(torch.ones(self.irreps.num_irreps))
            self.affine_bias = nn.Parameter(torch.zeros(num_scalar))
        else:
            self.register_parameter("affine_weight", None)
            self.register_parameter("affine_bias", None)
        assert isinstance(reduce, str), "reduce should be passed as a string value"
        assert reduce in ["mean", "max"], "reduce needs to be 'mean' or 'max'"
        self.reduce = reduce
        assert normalization in ["norm", "component"], "normalization needs to be 'norm' or 'component'"
        self.normalization = normalization
        self._layout = SegNormLayout([(mul, ir.dim, ir.l == 0 and ir.p == 1) for mul, ir in self.irreps], eps,
                                     normalization == "component")

    def __repr__(self) -> str:
        return f"{self.__class__.__name__} ({self.irreps}, eps={self.eps})"

    @property
    def supports_planar(self) -> bool:
        return True

    def _args(self):
        return self.affine_weight, self.affine_bias, (self.mean_shift if self._mean_shift else None)

    @staticmethod
    def _batch(batch, n_graphs, like):
        """``batch=None``: every node belongs to one graph (as ``global_mean_pool`` reads a missing ``batch``)."""
        if batch is not None:
            return batch, n_graphs
        return torch.zeros(like.shape[0], dtype=torch.int64, device=like.device), 1

    def planar(self, xs, batch=None, n_graphs=None, graph_ptr=None, **kwargs):
        """The same normalisation on planar blocks (one ``[N, 2l+1, mul]`` tensor per irreps entry); ``graph_ptr`` (the
        first node of each graph, ``[n_graphs + 1]``) is built from ``batch`` when not given."""
        if batch is None:
            graph_ptr = None
        batch, n_graphs = self._batch(batch, n_graphs, xs[0])
        seg = ops.GraphSegments(batch, n_graphs, graph_ptr)
        return ops.segment_norm_planar(self._layout, list(xs), seg, *self._args(), reduce=self.reduce)

    def forward(self, node_input, batch=None, **kwargs):
        x = node_input
        if x.shape[-1] != self.irreps.dim:
            raise AssertionError(f"`ix` should have reached node_input.size(-1) ({x.shape[-1]}), "
                                 f"but it ended at {self.irreps.dim}")
        if ops.fused_ok(x) and x.dim() == 2 and self.affine and self.reduce == "mean" and self._layout.c is not None:
            return ops.from_planar(self.planar(ops.to_planar(x, self.irreps), batch, kwargs.get("n_graphs"),
                                               kwargs.get("graph_ptr")))
        batch, n_graphs = self._batch(batch, kwargs.get("n_graphs"), x)
        if n_graphs is None:
            n_graphs = int(batch.max()) + 1 if batch.numel() else 0
        fields, off = [], 0
        for mul, ir in self.irreps:
            fields.append(x.narrow(1, off, mul * ir.dim).reshape(-1, mul, ir.dim))
            off += mul * ir.dim
        out = ops.segment_norm_torch(self._layout, fields, batch, n_graphs, *self._args(), reduce=self.reduce)
        return torch.cat([f.reshape(x.shape[0], -1) for f in out], dim=-1)
