"""Equivariant layer normalisation with ``F.layer_norm`` on the scalars (drop-in for ``EquivariantLayerNormFast``,
``nets/fast_layer_norm.py:9-85``).

Algebraically the same map as ``EquivariantLayerNormV2``: the 0e entry is centred over its channels and divided by
the square root of the biased variance plus eps (``F.layer_norm``), which is the V2 scale of a ``2l+1 = 1`` entry.  So
the affine 'component' norm of at most 8 entries runs on the same fused kernels (``ops.equivariant_layer_norm`` and
its planar form); the torch statement below is the reference's.  ``state_dict`` keys ``affine_weight`` /
``affine_bias``.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

from .. import ops
from ..o3 import Irreps


class EquivariantLayerNormFast(nn.Module):
    def __init__(self, irreps, eps=1e-5, affine=True, normalization="component"):
        super().__init__()
        self.irreps = Irreps(irreps)
        self.eps = eps
        self.affine = affine
        num_scalar = sum(mul for mul, ir in self.irreps if ir.l == 0 and ir.p == 1)
        if affine:
            self.affine_weight = nn.Parameter(torch.ones(self.irreps.num_irreps))
            self.affine_bias = nn.Parameter(torch.zeros(num_scalar))
        else:
            self.register_parameter("affine_weight", None)
            self.register_parameter("affine_bias", None)
        assert normalization in ["norm", "component"], "normalization needs to be 'norm' or 'component'"
        self.normalization = normalization
        self._layout = None
        if affine and normalization == "component" and len(self.irreps) <= 8:
            self._layout = ops.NormLayout([(mul, ir.dim, ir.l == 0 and ir.p == 1) for mul, ir in self.irreps], eps)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__} ({self.irreps}, eps={self.eps})"

    @property
    def supports_planar(self) -> bool:
        return self._layout is not None

    def planar(self, xs, **kwargs):
        """The same normalisation on planar blocks (one ``[N, 2l+1, mul]`` tensor per irreps entry)."""
        if self._layout is None:
            raise NotImplementedError("planar EquivariantLayerNormFast needs the affine 'component' configuration")
        return ops.equivariant_layer_norm_planar(self._layout, xs, self.affine_weight, self.affine_bias)

    def forward(self, node_input, **kwargs):
        if self._layout is not None and ops.fused_ok(node_input) and node_input.dim() == 2:
            return ops.equivariant_layer_norm(self._layout, node_input, self.affine_weight, self.affine_bias)
        fields, ix, iw, ib = [], 0, 0, 0
        for mul, ir in self.irreps:
            d = ir.dim
            field = node_input.narrow(1, ix, mul * d)
            ix += mul * d
            if ir.l == 0 and ir.p == 1:
                weight = self.affine_weight[iw:iw + mul] if self.affine else None
                bias = self.affine_bias[ib:ib + mul] if self.affine else None
                iw += mul
                ib += mul
                fields.append(F.layer_norm(field, (mul,), weight, bias, self.eps).reshape(-1, mul * d))
                continue
            field = field.reshape(-1, mul, d)
            sq = field.pow(2)
            field_norm = sq.sum(-1) if self.normalization == "norm" else sq.mean(-1)
            field_norm = 1.0 / (field_norm.mean(dim=1, keepdim=True) + self.eps).sqrt()
            if self.affine:
                field_norm = field_norm * self.affine_weight[None, iw:iw + mul]
                iw += mul
            fields.append((field * field_norm.reshape(-1, mul, 1)).reshape(-1, mul * d))
        assert ix == node_input.shape[-1]
        return torch.cat(fields, dim=-1)
