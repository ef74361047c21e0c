"""Equivariant layer normalisation (drop-in for ``EquivariantLayerNormV2``, ``nets/layer_norm.py:62-152``).

Node-level, O(N*D) work; the affine 'component' case runs as one fused kernel forward and one backward
(``ops.equivariant_layer_norm`` -> ``eqf_eln_fwd/bwd``), everything else as the torch statement below.  Per irreps entry ``[N, mul, 2l+1]``: scalars are
mean-centred over channels; every entry is divided by the RMS over (channels, components)
(``normalization='component'``) or the channel mean of squared norms (``'norm'``), scaled by a per-channel
affine weight; scalars get an affine bias.  ``state_dict`` keys ``affine_weight`` / ``affine_bias``.
"""
from __future__ import annotations

import torch
from torch import nn

from .. import ops
from ..o3 import Irreps


class EquivariantLayerNormV2(nn.Module):
    def __init__(self, irreps, eps: float = 1e-5, affine: bool = True, normalization: str = "component"):
        super().__init__()
        self.irreps = Irreps(irreps)
        self.eps = eps
        self.affine = affine
        n_scalar = sum(mul for mul, ir in self.irreps if ir.l == 0 and ir.p == 1)
        if affine:
            self.affine_weight = nn.Parameter(torch.ones(self.irreps.num_irreps))
            self.affine_bias = nn.Parameter(torch.zeros(n_scalar))
        else:
            self.register_parameter("affine_weight", None)
            self.register_parameter("affine_bias", None)
        if normalization not in ("norm", "component"):
            raise AssertionError("normalization needs to be 'norm' or 'component'")
        self.normalization = normalization
        self._layout = None
        if affine and normalization == "component" and len(self.irreps) <= 8:
            self._layout = ops.NormLayout([(mul, ir.dim, ir.l == 0 and ir.p == 1) for mul, ir in self.irreps], eps)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.irreps}, eps={self.eps})"

    @property
    def supports_planar(self) -> bool:
        return self._layout is not None

    def planar(self, xs, **kwargs):
        """The same normalisation on planar blocks (one ``[N, 2l+1, mul]`` tensor per irreps entry); the per-graph
        arguments the transformer blocks hand every norm (``batch``, ``n_graphs``, ``graph_ptr``) are not used."""
        if self._layout is None:
            raise NotImplementedError("planar LayerNorm needs the affine 'component' configuration")
        return ops.equivariant_layer_norm_planar(self._layout, xs, self.affine_weight, self.affine_bias)

    def forward(self, node_input, **kwargs):
        x = node_input.float() if node_input.dtype in (torch.float16, torch.bfloat16) else node_input
        if x.shape[-1] != self.irreps.dim:
            raise AssertionError(f"`ix` should have reached node_input.size(-1) ({x.shape[-1]}), "
                                 f"but it ended at {self.irreps.dim}")
        if self._layout is not None and x.dim() == 2:
            return ops.equivariant_layer_norm(self._layout, x, self.affine_weight, self.affine_bias)
        out, off, iw, ib = [], 0, 0, 0
        for mul, ir in self.irreps:
            d = ir.dim
            f = x.narrow(1, off, mul * d).reshape(-1, mul, d)
            off += mul * d
            scalar = ir.l == 0 and ir.p == 1
            if scalar:
                f = f - f.mean(dim=1, keepdim=True)
            sq = f.pow(2)
            per_chan = sq.sum(-1) if self.normalization == "norm" else sq.mean(-1)
            scale = (per_chan.mean(dim=1, keepdim=True) + self.eps).pow(-0.5)
            if self.affine:
                scale = scale * self.affine_weight[None, iw:iw + mul]
                iw += mul
            f = f * scale.unsqueeze(-1)
            if self.affine and scalar:
                f = f + self.affine_bias[ib:ib + mul].reshape(mul, 1)
                ib += mul
            out.append(f.reshape(-1, mul * d))
        return torch.cat(out, dim=-1)
