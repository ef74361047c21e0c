"""Radial profile MLP producing the per-edge DTP weights (drop-in for ``nets/radial_func.py``).

``Linear -> LayerNorm -> SiLU`` per hidden width, then ``Linear(no bias) + offset`` (``radial_func.py:9-50``);
``state_dict`` keys ``net.{0,1,3,4,6}.*`` and ``offset`` as in the reference.
"""
from __future__ import annotations

import math

import torch
from torch import nn


def hoist_first_layers(modules, x: torch.Tensor):
    """One GEMM for the FIRST Linear of every radial MLP that reads the same edge scalars.

    The reference evaluates one ``RadialProfile`` MLP per block (``graph_attention_transformer.py:487``) plus the degree
    embedding's on the same ``[E, number_of_basis]`` embedding - 7 per QM9 step: 7 products ``[E, 128] x [128, 64]`` that each
    re-read the input, 7 data-gradient products whose results are summed, 7 weight-gradient reductions over all edges.
    Stacking the weights gives one ``[E, 128] x [128, 7 * 64]`` product each way; the modules pick their column block up in
    ``forward`` (same parameters, same ``state_dict``).  Returns the modules it served.  The QM9 and OC20 steps gain from
    it; the MD17 energy + force step (2 100 edges, second-order graph) got slower, so the MD17 / DeNS models do not hoist."""
    from .. import ops
    if not ops.fused_ok(x) or x.dim() != 2:
        return []
    mods = []
    for m in modules:
        net = list(m.net)
        if (len(net) >= 3 and isinstance(net[0], nn.Linear) and isinstance(net[1], nn.LayerNorm) and isinstance(net[2], nn.SiLU)
                and net[0].in_features == x.shape[1] and net[0].out_features % 4 == 0):
            mods.append(m)
    if len(mods) < 2:
        return []
    W = torch.cat([m.net[0].weight for m in mods], 0)
    pre = ops.split_columns(ops.linear_f32(x, W, None), [m.net[0].out_features for m in mods])
    for m, c in zip(mods, pre):
        m._hoisted = (x, c)
    return mods


def clear_hoisted(mods) -> None:
    for m in mods:
        m._hoisted = None


class RadialProfile(nn.Module):
    def __init__(self, ch_list, use_layer_norm: bool = True, use_offset: bool = True):
        super().__init__()
        layers = []
        last = len(ch_list) - 1
        for i in range(1, len(ch_list)):
            is_last = i == last
            layers.append(nn.Linear(ch_list[i - 1], ch_list[i], bias=not (is_last and use_offset)))
            if is_last:
                break
            if use_layer_norm:
                layers.append(nn.LayerNorm(ch_list[i]))
            layers.append(nn.SiLU())
        self.net = nn.Sequential(*layers)
        self.offset = None
        if use_offset:
            self.offset = nn.Parameter(torch.zeros(ch_list[-1]))
            fan_in = ch_list[-2]
            bound = 1.0 / math.sqrt(fan_in) if fan_in > 0 else 0.0
            nn.init.uniform_(self.offset, -bound, bound)

    def forward(self, f_in, add_offset: bool = True):
        """``add_offset=False`` returns the MLP output without ``offset``: the caller hands ``self.offset`` to the
        tensor-product kernel, which adds it while loading the weights (no extra pass over ``[E, weight_numel]``)."""
        from .. import ops
        out = f_in
        mods = list(self.net)    # same modules / state_dict keys as nn.Sequential; executed with fused kernels on CUDA
        i = 0
        hoisted = getattr(self, "_hoisted", None)
        if hoisted is not None:
            self._hoisted = None
            if hoisted[0] is f_in:      # the first Linear (without bias) was computed with the other MLPs' (hoist_first_layers)
                nxt = mods[1]
                out = ops.ln_silu(hoisted[1], nxt.weight, nxt.bias, nxt.eps, bias=mods[0].bias)
                i = 3
        while i < len(mods):
            m = mods[i]
            nxt = mods[i + 1] if i + 1 < len(mods) else None
            nxt2 = mods[i + 2] if i + 2 < len(mods) else None
            fuse_ln = (isinstance(nxt, nn.LayerNorm) and isinstance(nxt2, nn.SiLU) and nxt.elementwise_affine
                       and len(nxt.normalized_shape) == 1)
            if isinstance(m, nn.Linear) and fuse_ln:
                # Linear -> LayerNorm -> SiLU: GEMM without bias, then ONE kernel for bias + LayerNorm + SiLU
                out = ops.ln_silu(ops.linear_f32(out, m.weight, None), nxt.weight, nxt.bias, nxt.eps, bias=m.bias)
                i += 3
            elif isinstance(m, nn.Linear):
                out = ops.linear_f32(out, m.weight, m.bias)
                i += 1
            elif isinstance(m, nn.LayerNorm) and isinstance(nxt, nn.SiLU) and m.elementwise_affine \
                    and len(m.normalized_shape) == 1:
                out = ops.ln_silu(out, m.weight, m.bias, m.eps)      # LayerNorm + SiLU in one pass
                i += 2
            else:
                out = m(out)
                i += 1
        if self.offset is not None and add_offset:
            out = ops.add_bias(out, self.offset)
        return out
