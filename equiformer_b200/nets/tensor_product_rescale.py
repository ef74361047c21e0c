"""Drop-in for the reference's ``nets/tensor_product_rescale.py`` (operator boundary, SURVEY.md 8b).

Same classes, constructor arguments, attributes (``.tp``, ``.irreps_*``, ``.slices_sqrt_k``, ``.bias``) and
``state_dict`` keys as the reference; the tensor product underneath is
:class:`equiformer_b200.o3.TensorProduct`, i.e. the sm_90a depth-wise kernels for ``'uvu'`` and planar
per-degree GEMMs for the scalar-``in2`` ``'uvw'`` case.

Behaviour restated from the reference (not copied):
* ``path_normalization='none'`` tensor product (``tensor_product_rescale.py:33-37``);
* at construction, internal weights are scaled by ``1/sqrt(fan_in)`` where ``fan_in`` is accumulated over all
  instructions writing the same output entry (``:84-110``); forward applies no further normalisation;
* one zero-initialised bias per ``0e`` entry of ``irreps_out.simplify()`` when ``bias=True`` (``:72-82``),
  added after the product (``:126-136``).

In addition to the e3nn-layout ``forward`` every class has a ``planar`` entry used by the fused
``GraphAttention`` path, which keeps edge tensors in the channel-innermost layout end to end.
"""
from __future__ import annotations

import collections
from typing import List, Optional, Sequence

import torch

from .. import o3
from .. import ops
from ..o3 import Irreps


def _fan_in(tp: o3.TensorProduct, ins) -> int:
    m1 = tp.irreps_in1[ins.i_in1].mul
    m2 = tp.irreps_in2[ins.i_in2].mul
    table = {"uvw": m1 * m2, "uvu": m2, "uvv": m1, "uuw": m1, "uuu": 1, "uvuv": 1,
             "uvu<v": 1, "u<vw": m1 * (m2 - 1) // 2}
    return table[ins.connection_mode]


class TensorProductRescale(torch.nn.Module):
    def __init__(self, irreps_in1, irreps_in2, irreps_out, instructions, bias=True, rescale=True,
                 internal_weights=None, shared_weights=None, normalization=None):
        super().__init__()
        self.irreps_in1 = Irreps(irreps_in1)
        self.irreps_in2 = Irreps(irreps_in2)
        self.irreps_out = Irreps(irreps_out)
        self.rescale = rescale
        self.use_bias = bias
        self.tp = o3.TensorProduct(self.irreps_in1, self.irreps_in2, self.irreps_out, instructions,
                                   normalization=normalization, internal_weights=internal_weights,
                                   shared_weights=shared_weights, path_normalization="none")
        self.init_rescale_bias()

    def calculate_fan_in(self, ins) -> int:
        return _fan_in(self.tp, ins)

    def init_rescale_bias(self) -> None:
        out = self.irreps_out
        self.irreps_out_orders = [ir.l for _, ir in out]
        self.irreps_out_dims = [mul for mul, _ in out]
        self.irreps_out_slices = out.slices()

        simplified = out.simplify()
        self.irreps_bias = simplified
        self.irreps_bias_orders = [ir.l for _, ir in simplified]
        self.irreps_bias_parity = ["e" if ir.p == 1 else "o" for _, ir in simplified]
        self.irreps_bias_dims = [mul for mul, _ in simplified]
        self.bias_slices, self.bias_slice_idx = [], []
        params = []
        if self.use_bias:
            dtype = self.tp.weight.dtype
            for idx, ((mul, ir), sl) in enumerate(zip(simplified, simplified.slices())):
                if ir.l == 0 and ir.p == 1:
                    params.append(torch.nn.Parameter(torch.zeros(mul, dtype=dtype)))
                    self.bias_slices.append(sl)
                    self.bias_slice_idx.append(idx)
        self.bias = torch.nn.ParameterList(params)

        fan = collections.defaultdict(int)
        for ins in self.tp.instructions:
            fan[ins.i_out] += _fan_in(self.tp, ins)
        self.slices_sqrt_k = {}
        for ins in self.tp.instructions:
            k = fan[ins.i_out] ** -0.5 if self.rescale else 1.0
            self.slices_sqrt_k[ins.i_out] = (self.irreps_out_slices[ins.i_out], k)
        if self.tp.internal_weights and self.rescale:
            with torch.no_grad():
                for view, ins in zip(self.tp.weight_views(), [i for i in self.tp.instructions if i.has_weight]):
                    view.mul_(fan[ins.i_out] ** -0.5)

        # planar bookkeeping: which bias (and channel offset) feeds each irreps_out entry
        self._entry_bias = []
        run_idx, run_off, prev = -1, 0, None
        bias_of_run = {idx: b for b, idx in enumerate(self.bias_slice_idx)}
        for mul, ir in out:
            if prev is None or ir != prev:
                run_idx, run_off, prev = run_idx + 1, 0, ir
            self._entry_bias.append((bias_of_run.get(run_idx), run_off))
            run_off += mul

    # ------------------------------------------------------------------ e3nn layout
    def forward_tp_rescale_bias(self, x, y, weight=None):
        out = self.tp(x, y, weight)
        if self.use_bias and len(self.bias) > 0:
            pieces, pos = [], 0
            for sl, b in zip(self.bias_slices, self.bias):
                if sl.start > pos:
                    pieces.append(out.narrow(-1, pos, sl.start - pos))
                pieces.append(out.narrow(-1, sl.start, sl.stop - sl.start) + b)
                pos = sl.stop
            if pos < out.shape[-1]:
                pieces.append(out.narrow(-1, pos, out.shape[-1] - pos))
            out = torch.cat(pieces, dim=-1) if len(pieces) > 1 else pieces[0]
        return out

    def forward(self, x, y, weight=None):
        return self.forward_tp_rescale_bias(x, y, weight)

    # ------------------------------------------------------------------ planar layout
    def _planar_bias(self, outs: List[torch.Tensor]) -> List[torch.Tensor]:
        if not (self.use_bias and len(self.bias) > 0):
            return outs
        res = []
        for t, (b_idx, off) in zip(outs, self._entry_bias):
            if b_idx is not None:
                t = ops.add_bias(t, self.bias[b_idx].narrow(0, off, t.shape[-1]))
            res.append(t)
        return res

    def planar(self, xs: Sequence[torch.Tensor], y: Optional[torch.Tensor] = None, weight=None):
        """Planar forward.  Depth-wise kind: in1 blocks -> output *groups*; linear kind: entries -> entries."""
        if self.tp._kind == "depthwise":
            if self.use_bias and len(self.bias) > 0:
                raise NotImplementedError("bias on a depth-wise product is unused by the reference (bias=False)")
            return self.tp.planar_depthwise(xs, y, weight)
        return self._planar_bias(self.tp.planar_linear(xs, y, weight))


class FullyConnectedTensorProductRescale(TensorProductRescale):
    def __init__(self, irreps_in1, irreps_in2, irreps_out, bias=True, rescale=True,
                 internal_weights=None, shared_weights=None, normalization=None):
        irreps_in1, irreps_in2, irreps_out = Irreps(irreps_in1), Irreps(irreps_in2), Irreps(irreps_out)
        instructions = []
        for i1, (_, ir1) in enumerate(irreps_in1):
            for i2, (_, ir2) in enumerate(irreps_in2):
                allowed = ir1 * ir2
                for io, (_, iro) in enumerate(irreps_out):
                    if iro in allowed:
                        instructions.append((i1, i2, io, "uvw", True, 1.0))
        super().__init__(irreps_in1, irreps_in2, irreps_out, instructions, bias=bias, rescale=rescale,
                         internal_weights=internal_weights, shared_weights=shared_weights,
                         normalization=normalization)


class LinearRS(FullyConnectedTensorProductRescale):
    """Equivariant linear map: FCTP against the constant scalar 1."""

    def __init__(self, irreps_in, irreps_out, bias=True, rescale=True):
        super().__init__(irreps_in, Irreps("1x0e"), irreps_out, bias=bias, rescale=rescale,
                         internal_weights=True, shared_weights=True, normalization=None)

    def forward(self, x):
        return self.forward_tp_rescale_bias(x, torch.ones_like(x[:, 0:1]))

    def planar(self, xs, y=None, weight=None):
        return self._planar_bias(self.tp.planar_linear(xs, None, weight))


def irreps2gate(irreps):
    """Split ``irreps`` into (scalars 0e, one 0e gate per gated channel, gated non-scalars)."""
    scalars, gated = [], []
    for mul, ir in Irreps(irreps):
        (scalars if ir.l == 0 and ir.p == 1 else gated).append((mul, ir))
    irreps_scalars = Irreps(scalars).simplify()
    irreps_gated = Irreps(gated).simplify()
    gate_ir = "0e" if irreps_gated.dim > 0 else None
    irreps_gates = Irreps([(mul, gate_ir) for mul, _ in irreps_gated]).simplify()
    return irreps_scalars, irreps_gates, irreps_gated


class FullyConnectedTensorProductRescaleSwishGate(FullyConnectedTensorProductRescale):
    """FCTP followed by SiLU on scalars / sigmoid gates on the rest (``graph_attention_transformer.py:128-154``)."""

    def __init__(self, irreps_in1, irreps_in2, irreps_out, bias=True, rescale=True,
                 internal_weights=None, shared_weights=None, normalization=None):
        from .fast_activation import Activation, Gate
        irreps_scalars, irreps_gates, irreps_gated = irreps2gate(irreps_out)
        if irreps_gated.num_irreps == 0:
            gate = Activation(irreps_out, acts=[torch.nn.SiLU()])
        else:
            gate = Gate(irreps_scalars, [torch.nn.SiLU() for _ in irreps_scalars],
                        irreps_gates, [torch.sigmoid for _ in irreps_gates], irreps_gated)
        super().__init__(irreps_in1, irreps_in2, gate.irreps_in, bias=bias, rescale=rescale,
                         internal_weights=internal_weights, shared_weights=shared_weights,
                         normalization=normalization)
        self.gate = gate

    def forward(self, x, y, weight=None):
        return self.gate(self.forward_tp_rescale_bias(x, y, weight))


def sort_irreps_even_first(irreps):
    """Stable sort by degree with even parity before odd (the reference's replacement for ``Irreps.sort``)."""
    Ret = collections.namedtuple("sort", ["irreps", "p", "inv"])
    irreps = Irreps(irreps)
    keyed = sorted((ir.l, -ir.p, i, mul) for i, (mul, ir) in enumerate(irreps))
    inv = tuple(i for _, _, i, _ in keyed)
    p = [0] * len(inv)
    for new, old in enumerate(inv):
        p[old] = new
    return Ret(Irreps([(mul, (l, -negp)) for l, negp, _, mul in keyed]), tuple(p), inv)
