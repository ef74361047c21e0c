"""``o3.TensorProduct`` as far as the Equiformer hot path uses it.

Same constructor surface as ``e3nn.o3.TensorProduct`` (0.4.4) for the two instruction kinds the
reference instantiates through ``TensorProductRescale`` (``nets/tensor_product_rescale.py:33-37``):

* weighted ``'uvu'`` with multiplicity-1 second operand - the depth-wise tensor product; executed by
  the sm_90a kernels in ``csrc/eqf_dtp.cu`` (no other implementation exists here);
* weighted ``'uvw'`` whose second operand is scalar (``1x0e`` node attributes / the constant 1 of
  ``LinearRS``) - a per-degree dense channel mix, executed as row-major GEMMs on planar blocks.

Semantics fixed by the reference: ``irrep_normalization='component'`` (e3nn default),
``path_normalization='none'`` -> each path is scaled by ``sqrt(2 l_out + 1)`` only; flat weights are
consumed in instruction order; default initialisation ``randn``.  ``state_dict`` keys match e3nn's
(``weight``, ``output_mask``) so reference checkpoints load.
"""
from __future__ import annotations

import collections
import math
from typing import List, Optional, Sequence

import torch

from .irreps import Irreps
from .wigner import wigner_3j_np

Instruction = collections.namedtuple(
    "Instruction", ["i_in1", "i_in2", "i_out", "connection_mode", "has_weight", "path_weight", "path_shape"])


def _prod(shape) -> int:
    out = 1
    for s in shape:
        out *= s
    return out


class TensorProduct(torch.nn.Module):
    def __init__(self, irreps_in1, irreps_in2, irreps_out, instructions: Sequence[tuple],
                 in1_var=None, in2_var=None, out_var=None, irrep_normalization: Optional[str] = None,
                 path_normalization: Optional[str] = None, internal_weights: Optional[bool] = None,
                 shared_weights: Optional[bool] = None, normalization: Optional[str] = None, **_ignored):
        super().__init__()
        if normalization is not None:
            irrep_normalization = normalization
        if irrep_normalization is None:
            irrep_normalization = "component"
        if path_normalization is None:
            path_normalization = "element"
        if irrep_normalization not in ("component", "norm", "none"):
            raise ValueError("irrep_normalization must be 'component', 'norm' or 'none'")
        if path_normalization not in ("element", "path", "none"):
            raise ValueError("path_normalization must be 'element', 'path' or 'none'")
        if in1_var is not None or in2_var is not None or out_var is not None:
            raise NotImplementedError("custom variances are outside the Equiformer hot path")
        self.irreps_in1 = Irreps(irreps_in1)
        self.irreps_in2 = Irreps(irreps_in2)
        self.irreps_out = Irreps(irreps_out)

        norm_ins = []
        for ins in instructions:
            ins = tuple(ins)
            if len(ins) == 5:
                ins = ins + (1.0,)
            i1, i2, io, mode, has_weight, pw = ins[:6]
            m1, m2, mo = self.irreps_in1[i1].mul, self.irreps_in2[i2].mul, self.irreps_out[io].mul
            shape = {"uvw": (m1, m2, mo), "uvu": (m1, m2), "uvv": (m1, m2), "uuw": (m1, mo), "uuu": (m1,),
                     "uvuv": (m1, m2)}.get(mode)
            if shape is None:
                raise ValueError(f"unsupported connection mode {mode!r}")
            norm_ins.append(Instruction(i1, i2, io, mode, bool(has_weight), float(pw), shape))

        def num_elements(ins):
            return {"uvw": self.irreps_in1[ins.i_in1].mul * self.irreps_in2[ins.i_in2].mul,
                    "uvu": self.irreps_in2[ins.i_in2].mul, "uvv": self.irreps_in1[ins.i_in1].mul,
                    "uuw": self.irreps_in1[ins.i_in1].mul, "uuu": 1, "uvuv": 1}[ins.connection_mode]

        final = []
        for ins in norm_ins:
            ir1, ir2, iro = self.irreps_in1[ins.i_in1].ir, self.irreps_in2[ins.i_in2].ir, self.irreps_out[ins.i_out].ir
            if iro not in ir1 * ir2:
                raise ValueError(f"instruction {ins} violates the O(3) selection rule")
            alpha = {"component": iro.dim, "norm": ir1.dim * ir2.dim, "none": 1}[irrep_normalization]
            if path_normalization == "element":
                x = sum(num_elements(i) for i in norm_ins if i.i_out == ins.i_out)
            elif path_normalization == "path":
                x = num_elements(ins) * len([i for i in norm_ins if i.i_out == ins.i_out])
            else:
                x = 1
            if x > 0:
                alpha = alpha / x
            alpha = alpha * ins.path_weight
            final.append(ins._replace(path_weight=math.sqrt(alpha)))
        self.instructions: List[Instruction] = final

        if shared_weights is False and internal_weights is None:
            internal_weights = False
        if shared_weights is None:
            shared_weights = True
        if internal_weights is None:
            internal_weights = shared_weights and any(i.has_weight for i in self.instructions)
        if internal_weights and not shared_weights:
            raise ValueError("internal weights must be shared")
        self.internal_weights = internal_weights
        self.shared_weights = shared_weights
        self.weight_numel = sum(_prod(i.path_shape) for i in self.instructions if i.has_weight)
        if internal_weights and self.weight_numel > 0:
            self.weight = torch.nn.Parameter(torch.randn(self.weight_numel))
        else:
            self.register_buffer("weight", torch.Tensor())
        mask = torch.zeros(self.irreps_out.dim)
        for ins in self.instructions:
            if ins.path_weight != 0:
                mask[self.irreps_out.slices()[ins.i_out]] = 1.0
        self.register_buffer("output_mask", mask)

        modes = {i.connection_mode for i in self.instructions}
        self._kind = None
        self._plan = None
        if modes == {"uvu"} and all(i.has_weight for i in self.instructions) and \
                all(mul == 1 for mul, _ in self.irreps_in2):
            self._kind = "depthwise"
        elif modes == {"uvw"} and all(i.has_weight for i in self.instructions) and \
                all(ir.l == 0 and ir.p == 1 for _, ir in self.irreps_in2):
            self._kind = "linear"

    # ------------------------------------------------------------------ weights
    def weight_views(self, weight: Optional[torch.Tensor] = None, yield_instruction: bool = False):
        from .. import ops
        w = self._get_weights(weight)
        batch = w.shape[:-1]
        weighted = [(idx, ins) for idx, ins in enumerate(self.instructions) if ins.has_weight]
        chunks = ops.split_flat(w, [_prod(ins.path_shape) for _, ins in weighted])
        for (idx, ins), chunk in zip(weighted, chunks):
            view = chunk.view(batch + ins.path_shape)
            yield (idx, ins, view) if yield_instruction else view

    def _get_weights(self, weight: Optional[torch.Tensor]) -> torch.Tensor:
        if weight is None:
            if self.weight_numel > 0 and not self.internal_weights:
                raise RuntimeError("Weights must be provided when the TensorProduct does not have internal_weights")
            return self.weight
        if self.shared_weights:
            if weight.shape != (self.weight_numel,):
                raise ValueError(f"Invalid weight shape {tuple(weight.shape)}")
        else:
            if weight.shape[-1] != self.weight_numel or weight.dim() < 2:
                raise ValueError(f"Invalid weight shape {tuple(weight.shape)}")
        return weight

    # ------------------------------------------------------------------ depth-wise plan
    @property
    def plan(self):
        """Path tables for the edge kernels (only for the depth-wise kind)."""
        if self._kind != "depthwise":
            raise NotImplementedError("only the depth-wise ('uvu', mul(in2)=1) tensor product has an edge-kernel plan")
        if self._plan is None:
            from ..plan import DtpPlan
            raw = []
            for ins in self.instructions:
                iro = self.irreps_out[ins.i_out].ir
                # DtpPlan multiplies by ir_out.dim itself; hand it the residual factor
                raw.append((ins.i_in1, ins.i_in2, ins.i_out, ins.connection_mode, ins.has_weight,
                            ins.path_weight ** 2 / iro.dim))
            self._plan = DtpPlan(self.irreps_in1, self.irreps_in2, self.irreps_out, raw)
        return self._plan

    # ------------------------------------------------------------------ planar entry points
    def planar_depthwise(self, xs, y, weight=None):
        """Planar DTP: in1 blocks ``[E, 2l+1, mul]`` -> output groups ``[E, 2l+1, K]`` (sm_90a kernels)."""
        from .. import ops
        w = self._get_weights(weight)
        return ops.depthwise_tensor_product(self.plan, xs, y, w)

    def planar_depthwise_gathered(self, graph, As, Bs, y, weight=None, weight_offset=None):
        """Planar DTP on ``A[src] (+ B[dst])`` with the gather folded into the kernel's operand load; the weights are
        ``weight (+ weight_offset)`` with the ``[weight_numel]`` offset added inside the kernel when it can be."""
        from .. import ops
        w = self._get_weights(weight)
        return ops.depthwise_tensor_product_gathered(self.plan, graph, As, Bs, y, w, weight_offset)

    def linear_weight_blocks(self, weight=None):
        """``[(i_in1, i_in2, i_out, W[mul_in, mul_in2, mul_out] * path constant)]`` for the scalar-in2 'uvw' kind."""
        if self._kind != "linear":
            raise NotImplementedError("not a scalar-in2 'uvw' tensor product")
        out = []
        for _idx, ins, view in self.weight_views(weight, yield_instruction=True):
            ir1 = self.irreps_in1[ins.i_in1].ir
            c = ins.path_weight * float(wigner_3j_np(ir1.l, 0, ir1.l)[0, 0, 0])  # w3j(l,0,l) = delta / sqrt(2l+1)
            if abs(c - 1.0) < 1e-12:     # sqrt(2l+1) / sqrt(2l+1) in floating point: not a reason for an extra pass
                c = 1.0
            out.append((ins.i_in1, ins.i_in2, ins.i_out, view, c))
        return out

    def _linear_spec(self):
        """``ops.LinearSpec`` of the scalar-in2 'uvw' paths (None when a path has a non-scalar second operand)."""
        if getattr(self, "_lin_spec", False) is False:
            from .. import ops
            paths, off = [], 0
            ok = self._kind == "linear"
            for ins in (i for i in self.instructions if i.has_weight):
                mul_in, m2, mul_out = ins.path_shape
                ir1 = self.irreps_in1[ins.i_in1].ir
                c = ins.path_weight * float(wigner_3j_np(ir1.l, 0, ir1.l)[0, 0, 0])
                ok = ok and m2 == 1
                paths.append((ins.i_in1, ins.i_out, off, mul_in, mul_out, 1.0 if abs(c - 1.0) < 1e-12 else c))
                off += mul_in * m2 * mul_out
            self._lin_spec = ops.LinearSpec(paths, off) if ok and off == self.weight_numel else None
        return self._lin_spec

    def planar_linear(self, xs, y=None, weight=None):
        """Per-degree channel mix on planar blocks: one ``[R*(2l+1), mul_in] @ [mul_in, mul_out]`` GEMM per path.

        ``xs``: one block ``[R, 2l+1, mul]`` per ``irreps_in1`` entry; ``y``: ``[R, irreps_in2.dim]`` or None (== 1).
        Returns one block per ``irreps_out`` entry.
        """
        from .. import ops
        w = self._get_weights(weight)
        if w.dim() != 1:
            raise NotImplementedError("per-row weights for 'uvw' are outside the hot path")
        in2_off = [s.start for s in self.irreps_in2.slices()]
        outs: List[Optional[torch.Tensor]] = [None] * len(self.irreps_out)
        R = xs[0].shape[0]
        if y is None:
            # small products (node-level linears, every linear of the small-graph models): all degrees in one launch
            spec = self._linear_spec()
            if spec is not None and ops.planar_linear_grouped_ok(spec, w, [xs[p[0]] for p in spec.paths]):
                ts = ops.planar_linear_grouped(spec, w, [xs[p[0]] for p in spec.paths])
                for p, t in zip(spec.paths, ts):
                    outs[p[1]] = t
                for io, (mul, ir) in enumerate(self.irreps_out):
                    if outs[io] is None:
                        outs[io] = xs[0].new_zeros((R, ir.dim, mul))
                return outs
        for i1, i2, io, W, c in self.linear_weight_blocks(w):
            x = xs[i1]
            d = x.shape[1]
            m2 = W.shape[1]
            if c != 1.0:
                W = W * c                    # the path constant goes onto the [mul_in, mul_out] weights, not the rows
            if y is None:
                if m2 != 1:
                    raise ValueError("second operand required")
                Weff = W.reshape(W.shape[0], W.shape[2])    # a view: `W[:, 0, :]` costs a zero-fill + copy in its backward
                t = ops.matmul_f32(x.reshape(R * d, -1), Weff).view(R, d, -1)
            elif m2 == 1:
                t = ops.matmul_f32(x.reshape(R * d, -1), W.reshape(W.shape[0], W.shape[2])).view(R, d, -1)
                t = t * y[:, in2_off[i2]].view(R, 1, 1)
            else:
                yy = y[:, in2_off[i2]:in2_off[i2] + m2]
                t = torch.einsum("rdu,rv,uvw->rdw", x, yy, W)
            outs[io] = t if outs[io] is None else outs[io] + t
        for io, (mul, ir) in enumerate(self.irreps_out):
            if outs[io] is None:
                outs[io] = xs[0].new_zeros((R, ir.dim, mul))
        return outs

    # ------------------------------------------------------------------ e3nn-layout forward
    def forward(self, x, y, weight: Optional[torch.Tensor] = None):
        from .. import ops
        if x.shape[-1] != self.irreps_in1.dim or y.shape[-1] != self.irreps_in2.dim:
            raise ValueError("input dimensions do not match irreps")
        lead = x.shape[:-1]
        x2 = x.reshape(-1, self.irreps_in1.dim)
        y2 = y.reshape(-1, self.irreps_in2.dim)
        if self._kind == "depthwise":
            w = self._get_weights(weight)
            if w.dim() > 1:
                w = w.reshape(-1, self.weight_numel)
            groups = self.planar_depthwise(ops.to_planar(x2, self.irreps_in1), y2.contiguous(), w)
            out = ops.from_planar(groups)  # groups follow irreps_out order, channels concatenated per run
        elif self._kind == "linear":
            outs = self.planar_linear(ops.to_planar(x2, self.irreps_in1), y2, weight)
            out = ops.from_planar(outs)
        else:
            raise NotImplementedError(
                "this TensorProduct configuration is outside the Equiformer hot path "
                "(supported: weighted 'uvu' with mul-1 in2, weighted 'uvw' with scalar in2)")
        return out.reshape(*lead, self.irreps_out.dim)

    def extra_repr(self) -> str:
        return (f"{self.irreps_in1} x {self.irreps_in2} -> {self.irreps_out} | "
                f"{len(self.instructions)} paths | {self.weight_numel} weights")
