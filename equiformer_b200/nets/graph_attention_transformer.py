"""Equivariant graph attention blocks and the QM9 model (drop-in for ``nets/graph_attention_transformer.py``).

Same classes, constructor arguments, forward signatures and ``state_dict`` keys as the reference.  What differs
is the body of the per-edge hot path (``GraphAttention.forward``, reference ``:482-527``, and
``EdgeDegreeEmbeddingNetwork.forward``, ``:725-733``):

* edge tensors stay in the planar (channel-innermost, one buffer per degree) layout from the merge linears to
  the aggregated node output; the head reshapes ``Vec2AttnHeads`` / ``AttnHeads2Vec`` become index arithmetic;
* both depth-wise tensor products run on the sm_90a kernels of ``csrc/eqf_dtp.cu`` (forward, and the hand
  derived gradient family, twice differentiable);
* softmax over destination segments and the attention-weighted scatter run on ``csrc/eqf_attn.cu`` over the
  destination-sorted edge list (no atomics);
* the per-degree channel-mixing linears are row-major GEMMs on the planar buffers.

There is no CPU implementation of these two forwards: CPU tensors raise (``equiformer_b200._lib.EqfError``).
"""
from __future__ import annotations

import math
from typing import List, Sequence

import torch

from .. import o3, ops
from ..graph import radius_graph, scatter_sum
from ..o3 import Irreps
from .drop import EquivariantDropout, GraphDropPath
from .fast_activation import Activation, Gate
from .gaussian_rbf import GaussianRadialBasisLayer
from .layer_norm import EquivariantLayerNormV2
from .radial_func import RadialProfile, clear_hoisted, hoist_first_layers
from .registry import register_model
from .tensor_product_rescale import (FullyConnectedTensorProductRescale,
                                     FullyConnectedTensorProductRescaleSwishGate, LinearRS, TensorProductRescale,
                                     irreps2gate, sort_irreps_even_first)

_RESCALE = True
_USE_BIAS = True

# QM9 statistics with cutoff radius 5 (reference :34-36)
_MAX_ATOM_TYPE = 5
_AVG_NUM_NODES = 18.03065905448718
_AVG_DEGREE = 15.57930850982666


def get_norm_layer(norm_type):
    if norm_type == "layer":
        return EquivariantLayerNormV2
    if norm_type is None:
        return None
    if norm_type in ("graph", "instance", "fast_layer"):
        raise NotImplementedError(f"norm '{norm_type}' is not used by any shipped Equiformer config (out of scope)")
    raise ValueError(f"Norm type {norm_type} not supported.")


class SmoothLeakyReLU(torch.nn.Module):
    """``(1+a)/2 x + (1-a)/2 x (2 sigmoid(x) - 1)`` (reference :54-63)."""

    def __init__(self, negative_slope: float = 0.2):
        super().__init__()
        self.alpha = negative_slope

    def forward(self, x):
        return 0.5 * (1 + self.alpha) * x + 0.5 * (1 - self.alpha) * x * (2 * torch.sigmoid(x) - 1)

    def extra_repr(self) -> str:
        return f"negative_slope={self.alpha}"


def get_mul_0(irreps) -> int:
    return sum(mul for mul, ir in Irreps(irreps) if ir.l == 0 and ir.p == 1)


def DepthwiseTensorProduct(irreps_node_input, irreps_edge_attr, irreps_node_output, internal_weights=False, bias=True):
    """One 'uvu' path per allowed (input irrep, edge irrep, output irrep); outputs sorted even-first (ref :157-183)."""
    irreps_node_input, irreps_edge_attr = Irreps(irreps_node_input), Irreps(irreps_edge_attr)
    irreps_node_output = Irreps(irreps_node_output)
    entries, raw = [], []
    scalar = o3.Irrep(0, 1)
    for i, (mul, ir_in) in enumerate(irreps_node_input):
        for j, (_, ir_edge) in enumerate(irreps_edge_attr):
            for ir_out in ir_in * ir_edge:
                if ir_out in irreps_node_output or ir_out == scalar:
                    raw.append((i, j, len(entries), "uvu", True))
                    entries.append((mul, ir_out))
    irreps_output, perm, _ = sort_irreps_even_first(Irreps(entries))
    instructions = [(i1, i2, perm[io], mode, train) for i1, i2, io, mode, train in raw]
    return TensorProductRescale(irreps_node_input, irreps_edge_attr, irreps_output, instructions,
                                internal_weights=internal_weights, shared_weights=internal_weights,
                                bias=bias, rescale=_RESCALE)


class SeparableFCTP(torch.nn.Module):
    """Depth-wise TP (radial weights) followed by a per-degree linear (+ optional norm / gate) (ref :186-248)."""

    def __init__(self, irreps_node_input, irreps_edge_attr, irreps_node_output, fc_neurons,
                 use_activation=False, norm_layer="graph", internal_weights=False):
        super().__init__()
        self.irreps_node_input = Irreps(irreps_node_input)
        self.irreps_edge_attr = Irreps(irreps_edge_attr)
        self.irreps_node_output = Irreps(irreps_node_output)
        norm = get_norm_layer(norm_layer)
        self.dtp = DepthwiseTensorProduct(self.irreps_node_input, self.irreps_edge_attr, self.irreps_node_output,
                                          bias=False, internal_weights=internal_weights)
        self.dtp_rad = None
        if fc_neurons is not None:
            self.dtp_rad = RadialProfile(fc_neurons + [self.dtp.tp.weight_numel])
            with torch.no_grad():  # rows indexed by *output feature* slices, factor is 1 for 'uvu' (ref :205-208)
                for sl, k in self.dtp.slices_sqrt_k.values():
                    self.dtp_rad.net[-1].weight.data[sl, :] *= k
                    self.dtp_rad.offset.data[sl] *= k
        irreps_lin_output = self.irreps_node_output
        irreps_scalars, irreps_gates, irreps_gated = irreps2gate(self.irreps_node_output)
        if use_activation:
            irreps_lin_output = (irreps_scalars + irreps_gates + irreps_gated).simplify()
        self.lin = LinearRS(self.dtp.irreps_out.simplify(), irreps_lin_output)
        self.norm = norm(self.lin.irreps_out) if norm_layer is not None else None
        self.gate = None
        if use_activation:
            if irreps_gated.num_irreps == 0:
                self.gate = Activation(self.irreps_node_output, acts=[torch.nn.SiLU()])
            else:
                self.gate = Gate(irreps_scalars, [torch.nn.SiLU() for _ in irreps_scalars],
                                 irreps_gates, [torch.sigmoid for _ in irreps_gates], irreps_gated)

    def forward(self, node_input, edge_attr, edge_scalars, batch=None, **kwargs):
        weight = None
        if self.dtp_rad is not None and edge_scalars is not None:
            weight = self.dtp_rad(edge_scalars)
        out = self.lin(self.dtp(node_input, edge_attr, weight))
        if self.norm is not None:
            out = self.norm(out, batch=batch)
        if self.gate is not None:
            out = self.gate(out)
        return out

    def planar(self, xs: Sequence[torch.Tensor], edge_attr, edge_scalars):
        """Planar forward: in1 blocks -> entries of the output irreps (gate applied when present)."""
        if self.norm is not None:
            raise NotImplementedError("planar SeparableFCTP with a norm layer is unused by the reference")
        weight = self.dtp_rad(edge_scalars) if (self.dtp_rad is not None and edge_scalars is not None) else None
        out = self.lin.planar(self.dtp.planar(xs, edge_attr, weight))
        if self.gate is not None:
            out = self.gate.planar(out) if isinstance(self.gate, Gate) else [self.gate(o) for o in out]
        return out


class Vec2AttnHeads(torch.nn.Module):
    """``[N, irreps_head * H]`` -> ``[N, H, irreps_head]`` (ref :252-285); e3nn-layout compatibility op."""

    def __init__(self, irreps_head, num_heads):
        super().__init__()
        self.num_heads = num_heads
        self.irreps_head = Irreps(irreps_head)
        self.irreps_mid_in = Irreps([(mul * num_heads, ir) for mul, ir in self.irreps_head])
        self.mid_in_indices = [(s.start, s.stop) for s in self.irreps_mid_in.slices()]

    def forward(self, x):
        n = x.shape[0]
        return torch.cat([x.narrow(1, a, b - a).reshape(n, self.num_heads, -1) for a, b in self.mid_in_indices], dim=2)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(irreps_head={self.irreps_head}, num_heads={self.num_heads})"


class AttnHeads2Vec(torch.nn.Module):
    """Inverse of :class:`Vec2AttnHeads` (ref :289-316)."""

    def __init__(self, irreps_head):
        super().__init__()
        self.irreps_head = Irreps(irreps_head)
        self.head_indices = [(s.start, s.stop) for s in self.irreps_head.slices()]

    def forward(self, x):
        n = x.shape[0]
        return torch.cat([x.narrow(2, a, b - a).reshape(n, -1) for a, b in self.head_indices], dim=1)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(irreps_head={self.irreps_head})"


_GRAPH_CACHE = {}


def _graph_for(edge_src, edge_dst, n_nodes, kwargs) -> ops.Graph:
    g = kwargs.get("graph")
    if isinstance(g, ops.Graph) and g.n_nodes == n_nodes:
        return g
    key = (edge_src.data_ptr(), edge_dst.data_ptr(), edge_dst.numel(), n_nodes, edge_dst._version, edge_src._version)
    hit = _GRAPH_CACHE.get("last")
    if hit is not None and hit[0] == key:
        return hit[1]
    g = ops.Graph(edge_src, edge_dst, n_nodes)
    _GRAPH_CACHE["last"] = (key, g, edge_src, edge_dst)  # keep the index tensors alive with the key
    return g


def _is_sorted_simplified(irreps: Irreps) -> bool:
    keys = [(ir.l, -ir.p) for _, ir in irreps]
    return keys == sorted(keys) and len(set(keys)) == len(keys)


def _entries_from_groups(groups: Sequence[torch.Tensor], plan) -> List[torch.Tensor]:
    """Views of the DTP output groups, one per (unsimplified) ``irreps_out`` entry."""
    return [groups[plan.group_of_entry[io]].narrow(2, plan.chan_off_of_entry[io], mul)
            for io, (mul, _ir) in enumerate(plan.irreps_out)]


def _reblock(blocks: Sequence[torch.Tensor], irreps_from: Irreps, irreps_to: Irreps) -> List[torch.Tensor]:
    if list(irreps_from) == list(irreps_to):
        return list(blocks)
    if irreps_from.dim != irreps_to.dim:
        raise ValueError(f"cannot reinterpret {irreps_from} as {irreps_to}")
    return ops.to_planar(ops.from_planar(blocks), irreps_to)


def _group_weight_matrices(lin, n_groups: int):
    """``[K_g, N_g]`` weight views of a per-degree linear whose entries map one to one onto the ``n_groups`` output
    groups of the depth-wise product in front of it (instruction g: group g -> entry g, path constant 1), or None when
    the linear does not have that canonical structure (then the unfused route is taken)."""
    try:
        ins = [(i.i_in1, i.i_in2, i.i_out) for i in lin.tp.instructions]
        if ins != [(g, 0, g) for g in range(n_groups)] or len(lin.irreps_out) != n_groups:
            return None
        blocks = lin.tp.linear_weight_blocks()
        if any(c != 1.0 for *_i, _W, c in blocks):
            return None
        return [W.reshape(W.shape[0], W.shape[2]) for _i1, _i2, _io, W, _c in blocks]
    except (AttributeError, NotImplementedError):
        return None


def _fused_linear_possible(lin, dtp) -> bool:
    return _group_weight_matrices(lin, len(dtp.tp.plan.out_groups)) is not None


class GraphAttention(torch.nn.Module):
    """Multi-head equivariant graph attention (ref :403-533): message = alpha * value, aggregated at the target."""

    def __init__(self, irreps_node_input, irreps_node_attr, irreps_edge_attr, irreps_node_output, fc_neurons,
                 irreps_head, num_heads, irreps_pre_attn=None, rescale_degree=False, nonlinear_message=False,
                 alpha_drop=0.1, proj_drop=0.1):
        super().__init__()
        self.irreps_node_input = Irreps(irreps_node_input)
        self.irreps_node_attr = Irreps(irreps_node_attr)
        self.irreps_edge_attr = Irreps(irreps_edge_attr)
        self.irreps_node_output = Irreps(irreps_node_output)
        self.irreps_pre_attn = self.irreps_node_input if irreps_pre_attn is None else Irreps(irreps_pre_attn)
        self.irreps_head = Irreps(irreps_head)
        self.num_heads = num_heads
        self.rescale_degree = rescale_degree
        self.nonlinear_message = nonlinear_message

        self.merge_src = LinearRS(self.irreps_node_input, self.irreps_pre_attn, bias=True)
        self.merge_dst = LinearRS(self.irreps_node_input, self.irreps_pre_attn, bias=False)

        irreps_attn_heads = self.irreps_head * num_heads
        irreps_attn_heads, _, _ = sort_irreps_even_first(irreps_attn_heads)
        irreps_attn_heads = irreps_attn_heads.simplify()
        mul_alpha = get_mul_0(irreps_attn_heads)
        mul_alpha_head = mul_alpha // num_heads
        irreps_alpha = Irreps(f"{mul_alpha}x0e")
        irreps_attn_all = (irreps_alpha + irreps_attn_heads).simplify()
        self.irreps_attn_heads = irreps_attn_heads

        self.sep_act = None
        if self.nonlinear_message:
            self.sep_act = SeparableFCTP(self.irreps_pre_attn, self.irreps_edge_attr, self.irreps_pre_attn, fc_neurons,
                                         use_activation=True, norm_layer=None, internal_weights=False)
            self.sep_alpha = LinearRS(self.sep_act.dtp.irreps_out, irreps_alpha)
            self.sep_value = SeparableFCTP(self.irreps_pre_attn, self.irreps_edge_attr, irreps_attn_heads,
                                           fc_neurons=None, use_activation=False, norm_layer=None,
                                           internal_weights=True)
            self.vec2heads_alpha = Vec2AttnHeads(Irreps(f"{mul_alpha_head}x0e"), num_heads)
            self.vec2heads_value = Vec2AttnHeads(self.irreps_head, num_heads)
        else:
            self.sep = SeparableFCTP(self.irreps_pre_attn, self.irreps_edge_attr, irreps_attn_all, fc_neurons,
                                     use_activation=False, norm_layer=None)
            self.vec2heads = Vec2AttnHeads((Irreps(f"{mul_alpha_head}x0e") + self.irreps_head).simplify(), num_heads)

        self.alpha_act = Activation(Irreps(f"{mul_alpha_head}x0e"), [SmoothLeakyReLU(0.2)])
        self.heads2vec = AttnHeads2Vec(self.irreps_head)
        self.mul_alpha_head = mul_alpha_head
        self.alpha_dot = torch.nn.Parameter(torch.randn(1, num_heads, mul_alpha_head))
        bound = math.sqrt(6.0 / (num_heads + mul_alpha_head))  # torch_geometric.nn.inits.glorot (GATv2 style)
        with torch.no_grad():
            self.alpha_dot.uniform_(-bound, bound)
        self.alpha_dropout = torch.nn.Dropout(alpha_drop) if alpha_drop != 0.0 else None
        self.proj = LinearRS(irreps_attn_heads, self.irreps_node_output)
        self.proj_drop = EquivariantDropout(self.irreps_node_input, drop_prob=proj_drop) if proj_drop != 0.0 else None

        # sep_alpha reads only the 0e entries of the DTP output; when they form the first output group (always, after the
        # even-first sort) its per-entry weights are one contiguous [K0, mul_alpha] matrix -> a single GEMM
        self._alpha_single_gemm = False
        if self.nonlinear_message:
            plan_out = self.sep_act.dtp.irreps_out
            n0 = sum(1 for _, ir in plan_out if ir.is_scalar())
            ins = [(i.i_in1, i.i_in2, i.i_out) for i in self.sep_alpha.tp.instructions]
            if (n0 > 0 and all(ir.is_scalar() for _, ir in plan_out[:n0]) and ins == [(i, 0, 0) for i in range(n0)]
                    and all(c == 1.0 for *_i, _W, c in self.sep_alpha.tp.linear_weight_blocks())):
                self._alpha_single_gemm = True

        # fused bias + Gate + logits kernel (ops.GateLogits) when the layer has the canonical structure:
        # lin outputs [(scalars+gates) x 0e | gated entries], one instruction per output entry, single-GEMM alpha
        self._gate_layout = None
        if self.nonlinear_message and self._alpha_single_gemm and isinstance(self.sep_act.gate, Gate):
            gate, lin = self.sep_act.gate, self.sep_act.lin
            ins = [(i.i_in1, i.i_out) for i in lin.tp.instructions]
            n_out = len(lin.irreps_out)
            canonical = (len(gate.irreps_scalars) == 1 and ins == [(i, i) for i in range(n_out)]
                         and lin.irreps_out[0].ir.is_scalar()
                         and lin.irreps_out[0].mul == gate.irreps_scalars.dim + gate.irreps_gates.dim
                         and [m for m, _ in lin.irreps_out[1:]] == [m for m, _ in gate.irreps_gated]
                         and len(lin.bias) == 1 and len(self.sep_alpha.bias) == 1 and mul_alpha_head <= 32
                         # the fused path feeds the raw weight blocks to the GEMMs: every path constant must be 1
                         and all(c == 1.0 for *_i, _W, c in lin.tp.linear_weight_blocks())
                         and all(c == 1.0 for *_i, _W, c in self.sep_alpha.tp.linear_weight_blocks()))
            if canonical:
                self._gate_layout = ops.GateLayout(
                    mul_alpha, gate.irreps_scalars.dim, num_heads, [ir.dim for _, ir in gate.irreps_gated],
                    [m for m, _ in gate.irreps_gated], gate.act_scalars.acts[0].cst, gate.act_gates.acts[0].cst,
                    self.alpha_act.acts[0].cst, 0.2)

        if not _is_sorted_simplified(self.irreps_head):
            raise NotImplementedError("irreps_head must be sorted (l ascending, even first) with one entry per irrep")
        self._head_layout = ops.HeadLayout([ir.dim for _, ir in irreps_attn_heads],
                                           [mul for mul, _ in irreps_attn_heads], num_heads)
        # K1 (ops.DtpLinear): both depth-wise products feed their per-degree linears on chip when the linears are canonical
        self._fuse_act = (self._gate_layout is not None and _fused_linear_possible(self.sep_act.lin, self.sep_act.dtp))
        self._fuse_value = (self.nonlinear_message and _fused_linear_possible(self.sep_value.lin, self.sep_value.dtp))

    # ---------------------------------------------------------------------------------------------
    @property
    def supports_planar(self) -> bool:
        """True when the block can stay in the planar layout (no output dropout to apply on e3nn-layout features)."""
        return self.proj_drop is None or not self.training or getattr(self.proj_drop, "drop_prob", 1.0) == 0.0

    def forward(self, node_input, node_attr, edge_src, edge_dst, edge_attr, edge_scalars, batch, **kwargs):
        xs = ops.to_planar(node_input, self.irreps_node_input)
        node = self.forward_planar(xs, node_attr, edge_src, edge_dst, edge_attr, edge_scalars, batch, **kwargs)
        node_output = ops.from_planar(node)                                               # [ref :522]
        if self.proj_drop is not None:
            node_output = self.proj_drop(node_output)
        return node_output

    def forward_planar(self, xs, node_attr, edge_src, edge_dst, edge_attr, edge_scalars, batch, **kwargs):
        """The layer on planar node blocks (one ``[N, 2l+1, mul]`` tensor per input entry) -> planar output blocks,
        before the output dropout."""
        n_nodes = xs[0].shape[0]
        graph = _graph_for(edge_src, edge_dst, n_nodes, kwargs)
        edge_attr = graph.sort_edges(edge_attr).contiguous()
        edge_scalars = graph.sort_edges(edge_scalars)
        E, H, A = graph.n_edges, self.num_heads, self.mul_alpha_head

        # merge (node level, per-degree GEMMs) then gather + add along the edge list      [ref :485-487]
        m_src = self.merge_src.planar(xs)
        m_dst = self.merge_dst.planar(xs)
        # the gather + add of ref :487 happens inside the DTP kernel's operand load (node tables stay L2-resident)

        if self.nonlinear_message:
            sa = self.sep_act
            # [ref :490] radial weights; the radial offset is added inside the DTP kernel's weight load
            weight = sa.dtp_rad(edge_scalars, add_offset=False)
            plan1 = sa.dtp.tp.plan
            fuse1 = self._fuse_act and ops.dtp_linear_ok(plan1, edge_attr, weight)
            f = None
            if not fuse1:
                f = sa.dtp.tp.planar_depthwise_gathered(graph, m_src, m_dst, edge_attr, weight,
                                                        sa.dtp_rad.offset)                # [ref :487+:491]  DTP #1
            logits = None
            if self._gate_layout is not None and (fuse1 or ops.fused_ok(f[0])):
                # one GEMM for alpha and the 0e part of the value linear ([K0, A0 | S + Gates]), then ONE kernel for
                # the bias adds, the gate and the attention logits                           [ref :492-495, :506-507]
                lay = self._gate_layout
                blocks = {io: (W, c) for _i1, _i2, io, W, c in sa.lin.tp.linear_weight_blocks()}
                k0 = plan1.out_groups[0][2]
                w_cat = torch.cat([self.sep_alpha.tp.weight.view(k0, -1), blocks[0][0].reshape(k0, -1)], dim=1)
                bias = torch.cat([self.sep_alpha.bias[0], sa.lin.bias[0]])
                if fuse1:
                    # K1: DTP #1 is the on-chip A operand of the three per-degree GEMMs - [E, 3136] never reaches HBM
                    Ws = [w_cat] + [blocks[g][0].reshape(blocks[g][0].shape[0], -1) for g in range(1, len(plan1.out_groups))]
                    outs = ops.dtp_linear(plan1, graph, m_src, m_dst, edge_attr, weight, sa.dtp_rad.offset, Ws)
                    t0, gated = outs[0].reshape(E, -1), outs[1:]
                else:
                    t0 = ops.matmul_f32(f[0].reshape(E, k0), w_cat)
                    gated = [ops.matmul_f32(f[g].reshape(E * f[g].shape[1], f[g].shape[2]), blocks[g][0].reshape(f[g].shape[2], -1))
                             .view(E, f[g].shape[1], -1) for g in range(1, len(f))]
                logits, v0, *vs = ops.GateLogits.apply(lay, t0, bias, self.alpha_dot.view(H, A), *gated)
                value = _reblock([v0.view(E, 1, -1), *vs], sa.gate.irreps_out, self.sep_value.irreps_node_input)
                value = self._value_linear(value, edge_attr)                              # [ref :496]  DTP #2 + lin
                alpha = None
            elif self._alpha_single_gemm:                                                 # [ref :492]
                k0 = f[0].shape[2]
                w_alpha = self.sep_alpha.tp.weight.view(k0, -1)
                alpha = ops.matmul_f32(f[0].reshape(E, k0), w_alpha)
                if len(self.sep_alpha.bias) > 0:
                    alpha = alpha + self.sep_alpha.bias[0]
            else:
                alpha = self.sep_alpha.planar(_entries_from_groups(f, sa.dtp.tp.plan))[0]
            if logits is None:
                value = sa.lin.planar(f)                                                  # [ref :494]
                value = sa.gate.planar(value) if isinstance(sa.gate, Gate) else [sa.gate(v) for v in value]  # [:495]
                value = _reblock(value, sa.gate.irreps_out, self.sep_value.irreps_node_input)
                value = self._value_linear(value, edge_attr)                              # [ref :496]  DTP #2 + lin
                alpha = alpha.reshape(E, H, A)                                            # [ref :493]
        else:
            weight = self.sep.dtp_rad(edge_scalars, add_offset=False)
            logits = None
            out = self.sep.lin.planar(self.sep.dtp.tp.planar_depthwise_gathered(
                graph, m_src, m_dst, edge_attr, weight, self.sep.dtp_rad.offset))         # [ref :487+:499]
            first = out[0]                                                                # 0e entry: alpha | value scalars
            if first.shape[1] != 1:
                raise NotImplementedError("attention logits need a leading 0e entry")
            per_head = first.reshape(E, H, -1)
            alpha = per_head.narrow(2, 0, A)
            rest = per_head.shape[2] - A
            value = ([per_head.narrow(2, A, rest).reshape(E, 1, H * rest)] if rest > 0 else []) + list(out[1:])

        # logits -> segment softmax -> weighted aggregation                               [ref :506-513]
        z = logits if logits is not None else (self.alpha_act(alpha) * self.alpha_dot).sum(dim=-1)
        no_drop = self.alpha_dropout is None or not self.training or self.alpha_dropout.p == 0.0
        if no_drop and ops.softmax_aggregate_ok(self._head_layout, z):
            # K2: softmax over the destination segment and the weighted aggregation in one kernel
            node = list(ops.SoftmaxAggregate.apply(self._head_layout, graph, z.contiguous(), *[v.contiguous() for v in value]))
        else:
            attn = ops.segment_softmax(z.contiguous(), graph)
            if self.alpha_dropout is not None:
                attn = self.alpha_dropout(attn)
            node = ops.attention_aggregate(self._head_layout, graph, attn.contiguous(), [v.contiguous() for v in value])

        if self.rescale_degree:                                                           # [ref :516-520]
            degree = (graph.row_ptr[1:] - graph.row_ptr[:-1]).to(node[0].dtype).view(-1, 1, 1)
            node = [t * degree for t in node]
        return self.proj.planar(node)

    def _value_linear(self, value, edge_attr):
        """``sep_value``: depth-wise product with the shared (internal) weights, then the per-degree linear [ref :496]."""
        sv = self.sep_value
        plan2 = sv.dtp.tp.plan
        w2 = sv.dtp.tp.weight
        if self._fuse_value and ops.dtp_linear_ok(plan2, edge_attr, w2):
            Ws = _group_weight_matrices(sv.lin, len(plan2.out_groups))
            return sv.lin._planar_bias(ops.dtp_linear(plan2, None, [v.contiguous() for v in value], None, edge_attr, w2,
                                                      None, Ws))
        return sv.lin.planar(sv.dtp.planar(value, edge_attr, None))

    def extra_repr(self) -> str:
        return f"rescale_degree={self.rescale_degree}, "


class FeedForwardNetwork(torch.nn.Module):
    """Two node-level FCTPs with a gate in between (ref :537-571)."""

    def __init__(self, irreps_node_input, irreps_node_attr, irreps_node_output, irreps_mlp_mid=None, proj_drop=0.1):
        super().__init__()
        self.irreps_node_input = Irreps(irreps_node_input)
        self.irreps_node_attr = Irreps(irreps_node_attr)
        self.irreps_mlp_mid = Irreps(irreps_mlp_mid) if irreps_mlp_mid is not None else self.irreps_node_input
        self.irreps_node_output = Irreps(irreps_node_output)
        self.fctp_1 = FullyConnectedTensorProductRescaleSwishGate(
            self.irreps_node_input, self.irreps_node_attr, self.irreps_mlp_mid, bias=True, rescale=_RESCALE)
        self.fctp_2 = FullyConnectedTensorProductRescale(
            self.irreps_mlp_mid, self.irreps_node_attr, self.irreps_node_output, bias=True, rescale=_RESCALE)
        self.proj_drop = EquivariantDropout(self.irreps_node_output, drop_prob=proj_drop) if proj_drop != 0.0 else None
        # bias + Gate in one kernel when fctp_1 has the canonical structure (one instruction per output entry)
        self._gate_layout = None
        gate, f1 = self.fctp_1.gate, self.fctp_1
        ins = [(i.i_in1, i.i_out) for i in f1.tp.instructions]
        if (isinstance(gate, Gate) and ins == [(i, i) for i in range(len(f1.irreps_out))] and len(f1.bias) == 1
                and self.irreps_node_attr.dim == 1):
            lay = ops.gate_only_layout(gate, f1.irreps_out)
            self._gate_layout = lay if (lay is not None and f1.bias[0].numel() == lay.width) else None

    @property
    def supports_planar(self) -> bool:
        return self.proj_drop is None or not self.training or getattr(self.proj_drop, "drop_prob", 1.0) == 0.0

    def forward(self, node_input, node_attr, **kwargs):
        node_output = ops.from_planar(self.forward_planar(ops.to_planar(node_input, self.irreps_node_input), node_attr))
        if self.proj_drop is not None:
            node_output = self.proj_drop(node_output)
        return node_output

    def forward_planar(self, xs, node_attr, **kwargs):
        # planar end to end: entries of fctp_1's gate input -> gate -> fctp_2
        # the models feed the constant scalar 1 as node_attr (ref :869): the multiply by it is skipped when marked so
        y = None if (getattr(node_attr, "_eqf_all_ones", False) and self.irreps_node_attr.dim == 1) else node_attr
        gate = self.fctp_1.gate
        if self._gate_layout is not None and y is None and ops.fused_ok(xs[0]):
            pre = self.fctp_1.tp.planar_linear(xs, None, None)                  # bias is added inside the gate kernel
            N = pre[0].shape[0]
            h = ops.gate_fused(self._gate_layout, pre[0].reshape(N, -1), self.fctp_1.bias[0], pre[1:])
            h = _reblock([h[0].view(N, 1, -1), *h[1:]], gate.irreps_out, self.fctp_2.irreps_in1)
        else:
            h = self.fctp_1.planar(xs, y)
            if isinstance(gate, Gate):
                h = _reblock(gate.planar(h), gate.irreps_out, self.fctp_2.irreps_in1)
            else:
                h = [gate(t) for t in h]
        return self.fctp_2.planar(h, y)


class TransBlock(torch.nn.Module):
    """Pre-norm block: LayerNorm -> GraphAttention -> residual -> LayerNorm -> FFN -> residual (ref :575-667)."""

    def __init__(self, irreps_node_input, irreps_node_attr, irreps_edge_attr, irreps_node_output, fc_neurons,
                 irreps_head, num_heads, irreps_pre_attn=None, rescale_degree=False, nonlinear_message=False,
                 alpha_drop=0.1, proj_drop=0.1, drop_path_rate=0.0, irreps_mlp_mid=None, norm_layer="layer"):
        super().__init__()
        self.irreps_node_input = Irreps(irreps_node_input)
        self.irreps_node_attr = Irreps(irreps_node_attr)
        self.irreps_edge_attr = Irreps(irreps_edge_attr)
        self.irreps_node_output = Irreps(irreps_node_output)
        self.irreps_pre_attn = self.irreps_node_input if irreps_pre_attn is None else Irreps(irreps_pre_attn)
        self.irreps_head = Irreps(irreps_head)
        self.num_heads = num_heads
        self.rescale_degree = rescale_degree
        self.nonlinear_message = nonlinear_message
        self.irreps_mlp_mid = Irreps(irreps_mlp_mid) if irreps_mlp_mid is not None else self.irreps_node_input

        self.norm_1 = get_norm_layer(norm_layer)(self.irreps_node_input)
        # the attention sub-layer registers under the reference's attribute name ("ga"; "dpa" in DPTransBlock)
        setattr(self, self._attn_name, self._make_attention(fc_neurons, alpha_drop, proj_drop))
        self.drop_path = GraphDropPath(drop_path_rate) if drop_path_rate > 0.0 else None
        self.norm_2 = get_norm_layer(norm_layer)(self.irreps_node_input)
        self.ffn = FeedForwardNetwork(irreps_node_input=self.irreps_node_input, irreps_node_attr=self.irreps_node_attr,
                                      irreps_node_output=self.irreps_node_output, irreps_mlp_mid=self.irreps_mlp_mid,
                                      proj_drop=proj_drop)
        self.ffn_shortcut = None
        if self.irreps_node_input != self.irreps_node_output:
            self.ffn_shortcut = FullyConnectedTensorProductRescale(
                self.irreps_node_input, self.irreps_node_attr, self.irreps_node_output, bias=True, rescale=_RESCALE)

    _attn_name = "ga"

    def _make_attention(self, fc_neurons, alpha_drop, proj_drop):
        return GraphAttention(irreps_node_input=self.irreps_node_input, irreps_node_attr=self.irreps_node_attr,
                              irreps_edge_attr=self.irreps_edge_attr, irreps_node_output=self.irreps_node_input,
                              fc_neurons=fc_neurons, irreps_head=self.irreps_head, num_heads=self.num_heads,
                              irreps_pre_attn=self.irreps_pre_attn, rescale_degree=self.rescale_degree,
                              nonlinear_message=self.nonlinear_message, alpha_drop=alpha_drop, proj_drop=proj_drop)

    @property
    def attention(self):
        return getattr(self, self._attn_name)

    def forward(self, node_input, node_attr, edge_src, edge_dst, edge_attr, edge_scalars, batch, **kwargs):
        features = self.norm_1(node_input, batch=batch)
        features = self.attention(node_input=features, node_attr=node_attr, edge_src=edge_src, edge_dst=edge_dst,
                                  edge_attr=edge_attr, edge_scalars=edge_scalars, batch=batch, **kwargs)
        if self.drop_path is not None:
            features = self.drop_path(features, batch)
        node_output = node_input + features

        features = self.ffn(self.norm_2(node_output, batch=batch), node_attr)
        if self.ffn_shortcut is not None:
            node_output = self.ffn_shortcut(node_output, node_attr)
        if self.drop_path is not None:
            features = self.drop_path(features, batch)
        return node_output + features

    @property
    def supports_planar(self) -> bool:
        """The whole block can run on planar node blocks: fused LayerNorms, no shortcut projection, no stochastic depth
        or output dropout in effect."""
        return (getattr(self.norm_1, "supports_planar", False) and getattr(self.norm_2, "supports_planar", False)
                and self.ffn_shortcut is None and (self.drop_path is None or not self.training)
                and self.attention.supports_planar and self.ffn.supports_planar
                and self.irreps_node_input == self.irreps_node_output)

    def forward_planar(self, xs, node_attr, edge_src, edge_dst, edge_attr, edge_scalars, batch, **kwargs):
        """``forward`` on planar node blocks -> planar node blocks: the features never pass through the e3nn layout
        (saves the layout copies at every sub-layer boundary, ~24 small launches per block and step)."""
        f = self.attention.forward_planar(self.norm_1.planar(xs), node_attr, edge_src, edge_dst, edge_attr, edge_scalars,
                                          batch, **kwargs)
        xs = [a + b for a, b in zip(xs, f)]
        f = self.ffn.forward_planar(self.norm_2.planar(xs), node_attr)
        return [a + b for a, b in zip(xs, f)]


class NodeEmbeddingNetwork(torch.nn.Module):
    def __init__(self, irreps_node_embedding, max_atom_type=_MAX_ATOM_TYPE, bias=True):
        super().__init__()
        self.max_atom_type = max_atom_type
        self.irreps_node_embedding = Irreps(irreps_node_embedding)
        self.atom_type_lin = LinearRS(Irreps(f"{self.max_atom_type}x0e"), self.irreps_node_embedding, bias=bias)
        self.atom_type_lin.tp.weight.data.mul_(self.max_atom_type ** 0.5)

    def forward(self, node_atom):
        # one-hot without torch's range check (that check is a device synchronisation; keeps the step graph-capturable)
        classes = torch.arange(self.max_atom_type, device=node_atom.device)
        onehot = (node_atom.unsqueeze(-1) == classes).to(self.atom_type_lin.tp.weight.dtype)
        return self.atom_type_lin(onehot), onehot, onehot


class ScaledScatter(torch.nn.Module):
    def __init__(self, avg_aggregate_num):
        super().__init__()
        self.avg_aggregate_num = avg_aggregate_num + 0.0

    def forward(self, x, index, **kwargs):
        return scatter_sum(x, index, **kwargs).div(self.avg_aggregate_num ** 0.5)

    def extra_repr(self) -> str:
        return f"avg_aggregate_num={self.avg_aggregate_num}"


class EdgeDegreeEmbeddingNetwork(torch.nn.Module):
    """Initial node features from the neighbourhood geometry: gather -> DTP -> linear -> scaled scatter (ref :709-733)."""

    def __init__(self, irreps_node_embedding, irreps_edge_attr, fc_neurons, avg_aggregate_num):
        super().__init__()
        irreps_node_embedding = Irreps(irreps_node_embedding)
        self.exp = LinearRS(Irreps("1x0e"), irreps_node_embedding, bias=_USE_BIAS, rescale=_RESCALE)
        self.dw = DepthwiseTensorProduct(irreps_node_embedding, irreps_edge_attr, irreps_node_embedding,
                                         internal_weights=False, bias=False)
        self.rad = RadialProfile(fc_neurons + [self.dw.tp.weight_numel])
        with torch.no_grad():
            for sl, k in self.dw.slices_sqrt_k.values():
                self.rad.net[-1].weight.data[sl, :] *= k
                self.rad.offset.data[sl] *= k
        self.proj = LinearRS(self.dw.irreps_out.simplify(), irreps_node_embedding)
        self.scale_scatter = ScaledScatter(avg_aggregate_num)
        self._sum_layout = ops.HeadLayout([ir.dim for _, ir in self.proj.irreps_out],
                                          [mul for mul, _ in self.proj.irreps_out], 1)
        self._fuse_proj = _fused_linear_possible(self.proj, self.dw)

    def forward(self, node_input, edge_attr, edge_scalars, edge_src, edge_dst, batch, **kwargs):
        n_nodes = node_input.shape[0]
        graph = _graph_for(edge_src, edge_dst, n_nodes, kwargs)
        edge_attr = graph.sort_edges(edge_attr).contiguous()
        edge_scalars = graph.sort_edges(edge_scalars)
        ones = torch.ones((n_nodes, 1, 1), dtype=node_input.dtype, device=node_input.device)
        node_feats = self.exp.planar([ones])
        weight = self.rad(edge_scalars, add_offset=False)        # the radial offset is added inside the DTP kernel
        plan = self.dw.tp.plan
        if self._fuse_proj and ops.dtp_linear_ok(plan, edge_attr, weight):        # K1: DTP -> proj on chip
            Ws = _group_weight_matrices(self.proj, len(plan.out_groups))
            edge_feats = self.proj._planar_bias(ops.dtp_linear(plan, graph, node_feats, None, edge_attr, weight,
                                                               self.rad.offset, Ws))
        else:
            edge_feats = self.dw.tp.planar_depthwise_gathered(graph, node_feats, None, edge_attr, weight, self.rad.offset)
            edge_feats = self.proj.planar(edge_feats)
        summed = ops.attention_aggregate(self._sum_layout, graph, None, [t.contiguous() for t in edge_feats])
        return ops.from_planar(summed).div(self.scale_scatter.avg_aggregate_num ** 0.5)


class GraphAttentionTransformer(torch.nn.Module):
    """The QM9 Equiformer (ref :736-899)."""

    def __init__(self, irreps_in="5x0e", irreps_node_embedding="128x0e+64x1e+32x2e", num_layers=6,
                 irreps_node_attr="1x0e", irreps_sh="1x0e+1x1e+1x2e", max_radius=5.0, number_of_basis=128,
                 basis_type="gaussian", fc_neurons=[64, 64], irreps_feature="512x0e",
                 irreps_head="32x0e+16x1o+8x2e", num_heads=4, irreps_pre_attn=None, rescale_degree=False,
                 nonlinear_message=False, irreps_mlp_mid="128x0e+64x1e+32x2e", norm_layer="layer",
                 alpha_drop=0.2, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0,
                 mean=None, std=None, scale=None, atomref=None):
        super().__init__()
        self.max_radius = max_radius
        self.number_of_basis = number_of_basis
        self.alpha_drop, self.proj_drop, self.out_drop = alpha_drop, proj_drop, out_drop
        self.drop_path_rate = drop_path_rate
        self.norm_layer = norm_layer
        self.task_mean, self.task_std, self.scale = mean, std, scale
        self.register_buffer("atomref", atomref)

        self.irreps_node_attr = Irreps(irreps_node_attr)
        self.irreps_node_input = Irreps(irreps_in)
        self.irreps_node_embedding = Irreps(irreps_node_embedding)
        self.lmax = self.irreps_node_embedding.lmax
        self.irreps_feature = Irreps(irreps_feature)
        self.num_layers = num_layers
        self.irreps_edge_attr = Irreps(irreps_sh) if irreps_sh is not None else Irreps.spherical_harmonics(self.lmax)
        self.fc_neurons = [self.number_of_basis] + list(fc_neurons)
        self.irreps_head = Irreps(irreps_head)
        self.num_heads = num_heads
        self.irreps_pre_attn = irreps_pre_attn
        self.rescale_degree = rescale_degree
        self.nonlinear_message = nonlinear_message
        self.irreps_mlp_mid = Irreps(irreps_mlp_mid)

        self.atom_embed = NodeEmbeddingNetwork(self.irreps_node_embedding, _MAX_ATOM_TYPE)
        self.basis_type = basis_type
        if basis_type == "gaussian":
            self.rbf = GaussianRadialBasisLayer(self.number_of_basis, cutoff=self.max_radius)
        elif basis_type == "bessel":
            raise NotImplementedError("Bessel basis comes from ocpmodels (absent dependency; out of scope, SURVEY.md 2#5)")
        else:
            raise ValueError(basis_type)
        self.edge_deg_embed = EdgeDegreeEmbeddingNetwork(self.irreps_node_embedding, self.irreps_edge_attr,
                                                         self.fc_neurons, _AVG_DEGREE)
        self.blocks = torch.nn.ModuleList()
        self.build_blocks()
        self.norm = get_norm_layer(self.norm_layer)(self.irreps_feature)
        self.out_dropout = EquivariantDropout(self.irreps_feature, self.out_drop) if self.out_drop != 0.0 else None
        self.head = torch.nn.Sequential(
            LinearRS(self.irreps_feature, self.irreps_feature, rescale=_RESCALE),
            Activation(self.irreps_feature, acts=[torch.nn.SiLU()]),
            LinearRS(self.irreps_feature, Irreps("1x0e"), rescale=_RESCALE))
        self.scale_scatter = ScaledScatter(_AVG_NUM_NODES)
        self.register_buffer("_atom_remap", torch.tensor([-1, 0, -1, -1, -1, -1, 1, 2, 3, 4]), persistent=False)
        self.apply(self._init_weights)

    _block_cls = TransBlock

    def build_blocks(self):
        for i in range(self.num_layers):
            out = self.irreps_node_embedding if i != self.num_layers - 1 else self.irreps_feature
            self.blocks.append(self._block_cls(
                irreps_node_input=self.irreps_node_embedding, irreps_node_attr=self.irreps_node_attr,
                irreps_edge_attr=self.irreps_edge_attr, irreps_node_output=out, fc_neurons=self.fc_neurons,
                irreps_head=self.irreps_head, num_heads=self.num_heads, irreps_pre_attn=self.irreps_pre_attn,
                rescale_degree=self.rescale_degree, nonlinear_message=self.nonlinear_message,
                alpha_drop=self.alpha_drop, proj_drop=self.proj_drop, drop_path_rate=self.drop_path_rate,
                irreps_mlp_mid=self.irreps_mlp_mid, norm_layer=self.norm_layer))

    def _init_weights(self, m):
        if isinstance(m, torch.nn.Linear):
            if m.bias is not None:
                torch.nn.init.constant_(m.bias, 0)
        elif isinstance(m, torch.nn.LayerNorm):
            torch.nn.init.constant_(m.bias, 0)
            torch.nn.init.constant_(m.weight, 1.0)

    @torch.jit.ignore
    def no_weight_decay(self):
        skip = set()
        names = {n for n, _ in self.named_parameters()}
        for mod_name, mod in self.named_modules():
            if isinstance(mod, (torch.nn.Linear, torch.nn.LayerNorm, EquivariantLayerNormV2, GaussianRadialBasisLayer)):
                for p_name, _ in mod.named_parameters():
                    if isinstance(mod, torch.nn.Linear) and "weight" in p_name:
                        continue
                    full = f"{mod_name}.{p_name}"
                    assert full in names
                    skip.add(full)
        return skip

    def forward(self, f_in, pos, batch, node_atom, **kwargs) -> torch.Tensor:
        edge_src, edge_dst = radius_graph(pos, r=self.max_radius, batch=batch, max_num_neighbors=1000)
        # radius_graph emits the edge list sorted by destination: skip the (host-synchronising) sortedness check
        return self.forward_edges(pos, batch, node_atom, edge_src, edge_dst, n_graphs=kwargs.get("n_graphs"),
                                  edges_sorted=True)

    def forward_edges(self, pos, batch, node_atom, edge_src, edge_dst, graph=None, n_graphs=None,
                      edges_sorted: bool = False, edge_vec=None) -> torch.Tensor:
        """Everything after neighbour search (ref :868-899); free of host synchronisation when ``graph`` (the CSR of
        the destination-sorted edge list) and ``n_graphs`` are supplied, so it can be captured in a CUDA graph.
        Contract: the kernels need the edge list sorted by destination.  A caller-supplied ``graph`` carries its own
        order; otherwise the list is checked (one host synchronisation) and, when unsorted, everything per-edge is
        permuted - unless the caller vouches for the order with ``edges_sorted=True``.  ``edge_vec`` overrides
        ``pos[src] - pos[dst]`` (periodic cells: the caller adds the image offsets; needs a sorted edge list)."""
        if edge_vec is not None and not (edges_sorted or graph is not None):
            raise ValueError("edge_vec needs a destination-sorted edge list (edges_sorted=True or a graph)")
        if graph is None:
            graph = ops.Graph(edge_src, edge_dst, pos.shape[0], check_sorted=not edges_sorted)
            if graph.perm is not None:      # unsorted input: work on the sorted copy
                edge_src, edge_dst = graph.src, graph.dst
                graph.perm = None
        edge_vec, edge_length, edge_sh = edge_features(self.irreps_edge_attr, pos, graph, edge_vec)
        atom_embedding, _attr, _onehot = self.atom_embed(self._atom_remap[node_atom])
        edge_length_embedding = self.rbf(edge_length)
        served = hoist_radial(self, edge_length_embedding)     # first Linear of all radial MLPs: one GEMM
        try:
            edge_degree_embedding = self.edge_deg_embed(atom_embedding, edge_sh, edge_length_embedding, edge_src, edge_dst,
                                                        batch, graph=graph)
            node_features = atom_embedding + edge_degree_embedding
            node_attr = torch.ones_like(node_features.narrow(1, 0, 1))
            node_attr._eqf_all_ones = True          # lets the node-level FCTPs skip the multiply by the constant 1
            node_features = _run_blocks(self.blocks, node_features, self.irreps_node_embedding, node_attr, edge_src, edge_dst,
                                        edge_sh, edge_length_embedding, batch, graph)
        finally:
            clear_hoisted(served)
        node_features = self.norm(node_features, batch=batch)
        if self.out_dropout is not None:
            node_features = self.out_dropout(node_features)
        outputs = self.head(node_features)
        outputs = self.scale_scatter(outputs, batch, dim=0, dim_size=n_graphs)
        if self.scale is not None:
            outputs = self.scale * outputs
        return outputs


def edge_features(irreps_edge_attr, pos, graph, edge_vec=None):
    """``(edge_vec, edge_length, edge_sh)`` of a destination-sorted graph (ref :866-870).  When the edge irreps are the plain
    harmonics ``0 .. lmax <= 3`` and the vector is ``pos[src] - pos[dst]`` this is ONE kernel (``ops.EdgeGeometry``; its
    backward scatters to ``pos``); a caller-supplied ``edge_vec`` (periodic images) or other irreps take the torch chain."""
    ls = [ir.l for mul, ir in irreps_edge_attr for _ in range(mul)]
    if (edge_vec is None and ls == list(range(len(ls))) and 1 <= len(ls) <= 4 and pos.is_cuda and pos.dtype == torch.float32
            and graph.perm is None and graph.n_edges > 0):
        return ops.edge_geometry(pos, graph, len(ls) - 1)
    if edge_vec is None:
        edge_vec = pos.index_select(0, graph.src) - pos.index_select(0, graph.dst)
    edge_sh = o3.spherical_harmonics(l=irreps_edge_attr, x=edge_vec, normalize=True, normalization="component")
    return edge_vec, edge_vec.norm(dim=1), edge_sh


def hoist_radial(model, edge_scalars):
    """``radial_func.hoist_first_layers`` over every ``RadialProfile`` of ``model`` (list cached on the instance)."""
    mods = model.__dict__.get("_rad_modules")
    if mods is None:
        mods = [m for m in model.modules() if isinstance(m, RadialProfile)]
        model.__dict__["_rad_modules"] = mods
    return hoist_first_layers(mods, edge_scalars)


def _run_blocks(blocks, node_features, irreps, node_attr, edge_src, edge_dst, edge_sh, edge_scalars, batch, graph):
    """The transformer blocks; consecutive blocks that support it keep the node features in planar blocks."""
    planar = None
    for blk in blocks:
        kw = dict(node_attr=node_attr, edge_src=edge_src, edge_dst=edge_dst, edge_attr=edge_sh, edge_scalars=edge_scalars,
                  batch=batch, graph=graph)
        if getattr(blk, "supports_planar", False) and ops.fused_ok(node_features if planar is None else planar[0]):
            if planar is None:
                planar = ops.to_planar(node_features, Irreps(irreps))
            planar = blk.forward_planar(planar, **kw)
        else:
            if planar is not None:
                node_features, planar = ops.from_planar(planar), None
            node_features = blk(node_input=node_features, **kw)
    return ops.from_planar(planar) if planar is not None else node_features


def _qm9(irreps_in, radius, num_basis, atomref, task_mean, task_std, **over):
    cfg = dict(irreps_in=irreps_in, irreps_node_embedding="128x0e+64x1e+32x2e", num_layers=6,
               irreps_node_attr="1x0e", irreps_sh="1x0e+1x1e+1x2e", max_radius=radius, number_of_basis=num_basis,
               fc_neurons=[64, 64], irreps_feature="512x0e", irreps_head="32x0e+16x1e+8x2e", num_heads=4,
               irreps_pre_attn=None, rescale_degree=False, nonlinear_message=False,
               irreps_mlp_mid="384x0e+192x1e+96x2e", norm_layer="layer", alpha_drop=0.2, proj_drop=0.0,
               out_drop=0.0, drop_path_rate=0.0, mean=task_mean, std=task_std, scale=None, atomref=atomref)
    cfg.update(over)
    return GraphAttentionTransformer(**cfg)


@register_model
def graph_attention_transformer_l2(irreps_in, radius, num_basis=128, atomref=None, task_mean=None, task_std=None, **kwargs):
    return _qm9(irreps_in, radius, num_basis, atomref, task_mean, task_std)


@register_model
def graph_attention_transformer_nonlinear_l2(irreps_in, radius, num_basis=128, atomref=None, task_mean=None,
                                             task_std=None, **kwargs):
    return _qm9(irreps_in, radius, num_basis, atomref, task_mean, task_std, nonlinear_message=True)


@register_model
def graph_attention_transformer_nonlinear_l2_e3(irreps_in, radius, num_basis=128, atomref=None, task_mean=None,
                                                task_std=None, **kwargs):
    return _qm9(irreps_in, radius, num_basis, atomref, task_mean, task_std, nonlinear_message=True,
                irreps_node_embedding="128x0e+32x0o+32x1e+32x1o+16x2e+16x2o", irreps_sh="1x0e+1x1o+1x2e",
                irreps_head="32x0e+8x0o+8x1e+8x1o+4x2e+4x2o", irreps_mlp_mid="384x0e+96x0o+96x1e+96x1o+48x2e+48x2o")


@register_model
def graph_attention_transformer_nonlinear_bessel_l2(irreps_in, radius, num_basis=128, atomref=None, task_mean=None,
                                                    task_std=None, **kwargs):
    return _qm9(irreps_in, radius, num_basis, atomref, task_mean, task_std, nonlinear_message=True, basis_type="bessel")


@register_model
def graph_attention_transformer_nonlinear_bessel_l2_drop01(irreps_in, radius, num_basis=128, atomref=None,
                                                           task_mean=None, task_std=None, **kwargs):
    return _qm9(irreps_in, radius, num_basis, atomref, task_mean, task_std, nonlinear_message=True,
                basis_type="bessel", alpha_drop=0.1)


@register_model
def graph_attention_transformer_nonlinear_bessel_l2_drop00(irreps_in, radius, num_basis=128, atomref=None,
                                                           task_mean=None, task_std=None, **kwargs):
    return _qm9(irreps_in, radius, num_basis, atomref, task_mean, task_std, nonlinear_message=True,
                basis_type="bessel", alpha_drop=0.0)
