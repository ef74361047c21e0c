"""Dot-product-attention variant (drop-in for ``nets/dp_attention_transformer.py``; SURVEY.md 8f-4).

Same machinery as the graph-attention path - node-level per-degree GEMMs, the fused gather + depth-wise tensor product,
the per-degree edge linears, segment softmax and the segment sum - with the MLP attention logits replaced by scaled
``q . k``.  On CUDA the logits, the segment softmax, the attention dropout and the weighted sum run as one kernel pair
(``ops.DotSoftmaxAggregate``: ``eqf_attn_dot_softmax_aggregate`` and its backward), which reads the keys and values in
place from the key / value blocks; under ``create_graph`` (forces) its backward is rebuilt from the closed family.  The
chain it replaces - ``ops.EdgeDot`` (per edge and head, the dot product of an edge row with a node row), segment softmax,
``nn.Dropout``, ``ops.attention_aggregate`` on contiguous key and value halves - remains the route for CPU tensors and
layouts the kernel does not take.

Key / value layout: ``key_value`` emits ``irreps_head x 2H`` sorted and simplified, i.e. per degree a block of
``2 H m_l`` channels in which head ``g`` owns channels ``[g m_l, (g + 1) m_l)`` (``Vec2AttnHeads`` :252-285); the first
``H`` heads are the keys, the last ``H`` the values (ref :141-142) - a contiguous channel split of every planar block.
"""
from __future__ import annotations

import torch

from .. import ops
from ..o3 import Irreps
from .drop import EquivariantDropout
from .graph_attention_transformer import (_AVG_DEGREE, _RESCALE, AttnHeads2Vec, GraphAttentionTransformer, SeparableFCTP, TransBlock,
                                          Vec2AttnHeads, _graph_for, _is_sorted_simplified)
from .graph_attention_transformer_md17 import GraphAttentionTransformerMD17
from .registry import register_model
from .tensor_product_rescale import LinearRS

assert _RESCALE


class ScaleFactor(torch.nn.Module):
    """``x_l / (sqrt(num_irreps) sqrt(2l+1))`` on a head vector (ref :49-66)."""

    def __init__(self, irreps, normalization="component"):
        super().__init__()
        self.irreps = Irreps(irreps)
        self.channel_norm_factor = 1 / (self.irreps.num_irreps ** 0.5)

    def factors(self):
        return [self.channel_norm_factor / (ir.dim ** 0.5) for _, ir in self.irreps]

    def forward(self, x):
        out, idx = [], 0
        for (mul, ir), f in zip(self.irreps, self.factors()):
            out.append(x.narrow(-1, idx, mul * ir.dim) * f)
            idx += mul * ir.dim
        return torch.cat(out, dim=-1)


class DotProductAttention(torch.nn.Module):
    """Multi-head scaled dot-product attention over the edges of the radius graph (ref :70-165)."""

    def __init__(self, irreps_node_input, irreps_node_attr, irreps_edge_attr, irreps_node_output, fc_neurons,
                 irreps_head, num_heads, irreps_pre_attn=None, rescale_degree=False, alpha_drop=0.1, proj_drop=0.1):
        super().__init__()
        self.irreps_node_input = Irreps(irreps_node_input)
        self.irreps_node_attr = Irreps(irreps_node_attr)
        self.irreps_edge_attr = Irreps(irreps_edge_attr)
        self.irreps_node_output = Irreps(irreps_node_output)
        self.irreps_pre_attn = self.irreps_node_input if irreps_pre_attn is None else Irreps(irreps_pre_attn)
        self.irreps_head = Irreps(irreps_head)
        self.num_heads = num_heads
        self.rescale_degree = rescale_degree

        # the reference uses e3nn's plain ``Irreps.sort()`` here (odd before even; ref :90-97), not the even-first sort of
        # GraphAttention; the planar kernels need one entry per irrep in (l ascending, even first) order, so head irreps
        # that mix parities (where the two sorts differ) are refused rather than laid out differently from the reference
        if any(ir.p != 1 for _, ir in self.irreps_head):
            raise NotImplementedError("DotProductAttention with odd-parity head irreps: the reference's Irreps.sort() "
                                      "layout (odd before even) is not supported by the planar kernels")
        irreps_attn_heads, _, _ = (self.irreps_head * num_heads).sort()
        irreps_attn_heads = irreps_attn_heads.simplify()
        self.query = LinearRS(self.irreps_node_input, irreps_attn_heads)
        irreps_kv_heads, _, _ = (self.irreps_head * num_heads * 2).sort()
        irreps_kv_heads = irreps_kv_heads.simplify()
        self.merge_src = LinearRS(self.irreps_node_input, self.irreps_pre_attn, bias=True)
        self.merge_dst = LinearRS(self.irreps_node_input, self.irreps_pre_attn, bias=False)
        self.key_value = SeparableFCTP(self.irreps_pre_attn, self.irreps_edge_attr, irreps_kv_heads, fc_neurons,
                                       use_activation=False, norm_layer=None)
        self.vec2heads_q = Vec2AttnHeads(self.irreps_head, num_heads)
        self.vec2heads_kv = Vec2AttnHeads(self.irreps_head, num_heads * 2)
        self.scale_factor = ScaleFactor(self.irreps_head)
        self.heads2vec = AttnHeads2Vec(self.irreps_head)
        self.alpha_dropout = torch.nn.Dropout(alpha_drop) if alpha_drop != 0.0 else None
        self.proj = LinearRS(irreps_attn_heads, self.irreps_node_output)
        self.proj_drop = EquivariantDropout(self.irreps_node_output, drop_prob=proj_drop) if proj_drop != 0.0 else None

        if not _is_sorted_simplified(self.irreps_head):
            raise NotImplementedError("irreps_head must be sorted (l ascending, even first) with one entry per irrep")
        self._head_layout = ops.HeadLayout([ir.dim for _, ir in irreps_attn_heads], [mul for mul, _ in irreps_attn_heads],
                                           num_heads)

    @property
    def supports_planar(self) -> bool:
        return self.proj_drop is None or not self.training or getattr(self.proj_drop, "drop_prob", 1.0) == 0.0

    def forward(self, node_input, node_attr, edge_src, edge_dst, edge_attr, edge_scalars, batch, **kwargs):
        xs = ops.to_planar(node_input, self.irreps_node_input)
        node_output = ops.from_planar(self.forward_planar(xs, node_attr, edge_src, edge_dst, edge_attr, edge_scalars, batch,
                                                          **kwargs))
        if self.proj_drop is not None:
            node_output = self.proj_drop(node_output)
        return node_output

    def forward_planar(self, xs, node_attr, edge_src, edge_dst, edge_attr, edge_scalars, batch, **kwargs):
        n_nodes = xs[0].shape[0]
        graph = _graph_for(edge_src, edge_dst, n_nodes, kwargs)
        edge_attr = graph.sort_edges(edge_attr).contiguous()
        edge_scalars = graph.sort_edges(edge_scalars)

        q = [t * f for t, f in zip(self.query.planar(xs), self.scale_factor.factors())]          # [ref :131-133]
        m_src = self.merge_src.planar(xs)                                                        # [ref :135-136]
        m_dst = self.merge_dst.planar(xs)
        kv = self.key_value                                                                      # [ref :137-138]
        weight = kv.dtp_rad(edge_scalars, add_offset=False)
        out = kv.lin.planar(kv.dtp.tp.planar_depthwise_gathered(graph, m_src, m_dst, edge_attr, weight, kv.dtp_rad.offset))
        lay = self._head_layout
        if ops.dot_softmax_aggregate_ok(lay, q[0], graph):
            # [ref :139-152] q[dst] . k, segment softmax, dropout and the weighted sum in one kernel that reads the keys
            # and values in place; the mask is drawn as nn.Dropout draws it on the [E, H] weights (same generator use)
            keep = None
            if self.alpha_dropout is not None and self.training and self.alpha_dropout.p != 0.0:
                ones = torch.ones((graph.n_edges, lay.n_heads), device=q[0].device, dtype=q[0].dtype)
                keep = torch.nn.functional.dropout(ones, self.alpha_dropout.p, True)
            node = list(ops.DotSoftmaxAggregate.apply(lay, graph, keep, *[t.contiguous() for t in q],
                                                      *[t.contiguous() for t in out]))
        else:
            k = [t.narrow(2, 0, t.shape[2] // 2).contiguous() for t in out]                      # [ref :139-142]
            v = [t.narrow(2, t.shape[2] // 2, t.shape[2] // 2).contiguous() for t in out]
            z = ops.EdgeDot.apply(lay, graph, *k, *[t.contiguous() for t in q])                  # [ref :145]  q[dst] . k
            attn = ops.segment_softmax(z.contiguous(), graph)                                    # [ref :146]
            if self.alpha_dropout is not None:
                attn = self.alpha_dropout(attn)
            node = ops.attention_aggregate(lay, graph, attn.contiguous(), v)                     # [ref :149-152]
        if self.rescale_degree:                                                                  # [ref :154-158]
            degree = (graph.row_ptr[1:] - graph.row_ptr[:-1]).to(node[0].dtype).view(-1, 1, 1)
            node = [t * (degree / _AVG_DEGREE) for t in node]                                    # [ref :152] DP variant only
        return self.proj.planar(node)                                                            # [ref :160]

    def extra_repr(self) -> str:
        return f"rescale_degree={self.rescale_degree}"


class DPTransBlock(TransBlock):
    """LayerNorm -> DotProductAttention -> residual -> LayerNorm -> FFN -> residual (ref :167-255)."""

    _attn_name = "dpa"

    def _make_attention(self, fc_neurons, alpha_drop, proj_drop):
        return DotProductAttention(irreps_node_input=self.irreps_node_input, irreps_node_attr=self.irreps_node_attr,
                                   irreps_edge_attr=self.irreps_edge_attr, irreps_node_output=self.irreps_node_input,
                                   fc_neurons=fc_neurons, irreps_head=self.irreps_head, num_heads=self.num_heads,
                                   irreps_pre_attn=self.irreps_pre_attn, rescale_degree=self.rescale_degree,
                                   alpha_drop=alpha_drop, proj_drop=proj_drop)


class DotProductAttentionTransformer(GraphAttentionTransformer):
    """The QM9 model with ``DPTransBlock`` s (ref :258-413); Gaussian radial basis only, as in the reference."""

    _block_cls = DPTransBlock

    def __init__(self, irreps_in="5x0e", irreps_node_embedding="128x0e+64x1e+32x2e", num_layers=6, irreps_node_attr="1x0e",
                 irreps_sh="1x0e+1x1e+1x2e", max_radius=5.0, number_of_basis=128, fc_neurons=[64, 64],
                 irreps_feature="512x0e", irreps_head="32x0e+16x1o+8x2e", num_heads=4, irreps_pre_attn=None,
                 rescale_degree=False, nonlinear_message=False, irreps_mlp_mid="128x0e+64x1e+32x2e", norm_layer="layer",
                 alpha_drop=0.2, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0, mean=None, std=None, scale=None,
                 atomref=None):
        super().__init__(irreps_in=irreps_in, irreps_node_embedding=irreps_node_embedding, num_layers=num_layers,
                         irreps_node_attr=irreps_node_attr, irreps_sh=irreps_sh, max_radius=max_radius,
                         number_of_basis=number_of_basis, basis_type="gaussian", fc_neurons=fc_neurons,
                         irreps_feature=irreps_feature, irreps_head=irreps_head, num_heads=num_heads,
                         irreps_pre_attn=irreps_pre_attn, rescale_degree=rescale_degree, nonlinear_message=nonlinear_message,
                         irreps_mlp_mid=irreps_mlp_mid, norm_layer=norm_layer, alpha_drop=alpha_drop, proj_drop=proj_drop,
                         out_drop=out_drop, drop_path_rate=drop_path_rate, mean=mean, std=std, scale=scale, atomref=atomref)


@register_model
def dot_product_attention_transformer_l2(irreps_in, radius, num_basis=128, atomref=None, task_mean=None, task_std=None,
                                         **kwargs):
    return DotProductAttentionTransformer(
        irreps_in=irreps_in, irreps_node_embedding="128x0e+64x1e+32x2e", num_layers=6, irreps_node_attr="1x0e",
        irreps_sh="1x0e+1x1e+1x2e", max_radius=radius, number_of_basis=num_basis, fc_neurons=[64, 64],
        irreps_feature="512x0e", irreps_head="32x0e+16x1e+8x2e", num_heads=4, irreps_pre_attn=None, rescale_degree=False,
        nonlinear_message=False, irreps_mlp_mid="384x0e+192x1e+96x2e", norm_layer="layer", alpha_drop=0.2, proj_drop=0.0,
        out_drop=0.0, drop_path_rate=0.0, mean=task_mean, std=task_std, scale=None, atomref=atomref)


class DotProductAttentionTransformerMD17(GraphAttentionTransformerMD17):
    """The MD17 energy + force model with ``DPTransBlock`` s (drop-in for ``nets/dp_attention_transformer_md17.py`` :57-236)."""

    _block_cls = DPTransBlock

    def __init__(self, irreps_in="64x0e", irreps_node_embedding="128x0e+64x1e+32x2e", num_layers=6, irreps_node_attr="1x0e",
                 irreps_sh="1x0e+1x1e+1x2e", max_radius=5.0, number_of_basis=128, basis_type="gaussian", fc_neurons=[64, 64],
                 irreps_feature="512x0e", irreps_head="32x0e+16x1o+8x2e", num_heads=4, irreps_pre_attn=None,
                 rescale_degree=False, nonlinear_message=False, irreps_mlp_mid="128x0e+64x1e+32x2e", norm_layer="layer",
                 alpha_drop=0.2, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0, mean=None, std=None, scale=None,
                 atomref=None):
        super().__init__(irreps_in=irreps_in, irreps_node_embedding=irreps_node_embedding, num_layers=num_layers,
                         irreps_node_attr=irreps_node_attr, irreps_sh=irreps_sh, max_radius=max_radius,
                         number_of_basis=number_of_basis, basis_type=basis_type, fc_neurons=fc_neurons,
                         irreps_feature=irreps_feature, irreps_head=irreps_head, num_heads=num_heads,
                         irreps_pre_attn=irreps_pre_attn, rescale_degree=rescale_degree, nonlinear_message=nonlinear_message,
                         irreps_mlp_mid=irreps_mlp_mid, use_attn_head=False, norm_layer=norm_layer, alpha_drop=alpha_drop,
                         proj_drop=proj_drop, out_drop=out_drop, drop_path_rate=drop_path_rate, mean=mean, std=std,
                         scale=scale, atomref=atomref)


def _dp_md17(irreps_in, radius, num_basis, atomref, task_mean, task_std, **family):
    return DotProductAttentionTransformerMD17(
        irreps_in=irreps_in, num_layers=6, irreps_node_attr="1x0e", max_radius=radius, number_of_basis=num_basis,
        fc_neurons=[64, 64], basis_type="exp", irreps_feature="512x0e", num_heads=4, irreps_pre_attn=None,
        rescale_degree=False, nonlinear_message=False, norm_layer="layer", alpha_drop=0.0, proj_drop=0.0, out_drop=0.0,
        drop_path_rate=0.0, mean=task_mean, std=task_std, scale=None, atomref=atomref, **family)


@register_model
def dot_product_attention_transformer_exp_l2_md17(irreps_in, radius, num_basis=128, atomref=None, task_mean=None,
                                                  task_std=None, **kwargs):
    return _dp_md17(irreps_in, radius, num_basis, atomref, task_mean, task_std,
                    irreps_node_embedding="128x0e+64x1e+32x2e", irreps_sh="1x0e+1x1e+1x2e",
                    irreps_head="32x0e+16x1e+8x2e", irreps_mlp_mid="384x0e+192x1e+96x2e")


@register_model
def dot_product_attention_transformer_exp_l3_md17(irreps_in, radius, num_basis=128, atomref=None, task_mean=None,
                                                  task_std=None, **kwargs):
    return _dp_md17(irreps_in, radius, num_basis, atomref, task_mean, task_std,
                    irreps_node_embedding="128x0e+64x1e+64x2e+32x3e", irreps_sh="1x0e+1x1e+1x2e+1x3e",
                    irreps_head="32x0e+16x1e+16x2e+8x3e", irreps_mlp_mid="384x0e+192x1e+192x2e+96x3e")
