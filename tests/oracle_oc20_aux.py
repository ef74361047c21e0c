"""ORACLE extension (test infrastructure, never on the product path): the OC20 model with the IS2RS auxiliary head,
restated op-for-op on CPU torch from ``nets/graph_attention_transformer_oc20.py`` (paths relative to the reference tree).

``oracle.equiformer_ref.model_forward_oc20`` stops at the energy.  The ``*_aux_*`` OC20 configurations add two things it
does not state, and this module states them on top of its primitives:

* ``graph_attention_pre`` - ``GraphAttention.forward`` (graph_attention_transformer.py:482-527) with an ``irreps_pre_attn``
  that differs from the input irreps: the auxiliary head reads ``irreps_feature`` (e.g. ``512x0e+256x1e``) and merges it
  down to ``irreps_pre_attn`` (``256x0e+128x1e``) before the depth-wise products.  The blocks' oracle
  (``equiformer_ref.graph_attention``) assumes the two are equal.
* ``model_forward_oc20_aux`` - the forward of :305-380 with ``use_auxiliary_task=True``: blocks, final norm, the
  feed-forward energy head on the ``0e`` part of the feature (:169-179; a ``1e`` block of ``irreps_feature`` has no path
  to it) and the auxiliary head on the normed features (:372-379), returning ``(energy [G, 1], aux [N, 3])``.

Pinned by ``tests/golden/reference_model_oc20_aux_small.npz`` (the reference file itself, float64) in
``tests/test_oc20_aux.py``.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import e3nn_ref as e3
from oracle import equiformer_ref as R


def graph_attention_pre(params, prefix: str, irreps_in, irreps_pre, irreps_edge, irreps_head, num_heads, irreps_node_output,
                        nonlinear_message, x, edge_src, edge_dst, edge_sh, edge_scalars):
    """GraphAttention.forward - graph_attention_transformer.py:482-527 (eval mode), ``irreps_pre_attn = irreps_pre``."""
    n = x.shape[0]
    pre = irreps_pre
    heads_all, _ = R.sort_irreps_even_first([(m, l, p) for _ in range(num_heads) for m, l, p in irreps_head])
    heads_all = e3.simplify(heads_all)
    mul_alpha = sum(m for m, l, p in heads_all if l == 0 and p == 1)
    a_head = mul_alpha // num_heads
    irreps_alpha = [(mul_alpha, 0, 1)]

    msg_src = R.linear_rs(params, f"{prefix}.merge_src", irreps_in, pre, x)                     # :485
    msg_dst = R.linear_rs(params, f"{prefix}.merge_dst", irreps_in, pre, x, bias=False)         # :486
    message = msg_src.index_select(0, edge_src) + msg_dst.index_select(0, edge_dst)             # :487

    if nonlinear_message:
        dtp_out, dtp_ins = R.dtp_instructions(pre, irreps_edge, pre)
        weight = R.radial_profile(params, f"{prefix}.sep_act.dtp_rad", edge_scalars)            # :490
        message = e3.tensor_product(message, edge_sh, weight, pre, irreps_edge, dtp_out, dtp_ins, False)   # :491
        alpha = R.linear_rs(params, f"{prefix}.sep_alpha", dtp_out, irreps_alpha, message)      # :492
        alpha = R.vec2heads(alpha, [(a_head, 0, 1)], num_heads)                                 # :493
        scalars, gates, gated = R.irreps2gate(pre)
        lin_out = e3.simplify(scalars + gates + gated)
        value = R.linear_rs(params, f"{prefix}.sep_act.lin", e3.simplify(dtp_out), lin_out, message)   # :494
        value = R.gate(value, scalars, gates, gated)                                            # :495
        v_out, v_ins = R.dtp_instructions(pre, irreps_edge, heads_all)
        value = e3.tensor_product(value, edge_sh, params[f"{prefix}.sep_value.dtp.tp.weight"], pre, irreps_edge,
                                  v_out, v_ins, True)                                           # :496
        value = R.linear_rs(params, f"{prefix}.sep_value.lin", e3.simplify(v_out), heads_all, value)
        value = R.vec2heads(value, irreps_head, num_heads)                                      # :497
    else:
        attn_all = e3.simplify(irreps_alpha + heads_all)
        s_out, s_ins = R.dtp_instructions(pre, irreps_edge, attn_all)
        weight = R.radial_profile(params, f"{prefix}.sep.dtp_rad", edge_scalars)
        message = e3.tensor_product(message, edge_sh, weight, pre, irreps_edge, s_out, s_ins, False)   # :499
        message = R.linear_rs(params, f"{prefix}.sep.lin", e3.simplify(s_out), attn_all, message)
        message = R.vec2heads(message, e3.simplify([(a_head, 0, 1)] + list(irreps_head)), num_heads)  # :500
        alpha = message[:, :, :a_head]                                                          # :502
        value = message[:, :, a_head:]                                                          # :503

    alpha = e3.smooth_leaky_relu(alpha, 0.2) * e3.NORMALIZE2MOM["smooth_leaky_relu_0.2"]        # :506
    alpha = torch.einsum("bik,aik->bi", alpha, params[f"{prefix}.alpha_dot"])                   # :507
    alpha = R.pyg_softmax(alpha, edge_dst, n).unsqueeze(-1)                                     # :508-509
    attn = R.scatter_sum(value * alpha, edge_dst, n)                                            # :512-513
    attn = R.heads2vec(attn, irreps_head)                                                       # :514
    return R.linear_rs(params, f"{prefix}.proj", heads_all, irreps_node_output, attn)           # :522


def model_forward_oc20_aux(params, cfg: R.Config, pos, cell, batch, atomic_numbers, tags, n_graphs: int, edge_src, edge_dst,
                           cell_offsets, irreps_pre_attn: str):
    """GraphAttentionTransformerOC20.forward with ``use_auxiliary_task=True`` - graph_attention_transformer_oc20.py:305-380
    (eval mode, feed-forward energy head).  Returns ``(energy [G, 1], aux [N, 3])``."""
    dtype = pos.dtype
    emb = e3.parse_irreps(cfg.irreps_node_embedding)
    feat = e3.parse_irreps(cfg.irreps_feature)
    irreps_edge = e3.parse_irreps(cfg.irreps_sh)
    edge_vec = R.pbc_edge_vectors(pos, cell, batch, edge_src, edge_dst, cell_offsets)                # :283-296
    edge_sh = e3.spherical_harmonics([l for _, l, _ in irreps_edge], edge_vec, True, "component")   # :311-312
    onehot = F.one_hot(atomic_numbers, cfg.max_atom_type).to(dtype)
    atom_embedding = R.linear_rs(params, "atom_embed.atom_type_lin", [(cfg.max_atom_type, 0, 1)], emb, onehot)   # :316
    tag_embedding = R.linear_rs(params, "tag_embed.atom_type_lin", [(3, 0, 1)], emb, F.one_hot(tags, 3).to(dtype))  # :318
    edge_scalars = R.gaussian_rbf(params, "rbf", edge_vec.norm(dim=1), cfg.max_radius)              # :320-321
    deg = R.edge_degree_embedding(params, "edge_deg_embed", cfg, pos.shape[0], edge_sh, edge_scalars, edge_src, edge_dst,
                                  dtype)
    x = atom_embedding + tag_embedding + deg                                                        # :329
    node_attr = torch.ones_like(x[:, 0:1])
    for i in range(cfg.num_layers):                                                                 # :337-341
        out_irreps = emb if i != cfg.num_layers - 1 else feat
        x = R.trans_block(params, f"blocks.{i}", cfg, emb, out_irreps, x, node_attr, edge_src, edge_dst, edge_sh,
                          edge_scalars)
    x = R.layer_norm_v2(params, "norm", feat, x)                                                    # :343
    scalars = [(m, l, p) for m, l, p in feat if l == 0 and p == 1]                                  # :169-173
    h = R.linear_rs(params, "head.0", feat, scalars, x)                                             # :175-178, :369
    h = F.silu(h) * e3.NORMALIZE2MOM["silu"]
    h = R.linear_rs(params, "head.2", scalars, [(1, 0, 1)], h)
    energy = R.scatter_sum(h, batch, n_graphs) / math.sqrt(cfg.avg_num_nodes)                       # :370
    aux_irreps = [(1, 1, -1)] if any(l == 1 and p == -1 for _, l, p in feat) else [(1, 1, 1)]       # :184-186
    aux = graph_attention_pre(params, "auxiliary_head", feat, e3.parse_irreps(irreps_pre_attn), irreps_edge,
                              e3.parse_irreps(cfg.irreps_head), cfg.num_heads, aux_irreps, cfg.nonlinear_message, x,
                              edge_src, edge_dst, edge_sh, edge_scalars)                            # :373-377
    return energy, aux
