"""ORACLE (test infrastructure, never on the product path): the reference's graph-attention path restated
op-for-op on CPU torch, parameterised by a ``state_dict`` with the reference's key names.

PINNED to outputs of the reference's own code, produced here by ``tests/golden/make_reference_golden.py`` and checked in
``tests/test_reference_golden.py``:
  * ``gaussian_rbf``, ``expnorm_rbf``, ``radial_profile``, ``layer_norm_v2`` - the reference modules run as they are
    (stub e3nn for ``Irreps`` parsing only): 1e-12;
  * ``model_forward`` / ``energy_and_forces`` and everything they call (``graph_attention``, ``trans_block``,
    ``feed_forward``, ``linear_rs``, ``edge_degree_embedding`` ...) - the reference's model files
    (``nets/graph_attention_transformer.py``, ``..._md17.py``, ``tensor_product_rescale.py``, ``fast_activation.py``,
    ``drop.py``) executed end to end on small configurations: energy 1e-11, forces 1e-10.
PARITY UNPINNED below that line: in those end-to-end runs the third-party calls (``o3.TensorProduct``,
``o3.spherical_harmonics``, ``e3nn.nn.Gate``, ``torch_scatter.scatter``, ``torch_geometric.utils.softmax``,
``torch_cluster.radius_graph``) are served by stubs built on ``oracle/e3nn_ref.py`` and the primitives of this file,
because e3nn / torch_scatter / PyG / torch_cluster are absent from the image - their numerics remain restated from
published behaviour (see ``oracle/e3nn_ref.py``).

Each function cites the reference lines it follows (paths relative to ``/root/reference``).  The execution style
mirrors the reference on purpose - one einsum per tensor-product instruction + ``cat``, ``index_select`` gathers,
``index_add_`` scatters, separate softmax passes - because this file is also the "reference-style" CPU baseline that
``bench.py`` times.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from . import e3nn_ref as e3

Params = Dict[str, torch.Tensor]


# ----------------------------------------------------------------------------------------------------------------
# primitives


def scatter_sum(x, index, dim_size):
    """torch_scatter.scatter(..., reduce='sum') - nets/graph_attention_transformer.py:513,700"""
    out = x.new_zeros((dim_size,) + tuple(x.shape[1:]))
    out.index_add_(0, index, x)
    return out


def pyg_softmax(src, index, num_nodes):
    """torch_geometric.utils.softmax (2.0.3): (src - max).exp() / (scatter_sum + 1e-16) - :508"""
    expanded = index.view(-1, *([1] * (src.dim() - 1))).expand_as(src)
    src_max = torch.full((num_nodes,) + tuple(src.shape[1:]), float("-inf"), dtype=src.dtype, device=src.device)
    src_max = src_max.scatter_reduce(0, expanded, src, reduce="amax", include_self=True)
    out = (src - src_max.index_select(0, index)).exp()
    out_sum = scatter_sum(out, index, num_nodes).index_select(0, index)
    return out / (out_sum + 1e-16)


def sort_irreps_even_first(irreps):
    """nets/tensor_product_rescale.py:224-231"""
    keyed = sorted((l, -p, i, mul) for i, (mul, l, p) in enumerate(irreps))
    inv = [i for _, _, i, _ in keyed]
    perm = [0] * len(inv)
    for new, old in enumerate(inv):
        perm[old] = new
    return [(mul, l, -negp) for l, negp, _, mul in keyed], perm


def dtp_instructions(irreps_in, irreps_edge, irreps_target):
    """DepthwiseTensorProduct - nets/graph_attention_transformer.py:157-183.  Returns (irreps_out_sorted, instructions)."""
    out, ins = [], []
    target = {(l, p) for _, l, p in irreps_target}
    for i, (mul, l1, p1) in enumerate(irreps_in):
        for j, (_, l2, p2) in enumerate(irreps_edge):
            for lo, po in e3.product_irreps(l1, p1, l2, p2):
                if (lo, po) in target or (lo, po) == (0, 1):
                    ins.append((i, j, len(out), "uvu"))
                    out.append((mul, lo, po))
    out_sorted, perm = sort_irreps_even_first(out)
    return out_sorted, [(i, j, perm[k], m) for i, j, k, m in ins]


def fctp_instructions(irreps_in1, irreps_in2, irreps_out):
    """FullyConnectedTensorProductRescale - nets/tensor_product_rescale.py:151-157"""
    return [(i1, i2, io, "uvw")
            for i1, (_, l1, p1) in enumerate(irreps_in1)
            for i2, (_, l2, p2) in enumerate(irreps_in2)
            for io, (_, lo, po) in enumerate(irreps_out)
            if (lo, po) in e3.product_irreps(l1, p1, l2, p2)]


def add_bias(out, irreps_out, params: Params, prefix: str):
    """forward_tp_rescale_bias - nets/tensor_product_rescale.py:126-136 (one bias per 0e entry of simplify())"""
    simp = e3.simplify(irreps_out)
    b = 0
    out = out.clone()
    for (mul, l, p), sl in zip(simp, e3.irreps_slices(simp)):
        if l == 0 and p == 1:
            key = f"{prefix}.bias.{b}"
            if key in params:
                out[:, sl] = out[:, sl] + params[key]
            b += 1
    return out


def linear_rs(params: Params, prefix: str, irreps_in, irreps_out, x, bias=True, y=None):
    """LinearRS / FCTP against a scalar second operand - nets/tensor_product_rescale.py:144-174"""
    in2 = [(1, 0, 1)]
    if y is None:
        y = torch.ones_like(x[:, 0:1])
    out = e3.tensor_product(x, y, params[f"{prefix}.tp.weight"], irreps_in, in2, irreps_out,
                            fctp_instructions(irreps_in, in2, irreps_out), shared_weights=True)
    return add_bias(out, irreps_out, params, prefix) if bias else out


def radial_profile(params: Params, prefix: str, x):
    """RadialProfile - nets/radial_func.py:9-50 (Linear, LayerNorm, SiLU) x2, Linear(no bias) + offset"""
    h = F.linear(x, params[f"{prefix}.net.0.weight"], params[f"{prefix}.net.0.bias"])
    h = F.silu(F.layer_norm(h, h.shape[-1:], params[f"{prefix}.net.1.weight"], params[f"{prefix}.net.1.bias"], 1e-5))
    h = F.linear(h, params[f"{prefix}.net.3.weight"], params[f"{prefix}.net.3.bias"])
    h = F.silu(F.layer_norm(h, h.shape[-1:], params[f"{prefix}.net.4.weight"], params[f"{prefix}.net.4.bias"], 1e-5))
    h = F.linear(h, params[f"{prefix}.net.6.weight"])
    return h + params[f"{prefix}.offset"].reshape(1, -1)


def irreps2gate(irreps):
    """nets/tensor_product_rescale.py:177-192"""
    scalars = e3.simplify([(m, l, p) for m, l, p in irreps if l == 0 and p == 1])
    gated = e3.simplify([(m, l, p) for m, l, p in irreps if not (l == 0 and p == 1)])
    gates = e3.simplify([(m, 0, 1) for m, _, _ in gated])
    return scalars, gates, gated


def gate(x, scalars, gates, gated):
    """Gate - nets/fast_activation.py:132-148 with normalize2mom-wrapped SiLU / sigmoid"""
    ns, ng = e3.irreps_dim(scalars), e3.irreps_dim(gates)
    s = F.silu(x[:, :ns]) * e3.NORMALIZE2MOM["silu"]
    if ng == 0:
        return s
    g = torch.sigmoid(x[:, ns:ns + ng]) * e3.NORMALIZE2MOM["sigmoid"]
    pieces, off, goff = [s], ns + ng, 0
    for mul, l, _ in gated:
        d = 2 * l + 1
        blk = x[:, off:off + mul * d].reshape(-1, mul, d)
        pieces.append((blk * g[:, goff:goff + mul].unsqueeze(-1)).reshape(-1, mul * d))
        off += mul * d
        goff += mul
    return torch.cat(pieces, dim=1)


def vec2heads(x, irreps_head, num_heads):
    """Vec2AttnHeads - nets/graph_attention_transformer.py:252-285"""
    n = x.shape[0]
    mid = [(mul * num_heads, l, p) for mul, l, p in irreps_head]
    return torch.cat([x[:, sl].reshape(n, num_heads, -1) for sl in e3.irreps_slices(mid)], dim=2)


def heads2vec(x, irreps_head):
    """AttnHeads2Vec - :289-316"""
    n = x.shape[0]
    return torch.cat([x[:, :, sl].reshape(n, -1) for sl in e3.irreps_slices(irreps_head)], dim=1)


def layer_norm_v2(params: Params, prefix: str, irreps, x, eps=1e-5):
    """EquivariantLayerNormV2 ('component') - nets/layer_norm.py:89-152"""
    w, b = params[f"{prefix}.affine_weight"], params[f"{prefix}.affine_bias"]
    out, off, iw, ib = [], 0, 0, 0
    for mul, l, p in irreps:
        d = 2 * l + 1
        f = x[:, off:off + mul * d].reshape(-1, mul, d)
        off += mul * d
        if l == 0 and p == 1:
            f = f - f.mean(dim=1, keepdim=True)
        norm = f.pow(2).mean(-1).mean(dim=1, keepdim=True)
        norm = (norm + eps).pow(-0.5) * w[None, iw:iw + mul]
        iw += mul
        f = f * norm.reshape(-1, mul, 1)
        if d == 1 and p == 1:
            f = f + b[ib:ib + mul].reshape(mul, 1)
            ib += mul
        out.append(f.reshape(-1, mul * d))
    return torch.cat(out, dim=-1)


# ----------------------------------------------------------------------------------------------------------------
# blocks


@dataclass
class Config:
    """Hyper-parameters of one registered model (nets/graph_attention_transformer.py:902-1016, ..._md17.py:330-519)."""
    irreps_node_embedding: str = "128x0e+64x1e+32x2e"
    irreps_sh: str = "1x0e+1x1e+1x2e"
    irreps_head: str = "32x0e+16x1e+8x2e"
    irreps_mlp_mid: str = "384x0e+192x1e+96x2e"
    irreps_feature: str = "512x0e"
    num_heads: int = 4
    num_layers: int = 6
    max_radius: float = 5.0
    number_of_basis: int = 128
    basis_type: str = "gaussian"
    nonlinear_message: bool = True
    max_atom_type: int = 5
    qm9_atom_remap: bool = True
    avg_degree: float = 15.57930850982666
    avg_num_nodes: float = 18.03065905448718
    attention: str = "graph"          # "graph": GraphAttention / TransBlock; "dot_product": nets/dp_attention_transformer.py


def graph_attention(params: Params, prefix: str, irreps_in, irreps_edge, irreps_head, num_heads, irreps_node_output,
                    nonlinear_message, x, edge_src, edge_dst, edge_sh, edge_scalars):
    """GraphAttention.forward - nets/graph_attention_transformer.py:482-527 (eval mode: dropouts are identity)."""
    n = x.shape[0]
    pre = irreps_in  # irreps_pre_attn=None in every shipped config
    heads_all, _ = sort_irreps_even_first([(m, l, p) for _ in range(num_heads) for m, l, p in irreps_head])
    heads_all = e3.simplify(heads_all)
    mul_alpha = sum(m for m, l, p in heads_all if l == 0 and p == 1)
    a_head = mul_alpha // num_heads
    irreps_alpha = [(mul_alpha, 0, 1)]

    msg_src = linear_rs(params, f"{prefix}.merge_src", irreps_in, pre, x)                       # :485
    msg_dst = linear_rs(params, f"{prefix}.merge_dst", irreps_in, pre, x, bias=False)           # :486
    message = msg_src.index_select(0, edge_src) + msg_dst.index_select(0, edge_dst)             # :487

    if nonlinear_message:
        dtp_out, dtp_ins = dtp_instructions(pre, irreps_edge, pre)
        weight = radial_profile(params, f"{prefix}.sep_act.dtp_rad", edge_scalars)              # :490
        message = e3.tensor_product(message, edge_sh, weight, pre, irreps_edge, dtp_out, dtp_ins, False)   # :491
        alpha = linear_rs(params, f"{prefix}.sep_alpha", dtp_out, irreps_alpha, message)        # :492
        alpha = vec2heads(alpha, [(a_head, 0, 1)], num_heads)                                   # :493
        scalars, gates, gated = irreps2gate(pre)
        lin_out = e3.simplify(scalars + gates + gated)
        value = linear_rs(params, f"{prefix}.sep_act.lin", e3.simplify(dtp_out), lin_out, message)   # :494
        value = gate(value, scalars, gates, gated)                                              # :495
        v_out, v_ins = dtp_instructions(pre, irreps_edge, heads_all)
        value = e3.tensor_product(value, edge_sh, params[f"{prefix}.sep_value.dtp.tp.weight"], pre, irreps_edge,
                                  v_out, v_ins, True)                                           # :496 (SeparableFCTP :239-243)
        value = linear_rs(params, f"{prefix}.sep_value.lin", e3.simplify(v_out), heads_all, value)
        value = vec2heads(value, irreps_head, num_heads)                                        # :497
    else:
        attn_all = e3.simplify(irreps_alpha + heads_all)
        s_out, s_ins = dtp_instructions(pre, irreps_edge, attn_all)
        weight = radial_profile(params, f"{prefix}.sep.dtp_rad", edge_scalars)
        message = e3.tensor_product(message, edge_sh, weight, pre, irreps_edge, s_out, s_ins, False)   # :499
        message = linear_rs(params, f"{prefix}.sep.lin", e3.simplify(s_out), attn_all, message)
        message = vec2heads(message, e3.simplify([(a_head, 0, 1)] + list(irreps_head)), num_heads)     # :500
        alpha = message[:, :, :a_head]                                                          # :502
        value = message[:, :, a_head:]                                                          # :503

    alpha = e3.smooth_leaky_relu(alpha, 0.2) * e3.NORMALIZE2MOM["smooth_leaky_relu_0.2"]        # :506
    alpha = torch.einsum("bik,aik->bi", alpha, params[f"{prefix}.alpha_dot"])                   # :507
    alpha = pyg_softmax(alpha, edge_dst, n).unsqueeze(-1)                                       # :508-509
    attn = scatter_sum(value * alpha, edge_dst, n)                                              # :512-513
    attn = heads2vec(attn, irreps_head)                                                         # :514
    return linear_rs(params, f"{prefix}.proj", heads_all, irreps_node_output, attn)             # :522


def dot_product_attention(params: Params, prefix: str, irreps_in, irreps_edge, irreps_head, num_heads, irreps_node_output,
                          x, edge_src, edge_dst, edge_sh, edge_scalars, rescale_degree: bool = False):
    """DotProductAttention.forward - nets/dp_attention_transformer.py:128-162 (eval mode; ``rescale_degree`` multiplies
    by degree / _AVG_DEGREE, :148-152 - the division belongs to this variant only)"""
    n = x.shape[0]
    pre = irreps_in
    heads_q, _ = sort_irreps_even_first([(m, l, p) for _ in range(num_heads) for m, l, p in irreps_head])
    heads_q = e3.simplify(heads_q)                                                              # :93-96
    heads_kv, _ = sort_irreps_even_first([(m, l, p) for _ in range(2 * num_heads) for m, l, p in irreps_head])
    heads_kv = e3.simplify(heads_kv)                                                            # :98-100
    q = linear_rs(params, f"{prefix}.query", irreps_in, heads_q, x)                             # :131
    q = vec2heads(q, irreps_head, num_heads)                                                    # :132
    norm = 1.0 / math.sqrt(sum(m for m, _, _ in irreps_head))                                   # ScaleFactor :49-66
    q = torch.cat([q[..., sl] * (norm / math.sqrt(2 * l + 1))
                   for sl, (_, l, _) in zip(e3.irreps_slices(irreps_head), irreps_head)], dim=-1)
    msg_src = linear_rs(params, f"{prefix}.merge_src", irreps_in, pre, x)                       # :135
    msg_dst = linear_rs(params, f"{prefix}.merge_dst", irreps_in, pre, x, bias=False)           # :136
    kv = msg_src.index_select(0, edge_src) + msg_dst.index_select(0, edge_dst)                  # :137
    s_out, s_ins = dtp_instructions(pre, irreps_edge, heads_kv)                                 # SeparableFCTP, no activation
    weight = radial_profile(params, f"{prefix}.key_value.dtp_rad", edge_scalars)
    kv = e3.tensor_product(kv, edge_sh, weight, pre, irreps_edge, s_out, s_ins, False)          # :138
    kv = linear_rs(params, f"{prefix}.key_value.lin", e3.simplify(s_out), heads_kv, kv)
    kv = vec2heads(kv, irreps_head, 2 * num_heads)                                              # :139
    k, v = kv[:, :num_heads], kv[:, num_heads:]                                                 # :141-142
    alpha = torch.einsum("bik,bik->bi", q.index_select(0, edge_dst), k)                         # :145
    alpha = pyg_softmax(alpha, edge_dst, n).unsqueeze(-1)                                       # :146-147
    attn = scatter_sum(v * alpha, edge_dst, n)                                                  # :150-151
    attn = heads2vec(attn, irreps_head)                                                         # :146
    if rescale_degree:                                                                          # :148-152
        degree = torch.zeros(n, dtype=x.dtype, device=x.device).index_add_(
            0, edge_dst, torch.ones(edge_dst.numel(), dtype=x.dtype, device=x.device))
        attn = attn * degree.view(-1, 1) / 15.57930850982666
    return linear_rs(params, f"{prefix}.proj", heads_q, irreps_node_output, attn)               # :154


def feed_forward(params: Params, prefix: str, irreps_in, irreps_mid, irreps_out, x, node_attr):
    """FeedForwardNetwork.forward - :566-571"""
    scalars, gates, gated = irreps2gate(irreps_mid)
    gate_in = e3.simplify(scalars + gates + gated) if e3.irreps_dim(gated) > 0 else irreps_mid
    h = linear_rs(params, f"{prefix}.fctp_1", irreps_in, gate_in, x, y=node_attr)
    h = gate(h, scalars, gates, gated)
    gate_out = scalars + gated
    return linear_rs(params, f"{prefix}.fctp_2", gate_out if e3.irreps_dim(gated) > 0 else irreps_mid, irreps_out, h,
                     y=node_attr)


def trans_block(params: Params, prefix: str, cfg: Config, irreps_in, irreps_out, x, node_attr, edge_src, edge_dst,
                edge_sh, edge_scalars):
    """TransBlock.forward - :639-667 (drop_path = 0)"""
    irreps_edge = e3.parse_irreps(cfg.irreps_sh)
    h = layer_norm_v2(params, f"{prefix}.norm_1", irreps_in, x)
    if cfg.attention == "dot_product":      # DPTransBlock.forward - nets/dp_attention_transformer.py:228-255, same skeleton
        h = dot_product_attention(params, f"{prefix}.dpa", irreps_in, irreps_edge, e3.parse_irreps(cfg.irreps_head),
                                  cfg.num_heads, irreps_in, h, edge_src, edge_dst, edge_sh, edge_scalars)
    else:
        h = graph_attention(params, f"{prefix}.ga", irreps_in, irreps_edge, e3.parse_irreps(cfg.irreps_head),
                            cfg.num_heads, irreps_in, cfg.nonlinear_message, h, edge_src, edge_dst, edge_sh, edge_scalars)
    y = x + h
    h = layer_norm_v2(params, f"{prefix}.norm_2", irreps_in, y)
    h = feed_forward(params, f"{prefix}.ffn", irreps_in, e3.parse_irreps(cfg.irreps_mlp_mid), irreps_out, h, node_attr)
    if irreps_in != irreps_out:
        y = linear_rs(params, f"{prefix}.ffn_shortcut", irreps_in, irreps_out, y, y=node_attr)
    return y + h


def edge_degree_embedding(params: Params, prefix: str, cfg: Config, n_nodes, edge_sh, edge_scalars, edge_src, edge_dst,
                          dtype):
    """EdgeDegreeEmbeddingNetwork.forward - :725-733"""
    emb = e3.parse_irreps(cfg.irreps_node_embedding)
    irreps_edge = e3.parse_irreps(cfg.irreps_sh)
    ones = torch.ones((n_nodes, 1), dtype=dtype, device=edge_sh.device)
    feats = linear_rs(params, f"{prefix}.exp", [(1, 0, 1)], emb, ones)
    weight = radial_profile(params, f"{prefix}.rad", edge_scalars)
    dw_out, dw_ins = dtp_instructions(emb, irreps_edge, emb)
    ef = e3.tensor_product(feats.index_select(0, edge_src), edge_sh, weight, emb, irreps_edge, dw_out, dw_ins, False)
    ef = linear_rs(params, f"{prefix}.proj", e3.simplify(dw_out), emb, ef)
    return scatter_sum(ef, edge_dst, n_nodes) / math.sqrt(cfg.avg_degree)


def gaussian_rbf(params: Params, prefix: str, dist, cutoff):
    """GaussianRadialBasisLayer.forward - nets/gaussian_rbf.py:32-40 (pi truncated to 3.14159 as in :6)"""
    x = (dist / cutoff).unsqueeze(-1)
    x = params[f"{prefix}.weight"] * x + params[f"{prefix}.bias"]
    std = params[f"{prefix}.std"].abs() + 1e-5
    a = (2 * 3.14159) ** 0.5
    return torch.exp(-0.5 * (((x - params[f"{prefix}.mean"]) / std) ** 2)) / (a * std)


def expnorm_rbf(params: Params, prefix: str, dist, cutoff):
    """ExpNormalSmearing.forward - nets/expnorm_rbf.py:73-78 with CosineCutoff(0, cutoff) :11-33"""
    d = dist.unsqueeze(-1)
    cut = 0.5 * (torch.cos(d * math.pi / cutoff) + 1.0) * (d < cutoff).to(d.dtype)
    alpha = 5.0 / cutoff
    return cut * torch.exp(-params[f"{prefix}.betas"] * (torch.exp(alpha * (-d)) - params[f"{prefix}.means"]) ** 2)


def radius_graph(pos, r, batch):
    """torch_cluster.radius_graph contract - :866-867: (src=neighbour, dst=centre ascending), no self loops, d < r."""
    d2 = (pos[:, None, :] - pos[None, :, :]).pow(2).sum(-1)
    mask = (d2 < r * r) & (batch[:, None] == batch[None, :])
    mask.fill_diagonal_(False)
    dst, src = mask.nonzero(as_tuple=True)
    return src, dst


def model_forward(params: Params, cfg: Config, pos, batch, node_atom, n_graphs: int,
                  edges: Optional[Tuple[torch.Tensor, torch.Tensor]] = None):
    """GraphAttentionTransformer.forward - :864-899 (QM9) / GraphAttentionTransformerMD17.forward energy part - md17 :276-314."""
    dtype = pos.dtype
    emb = e3.parse_irreps(cfg.irreps_node_embedding)
    feat = e3.parse_irreps(cfg.irreps_feature)
    irreps_edge = e3.parse_irreps(cfg.irreps_sh)
    if edges is None:
        edge_src, edge_dst = radius_graph(pos.detach(), cfg.max_radius, batch)
    else:
        edge_src, edge_dst = edges
    edge_vec = pos.index_select(0, edge_src) - pos.index_select(0, edge_dst)
    edge_sh = e3.spherical_harmonics([l for _, l, _ in irreps_edge], edge_vec, True, "component")   # :869-870
    if cfg.qm9_atom_remap:
        node_atom = node_atom.new_tensor([-1, 0, -1, -1, -1, -1, 1, 2, 3, 4])[node_atom]        # :872
    onehot = F.one_hot(node_atom, cfg.max_atom_type).to(dtype)
    atom_embedding = linear_rs(params, "atom_embed.atom_type_lin", [(cfg.max_atom_type, 0, 1)], emb, onehot)
    edge_length = edge_vec.norm(dim=1)
    if cfg.basis_type == "gaussian":
        edge_scalars = gaussian_rbf(params, "rbf", edge_length, cfg.max_radius)
    else:
        edge_scalars = expnorm_rbf(params, "rbf", edge_length, cfg.max_radius)
    deg = edge_degree_embedding(params, "edge_deg_embed", cfg, pos.shape[0], edge_sh, edge_scalars, edge_src, edge_dst,
                                dtype)
    x = atom_embedding + deg
    node_attr = torch.ones_like(x[:, 0:1])
    for i in range(cfg.num_layers):
        out_irreps = emb if i != cfg.num_layers - 1 else feat
        x = trans_block(params, f"blocks.{i}", cfg, emb, out_irreps, x, node_attr, edge_src, edge_dst, edge_sh,
                        edge_scalars)
    x = layer_norm_v2(params, "norm", feat, x)
    h = linear_rs(params, "head.0", feat, feat, x)
    h = F.silu(h) * e3.NORMALIZE2MOM["silu"]
    h = linear_rs(params, "head.2", feat, [(1, 0, 1)], h)
    return scatter_sum(h, batch, n_graphs) / math.sqrt(cfg.avg_num_nodes)                      # :894


def pbc_edge_vectors(pos, cell, batch, edge_src, edge_dst, cell_offsets):
    """ocpmodels ``get_pbc_distances`` as consumed at nets/graph_attention_transformer_oc20.py:283-296:
    ``pos[src] - pos[dst] + cell_offsets @ cell[frame]`` (rows of ``cell`` = lattice vectors)."""
    cells = cell.to(pos.dtype).index_select(0, batch.index_select(0, edge_dst))
    offsets = torch.bmm(cell_offsets.to(pos.dtype).view(-1, 1, 3), cells).view(-1, 3)
    return pos.index_select(0, edge_src) - pos.index_select(0, edge_dst) + offsets


def nearest_neighbours_mask(centre, d2, max_neighbors):
    """ocpmodels ``get_max_neighbors_mask``: keep the ``max_neighbors`` smallest ``d2`` of every centre; equal ``d2``
    keep list order.  An exact lexicographic sort on (centre, d2, list position)."""
    centre_np = centre.cpu().numpy()
    d2_np = d2.detach().cpu().double().numpy()
    keep = np.ones(centre_np.shape[0], dtype=bool)
    if max_neighbors is None or centre_np.size == 0:
        return torch.from_numpy(keep)
    order = np.lexsort((np.arange(centre_np.size), d2_np, centre_np))
    sorted_centre = centre_np[order]
    first = np.searchsorted(sorted_centre, sorted_centre, side="left")
    keep[order] = np.arange(order.size) - first < max_neighbors
    return torch.from_numpy(keep)


def radius_graph_pbc(pos, batch, cell, r, max_neighbors=None, budget=2 ** 25):
    """ocpmodels ``radius_graph_pbc`` (as consumed at nets/graph_attention_transformer_oc20.py:267-302) in float64, on
    the device of ``pos``: every (centre i, atom j, image n) of one frame with ``1e-4 < |pos_j + n . cell - pos_i|^2 <=
    r^2``; rows of ``cell [n_frames, 3, 3]`` are the lattice vectors.

    Each frame enumerates ``ceil(r / height) + 1`` images per lattice vector, one shell more than can hold a neighbour
    of an atom inside the cell, so that a short repetition count elsewhere shows up as missing pairs.  Hits are ordered
    by centre, then j, then image (a slowest, c fastest); with ``max_neighbors`` each centre keeps its nearest hits by
    exact ``d2`` (``nearest_neighbours_mask``).  Centres are evaluated in chunks of about ``budget`` float64 elements.
    Returns ``(edge_index [2, E] = (j, i), cell_offsets [E, 3] int64, d2 [E] float64)``."""
    pos, cell = pos.detach().double(), cell.detach().to(pos.device, torch.float64)
    r2 = float(r) ** 2
    srcs, dsts, offs, d2s = [], [], [], []
    for f in range(cell.shape[0]):
        idx = (batch == f).nonzero().flatten()
        if idx.numel() == 0:
            continue
        a, b, c = cell[f]
        volume = float(torch.dot(a, torch.linalg.cross(b, c)).abs())
        heights = [volume / float(torch.linalg.cross(u, v).norm()) for u, v in ((b, c), (c, a), (a, b))]
        reps = [math.ceil(float(r) / h) + 1 for h in heights]
        imgs = torch.tensor([(na, nb, nc) for na in range(-reps[0], reps[0] + 1) for nb in range(-reps[1], reps[1] + 1)
                             for nc in range(-reps[2], reps[2] + 1)], dtype=torch.int64, device=pos.device)
        shift = imgs.double() @ cell[f]                                                         # [n_img, 3]
        p = pos[idx]
        image_pos = (p[:, None, :] + shift[None, :, :]).reshape(-1, 3)                        # [(j, img), 3]
        chunk = max(1, budget // (3 * image_pos.shape[0]))
        for i0 in range(0, idx.numel(), chunk):
            centres = p[i0:i0 + chunk]
            d2 = (image_pos[None, :, :] - centres[:, None, :]).pow(2).sum(-1)                  # [i, (j, img)]
            i, t = ((d2 > 1e-4) & (d2 <= r2)).nonzero(as_tuple=True)
            srcs.append(idx[t // imgs.shape[0]])
            dsts.append(idx[i0 + i])
            offs.append(imgs[t % imgs.shape[0]])
            d2s.append(d2[i, t])
    if not srcs:
        return (torch.zeros(2, 0, dtype=torch.int64, device=pos.device), torch.zeros(0, 3, dtype=torch.int64, device=pos.device),
                torch.zeros(0, dtype=torch.float64, device=pos.device))
    src, dst, off, d2 = torch.cat(srcs), torch.cat(dsts), torch.cat(offs), torch.cat(d2s)
    order = torch.argsort(dst, stable=True)                                                     # frames in any order
    src, dst, off, d2 = src[order], dst[order], off[order], d2[order]
    keep = nearest_neighbours_mask(dst, d2, max_neighbors).to(pos.device)
    return torch.stack([src[keep], dst[keep]]), off[keep], d2[keep]


def model_forward_oc20(params: Params, cfg: Config, pos, cell, batch, atomic_numbers, tags, n_graphs: int, edge_src,
                       edge_dst, cell_offsets):
    """GraphAttentionTransformerOC20.forward - nets/graph_attention_transformer_oc20.py:305-380 (feed-forward energy head,
    no auxiliary task); the periodic neighbour list (ocpmodels ``radius_graph_pbc``) is an input.  ``cfg`` carries the OC20
    statistics (``avg_degree`` 23.395..., ``avg_num_nodes`` 77.81317, :60-66) and ``max_atom_type`` 84."""
    dtype = pos.dtype
    emb = e3.parse_irreps(cfg.irreps_node_embedding)
    feat = e3.parse_irreps(cfg.irreps_feature)
    irreps_edge = e3.parse_irreps(cfg.irreps_sh)
    edge_vec = pbc_edge_vectors(pos, cell, batch, edge_src, edge_dst, cell_offsets)                  # :283-296
    edge_sh = e3.spherical_harmonics([l for _, l, _ in irreps_edge], edge_vec, True, "component")   # :311-312
    onehot = F.one_hot(atomic_numbers, cfg.max_atom_type).to(dtype)
    atom_embedding = linear_rs(params, "atom_embed.atom_type_lin", [(cfg.max_atom_type, 0, 1)], emb, onehot)   # :316
    tag_embedding = linear_rs(params, "tag_embed.atom_type_lin", [(3, 0, 1)], emb, F.one_hot(tags, 3).to(dtype))  # :318
    edge_scalars = gaussian_rbf(params, "rbf", edge_vec.norm(dim=1), cfg.max_radius)                # :320-321
    deg = edge_degree_embedding(params, "edge_deg_embed", cfg, pos.shape[0], edge_sh, edge_scalars, edge_src, edge_dst,
                                dtype)
    x = atom_embedding + tag_embedding + deg                                                        # :329
    node_attr = torch.ones_like(x[:, 0:1])
    for i in range(cfg.num_layers):
        out_irreps = emb if i != cfg.num_layers - 1 else feat
        x = trans_block(params, f"blocks.{i}", cfg, emb, out_irreps, x, node_attr, edge_src, edge_dst, edge_sh,
                        edge_scalars)
    x = layer_norm_v2(params, "norm", feat, x)
    scalars = [(m, l, p) for m, l, p in feat if l == 0 and p == 1]
    h = linear_rs(params, "head.0", feat, scalars, x)                                               # :176-179
    h = F.silu(h) * e3.NORMALIZE2MOM["silu"]
    h = linear_rs(params, "head.2", scalars, [(1, 0, 1)], h)
    return scatter_sum(h, batch, n_graphs) / math.sqrt(cfg.avg_num_nodes)                          # :365-366


def energy_and_forces(params: Params, cfg: Config, pos, batch, node_atom, n_graphs: int, create_graph: bool = False):
    """GraphAttentionTransformerMD17.forward - nets/graph_attention_transformer_md17.py:276-327"""
    with torch.enable_grad():
        pos = pos.detach().clone().requires_grad_(True)
        energy = model_forward(params, cfg, pos, batch, node_atom, n_graphs)
        forces = -torch.autograd.grad(energy, pos, grad_outputs=torch.ones_like(energy), create_graph=create_graph)[0]
    return energy, forces


def cast_params(state_dict, dtype) -> Params:
    return {k: (v.detach().to("cpu", dtype) if v.is_floating_point() else v.detach().cpu()) for k, v in state_dict.items()}
