"""MD17 Equiformer: energies plus autograd forces (drop-in for ``nets/graph_attention_transformer_md17.py``).

Same blocks as the QM9 model with 64 one-hot atom types, the exp-normal radial basis and
``forces = -d energy / d pos`` with ``create_graph=True`` (reference ``:276-327``), which is what makes every
edge kernel need a differentiable backward (``equiformer_b200/ops.py`` families).
"""
from __future__ import annotations

import torch

from .. import ops
from ..o3 import Irreps
from .bessel_rbf import RadialBasis
from .drop import EquivariantDropout
from .fast_activation import Activation
from .gaussian_rbf import GaussianRadialBasisLayer
from .graph_attention_transformer import (_run_blocks, edge_features, EdgeDegreeEmbeddingNetwork, GraphAttention, NodeEmbeddingNetwork,
                                          ScaledScatter, TransBlock, get_norm_layer, norm_segments, radial_basis)
from .graph_norm import EquivariantGraphNorm
from .layer_norm import EquivariantLayerNormV2
from .registry import register_model
from .tensor_product_rescale import LinearRS
from ..graph import radius_graph

_RESCALE = True
_USE_BIAS = True
_MAX_ATOM_TYPE = 64
# QM9 statistics re-used for MD17 by the reference (:46-49)
_AVG_NUM_NODES = 18.03065905448718
_AVG_DEGREE = 15.57930850982666


class GraphAttentionTransformerMD17(torch.nn.Module):
    _block_cls = TransBlock      # DPTransBlock in the dot-product variant (nets/dp_attention_transformer.py)

    def __init__(self, irreps_in="64x0e", irreps_node_embedding="128x0e+64x1e+32x2e", num_layers=6,
                 irreps_node_attr="1x0e", irreps_sh="1x0e+1x1e+1x2e", max_radius=5.0, number_of_basis=128,
                 basis_type="gaussian", fc_neurons=[64, 64], irreps_feature="512x0e",
                 irreps_head="32x0e+16x1o+8x2e", num_heads=4, irreps_pre_attn=None, rescale_degree=False,
                 nonlinear_message=False, irreps_mlp_mid="128x0e+64x1e+32x2e", use_attn_head=False,
                 norm_layer="layer", alpha_drop=0.2, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0,
                 mean=None, std=None, scale=None, atomref=None):
        super().__init__()
        self.max_radius, self.number_of_basis = max_radius, number_of_basis
        self.alpha_drop, self.proj_drop, self.out_drop = alpha_drop, proj_drop, out_drop
        self.drop_path_rate, self.use_attn_head, self.norm_layer = drop_path_rate, use_attn_head, norm_layer
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
        self.rescale_degree, self.nonlinear_message = rescale_degree, nonlinear_message
        self.irreps_mlp_mid = Irreps(irreps_mlp_mid)

        self.atom_embed = NodeEmbeddingNetwork(self.irreps_node_embedding, _MAX_ATOM_TYPE)
        self.basis_type = basis_type
        self.rbf = radial_basis(basis_type, self.number_of_basis, self.max_radius, ("gaussian", "bessel", "exp"))
        self.edge_deg_embed = EdgeDegreeEmbeddingNetwork(self.irreps_node_embedding, self.irreps_edge_attr,
                                                         self.fc_neurons, _AVG_DEGREE)
        self.blocks = torch.nn.ModuleList()
        for i in range(num_layers):
            out = self.irreps_node_embedding if i != num_layers - 1 else self.irreps_feature
            self.blocks.append(self._block_cls(
                irreps_node_input=self.irreps_node_embedding, irreps_node_attr=self.irreps_node_attr,
                irreps_edge_attr=self.irreps_edge_attr, irreps_node_output=out, fc_neurons=self.fc_neurons,
                irreps_head=self.irreps_head, num_heads=num_heads, irreps_pre_attn=irreps_pre_attn,
                rescale_degree=rescale_degree, nonlinear_message=nonlinear_message, alpha_drop=alpha_drop,
                proj_drop=proj_drop, drop_path_rate=drop_path_rate, irreps_mlp_mid=self.irreps_mlp_mid,
                norm_layer=norm_layer))
        self.norm = get_norm_layer(norm_layer)(self.irreps_feature)
        self.out_dropout = EquivariantDropout(self.irreps_feature, out_drop) if out_drop != 0.0 else None
        if use_attn_head:
            self.head = GraphAttention(irreps_node_input=self.irreps_feature, irreps_node_attr=self.irreps_node_attr,
                                       irreps_edge_attr=self.irreps_edge_attr, irreps_node_output=Irreps("1x0e"),
                                       fc_neurons=self.fc_neurons, irreps_head=self.irreps_head, num_heads=num_heads,
                                       irreps_pre_attn=irreps_pre_attn, rescale_degree=rescale_degree,
                                       nonlinear_message=nonlinear_message, alpha_drop=alpha_drop, proj_drop=proj_drop)
        else:
            self.head = torch.nn.Sequential(
                LinearRS(self.irreps_feature, self.irreps_feature, rescale=_RESCALE),
                Activation(self.irreps_feature, acts=[torch.nn.SiLU()]),
                LinearRS(self.irreps_feature, Irreps("1x0e"), rescale=_RESCALE))
        self.scale_scatter = ScaledScatter(_AVG_NUM_NODES)
        self.apply(self._init_weights)

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
        for mod_name, mod in self.named_modules():
            if isinstance(mod, (torch.nn.Linear, torch.nn.LayerNorm, EquivariantLayerNormV2, EquivariantGraphNorm,
                                GaussianRadialBasisLayer, RadialBasis)):
                for p_name, _ in mod.named_parameters():
                    if isinstance(mod, torch.nn.Linear) and "weight" in p_name:
                        continue
                    skip.add(f"{mod_name}.{p_name}")
        return skip

    @torch.enable_grad()
    def forward(self, node_atom, pos, batch):
        pos = pos.requires_grad_(True)
        edge_src, edge_dst = radius_graph(pos, r=self.max_radius, batch=batch, max_num_neighbors=1000)
        return self.forward_edges(node_atom, pos, batch, edge_src, edge_dst)

    @torch.enable_grad()
    def forward_edges(self, node_atom, pos, batch, edge_src, edge_dst, graph=None, n_graphs=None):
        """Everything after the neighbour search (ref :283-327): energies and ``-dE/dpos`` with ``create_graph=True``.
        ``pos`` must require grad; with ``graph`` (CSR of the destination-sorted edge list) and ``n_graphs`` supplied nothing
        here synchronises with the host, so the whole energy + force step can be captured in a CUDA graph."""
        if graph is None:
            graph = ops.Graph(edge_src, edge_dst, pos.shape[0], check_sorted=False)
        _edge_vec, edge_length, edge_sh = edge_features(self.irreps_edge_attr, pos, graph)
        atom_embedding, _attr, _onehot = self.atom_embed(node_atom)
        edge_length_embedding = self.rbf(edge_length)
        edge_degree_embedding = self.edge_deg_embed(atom_embedding, edge_sh, edge_length_embedding, edge_src, edge_dst,
                                                    batch, graph=graph)
        node_features = atom_embedding + edge_degree_embedding
        node_attr = torch.ones_like(node_features.narrow(1, 0, 1))
        node_attr._eqf_all_ones = True
        seg = norm_segments(self, batch, n_graphs)
        node_features = _run_blocks(self.blocks, node_features, self.irreps_node_embedding, node_attr, edge_src, edge_dst,
                                    edge_sh, edge_length_embedding, batch, graph, **seg)
        node_features = self.norm(node_features, batch=batch, **seg)
        if self.out_dropout is not None:
            node_features = self.out_dropout(node_features)
        if self.use_attn_head:
            outputs = self.head(node_input=node_features, node_attr=node_attr, edge_src=edge_src, edge_dst=edge_dst,
                                edge_attr=edge_sh, edge_scalars=edge_length_embedding, batch=batch, graph=graph)
        else:
            outputs = self.head(node_features)
        outputs = self.scale_scatter(outputs, batch, dim=0, dim_size=n_graphs)
        if self.scale is not None:
            outputs = self.scale * outputs
        energy = outputs
        forces = -1 * torch.autograd.grad(energy, pos, grad_outputs=torch.ones_like(energy), create_graph=True)[0]
        return energy, forces


_L2 = dict(irreps_node_embedding="128x0e+64x1e+32x2e", irreps_sh="1x0e+1x1e+1x2e",
           irreps_head="32x0e+16x1e+8x2e", irreps_mlp_mid="384x0e+192x1e+96x2e")
_L2_E3 = dict(irreps_node_embedding="128x0e+32x0o+32x1e+32x1o+16x2e+16x2o", irreps_sh="1x0e+1x1o+1x2e",
              irreps_head="32x0e+8x0o+8x1e+8x1o+4x2e+4x2o", irreps_mlp_mid="384x0e+96x0o+96x1e+96x1o+48x2e+48x2o")
_L3 = dict(irreps_node_embedding="128x0e+64x1e+64x2e+32x3e", irreps_sh="1x0e+1x1e+1x2e+1x3e",
           irreps_head="32x0e+16x1e+16x2e+8x3e", irreps_mlp_mid="384x0e+192x1e+192x2e+96x3e")
_L3_E3 = dict(irreps_node_embedding="128x0e+64x0o+32x1e+32x1o+32x2e+32x2o+16x3e+16x3o",
              irreps_sh="1x0e+1x1o+1x2e+1x3o", irreps_head="32x0e+16x0o+8x1e+8x1o+8x2e+8x2o+4x3e+4x3o",
              irreps_mlp_mid="384x0e+192x0o+96x1e+96x1o+96x2e+96x2o+48x3e+48x3o")

# name -> (irreps family, overrides); hyper-parameters of record from the reference's registered configs (:330-519)
_CONFIGS = {
    "graph_attention_transformer_l2_md17": (_L2, dict(nonlinear_message=False, alpha_drop=0.2)),
    "graph_attention_transformer_nonlinear_l2_md17": (_L2, dict(alpha_drop=0.2)),
    "graph_attention_transformer_nonlinear_l2_e3_md17": (_L2_E3, dict(alpha_drop=0.2)),
    "graph_attention_transformer_nonlinear_bessel_l2_md17": (_L2, dict(basis_type="bessel", alpha_drop=0.0)),
    "graph_attention_transformer_nonlinear_exp_l2_md17": (_L2, dict(basis_type="exp", alpha_drop=0.0)),
    "graph_attention_transformer_nonlinear_exp_l3_md17": (_L3, dict(basis_type="exp", alpha_drop=0.0)),
    "graph_attention_transformer_nonlinear_attn_exp_l3_md17": (
        _L3, dict(basis_type="exp", alpha_drop=0.0, use_attn_head=True, irreps_feature="128x0e+64x1e+64x2e+32x3e")),
    "graph_attention_transformer_nonlinear_exp_l3_e3_md17": (_L3_E3, dict(basis_type="exp", alpha_drop=0.0)),
    "graph_attention_transformer_nonlinear_bessel_l3_md17": (_L3, dict(basis_type="bessel", alpha_drop=0.0)),
    "graph_attention_transformer_nonlinear_bessel_l3_e3_md17": (_L3_E3, dict(basis_type="bessel", alpha_drop=0.0)),
}


def _make(name):
    family, over = _CONFIGS[name]

    def build(irreps_in, radius, num_basis=128, atomref=None, task_mean=None, task_std=None, **kwargs):
        cfg = dict(irreps_in=irreps_in, num_layers=6, irreps_node_attr="1x0e", max_radius=radius,
                   number_of_basis=num_basis, fc_neurons=[64, 64], irreps_feature="512x0e", num_heads=4,
                   irreps_pre_attn=None, rescale_degree=False, nonlinear_message=True, norm_layer="layer",
                   proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0, mean=task_mean, std=task_std, scale=None,
                   atomref=atomref)
        cfg.update(family)
        cfg.update(over)
        return GraphAttentionTransformerMD17(**cfg)

    build.__name__ = name
    build.__qualname__ = name
    return register_model(build)


for _name in _CONFIGS:
    globals()[_name] = _make(_name)
