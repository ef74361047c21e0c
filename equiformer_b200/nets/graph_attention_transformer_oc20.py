"""OC20 IS2RE Equiformer (drop-in for ``nets/graph_attention_transformer_oc20.py``): the QM9 blocks with periodic
boundary conditions, 84 atom types plus a tag embedding (0 sub-surface, 1 surface, 2 adsorbate) and OC20 statistics.

Same constructor arguments, attribute / ``state_dict`` names and ``forward(data)`` contract as the reference
(``:72-117``, ``:296-380``); ``data`` is any object with ``pos, batch, atomic_numbers, tags, cell`` (+ ``edge_index,
cell_offsets`` when ``otf_graph=False``).  What the reference gets from ``ocpmodels`` - ``radius_graph_pbc`` and
``get_pbc_distances`` (``:267-302``) - is ``equiformer_b200.graph.radius_graph_pbc`` here: two sm_90a kernels around one
prefix sum, destination-sorted, same pair / image order and the same distance masks.  The energy head is the feed-forward
one of the shipped IS2RE configurations; the auxiliary-task and attention heads (``use_auxiliary_task``,
``use_attention_head``), learned node attributes and atom-pair edge attributes are outside the benchmarked path and raise.
"""
from __future__ import annotations

import torch

from .. import o3, ops
from ..graph import radius_graph, radius_graph_pbc
from ..o3 import Irreps
from .drop import EquivariantDropout
from .fast_activation import Activation
from .gaussian_rbf import GaussianRadialBasisLayer
from .graph_attention_transformer import (_run_blocks, clear_hoisted, hoist_radial, EdgeDegreeEmbeddingNetwork, NodeEmbeddingNetwork, ScaledScatter,
                                          TransBlock, get_norm_layer)
from .layer_norm import EquivariantLayerNormV2
from .registry import register_model
from .tensor_product_rescale import LinearRS

_RESCALE = True
_USE_BIAS = True
_MAX_ATOM_TYPE = 84
_NUM_TAGS = 3
# statistics of IS2RE 100k, max_radius = 5, max_neighbors = 100 (reference :60-66: the last assignment wins)
_AVG_NUM_NODES = 77.81317
_AVG_DEGREE = 23.395238876342773


class GraphAttentionTransformerOC20(torch.nn.Module):
    _block_cls = TransBlock

    def __init__(self, num_atoms=None, bond_feat_dim=None, num_targets=1, irreps_node_embedding="256x0e+128x1e",
                 num_layers=6, irreps_node_attr="1x0e", use_node_attr=False, irreps_sh="1x0e+1x1e", max_radius=6.0,
                 number_of_basis=128, fc_neurons=[64, 64], use_atom_edge_attr=False, irreps_atom_edge_attr="8x0e",
                 irreps_feature="512x0e", irreps_head="32x0e+16x1e", num_heads=8, irreps_pre_attn=None,
                 rescale_degree=False, nonlinear_message=False, irreps_mlp_mid="768x0e+384x1e", norm_layer="layer",
                 alpha_drop=0.2, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0, use_auxiliary_task=False,
                 auxiliary_head_dropout=True, use_attention_head=False, otf_graph=False, use_pbc=True, max_neighbors=50):
        super().__init__()
        if use_node_attr or use_atom_edge_attr or use_auxiliary_task or use_attention_head:
            raise NotImplementedError("learned node attributes, atom-pair edge attributes, the auxiliary task and the attention "
                                      "head are not used by the IS2RE configurations of the hot path (out of scope)")
        self.max_radius, self.number_of_basis = max_radius, number_of_basis
        self.alpha_drop, self.proj_drop, self.out_drop = alpha_drop, proj_drop, out_drop
        self.drop_path_rate, self.norm_layer = drop_path_rate, norm_layer
        self.otf_graph, self.use_pbc, self.max_neighbors = otf_graph, use_pbc, max_neighbors
        self.use_node_attr = use_node_attr
        self.irreps_node_attr = Irreps(irreps_node_attr)
        self.irreps_node_embedding = Irreps(irreps_node_embedding)
        self.lmax = self.irreps_node_embedding.lmax
        self.irreps_feature = Irreps(irreps_feature)
        self.num_layers = num_layers
        self.irreps_edge_attr = Irreps(irreps_sh) if irreps_sh is not None else Irreps.spherical_harmonics(self.lmax)
        self.use_atom_edge_attr = use_atom_edge_attr
        self.irreps_atom_edge_attr = Irreps(irreps_atom_edge_attr)
        self.fc_neurons = [self.number_of_basis] + list(fc_neurons)
        self.irreps_head = Irreps(irreps_head)
        self.num_heads = num_heads
        self.irreps_pre_attn = irreps_pre_attn
        self.rescale_degree, self.nonlinear_message = rescale_degree, nonlinear_message
        self.irreps_mlp_mid = Irreps(irreps_mlp_mid)

        self.atom_embed = NodeEmbeddingNetwork(self.irreps_node_embedding, _MAX_ATOM_TYPE)
        self.tag_embed = NodeEmbeddingNetwork(self.irreps_node_embedding, _NUM_TAGS)
        self.attr_embed = None
        self.rbf = GaussianRadialBasisLayer(self.number_of_basis, cutoff=self.max_radius)
        self.edge_deg_embed = EdgeDegreeEmbeddingNetwork(self.irreps_node_embedding, self.irreps_edge_attr,
                                                         self.fc_neurons, _AVG_DEGREE)
        self.edge_src_embed = self.edge_dst_embed = None
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
        self.irreps_feature_scalars = Irreps([(mul, ir) for mul, ir in self.irreps_feature if ir.l == 0 and ir.p == 1])
        self.head = torch.nn.Sequential(
            LinearRS(self.irreps_feature, self.irreps_feature_scalars, rescale=_RESCALE),
            Activation(self.irreps_feature_scalars, acts=[torch.nn.SiLU()]),
            LinearRS(self.irreps_feature_scalars, Irreps("1x0e")))
        self.scale_scatter = ScaledScatter(_AVG_NUM_NODES)
        self.use_auxiliary_task, self.use_attention_head = use_auxiliary_task, use_attention_head
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
            if isinstance(mod, (torch.nn.Linear, torch.nn.LayerNorm, EquivariantLayerNormV2, GaussianRadialBasisLayer)):
                for p_name, _ in mod.named_parameters():
                    if isinstance(mod, torch.nn.Linear) and "weight" in p_name:
                        continue
                    skip.add(f"{mod_name}.{p_name}")
        return skip

    # ---------------------------------------------------------------------------------------------- graph construction
    def build_graph(self, data):
        """``(edge_src, edge_dst, edge_vec)`` of the frame batch: on-the-fly periodic neighbour list (``otf_graph``) or the
        one carried by ``data`` (``edge_index``, ``cell_offsets``); without PBC the plain radius graph (ref :267-302)."""
        pos, batch = data.pos, data.batch
        if self.use_pbc:
            if self.otf_graph or getattr(data, "edge_index", None) is None:
                edge_index, cell_offsets, _d2 = radius_graph_pbc(pos, batch, data.cell, self.max_radius, self.max_neighbors)
            else:
                edge_index, cell_offsets = data.edge_index, data.cell_offsets
            edge_src, edge_dst = edge_index[0], edge_index[1]
            cell = data.cell.to(device=pos.device, dtype=pos.dtype)
            offsets = torch.bmm(cell_offsets.to(pos.dtype).view(-1, 1, 3), cell.index_select(0, batch.index_select(0, edge_dst))).view(-1, 3)
            edge_vec = pos.index_select(0, edge_src) - pos.index_select(0, edge_dst) + offsets
        else:
            edge_src, edge_dst = radius_graph(pos, r=self.max_radius, batch=batch, max_num_neighbors=self.max_neighbors)
            edge_vec = pos.index_select(0, edge_src) - pos.index_select(0, edge_dst)
        return edge_src, edge_dst, edge_vec

    def forward(self, data):
        edge_src, edge_dst, edge_vec = self.build_graph(data)
        n_graphs = getattr(data, "n_graphs", None)
        return self.forward_edges(edge_vec, data.batch, data.atomic_numbers.long(), data.tags.long(), edge_src, edge_dst,
                                  n_graphs=n_graphs)

    def forward_edges(self, edge_vec, batch, atomic_numbers, tags, edge_src, edge_dst, graph=None, n_graphs=None,
                      edges_sorted: bool = True):
        """Everything after the neighbour search (ref :305-380); host-synchronisation free when ``graph`` and ``n_graphs``
        are supplied (CUDA-graph capturable).  The periodic neighbour list is sorted by destination."""
        n_nodes = batch.shape[0]
        edge_sh = o3.spherical_harmonics(l=self.irreps_edge_attr, x=edge_vec, normalize=True, normalization="component")
        atom_embedding, _attr, _onehot = self.atom_embed(atomic_numbers)
        tag_embedding, _, _ = self.tag_embed(tags)
        edge_length_embedding = self.rbf(edge_vec.norm(dim=1), atomic_numbers, edge_src, edge_dst)
        if graph is None:
            graph = ops.Graph(edge_src, edge_dst, n_nodes, check_sorted=not edges_sorted)
            if graph.perm is not None:
                raise ValueError("forward_edges needs the edge list sorted by destination")
        served = hoist_radial(self, edge_length_embedding)     # first Linear of every radial MLP: one GEMM
        try:
            edge_degree_embedding = self.edge_deg_embed(atom_embedding, edge_sh, edge_length_embedding, edge_src, edge_dst,
                                                        batch, graph=graph)
            node_features = atom_embedding + tag_embedding + edge_degree_embedding
            node_attr = torch.ones_like(node_features.narrow(1, 0, 1))
            node_attr._eqf_all_ones = True
            node_features = _run_blocks(self.blocks, node_features, self.irreps_node_embedding, node_attr, edge_src, edge_dst,
                                        edge_sh, edge_length_embedding, batch, graph)
        finally:
            clear_hoisted(served)
        node_features = self.norm(node_features, batch=batch)
        outputs = self.out_dropout(node_features) if self.out_dropout is not None else node_features
        outputs = self.head(outputs)
        return self.scale_scatter(outputs, batch, dim=0, dim_size=n_graphs)


@register_model
def graph_attention_transformer_oc20(num_atoms=None, bond_feat_dim=None, num_targets=1, **kwargs):
    """The class ocpmodels registers as ``graph_attention_transformer`` (reference :69); keyword arguments are the ``model:``
    block of the OC20 configuration files, e.g. oc20/configs/is2re/all/graph_attention_transformer/l1_256_nonlinear_*.yml."""
    return GraphAttentionTransformerOC20(num_atoms, bond_feat_dim, num_targets, **kwargs)


# the model block of oc20/configs/is2re/all/graph_attention_transformer/l1_256_nonlinear_g@2_local.yml:5-31
OC20_L1_256_NONLINEAR = dict(
    irreps_node_embedding="256x0e+128x1e", num_layers=6, irreps_node_attr="1x0e", use_node_attr=False,
    irreps_sh="1x0e+1x1e", max_radius=5.0, number_of_basis=128, fc_neurons=[64, 64], use_atom_edge_attr=False,
    irreps_atom_edge_attr="1x0e", irreps_feature="512x0e", irreps_head="32x0e+16x1e", num_heads=8,
    irreps_pre_attn="256x0e+128x1e", rescale_degree=False, nonlinear_message=True, irreps_mlp_mid="768x0e+384x1e",
    norm_layer="layer", alpha_drop=0.2, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0, otf_graph=True, use_pbc=True,
    max_neighbors=500)
