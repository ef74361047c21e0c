"""OC20 IS2RE model with dot-product attention (drop-in for ``nets/dp_attention_transformer_oc20.py``).

The reference file is the graph-attention OC20 model (``graph_attention_transformer_oc20.py``) with ``DPTransBlock`` s in
place of ``TransBlock`` s, a ``DotProductAttention`` auxiliary head, and no ``auxiliary_head_dropout`` /
``use_attention_head`` arguments (``:86-103``); the statistics, embeddings, periodic neighbour list, energy head and
``no_weight_decay()`` are the same.  So is this mirror: ``GraphAttentionTransformerOC20`` with ``_block_cls =
DPTransBlock``, the same attribute / ``state_dict`` names and ``forward(data)`` / ``forward_edges`` contract.  The
attention of every block runs on ``ops.DotSoftmaxAggregate``.  The IS2RS auxiliary head, learned node attributes and
atom-pair edge attributes are not implemented and raise (no shipped dot-product configuration uses them).
"""
from __future__ import annotations

from .dp_attention_transformer import DPTransBlock
from .graph_attention_transformer_oc20 import GraphAttentionTransformerOC20
from .registry import register_model


class DotProductAttentionTransformerOC20(GraphAttentionTransformerOC20):
    _block_cls = DPTransBlock

    def __init__(self, num_atoms=None, bond_feat_dim=None, num_targets=1, irreps_node_embedding="256x0e+128x1e",
                 num_layers=6, irreps_node_attr="1x0e", use_node_attr=False, irreps_sh="1x0e+1x1e", max_radius=6.0,
                 number_of_basis=128, fc_neurons=[64, 64], use_atom_edge_attr=False, irreps_atom_edge_attr="8x0e",
                 irreps_feature="512x0e", irreps_head="32x0e+16x1e", num_heads=8, irreps_pre_attn=None,
                 rescale_degree=False, nonlinear_message=False, irreps_mlp_mid="768x0e+384x1e", norm_layer="layer",
                 alpha_drop=0.2, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0, use_auxiliary_task=False,
                 otf_graph=False, use_pbc=True, max_neighbors=50):
        if use_auxiliary_task or use_node_attr or use_atom_edge_attr:
            raise NotImplementedError("the IS2RS auxiliary head, learned node attributes and atom-pair edge attributes "
                                      "of the dot-product OC20 model are not implemented (no shipped configuration uses "
                                      "them)")
        super().__init__(num_atoms, bond_feat_dim, num_targets, irreps_node_embedding=irreps_node_embedding,
                         num_layers=num_layers, irreps_node_attr=irreps_node_attr, use_node_attr=use_node_attr,
                         irreps_sh=irreps_sh, max_radius=max_radius, number_of_basis=number_of_basis,
                         fc_neurons=fc_neurons, use_atom_edge_attr=use_atom_edge_attr,
                         irreps_atom_edge_attr=irreps_atom_edge_attr, irreps_feature=irreps_feature,
                         irreps_head=irreps_head, num_heads=num_heads, irreps_pre_attn=irreps_pre_attn,
                         rescale_degree=rescale_degree, nonlinear_message=nonlinear_message,
                         irreps_mlp_mid=irreps_mlp_mid, norm_layer=norm_layer, alpha_drop=alpha_drop,
                         proj_drop=proj_drop, out_drop=out_drop, drop_path_rate=drop_path_rate,
                         use_auxiliary_task=False, otf_graph=otf_graph, use_pbc=use_pbc, max_neighbors=max_neighbors)


@register_model
def dp_attention_transformer_oc20(num_atoms=None, bond_feat_dim=None, num_targets=1, **kwargs):
    """The class ocpmodels registers as ``dp_attention_transformer`` (reference :74); keyword arguments are the ``model:``
    block of oc20/configs/is2re/all/dp_attention_transformer/l1_256_g@2_local.yml."""
    return DotProductAttentionTransformerOC20(num_atoms, bond_feat_dim, num_targets, **kwargs)


# the model block of oc20/configs/is2re/all/dp_attention_transformer/l1_256_g@2_local.yml:5-31
OC20_DP_L1_256 = dict(
    irreps_node_embedding="256x0e+128x1e", num_layers=8, irreps_node_attr="1x0e", use_node_attr=False,
    irreps_sh="1x0e+1x1e", max_radius=5.0, number_of_basis=128, fc_neurons=[64, 64], use_atom_edge_attr=False,
    irreps_atom_edge_attr="1x0e", irreps_feature="512x0e", irreps_head="32x0e+16x1e", num_heads=8,
    irreps_pre_attn="256x0e+128x1e", rescale_degree=False, nonlinear_message=False, irreps_mlp_mid="768x0e+384x1e",
    norm_layer="layer", alpha_drop=0.2, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0, otf_graph=True, use_pbc=True,
    max_neighbors=500)
