"""Equiformer for MD17 with DeNS - denoising non-equilibrium structures (drop-in for ``nets/equiformer_md17_dens.py``).

The MD17 model with three additions (reference ``:55-176``, ``:238-354``): the (noised atoms') forces are encoded as
spherical harmonics scaled by ``|F| / sqrt(3)`` and added to the node embeddings through ``force_embed``; the energy head
reads the scalar channels of a wider equivariant feature (``512x0e+256x1e+128x2e``); a ``GraphAttention`` head
(``denoising_pos_head``, output ``1x1e``) predicts the position noise of the corrupted atoms, returned in place of their
forces.  Same constructor arguments, attribute / ``state_dict`` names and ``forward(data)`` contract; every edge-level op
is the hot path of this package (planar blocks, sm_90a kernels, closed autograd families for the ``create_graph`` forces).
"""
from __future__ import annotations

import math

import torch

from .. import o3, ops
from ..graph import radius_graph
from ..o3 import Irreps
from .bessel_rbf import RadialBasis
from .drop import EquivariantDropout
from .fast_activation import Activation
from .gaussian_rbf import GaussianRadialBasisLayer
from .graph_attention_transformer import (_run_blocks, edge_features, EdgeDegreeEmbeddingNetwork, GraphAttention,
                                          NodeEmbeddingNetwork, ScaledScatter, TransBlock, get_norm_layer, norm_segments,
                                          radial_basis)
from .graph_norm import EquivariantGraphNorm
from .layer_norm import EquivariantLayerNormV2
from .registry import register_model
from .tensor_product_rescale import LinearRS

_RESCALE = True
_MAX_ATOM_TYPE = 64
_AVG_NUM_NODES = 18.03065905448718
_AVG_DEGREE = 15.57930850982666


class Equiformer_MD17_DeNS(torch.nn.Module):
    def __init__(self, irreps_in="64x0e", irreps_equivariant_inputs="1x0e+1x1e+1x2e",
                 irreps_node_embedding="128x0e+64x1e+32x2e", num_layers=6, irreps_node_attr="1x0e",
                 irreps_sh="1x0e+1x1e+1x2e", max_radius=5.0, number_of_basis=32, basis_type="exp", fc_neurons=[64, 64],
                 irreps_feature="512x0e+256x1e+128x2e", irreps_head="32x0e+16x1o+8x2e", num_heads=4,
                 irreps_pre_attn="128x0e+64x1e+32x2e", rescale_degree=False, nonlinear_message=True,
                 irreps_mlp_mid="128x0e+64x1e+32x2e", norm_layer="layer", alpha_drop=0.0, proj_drop=0.0, out_drop=0.0,
                 drop_path_rate=0.0, mean=None, std=None, scale=None, atomref=None, use_force_encoding=True):
        super().__init__()
        self.max_radius, self.number_of_basis = max_radius, number_of_basis
        self.alpha_drop, self.proj_drop, self.out_drop = alpha_drop, proj_drop, out_drop
        self.drop_path_rate, self.norm_layer = drop_path_rate, norm_layer
        self.task_mean, self.task_std, self.scale = mean, std, scale
        self.register_buffer("atomref", atomref)
        self.use_force_encoding = use_force_encoding
        self.irreps_node_attr = Irreps(irreps_node_attr)
        self.irreps_node_input = Irreps(irreps_in)
        self.irreps_node_equivariant_inputs = Irreps(irreps_equivariant_inputs)
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
        self.force_embed = LinearRS(self.irreps_node_equivariant_inputs, self.irreps_node_embedding, rescale=_RESCALE)
        self.blocks = torch.nn.ModuleList()
        for i in range(num_layers):
            out = self.irreps_node_embedding if i != num_layers - 1 else self.irreps_feature
            self.blocks.append(TransBlock(
                irreps_node_input=self.irreps_node_embedding, irreps_node_attr=self.irreps_node_attr,
                irreps_edge_attr=self.irreps_edge_attr, irreps_node_output=out, fc_neurons=self.fc_neurons,
                irreps_head=self.irreps_head, num_heads=num_heads, irreps_pre_attn=irreps_pre_attn,
                rescale_degree=rescale_degree, nonlinear_message=nonlinear_message, alpha_drop=alpha_drop,
                proj_drop=proj_drop, drop_path_rate=drop_path_rate, irreps_mlp_mid=self.irreps_mlp_mid,
                norm_layer=norm_layer))
        self.norm = get_norm_layer(norm_layer)(self.irreps_feature)
        self.out_dropout = EquivariantDropout(self.irreps_feature, out_drop) if out_drop != 0.0 else None
        scalars = Irreps([(mul, ir) for mul, ir in self.irreps_feature if ir.l == 0 and ir.p == 1])
        self.energy_head = torch.nn.Sequential(
            LinearRS(self.irreps_feature, scalars, rescale=_RESCALE),
            Activation(scalars, acts=[torch.nn.SiLU()]),
            LinearRS(scalars, Irreps("1x0e"), rescale=_RESCALE))
        self.scale_scatter = ScaledScatter(_AVG_NUM_NODES)
        has_1e = any(ir.l == 1 and ir.p == 1 for _, ir in self.irreps_node_equivariant_inputs)
        self.denoising_pos_head = GraphAttention(
            irreps_node_input=self.irreps_feature, irreps_node_attr=self.irreps_node_attr,
            irreps_edge_attr=self.irreps_edge_attr, irreps_node_output=Irreps("1x1e" if has_1e else "1x1o"),
            fc_neurons=self.fc_neurons, irreps_head=self.irreps_head, num_heads=num_heads, irreps_pre_attn=irreps_pre_attn,
            rescale_degree=rescale_degree, nonlinear_message=nonlinear_message, alpha_drop=alpha_drop, proj_drop=proj_drop)
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
    def forward(self, data):
        """``(energy, dy)`` of a batch (ref :238-354).  The attributes present on ``data`` select the branches as in the
        reference: ``force`` the force encoding (with ``noise_mask``), ``noise_mask`` the denoising head, and, only when
        ``use_force_encoding=False``, ``denoising_mask`` / ``denoising_pos_mask`` the masking of energies / outputs."""
        node_atom, pos, batch = data.z, data.pos, data.batch
        pos = pos.requires_grad_(True)
        edge_src, edge_dst = radius_graph(pos, r=self.max_radius, batch=batch, max_num_neighbors=1000)
        force = noise_mask = denoising_mask = denoising_pos_mask = None
        if hasattr(data, "force") and self.use_force_encoding:
            force, noise_mask = data.force, data.noise_mask
        if hasattr(data, "noise_mask"):
            noise_mask = data.noise_mask
            if not self.use_force_encoding:
                denoising_pos_mask = data.denoising_pos_mask
        if hasattr(data, "denoising_mask") and not self.use_force_encoding:
            denoising_mask = data.denoising_mask
        return self.forward_edges(node_atom, pos, batch, edge_src, edge_dst, force=force, noise_mask=noise_mask,
                                  n_graphs=getattr(data, "n_graphs", None), denoising_mask=denoising_mask,
                                  denoising_pos_mask=denoising_pos_mask)

    @torch.enable_grad()
    def forward_edges(self, node_atom, pos, batch, edge_src, edge_dst, force=None, noise_mask=None, graph=None,
                      n_graphs=None, denoising_mask=None, denoising_pos_mask=None):
        """Everything after the neighbour search: ``(energy, dy)`` with ``dy = -dE/dpos`` (``create_graph=True``) for
        the clean atoms and the predicted noise for the atoms in ``noise_mask``.

        * ``force`` ``[N, 3]`` (with ``noise_mask``) is encoded for the atoms in ``noise_mask`` when
          ``use_force_encoding``; without it the encoding input is zero.
        * ``noise_mask`` ``[N]`` bool runs the denoising head; without it ``dy`` is the forces of every atom.
        * ``denoising_mask`` / ``denoising_pos_mask`` (only read when ``use_force_encoding=False``) zero the energies /
          outputs of the denoised atoms, as the reference does.

        ``pos`` must require grad.  With ``graph`` (CSR of the destination-sorted edge list) and ``n_graphs`` supplied
        nothing here synchronises with the host, so the whole energy + force + denoising step can be captured in a CUDA
        graph."""
        if graph is None:
            graph = ops.Graph(edge_src, edge_dst, pos.shape[0], check_sorted=False)
        _vec, edge_length, edge_sh = edge_features(self.irreps_edge_attr, pos, graph)
        atom_embedding, _attr, _onehot = self.atom_embed(node_atom)
        edge_length_embedding = self.rbf(edge_length)
        edge_degree_embedding = self.edge_deg_embed(atom_embedding, edge_sh, edge_length_embedding, edge_src, edge_dst,
                                                    batch, graph=graph)
        node_features = atom_embedding + edge_degree_embedding
        node_attr = torch.ones_like(node_features.narrow(1, 0, 1))
        node_attr._eqf_all_ones = True

        # forces of the corrupted atoms as an equivariant input (ref :273-292)
        if force is not None and self.use_force_encoding:
            if noise_mask is None:
                raise ValueError("the force encoding needs noise_mask (the atoms whose forces are encoded)")
            force_sh = o3.spherical_harmonics(l=self.irreps_node_equivariant_inputs, x=force, normalize=True,
                                              normalization="component")
            force_sh = force_sh * noise_mask.to(force_sh.dtype).unsqueeze(-1)
            force_sh = force_sh * (force.norm(dim=1, keepdim=True) / math.sqrt(3.0))
        else:
            force_sh = torch.zeros((node_features.shape[0], self.irreps_node_equivariant_inputs.dim),
                                   device=node_features.device, dtype=node_features.dtype)
        node_features = node_features + self.force_embed(force_sh)

        seg = norm_segments(self, batch, n_graphs)
        node_features = _run_blocks(self.blocks, node_features, self.irreps_node_embedding, node_attr, edge_src, edge_dst,
                                    edge_sh, edge_length_embedding, batch, graph, **seg)
        node_features = self.norm(node_features, batch=batch, **seg)
        if self.out_dropout is not None:
            node_features = self.out_dropout(node_features)

        energy = self.energy_head(node_features)
        if denoising_mask is not None and not self.use_force_encoding:
            energy = energy * (~denoising_mask).to(energy.dtype).view(-1, 1)
        energy = self.scale_scatter(energy, batch, dim=0, dim_size=n_graphs)
        if self.scale is not None:
            energy = self.scale * energy
        forces = -1 * torch.autograd.grad(energy, pos, grad_outputs=torch.ones_like(energy), create_graph=True)[0]

        if noise_mask is not None:
            noise = self.denoising_pos_head(node_input=node_features, node_attr=node_attr, edge_src=edge_src,
                                            edge_dst=edge_dst, edge_attr=edge_sh, edge_scalars=edge_length_embedding,
                                            batch=batch, graph=graph, n_graphs=n_graphs)
            mask = noise_mask.view(-1, 1)
            outputs_dy = torch.where(mask, noise, forces)          # forces of clean atoms, predicted noise of corrupted ones
            if not self.use_force_encoding:
                if denoising_pos_mask is None:
                    raise ValueError("use_force_encoding=False with a noise_mask needs denoising_pos_mask")
                outputs_dy = outputs_dy * (~denoising_pos_mask).to(outputs_dy.dtype).view(-1, 1)
            return energy, outputs_dy
        return energy, forces


@register_model
def equiformer_md17_dens(**kwargs):
    return Equiformer_MD17_DeNS(**kwargs)


# the model block of md17/configs/equiformer_dens/equiformer_dens_N@6_L@2_C@128-64-32.yml (scripts/train/md17/
# equiformer_dens/se_l2/: batch 8, lr 5e-4)
MD17_DENS_L2 = dict(
    irreps_in="64x0e", irreps_equivariant_inputs="1x0e+1x1e+1x2e", irreps_node_embedding="128x0e+64x1e+32x2e",
    num_layers=6, irreps_node_attr="1x0e", irreps_sh="1x0e+1x1e+1x2e", max_radius=5.0, number_of_basis=32,
    basis_type="exp", fc_neurons=[64, 64], irreps_feature="512x0e+256x1e+128x2e", irreps_head="32x0e+16x1e+8x2e",
    num_heads=4, irreps_pre_attn="128x0e+64x1e+32x2e", rescale_degree=False, nonlinear_message=True,
    irreps_mlp_mid="384x0e+192x1e+96x2e", norm_layer="layer", alpha_drop=0.0, proj_drop=0.0, out_drop=0.0,
    drop_path_rate=0.0, use_force_encoding=True)

# the model block of md17/configs/equiformer_dens/equiformer_dens_N@6_L@3_C@128-64-64-32.yml (se_l3/: batch 5, lr 2e-4);
# the file leaves use_force_encoding at its default, True
MD17_DENS_L3 = dict(
    irreps_in="64x0e", irreps_equivariant_inputs="1x0e+1x1e+1x2e+1x3e", irreps_node_embedding="128x0e+64x1e+64x2e+32x3e",
    num_layers=6, irreps_node_attr="1x0e", irreps_sh="1x0e+1x1e+1x2e+1x3e", max_radius=5.0, number_of_basis=32,
    basis_type="exp", fc_neurons=[64, 64], irreps_feature="512x0e+256x1e+256x2e+128x3e",
    irreps_head="32x0e+16x1e+16x2e+8x3e", num_heads=4, irreps_pre_attn="128x0e+64x1e+64x2e+32x3e", rescale_degree=False,
    nonlinear_message=True, irreps_mlp_mid="384x0e+192x1e+192x2e+96x3e", norm_layer="layer", alpha_drop=0.0,
    proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0, use_force_encoding=True)
