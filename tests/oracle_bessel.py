"""ORACLE extension (test infrastructure, never on the product path): the QM9 and MD17 models with the spherical Bessel
radial basis, restated op-for-op on CPU torch on top of the primitives of ``oracle.equiformer_ref``.

``oracle.equiformer_ref.model_forward`` states the Gaussian and exp-normal bases.  The ``*_bessel_*`` configurations build
ocpmodels 0.0.3's ``RadialBasis(num_basis, cutoff, rbf={'name': 'spherical_bessel'})`` instead
(nets/graph_attention_transformer.py:785-787, ..._md17.py:178-180).  ocpmodels is absent, so ``bessel_rbf`` restates it:
``PolynomialEnvelope(exponent 5) * SphericalBesselBasis``, parameter ``rbf.frequencies``.  ``model_forward_bessel`` is the
forward of :864-899 (QM9) / md17 :276-314 (energy part) with that basis; ``energy_and_forces_bessel`` adds the MD17 forces
(md17 :316-327).

Pinned by ``tests/golden/reference_model_bessel_small.npz`` (the reference's own model files run with a restated
``RadialBasis``, float64) in ``tests/test_bessel_basis.py``.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import e3nn_ref as e3
from oracle import equiformer_ref as R


def bessel_rbf(params, prefix: str, dist, cutoff):
    """RadialBasis.forward of ocpmodels 0.0.3 with rbf 'spherical_bessel' and the default polynomial envelope (p = 5)"""
    x = dist / cutoff
    p = 5
    a, b, c = -(p + 1) * (p + 2) / 2, p * (p + 2), -p * (p + 1) / 2
    env = torch.where(x < 1, 1 + a * x ** p + b * x ** (p + 1) + c * x ** (p + 2), torch.zeros_like(x))
    rbf = math.sqrt(2 / cutoff ** 3) / x[:, None] * torch.sin(params[f"{prefix}.rbf.frequencies"] * x[:, None])
    return env[:, None] * rbf


def model_forward_bessel(params, cfg: R.Config, pos, batch, node_atom, n_graphs: int):
    """GraphAttentionTransformer.forward - :864-899 / GraphAttentionTransformerMD17.forward energy part - md17 :276-314,
    with ``basis_type='bessel'``."""
    dtype = pos.dtype
    emb = e3.parse_irreps(cfg.irreps_node_embedding)
    feat = e3.parse_irreps(cfg.irreps_feature)
    irreps_edge = e3.parse_irreps(cfg.irreps_sh)
    edge_src, edge_dst = R.radius_graph(pos.detach(), cfg.max_radius, batch)
    edge_vec = pos.index_select(0, edge_src) - pos.index_select(0, edge_dst)
    edge_sh = e3.spherical_harmonics([l for _, l, _ in irreps_edge], edge_vec, True, "component")   # :869-870
    if cfg.qm9_atom_remap:
        node_atom = node_atom.new_tensor([-1, 0, -1, -1, -1, -1, 1, 2, 3, 4])[node_atom]        # :872
    onehot = F.one_hot(node_atom, cfg.max_atom_type).to(dtype)
    atom_embedding = R.linear_rs(params, "atom_embed.atom_type_lin", [(cfg.max_atom_type, 0, 1)], emb, onehot)
    edge_scalars = bessel_rbf(params, "rbf", edge_vec.norm(dim=1), cfg.max_radius)                # :877-878
    deg = R.edge_degree_embedding(params, "edge_deg_embed", cfg, pos.shape[0], edge_sh, edge_scalars, edge_src, edge_dst,
                                  dtype)
    x = atom_embedding + deg
    node_attr = torch.ones_like(x[:, 0:1])
    for i in range(cfg.num_layers):
        out_irreps = emb if i != cfg.num_layers - 1 else feat
        x = R.trans_block(params, f"blocks.{i}", cfg, emb, out_irreps, x, node_attr, edge_src, edge_dst, edge_sh,
                          edge_scalars)
    x = R.layer_norm_v2(params, "norm", feat, x)
    h = R.linear_rs(params, "head.0", feat, feat, x)
    h = F.silu(h) * e3.NORMALIZE2MOM["silu"]
    h = R.linear_rs(params, "head.2", feat, [(1, 0, 1)], h)
    return R.scatter_sum(h, batch, n_graphs) / math.sqrt(cfg.avg_num_nodes)                    # :894


def energy_and_forces_bessel(params, cfg: R.Config, pos, batch, node_atom, n_graphs: int, create_graph: bool = False):
    """GraphAttentionTransformerMD17.forward - md17 :276-327, with ``basis_type='bessel'``"""
    with torch.enable_grad():
        pos = pos.detach().clone().requires_grad_(True)
        energy = model_forward_bessel(params, cfg, pos, batch, node_atom, n_graphs)
        forces = -torch.autograd.grad(energy, pos, grad_outputs=torch.ones_like(energy), create_graph=create_graph)[0]
    return energy, forces
