"""Golden vectors from the reference's OWN model files for the E(3) (parity-carrying) Equiformer
-> ``tests/golden/reference_model_e3_small.npz``:

  * ``oc20/*`` - ``nets/graph_attention_transformer_oc20.py`` without the auxiliary head, small E(3) configuration
    (``0e``, ``0o``, ``1e``, ``1o`` node blocks, ``1x0e+1x1o`` spherical harmonics) on two triclinic periodic frames:
    energy, the parameter gradients of ``sum(energy ** 2)`` and the reference's periodic edge list;
  * ``qm9/*``  - ``nets/graph_attention_transformer.py`` (``GraphAttentionTransformer``), small E(3) configuration with
    ``2e`` / ``2o`` blocks and ``1x0e+1x1o+1x2e`` harmonics: the energies of a two-molecule batch and the parameter
    gradients of ``sum(energy ** 2)``;
  * ``md17/*`` - ``nets/graph_attention_transformer_md17.py`` (``GraphAttentionTransformerMD17``), the same small E(3)
    layout with the exp-normal basis: energy, forces (``-dE/dpos``) and the parameter gradients of
    ``energy.sum() + (forces ** 2).sum()`` (a second derivative through the forward);
  * ``oc20_full/state``, ``oc20_full/no_weight_decay`` - JSON of the parameter / buffer names and shapes and the
    ``no_weight_decay()`` set of the full-size model of oc20/configs/is2re/all/graph_attention_transformer/
    l1_256_e3_nonlinear_g@2_local.yml.

Every case stores ``state/*`` (the ``state_dict``), the inputs and ``cfg/*`` (the constructor arguments) under its prefix.
Every multiplicity per head is a multiple of 4, so on a GPU the mirrors run these cases on the float4 kernels.  The odd
blocks go through every layer of the reference with a parity branch: the depth-wise products' instruction lists and
their even-first sort, the gates (``0o`` is gated, not activated), the LayerNorm (no mean and no bias on ``0o``), the head
layout and the attention.  Same method and stand-ins as ``make_reference_golden.py`` and
``make_reference_golden_linear.py`` (the stand-ins already carry parity): the reference files are imported from where they
lie and run in float64.

Run in the build container only: ``python tests/golden/make_reference_golden_e3.py``.
"""
from __future__ import annotations

import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import make_reference_golden as G  # noqa: E402
import make_reference_golden_linear as GL  # noqa: E402
import make_reference_golden_oc20 as GO  # noqa: E402

OC20 = dict(irreps_node_embedding="16x0e+8x0o+8x1e+8x1o", num_layers=2, irreps_node_attr="1x0e", use_node_attr=False,
            irreps_sh="1x0e+1x1o", max_radius=5.0, number_of_basis=16, fc_neurons=[16, 16], use_atom_edge_attr=False,
            irreps_atom_edge_attr="1x0e", irreps_feature="32x0e", irreps_head="8x0e+4x0o+4x1e+4x1o", num_heads=2,
            irreps_pre_attn="16x0e+8x0o+8x1e+8x1o", rescale_degree=False, nonlinear_message=True,
            irreps_mlp_mid="48x0e+16x0o+16x1e+16x1o", norm_layer="layer", alpha_drop=0.0, proj_drop=0.0, out_drop=0.0,
            drop_path_rate=0.0, otf_graph=True, use_pbc=True, max_neighbors=500)
QM9 = dict(irreps_in="5x0e", irreps_node_embedding="16x0e+8x0o+8x1e+8x1o+4x2e+4x2o", num_layers=2,
           irreps_node_attr="1x0e", irreps_sh="1x0e+1x1o+1x2e", max_radius=5.0, number_of_basis=16, fc_neurons=[16, 16],
           irreps_feature="32x0e", irreps_head="8x0e+4x0o+4x1e+4x1o+4x2e+4x2o", num_heads=2, irreps_pre_attn=None,
           rescale_degree=False, nonlinear_message=True, irreps_mlp_mid="24x0e+8x0o+8x1e+8x1o+4x2e+4x2o",
           norm_layer="layer", alpha_drop=0.0, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0)
MD17 = dict(QM9, irreps_in="64x0e", basis_type="exp")
# the model block of oc20/configs/is2re/all/graph_attention_transformer/l1_256_e3_nonlinear_g@2_local.yml:5-31
FULL = dict(OC20, irreps_node_embedding="256x0e+64x0o+64x1e+64x1o", num_layers=6, number_of_basis=128,
            fc_neurons=[64, 64], irreps_feature="512x0e", irreps_head="32x0e+8x0o+8x1e+8x1o", num_heads=8,
            irreps_pre_attn="256x0e+64x0o+64x1e+64x1o", irreps_mlp_mid="768x0e+192x0o+192x1e+192x1o", alpha_drop=0.2)


def main():
    if not os.path.isdir(G.REF):
        raise SystemExit(f"{G.REF} is not here: this generator runs in the build container only")
    G._stub_e3nn()
    G._stub_third_party()
    GO._stub_ocpmodels()
    out: dict = {}

    # ---- OC20 model file without the auxiliary head, E(3), two periodic frames
    oc = G._reference_module("graph_attention_transformer_oc20")
    torch.manual_seed(53)
    model = oc.GraphAttentionTransformerOC20(None, None, 1, **OC20)
    gen = torch.Generator().manual_seed(5301)
    GL._move_off_init(model, gen)
    torch.set_default_dtype(torch.float64)
    model = model.double().eval()
    n_atoms = [9, 8]
    batch = torch.repeat_interleave(torch.arange(2), torch.tensor(n_atoms))
    cell = torch.tensor([[[6.4, 0.0, 0.0], [0.5, 6.3, 0.0], [-0.3, 0.4, 6.9]],
                         [[6.7, 0.2, 0.0], [0.0, 6.4, 0.4], [0.6, -0.2, 6.5]]], dtype=torch.float64)
    frac = torch.rand(sum(n_atoms), 3, generator=gen, dtype=torch.float64)
    pos = G._f32(torch.einsum("nk,nkd->nd", frac, cell[batch]))
    cell = G._f32(cell)
    z = torch.tensor([6, 8, 1, 29, 29, 78, 1, 7, 6, 13, 13, 8, 1, 47, 47, 47, 7])
    tags = torch.tensor([2, 2, 2, 1, 0, 0, 2, 2, 2, 1, 1, 2, 2, 0, 1, 0, 2])
    data = types.SimpleNamespace(pos=pos, batch=batch, cell=cell, atomic_numbers=z, tags=tags, natoms=torch.tensor(n_atoms))
    energy = model(data)
    model.zero_grad()
    (energy ** 2).sum().backward()
    torch.set_default_dtype(torch.float32)
    GL._store(out, "oc20", model, OC20, pos=pos.float(), batch=batch, cell=cell.float(), z=z, tags=tags, energy=energy,
              edge_index=data.edge_index, cell_offsets=data.cell_offsets)
    print(f"oc20: energy {energy.flatten().tolist()}; {data.edge_index.shape[1]} edges")

    # ---- QM9 model file, E(3)
    gat = G._reference_module("graph_attention_transformer")
    torch.manual_seed(59)
    model = gat.GraphAttentionTransformer(**QM9)
    gen = torch.Generator().manual_seed(5901)
    GL._move_off_init(model, gen)
    torch.set_default_dtype(torch.float64)
    model = model.double().eval()
    n_atoms = [8, 6]
    batch = torch.repeat_interleave(torch.arange(2), torch.tensor(n_atoms))
    pos = G._f32(2.0 * torch.randn(sum(n_atoms), 3, generator=gen, dtype=torch.float64))
    z = torch.tensor([6, 1, 1, 8, 7, 1, 9, 6, 6, 8, 1, 1, 7, 1])
    energy = model(f_in=None, pos=pos, batch=batch, node_atom=z)
    model.zero_grad()
    (energy ** 2).sum().backward()
    torch.set_default_dtype(torch.float32)
    GL._store(out, "qm9", model, QM9, pos=pos.float(), batch=batch, z=z, energy=energy)
    print(f"qm9: energy {energy.flatten().tolist()}")

    # ---- MD17 model file, E(3), exp-normal basis: energy, forces and the force-loss gradients
    md = G._reference_module("graph_attention_transformer_md17")
    torch.manual_seed(61)
    model = md.GraphAttentionTransformerMD17(**MD17)
    gen = torch.Generator().manual_seed(6101)
    GL._move_off_init(model, gen)
    torch.set_default_dtype(torch.float64)
    model = model.double().eval()
    z = torch.tensor([6, 6, 8, 1, 1, 1, 1, 6, 8, 1])
    batch = torch.zeros(10, dtype=torch.long)
    pos = G._f32(1.8 * torch.randn(10, 3, generator=gen, dtype=torch.float64))
    energy, forces = model(node_atom=z, pos=pos.clone(), batch=batch)
    model.zero_grad()
    (energy.sum() + (forces ** 2).sum()).backward()
    torch.set_default_dtype(torch.float32)
    GL._store(out, "md17", model, MD17, pos=pos.float(), batch=batch, z=z, energy=energy, forces=forces)
    print(f"md17: energy {energy.flatten().tolist()}")

    # ---- the full-size OC20 l1_256_e3_nonlinear model: names and shapes, no_weight_decay()
    torch.manual_seed(0)
    full = oc.GraphAttentionTransformerOC20(None, None, 1, **FULL)
    out["oc20_full/state"] = np.asarray(json.dumps({k: list(v.shape) for k, v in full.state_dict().items() if v is not None},
                                                   sort_keys=True))
    out["oc20_full/no_weight_decay"] = np.asarray(json.dumps(sorted(full.no_weight_decay())))
    print(f"oc20_full: {len(full.state_dict())} entries, {sum(p.numel() for p in full.parameters())} parameters")

    path = os.path.join(HERE, "reference_model_e3_small.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
