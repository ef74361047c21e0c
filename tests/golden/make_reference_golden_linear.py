"""Golden vectors from the reference's OWN model files for the linear-message graph attention
(``nonlinear_message=False``) -> ``tests/golden/reference_model_linear_small.npz``:

  * ``qm9/*``  - ``nets/graph_attention_transformer.py`` (``GraphAttentionTransformer``), small configuration: the energy
    of a two-molecule batch and the parameter gradients of ``sum(energy ** 2)``;
  * ``md17/*`` - ``nets/graph_attention_transformer_md17.py`` (``GraphAttentionTransformerMD17``), small L2 configuration:
    energy, forces (``-dE/dpos``) and the parameter gradients of ``energy.sum() + (forces ** 2).sum()`` (a second
    derivative through the forward);
  * ``oc20/*`` - ``nets/graph_attention_transformer_oc20.py`` without the auxiliary head, small configuration on two
    triclinic periodic frames: energy, the parameter gradients of ``sum(energy ** 2)`` and the reference's periodic edge
    list;
  * ``oc20_full/state``, ``oc20_full/no_weight_decay`` - JSON of the parameter / buffer names and shapes and the
    ``no_weight_decay()`` set of the full-size model of oc20/configs/is2re/all/graph_attention_transformer/
    l1_256_g@2_local.yml.

Every case stores ``state/*`` (the ``state_dict``), the inputs and ``cfg/*`` (the constructor arguments) under its prefix.
The channel counts per head are multiples of 4, so on a GPU the mirrors run these cases on the fused linear-message
attention kernel.  Same method and stand-ins as ``make_reference_golden.py`` and ``make_reference_golden_oc20.py``: the
reference files are imported from where they lie and run in float64.

Run in the build container only: ``python tests/golden/make_reference_golden_linear.py``.
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
import make_reference_golden_oc20 as GO  # noqa: E402

QM9 = dict(irreps_in="5x0e", irreps_node_embedding="16x0e+8x1e+8x2e", num_layers=2, irreps_node_attr="1x0e",
           irreps_sh="1x0e+1x1e+1x2e", max_radius=5.0, number_of_basis=16, fc_neurons=[16, 16], irreps_feature="32x0e",
           irreps_head="8x0e+4x1e+4x2e", num_heads=2, irreps_pre_attn=None, rescale_degree=False, nonlinear_message=False,
           irreps_mlp_mid="24x0e+12x1e+12x2e", norm_layer="layer", alpha_drop=0.0, proj_drop=0.0, out_drop=0.0,
           drop_path_rate=0.0)
MD17 = dict(irreps_in="64x0e", irreps_node_embedding="16x0e+8x1e+8x2e", num_layers=2, irreps_node_attr="1x0e",
            irreps_sh="1x0e+1x1e+1x2e", max_radius=5.0, number_of_basis=16, basis_type="exp", fc_neurons=[16, 16],
            irreps_feature="32x0e", irreps_head="8x0e+4x1e+4x2e", num_heads=2, irreps_pre_attn=None,
            rescale_degree=False, nonlinear_message=False, irreps_mlp_mid="24x0e+12x1e+12x2e", norm_layer="layer",
            alpha_drop=0.0, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0)
OC20 = dict(irreps_node_embedding="16x0e+8x1e", num_layers=2, irreps_node_attr="1x0e", use_node_attr=False,
            irreps_sh="1x0e+1x1e", max_radius=5.0, number_of_basis=16, fc_neurons=[16, 16], use_atom_edge_attr=False,
            irreps_atom_edge_attr="1x0e", irreps_feature="32x0e", irreps_head="8x0e+4x1e", num_heads=2,
            irreps_pre_attn="16x0e+8x1e", rescale_degree=False, nonlinear_message=False, irreps_mlp_mid="48x0e+24x1e",
            norm_layer="layer", alpha_drop=0.0, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0, otf_graph=True,
            use_pbc=True, max_neighbors=500)
# the model block of oc20/configs/is2re/all/graph_attention_transformer/l1_256_g@2_local.yml:5-31
FULL = dict(OC20, irreps_node_embedding="256x0e+128x1e", num_layers=8, number_of_basis=128, fc_neurons=[64, 64],
            irreps_feature="512x0e", irreps_head="32x0e+16x1e", num_heads=8, irreps_pre_attn="256x0e+128x1e",
            irreps_mlp_mid="768x0e+384x1e", alpha_drop=0.2)


def _move_off_init(model, gen):
    with torch.no_grad():                      # biases, offsets and norm shifts start at zero: move them
        for name, prm in model.named_parameters():
            if prm.abs().max() == 0 or "bias" in name or "offset" in name:
                prm.add_(0.1 * torch.randn(prm.shape, generator=gen))


def _store(out: dict, prefix: str, model, cfg: dict, **arrays):
    for k, v in model.state_dict().items():
        if v is None:
            continue
        if v.is_floating_point():
            assert torch.equal(v.float().double(), v), k
            out[f"{prefix}/state/{k}"] = v.detach().float().numpy()
        else:
            out[f"{prefix}/state/{k}"] = v.numpy()
    out.update({f"{prefix}/grad/{k}": p.grad.detach().numpy() for k, p in model.named_parameters() if p.grad is not None})
    for k, v in arrays.items():
        out[f"{prefix}/{k}"] = v.detach().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
    for k, v in cfg.items():
        if v is not None:
            out[f"{prefix}/cfg/{k}"] = np.asarray(v)


def main():
    if not os.path.isdir(G.REF):
        raise SystemExit(f"{G.REF} is not here: this generator runs in the build container only")
    G._stub_e3nn()
    G._stub_third_party()
    GO._stub_ocpmodels()
    out: dict = {}

    # ---- QM9 model file, linear message
    gat = G._reference_module("graph_attention_transformer")
    torch.manual_seed(31)
    model = gat.GraphAttentionTransformer(**QM9)
    gen = torch.Generator().manual_seed(3101)
    _move_off_init(model, gen)
    torch.set_default_dtype(torch.float64)
    model = model.double().eval()
    n_atoms = [7, 6]
    batch = torch.repeat_interleave(torch.arange(2), torch.tensor(n_atoms))
    pos = G._f32(2.1 * torch.randn(sum(n_atoms), 3, generator=gen, dtype=torch.float64))
    z = torch.tensor([6, 1, 1, 8, 7, 1, 9, 6, 6, 8, 1, 1, 7])
    energy = model(f_in=None, pos=pos, batch=batch, node_atom=z)
    model.zero_grad()
    (energy ** 2).sum().backward()
    torch.set_default_dtype(torch.float32)
    _store(out, "qm9", model, QM9, pos=pos.float(), batch=batch, z=z, energy=energy)
    print(f"qm9: energy {energy.flatten().tolist()}")

    # ---- MD17 model file (L2, exp-normal basis), linear message: energy, forces and the force-loss gradients
    md = G._reference_module("graph_attention_transformer_md17")
    torch.manual_seed(37)
    model = md.GraphAttentionTransformerMD17(**MD17)
    gen = torch.Generator().manual_seed(3701)
    _move_off_init(model, gen)
    torch.set_default_dtype(torch.float64)
    model = model.double().eval()
    z = torch.tensor([6, 6, 8, 1, 1, 1, 1, 6, 8])
    batch = torch.zeros(9, dtype=torch.long)
    pos = G._f32(1.8 * torch.randn(9, 3, generator=gen, dtype=torch.float64))
    energy, forces = model(node_atom=z, pos=pos.clone(), batch=batch)
    model.zero_grad()
    (energy.sum() + (forces ** 2).sum()).backward()
    torch.set_default_dtype(torch.float32)
    _store(out, "md17", model, MD17, pos=pos.float(), batch=batch, z=z, energy=energy, forces=forces)
    print(f"md17: energy {energy.flatten().tolist()}")

    # ---- OC20 model file without the auxiliary head, linear message, two periodic frames
    oc = G._reference_module("graph_attention_transformer_oc20")
    torch.manual_seed(41)
    model = oc.GraphAttentionTransformerOC20(None, None, 1, **OC20)
    gen = torch.Generator().manual_seed(4101)
    _move_off_init(model, gen)
    torch.set_default_dtype(torch.float64)
    model = model.double().eval()
    n_atoms = [8, 9]
    batch = torch.repeat_interleave(torch.arange(2), torch.tensor(n_atoms))
    cell = torch.tensor([[[6.3, 0.0, 0.0], [0.6, 6.5, 0.0], [0.2, -0.4, 7.0]],
                         [[6.9, 0.3, 0.0], [0.0, 6.2, 0.5], [0.4, 0.0, 6.6]]], dtype=torch.float64)
    frac = torch.rand(sum(n_atoms), 3, generator=gen, dtype=torch.float64)
    pos = G._f32(torch.einsum("nk,nkd->nd", frac, cell[batch]))
    cell = G._f32(cell)
    z = torch.tensor([6, 1, 8, 29, 29, 78, 1, 7, 13, 13, 8, 1, 6, 47, 47, 47, 7])
    tags = torch.tensor([2, 2, 2, 1, 0, 0, 2, 2, 1, 1, 2, 2, 2, 0, 1, 0, 2])
    data = types.SimpleNamespace(pos=pos, batch=batch, cell=cell, atomic_numbers=z, tags=tags, natoms=torch.tensor(n_atoms))
    energy = model(data)
    model.zero_grad()
    (energy ** 2).sum().backward()
    torch.set_default_dtype(torch.float32)
    _store(out, "oc20", model, OC20, pos=pos.float(), batch=batch, cell=cell.float(), z=z, tags=tags, energy=energy,
           edge_index=data.edge_index, cell_offsets=data.cell_offsets)
    print(f"oc20: energy {energy.flatten().tolist()}; {data.edge_index.shape[1]} edges")

    # ---- the full-size OC20 l1_256 model: names and shapes, no_weight_decay()
    torch.manual_seed(0)
    full = oc.GraphAttentionTransformerOC20(None, None, 1, **FULL)
    out["oc20_full/state"] = np.asarray(json.dumps({k: list(v.shape) for k, v in full.state_dict().items() if v is not None},
                                                   sort_keys=True))
    out["oc20_full/no_weight_decay"] = np.asarray(json.dumps(sorted(full.no_weight_decay())))
    print(f"oc20_full: {len(full.state_dict())} entries, {sum(p.numel() for p in full.parameters())} parameters")

    path = os.path.join(HERE, "reference_model_linear_small.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
