"""Golden vectors from the reference's OWN dot-product OC20 model file (``nets/dp_attention_transformer_oc20.py``):

  * ``reference_model_oc20_dp_small.npz`` - a small configuration run end to end in float64 on two triclinic periodic
    frames: ``state/*`` (the ``state_dict``), ``energy`` ``[2, 1]``, ``grad/*`` (the parameter gradients of
    ``sum(energy ** 2)``), the inputs (``pos``, ``batch``, ``cell``, ``z``, ``tags``), the reference's periodic edge list
    (``edge_index``, ``cell_offsets``) and ``cfg/*`` (the constructor arguments);
  * ``reference_state_shapes_oc20_dp.json`` - parameter / buffer names and shapes and the ``no_weight_decay()`` set of the
    full-size model of oc20/configs/is2re/all/dp_attention_transformer/l1_256_g@2_local.yml.

Same method and stand-ins as ``make_reference_golden_oc20.py`` (e3nn / torch_scatter / PyG from ``make_reference_golden.py``,
``ocpmodels.common`` from ``make_reference_golden_oc20.py``): the reference file is imported from where it lies.

Run in the build container only: ``python tests/golden/make_reference_golden_oc20_dp.py``.
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

CFG = dict(irreps_node_embedding="16x0e+8x1e", num_layers=2, irreps_node_attr="1x0e", use_node_attr=False,
           irreps_sh="1x0e+1x1e", max_radius=5.0, number_of_basis=16, fc_neurons=[16, 16], use_atom_edge_attr=False,
           irreps_atom_edge_attr="1x0e", irreps_feature="32x0e", irreps_head="8x0e+4x1e", num_heads=2,
           irreps_pre_attn="16x0e+8x1e", rescale_degree=False, nonlinear_message=False, irreps_mlp_mid="48x0e+24x1e",
           norm_layer="layer", alpha_drop=0.0, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0, otf_graph=True,
           use_pbc=True, max_neighbors=500)

# the model block of oc20/configs/is2re/all/dp_attention_transformer/l1_256_g@2_local.yml:5-31
FULL = dict(irreps_node_embedding="256x0e+128x1e", num_layers=8, irreps_node_attr="1x0e", use_node_attr=False,
            irreps_sh="1x0e+1x1e", max_radius=5.0, number_of_basis=128, fc_neurons=[64, 64], use_atom_edge_attr=False,
            irreps_atom_edge_attr="1x0e", irreps_feature="512x0e", irreps_head="32x0e+16x1e", num_heads=8,
            irreps_pre_attn="256x0e+128x1e", rescale_degree=False, nonlinear_message=False,
            irreps_mlp_mid="768x0e+384x1e", norm_layer="layer", alpha_drop=0.2, proj_drop=0.0, out_drop=0.0,
            drop_path_rate=0.0, otf_graph=True, use_pbc=True, max_neighbors=500)


def main():
    G._stub_e3nn()
    G._stub_third_party()
    GO._stub_ocpmodels()
    dp = G._reference_module("dp_attention_transformer_oc20")
    torch.manual_seed(23)
    model = dp.DotProductAttentionTransformerOC20(None, None, 1, **CFG)
    gen = torch.Generator().manual_seed(101)
    with torch.no_grad():
        for name, prm in model.named_parameters():
            if prm.abs().max() == 0 or "bias" in name or "offset" in name:
                prm.add_(0.1 * torch.randn(prm.shape, generator=gen))
    torch.set_default_dtype(torch.float64)
    model = model.double().eval()
    n_atoms = [7, 9]
    batch = torch.repeat_interleave(torch.arange(2), torch.tensor(n_atoms))
    cell = torch.tensor([[[6.2, 0.0, 0.0], [0.7, 6.6, 0.0], [0.3, -0.5, 7.1]],
                         [[7.0, 0.4, 0.0], [0.0, 6.1, 0.6], [0.5, 0.0, 6.4]]], dtype=torch.float64)
    frac = torch.rand(sum(n_atoms), 3, generator=gen, dtype=torch.float64)
    pos = G._f32(torch.einsum("nk,nkd->nd", frac, cell[batch]))
    cell = G._f32(cell)
    z = torch.tensor([6, 1, 8, 29, 29, 78, 1, 13, 13, 8, 1, 6, 47, 47, 47, 7])
    tags = torch.tensor([2, 2, 2, 1, 0, 0, 2, 1, 1, 2, 2, 2, 0, 1, 0, 2])
    data = types.SimpleNamespace(pos=pos, batch=batch, cell=cell, atomic_numbers=z, tags=tags, natoms=torch.tensor(n_atoms))
    energy = model(data)
    model.zero_grad()
    (energy ** 2).sum().backward()
    out = {f"state/{k}": (v.detach().float().numpy() if v.is_floating_point() else v.numpy())
           for k, v in model.state_dict().items() if v is not None}
    for k, v in model.state_dict().items():
        if v is not None and v.is_floating_point():
            assert torch.equal(v.float().double(), v), k
    out.update({f"grad/{k}": p.grad.detach().numpy() for k, p in model.named_parameters() if p.grad is not None})
    out.update({"pos": pos.float().numpy(), "batch": batch.numpy(), "cell": cell.float().numpy(), "z": z.numpy(),
                "tags": tags.numpy(), "energy": energy.detach().numpy(), "edge_index": data.edge_index.numpy(),
                "cell_offsets": data.cell_offsets.numpy()})
    for k, v in CFG.items():
        if v is not None:
            out[f"cfg/{k}"] = np.asarray(v)
    path = os.path.join(HERE, "reference_model_oc20_dp_small.npz")
    np.savez_compressed(path, **out)
    torch.set_default_dtype(torch.float32)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1024:.0f} KiB; energy {energy.flatten().tolist()}; "
          f"{data.edge_index.shape[1]} edges")

    torch.manual_seed(0)
    full = dp.DotProductAttentionTransformerOC20(None, None, 1, **FULL)
    table = {"state": {k: list(v.shape) for k, v in full.state_dict().items() if v is not None},
             "no_weight_decay": sorted(full.no_weight_decay())}
    path = os.path.join(HERE, "reference_state_shapes_oc20_dp.json")
    with open(path, "w") as f:
        json.dump(table, f, indent=0, sort_keys=True)
    print(f"wrote {path}: {len(table['state'])} entries, {sum(p.numel() for p in full.parameters())} parameters")


if __name__ == "__main__":
    main()
