"""Golden vector of the IS2RS auxiliary head, from the reference's OWN OC20 model file
(``nets/graph_attention_transformer_oc20.py`` with ``use_auxiliary_task=True``) -> ``tests/golden/reference_model_oc20_aux_small.npz``.

Same method and stand-ins as ``make_reference_golden_oc20.py`` (e3nn / torch_scatter / PyG from ``make_reference_golden.py``,
``ocpmodels.common`` from ``make_reference_golden_oc20.py``): the reference file is imported from where it lies and run end
to end in float64 on two triclinic periodic frames.  The configuration is small but has everything the ``*_aux_*`` OC20
configurations add: a final feature with a vector block (``irreps_feature='32x0e+16x1e'``, so the last block has an FFN
shortcut and the energy head a ``1e`` input without a path), and the ``auxiliary_head`` ``GraphAttention`` whose
``irreps_pre_attn`` differs from its input irreps.  Two cases, each under its own prefix:

  * ``nonlinear/`` - ``nonlinear_message=True`` (the shipped configurations);
  * ``linear/``    - ``nonlinear_message=False``.

Per case: ``state/*`` (the ``state_dict``), ``energy`` ``[2, 1]``, ``aux`` ``[16, 3]``, ``c`` ``[2, 1]`` and ``W`` ``[16, 3]``
(seeded cotangents) and ``grad/*``, the parameter gradients of ``sum(c * energy) + sum(W * aux)``.  Shared: ``pos``,
``batch``, ``cell``, ``z``, ``tags``, the reference's periodic edge list (``edge_index``, ``cell_offsets``) and ``cfg/*``
(the nonlinear case's constructor arguments; the linear case differs only in ``nonlinear_message``).

Run in the build container only: ``python tests/golden/make_reference_golden_oc20_aux.py``.
"""
from __future__ import annotations

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

CFG = dict(irreps_node_embedding="16x0e+8x1e", num_layers=3, irreps_node_attr="1x0e", use_node_attr=False,
           irreps_sh="1x0e+1x1e", max_radius=5.0, number_of_basis=16, fc_neurons=[16, 16], use_atom_edge_attr=False,
           irreps_atom_edge_attr="1x0e", irreps_feature="32x0e+16x1e", irreps_head="8x0e+4x1e", num_heads=2,
           irreps_pre_attn="16x0e+8x1e", rescale_degree=False, nonlinear_message=True, irreps_mlp_mid="48x0e+24x1e",
           norm_layer="layer", alpha_drop=0.0, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0, use_auxiliary_task=True,
           auxiliary_head_dropout=True, otf_graph=True, use_pbc=True, max_neighbors=500)


def _frames():
    gen = torch.Generator().manual_seed(77)
    n_atoms = [7, 9]
    batch = torch.repeat_interleave(torch.arange(2), torch.tensor(n_atoms))
    cell = torch.tensor([[[6.2, 0.0, 0.0], [0.7, 6.6, 0.0], [0.3, -0.5, 7.1]],
                         [[7.0, 0.4, 0.0], [0.0, 6.1, 0.6], [0.5, 0.0, 6.4]]], dtype=torch.float64)
    frac = torch.rand(sum(n_atoms), 3, generator=gen, dtype=torch.float64)
    pos = G._f32(torch.einsum("nk,nkd->nd", frac, cell[batch]))
    z = torch.tensor([6, 1, 8, 29, 29, 78, 1, 13, 13, 8, 1, 6, 47, 47, 47, 7])
    tags = torch.tensor([2, 2, 2, 1, 0, 0, 2, 1, 1, 2, 2, 2, 0, 1, 0, 2])
    return pos, batch, G._f32(cell), z, tags, n_atoms


def _case(oc, cfg, seed, pos, batch, cell, z, tags, n_atoms):
    torch.set_default_dtype(torch.float32)
    torch.manual_seed(seed)
    model = oc.GraphAttentionTransformerOC20(None, None, 1, **cfg)
    gen = torch.Generator().manual_seed(seed + 1000)
    with torch.no_grad():
        for name, prm in model.named_parameters():
            if prm.abs().max() == 0 or "bias" in name or "offset" in name:
                prm.add_(0.1 * torch.randn(prm.shape, generator=gen))
    torch.set_default_dtype(torch.float64)
    model = model.double().eval()
    data = types.SimpleNamespace(pos=pos, batch=batch, cell=cell, atomic_numbers=z, tags=tags, natoms=torch.tensor(n_atoms))
    energy, aux = model(data)
    c = G._f32(torch.randn(energy.shape, generator=gen, dtype=torch.float64))
    W = G._f32(torch.randn(aux.shape, generator=gen, dtype=torch.float64))
    model.zero_grad()
    ((c * energy).sum() + (W * aux).sum()).backward()
    out = {f"state/{k}": (v.detach().float().numpy() if v.is_floating_point() else v.numpy())
           for k, v in model.state_dict().items() if v is not None}
    for k, v in model.state_dict().items():
        if v is not None and v.is_floating_point():
            assert torch.equal(v.float().double(), v), k
    out.update({f"grad/{k}": p.grad.detach().numpy() for k, p in model.named_parameters() if p.grad is not None})
    out.update({"energy": energy.detach().numpy(), "aux": aux.detach().numpy(), "c": c.numpy(), "W": W.numpy()})
    torch.set_default_dtype(torch.float32)
    return out, data


def main():
    G._stub_e3nn()
    G._stub_third_party()
    GO._stub_ocpmodels()
    oc = G._reference_module("graph_attention_transformer_oc20")
    pos, batch, cell, z, tags, n_atoms = _frames()
    out = {}
    data = None
    for tag, seed, nonlinear in (("nonlinear", 31, True), ("linear", 32, False)):
        arrays, data = _case(oc, dict(CFG, nonlinear_message=nonlinear), seed, pos, batch, cell, z, tags, n_atoms)
        out.update({f"{tag}/{k}": v for k, v in arrays.items()})
        print(f"{tag}: energy {arrays['energy'].flatten().tolist()}, |aux| max {np.abs(arrays['aux']).max():.4f}")
    out.update({"pos": pos.float().numpy(), "batch": batch.numpy(), "cell": cell.float().numpy(), "z": z.numpy(),
                "tags": tags.numpy(), "edge_index": data.edge_index.numpy(), "cell_offsets": data.cell_offsets.numpy()})
    for k, v in CFG.items():
        if v is not None:
            out[f"cfg/{k}"] = np.asarray(v)
    path = os.path.join(HERE, "reference_model_oc20_aux_small.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1024:.0f} KiB; {data.edge_index.shape[1]} edges")


if __name__ == "__main__":
    main()
