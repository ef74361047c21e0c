"""Golden vectors from the reference's OWN model files at degree 4 -> ``tests/golden/reference_model_l4_small.npz``:

  * ``qm9/*``  - ``nets/graph_attention_transformer.py`` (``GraphAttentionTransformer``), a small SE(3) configuration with
    ``0e`` .. ``4e`` node blocks and ``1x0e+1x1e+1x2e+1x3e+1x4e`` harmonics: the energies of a two-molecule batch and the
    parameter gradients of ``sum(energy ** 2)``;
  * ``md17/*`` - ``nets/graph_attention_transformer_md17.py`` (``GraphAttentionTransformerMD17``), the same layout with the
    exp-normal basis: energy, forces (``-dE/dpos``) and the parameter gradients of ``energy.sum() + (forces ** 2).sum()``
    (a second derivative through the forward).

Every case stores ``state/*`` (the ``state_dict``), the inputs and ``cfg/*`` (the constructor arguments) under its prefix.
Every multiplicity per head is a multiple of 4, so on a GPU the mirrors run these cases on the float4 table-walk kernels.
Same method and stand-ins as ``make_reference_golden_e3.py``: the reference files are imported from where they lie and
run in float64; the stand-in ``o3.spherical_harmonics`` calls the oracle's, which ``tests/oracle_l4.py`` extends to l = 4.

Run in the build container only: ``python tests/golden/make_reference_golden_l4.py``.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import make_reference_golden as G  # noqa: E402
import make_reference_golden_linear as GL  # noqa: E402
from tests import oracle_l4  # noqa: E402

QM9 = dict(irreps_in="5x0e", irreps_node_embedding="8x0e+4x1e+4x2e+4x3e+4x4e", num_layers=2, irreps_node_attr="1x0e",
           irreps_sh="1x0e+1x1e+1x2e+1x3e+1x4e", max_radius=5.0, number_of_basis=8, fc_neurons=[8, 8],
           irreps_feature="16x0e", irreps_head="4x0e+4x1e+4x2e+4x3e+4x4e", num_heads=2, irreps_pre_attn=None,
           rescale_degree=False, nonlinear_message=True, irreps_mlp_mid="12x0e+4x1e+4x2e+4x3e+4x4e", norm_layer="layer",
           alpha_drop=0.0, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0)
MD17 = dict(QM9, irreps_in="64x0e", basis_type="exp")


def main():
    if not os.path.isdir(G.REF):
        raise SystemExit(f"{G.REF} is not here: this generator runs in the build container only")
    G._stub_e3nn()
    G._stub_third_party()
    out: dict = {}
    with oracle_l4.installed():
        # ---- QM9 model file, degree 4
        gat = G._reference_module("graph_attention_transformer")
        torch.manual_seed(67)
        model = gat.GraphAttentionTransformer(**QM9)
        gen = torch.Generator().manual_seed(6701)
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

        # ---- MD17 model file, degree 4, exp-normal basis: energy, forces and the force-loss gradients
        md = G._reference_module("graph_attention_transformer_md17")
        torch.manual_seed(71)
        model = md.GraphAttentionTransformerMD17(**MD17)
        gen = torch.Generator().manual_seed(7101)
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

    path = os.path.join(HERE, "reference_model_l4_small.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
