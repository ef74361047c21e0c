"""Golden vector from the reference's OWN DeNS model file (``nets/equiformer_md17_dens.py``) at Lmax = 3 ->
``tests/golden/reference_model_dens_l3_small.npz``: a small configuration shaped like the ``equiformer_dens`` L3 one
(``1x3e`` spherical harmonics, a ``3e`` block in the embedding, the final feature, the heads and the force encoding's
``1x0e+1x1e+1x2e+1x3e`` input), with the force encoding and the denoising head active.  Energies, the mixed forces /
predicted-noise output and the parameter gradients of an energy + output loss, in float64.  Same stubs as
``make_reference_golden.py`` and ``make_reference_golden_dens.py`` (third-party calls served by the oracle's primitives).

Run in the build container only: ``python tests/golden/make_reference_golden_dens_l3.py``.
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


def main():
    G._stub_e3nn()
    G._stub_third_party()
    dens = G._reference_module("equiformer_md17_dens")
    cfg = dict(irreps_in="64x0e", irreps_equivariant_inputs="1x0e+1x1e+1x2e+1x3e",
               irreps_node_embedding="16x0e+8x1e+4x2e+4x3e", num_layers=2, irreps_node_attr="1x0e",
               irreps_sh="1x0e+1x1e+1x2e+1x3e", max_radius=5.0, number_of_basis=16, basis_type="exp", fc_neurons=[16, 16],
               irreps_feature="32x0e+16x1e+8x2e+8x3e", irreps_head="8x0e+4x1e+2x2e+2x3e", num_heads=2,
               irreps_pre_attn="16x0e+8x1e+4x2e+4x3e", rescale_degree=False, nonlinear_message=True,
               irreps_mlp_mid="24x0e+12x1e+6x2e+6x3e", norm_layer="layer", alpha_drop=0.0, proj_drop=0.0, out_drop=0.0,
               drop_path_rate=0.0, use_force_encoding=True)
    torch.manual_seed(37)
    model = dens.Equiformer_MD17_DeNS(**cfg)
    gen = torch.Generator().manual_seed(919)
    with torch.no_grad():
        for name, prm in model.named_parameters():
            if prm.abs().max() == 0 or "bias" in name or "offset" in name:
                prm.add_(0.1 * torch.randn(prm.shape, generator=gen))
    torch.set_default_dtype(torch.float64)
    model = model.double().eval()
    z = torch.tensor([6, 6, 8, 1, 1, 1, 1, 6, 8, 1, 6])
    batch = torch.tensor([0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1])
    pos = G._f32(1.7 * torch.randn(11, 3, generator=gen, dtype=torch.float64))
    force = G._f32(torch.randn(11, 3, generator=gen, dtype=torch.float64))
    noise_mask = torch.tensor([False, True, True, False, False, True, False, True, False, False, True])
    data = types.SimpleNamespace(z=z, pos=pos.clone(), batch=batch, force=force, noise_mask=noise_mask)
    energy, dy = model(data)
    model.zero_grad()
    (energy.sum() + (dy ** 2).sum()).backward()
    out = {f"state/{k}": (v.detach().float().numpy() if v.is_floating_point() else v.numpy())
           for k, v in model.state_dict().items() if v is not None}
    for k, v in model.state_dict().items():
        if v is not None and v.is_floating_point():
            assert torch.equal(v.float().double(), v), k
    out.update({f"grad/{k}": p.grad.detach().numpy() for k, p in model.named_parameters() if p.grad is not None})
    out.update({"pos": pos.float().numpy(), "batch": batch.numpy(), "z": z.numpy(), "force": force.float().numpy(),
                "noise_mask": noise_mask.numpy(), "energy": energy.detach().numpy(), "dy": dy.detach().numpy()})
    for k, v in cfg.items():
        if v is not None:
            out[f"cfg/{k}"] = np.asarray(v)
    path = os.path.join(HERE, "reference_model_dens_l3_small.npz")
    np.savez_compressed(path, **out)
    torch.set_default_dtype(torch.float32)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1024:.0f} KiB; energy {energy.flatten().tolist()}")


if __name__ == "__main__":
    main()
