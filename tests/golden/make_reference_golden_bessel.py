"""Golden vectors from the reference's OWN model files with the spherical Bessel radial basis.

The reference takes ``RadialBasis`` from ocpmodels 0.0.3 (``ocpmodels/models/gemnet/layers/radial_basis.py``), which is not
installed here.  This script installs a restatement of it (``RadialBasis`` with ``envelope`` = ``PolynomialEnvelope(5)`` and
``rbf`` = ``SphericalBesselBasis``, parameter ``frequencies``) under that module name before any reference module is
imported, on top of the e3nn / PyG stubs of ``make_reference_golden.py``, and runs the reference's model files in float64:

  * ``reference_model_bessel_small.npz``
      - ``qm9/...``  : ``nets/graph_attention_transformer.py``, small channels, ``nonlinear_message=True``, 8 functions:
                       energies and the parameter gradients of sum(E^2), ``rbf.rbf.frequencies`` included;
      - ``md17/...`` : ``nets/graph_attention_transformer_md17.py``, Lmax 2, 16 functions: energy, forces and the parameter
                       gradients of an energy + force loss (a second derivative through the basis);
  * ``reference_state_shapes_bessel.json``: parameter / buffer names and shapes and the ``no_weight_decay()`` set of the six
    registered Bessel configurations at their real sizes (8 functions for QM9, as the reference's QM9 scripts run them;
    128 for MD17).

The Bessel numerics in these files are therefore the restatement's, not ocpmodels' own; ``tests/test_bessel_basis.py``
anchors the restatement to scipy's spherical Bessel function independently.  Run in the build container only:
``python tests/golden/make_reference_golden_bessel.py``.  No reference source is copied anywhere.
"""
from __future__ import annotations

import json
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import make_reference_golden as G  # noqa: E402

QM9_BESSEL = ["graph_attention_transformer_nonlinear_bessel_l2", "graph_attention_transformer_nonlinear_bessel_l2_drop01",
              "graph_attention_transformer_nonlinear_bessel_l2_drop00"]
MD17_BESSEL = ["graph_attention_transformer_nonlinear_bessel_l2_md17", "graph_attention_transformer_nonlinear_bessel_l3_md17",
               "graph_attention_transformer_nonlinear_bessel_l3_e3_md17"]


class PolynomialEnvelope(torch.nn.Module):
    def __init__(self, exponent):
        super().__init__()
        self.p = exponent
        self.a = -(self.p + 1) * (self.p + 2) / 2
        self.b = self.p * (self.p + 2)
        self.c = -self.p * (self.p + 1) / 2

    def forward(self, d_scaled):
        env = 1 + self.a * d_scaled ** self.p + self.b * d_scaled ** (self.p + 1) + self.c * d_scaled ** (self.p + 2)
        return torch.where(d_scaled < 1, env, torch.zeros_like(d_scaled))


class SphericalBesselBasis(torch.nn.Module):
    def __init__(self, num_radial, cutoff):
        super().__init__()
        self.norm_const = math.sqrt(2 / (cutoff ** 3))
        self.frequencies = torch.nn.Parameter(torch.tensor(np.pi * np.arange(1, num_radial + 1, dtype=np.float32)))

    def forward(self, d_scaled):
        return self.norm_const / d_scaled[:, None] * torch.sin(self.frequencies * d_scaled[:, None])


class RadialBasis(torch.nn.Module):
    def __init__(self, num_radial, cutoff, rbf={"name": "gaussian"}, envelope={"name": "polynomial", "exponent": 5},
                 scale_basis=False):
        super().__init__()
        assert rbf == {"name": "spherical_bessel"} and envelope == {"name": "polynomial", "exponent": 5} and not scale_basis
        self.inv_cutoff = 1 / cutoff
        self.envelope = PolynomialEnvelope(envelope["exponent"])
        self.rbf = SphericalBesselBasis(num_radial, cutoff)

    def forward(self, d):
        d_scaled = d * self.inv_cutoff
        return self.envelope(d_scaled)[:, None] * self.rbf(d_scaled)


def _perturb(model, gen):
    """Biases, offsets and norm shifts start at zero and the frequencies at pi * k: move them (float32 values)."""
    with torch.no_grad():
        for name, prm in model.named_parameters():
            if prm.abs().max() == 0 or "bias" in name or "offset" in name or "frequencies" in name:
                prm.add_(0.1 * torch.randn(prm.shape, generator=gen))


def _record(model, cfg, **arrays):
    out = {f"state/{k}": v.detach().float().numpy() if v.is_floating_point() else v.numpy()
           for k, v in model.state_dict().items() if v is not None}
    for k, v in model.state_dict().items():
        if v is not None and v.is_floating_point():
            assert torch.equal(v.float().double(), v), k
    out.update({f"grad/{k}": p.grad.detach().numpy() for k, p in model.named_parameters() if p.grad is not None})
    out.update({k: v.detach().numpy() for k, v in arrays.items()})
    out.update({f"cfg/{k}": np.asarray(v) for k, v in cfg.items() if v is not None})
    return out


def main():
    if not os.path.isdir(G.REF):
        raise SystemExit(f"{G.REF} is not here: this generator runs in the build container only")
    G._stub_e3nn()
    G._stub_third_party()
    sys.modules["ocpmodels.models.gemnet.layers.radial_basis"].RadialBasis = RadialBasis
    gat = G._reference_module("graph_attention_transformer")
    md = G._reference_module("graph_attention_transformer_md17")
    gen = torch.Generator().manual_seed(2468)
    fixture = {}

    # ---- the module alone: 128 functions, 5 A, frequencies moved off pi * k, some distances beyond the cutoff
    m = RadialBasis(128, 5.0, rbf={"name": "spherical_bessel"})
    _perturb(m, gen)
    m = m.double()
    dist = G._f32(0.05 + 5.3 * torch.rand(91, generator=gen, dtype=torch.float64))
    fixture.update({"module/dist": dist.float().numpy(), "module/state/rbf.frequencies": m.rbf.frequencies.detach().float().numpy(),
                    "module/y": m(dist).detach().numpy()})

    # ---- QM9 model file, 8 Bessel functions (the count the reference's QM9 scripts use)
    cfg = dict(irreps_in="5x0e", irreps_node_embedding="16x0e+8x1e+4x2e", num_layers=2, irreps_node_attr="1x0e",
               irreps_sh="1x0e+1x1e+1x2e", max_radius=5.0, number_of_basis=8, basis_type="bessel", fc_neurons=[16, 16],
               irreps_feature="32x0e", irreps_head="8x0e+4x1e+2x2e", num_heads=2, irreps_pre_attn=None,
               rescale_degree=False, nonlinear_message=True, irreps_mlp_mid="24x0e+12x1e+6x2e", norm_layer="layer",
               alpha_drop=0.0, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0)
    torch.manual_seed(41)
    model = gat.GraphAttentionTransformer(**cfg)
    _perturb(model, gen)
    torch.set_default_dtype(torch.float64)
    model = model.double().eval()
    n_atoms = [7, 6]
    batch = torch.repeat_interleave(torch.arange(2), torch.tensor(n_atoms))
    pos = G._f32(2.2 * torch.randn(sum(n_atoms), 3, generator=gen, dtype=torch.float64))
    z = torch.tensor([6, 1, 1, 8, 7, 1, 9, 6, 6, 8, 1, 1, 7])
    energy = model(f_in=None, pos=pos, batch=batch, node_atom=z)
    model.zero_grad()
    (energy ** 2).sum().backward()
    torch.set_default_dtype(torch.float32)
    qm9 = _record(model, cfg, pos=pos.float(), batch=batch, z=z, energy=energy)
    fixture.update({f"qm9/{k}": v for k, v in qm9.items()})
    print(f"qm9: energy {energy.flatten().tolist()}, {sum(k.startswith('grad/') for k in qm9)} gradients")

    # ---- MD17 model file, Lmax 2, 16 Bessel functions: energy, forces, gradients of an energy + force loss
    cfg = dict(irreps_in="64x0e", irreps_node_embedding="16x0e+8x1e+4x2e", num_layers=2, irreps_node_attr="1x0e",
               irreps_sh="1x0e+1x1e+1x2e", max_radius=5.0, number_of_basis=16, basis_type="bessel", fc_neurons=[16, 16],
               irreps_feature="32x0e", irreps_head="8x0e+4x1e+2x2e", num_heads=2, irreps_pre_attn=None,
               rescale_degree=False, nonlinear_message=True, irreps_mlp_mid="24x0e+12x1e+6x2e", norm_layer="layer",
               alpha_drop=0.0, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0)
    torch.manual_seed(43)
    model = md.GraphAttentionTransformerMD17(**cfg)
    _perturb(model, gen)
    torch.set_default_dtype(torch.float64)
    model = model.double().eval()
    z = torch.tensor([6, 6, 8, 1, 1, 1, 1, 6, 8, 1])
    batch = torch.zeros(10, dtype=torch.long)
    pos = G._f32(1.8 * torch.randn(10, 3, generator=gen, dtype=torch.float64))
    energy, forces = model(node_atom=z, pos=pos.clone(), batch=batch)
    model.zero_grad()
    (energy.sum() + (forces ** 2).sum()).backward()
    torch.set_default_dtype(torch.float32)
    md17 = _record(model, cfg, pos=pos.float(), batch=batch, z=z, energy=energy, forces=forces)
    fixture.update({f"md17/{k}": v for k, v in md17.items()})
    print(f"md17: energy {energy.flatten().tolist()}, {sum(k.startswith('grad/') for k in md17)} gradients")

    path = os.path.join(HERE, "reference_model_bessel_small.npz")
    np.savez_compressed(path, **fixture)
    print(f"wrote {path}: {len(fixture)} arrays, {os.path.getsize(path) / 1024:.0f} KiB")

    # ---- the six registered Bessel configurations at their real sizes: names, shapes, no_weight_decay()
    table = {}
    for mod, irreps_in, num_basis, names in ((gat, "5x0e", 8, QM9_BESSEL), (md, "64x0e", 128, MD17_BESSEL)):
        for name in names:
            torch.manual_seed(0)
            model = getattr(mod, name)(irreps_in=irreps_in, radius=5.0, num_basis=num_basis)
            table[name] = {"num_basis": num_basis,
                           "state": {k: list(v.shape) for k, v in model.state_dict().items() if v is not None},
                           "no_weight_decay": sorted(model.no_weight_decay())}
            print(f"  {name}: {len(table[name]['state'])} entries, {sum(p.numel() for p in model.parameters())} parameters")
    path = os.path.join(HERE, "reference_state_shapes_bessel.json")
    with open(path, "w") as f:
        json.dump(table, f, indent=0, sort_keys=True)
    print(f"wrote {path}: {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
