"""The reference-run model fixtures (``tests/golden/reference_*.npz``), read in one place.

``tests/golden/make_reference_golden*.py`` run the reference's own model files in float64.  Each run stores its
constructor arguments under ``cfg/``, its ``state_dict`` under ``state/``, the parameter gradients of its training loss
under ``grad/``, and its inputs and outputs as plain keys.  A file with several runs puts each under ``<case>/``; keys the
runs share (inputs, ``cfg/``) may stay at the top level.
"""
from __future__ import annotations

import os
import types

import numpy as np
import torch

from oracle import equiformer_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
OC20_STATS = dict(max_atom_type=84, qm9_atom_remap=False, avg_degree=23.395238876342773, avg_num_nodes=77.81317)
# what the oracle needs beyond the model's constructor arguments, per model family
ORACLE_EXTRAS = {"qm9": dict(basis_type="gaussian"),
                 "md17": dict(basis_type="exp", max_atom_type=64, qm9_atom_remap=False),
                 "oc20": OC20_STATS}
_ORACLE_KEYS = ("irreps_node_embedding", "irreps_sh", "irreps_head", "irreps_mlp_mid", "irreps_feature", "num_heads",
                "num_layers", "max_radius", "number_of_basis", "nonlinear_message")


class Case:
    """One run of a reference model file: ``arrays`` (its keys without the ``<case>/`` prefix), ``cfg`` (the constructor
    keyword arguments), ``state`` and ``grads`` (its ``state_dict`` and parameter gradients as tensors)."""

    def __init__(self, arrays: dict):
        self.arrays = arrays
        self.cfg = {k[len("cfg/"):]: v.tolist() for k, v in arrays.items() if k.startswith("cfg/")}
        self.state = {k[len("state/"):]: torch.from_numpy(v) for k, v in arrays.items() if k.startswith("state/")}
        self.grads = {k[len("grad/"):]: torch.from_numpy(v) for k, v in arrays.items() if k.startswith("grad/")}

    def t(self, key, dev=None, dtype=None):
        return torch.from_numpy(self.arrays[key]).to(device=dev, dtype=dtype)


def load(name: str, prefix: str = "") -> Case:
    """The run stored under ``<prefix>/`` of ``tests/golden/<name>``; a key it does not hold is read from the top level."""
    g = np.load(os.path.join(GOLDEN, name))
    arrays = {k: g[k] for k in g.files}
    if prefix:
        arrays.update({k[len(prefix) + 1:]: v for k, v in arrays.items() if k.startswith(prefix + "/")})
    return Case(arrays)


def oracle_config(family: str, cfg: dict, **overrides) -> R.Config:
    return R.Config(**{k: cfg[k] for k in _ORACLE_KEYS}, **dict(ORACLE_EXTRAS[family], **overrides))


def load_state(module, state):
    """``load_state_dict`` of a reference ``state_dict``: nothing unexpected, and nothing missing but the ``output_mask``
    buffers that e3nn's ``TensorProduct`` registers and the generators' stub e3nn does not."""
    res = module.load_state_dict(state, strict=False)
    assert not res.unexpected_keys and all(k.endswith("tp.output_mask") for k in res.missing_keys), res
    return module


def mirror(cls, cfg, state, *args):
    """The host-side mirror ``cls(*args, **cfg)`` loaded with the reference's ``state_dict``, in eval mode."""
    return load_state(cls(*args, **cfg), state).eval()


def oc20_data(case: Case, dev=None, dtype=torch.float64):
    """The batch of the two periodic OC20 frames as the OC20 models' ``forward(data)`` reads it."""
    return types.SimpleNamespace(pos=case.t("pos", dev, dtype), cell=case.t("cell", dev, dtype), batch=case.t("batch", dev),
                                 atomic_numbers=case.t("z", dev), tags=case.t("tags", dev), n_graphs=2)


def dens_setup(name: str, dev=None, dtype=torch.float64):
    """(case, mirror, data) of a DeNS fixture: ``Equiformer_MD17_DeNS`` with the reference's ``state_dict`` and the
    ``forward(data)`` batch (force encoding and noise mask included)."""
    from equiformer_b200.nets.equiformer_md17_dens import Equiformer_MD17_DeNS
    case = load(name)
    model = mirror(Equiformer_MD17_DeNS, case.cfg, case.state).to(dtype)
    if dev is not None:
        model = model.to(dev)
    data = types.SimpleNamespace(z=case.t("z", dev), pos=case.t("pos", dev, dtype), batch=case.t("batch", dev),
                                 force=case.t("force", dev, dtype), noise_mask=case.t("noise_mask", dev))
    return case, model, data


def run_oracle(family: str, case: Case, ocfg: R.Config):
    """The oracle on the case's inputs with its ``state_dict`` in float64 (every non-empty float tensor trainable), and the
    fixture's training loss backpropagated: sum E^2 for qm9 and oc20, E.sum() + sum F^2 for md17.  Returns (energy,
    forces or None, params)."""
    params = {k: v.requires_grad_(v.is_floating_point() and v.numel() > 0)
              for k, v in R.cast_params(case.state, torch.float64).items()}
    pos, batch, z = case.t("pos", dtype=torch.float64), case.t("batch"), case.t("z")
    forces = None
    if family == "qm9":
        energy = R.model_forward(params, ocfg, pos, batch, z, n_graphs=2)
        (energy ** 2).sum().backward()
    elif family == "md17":
        energy, forces = R.energy_and_forces(params, ocfg, pos, batch, z, 1, create_graph=True)
        (energy.sum() + (forces ** 2).sum()).backward()
    else:
        edge = case.t("edge_index")
        energy = R.model_forward_oc20(params, ocfg, pos, case.t("cell", dtype=torch.float64), batch, z, case.t("tags"), 2,
                                      edge[0], edge[1], case.t("cell_offsets"))
        (energy ** 2).sum().backward()
    return energy, forces, params


def run_mirror(family: str, model, case: Case, dev=None, dtype=torch.float64):
    """The mirror on the case's inputs and the fixture's training loss backpropagated into its parameters, as in
    ``run_oracle``.  Returns (energy, forces or None)."""
    pos, forces = case.t("pos", dev, dtype), None
    if family == "qm9":
        energy = model(f_in=None, pos=pos, batch=case.t("batch", dev), node_atom=case.t("z", dev))
        (energy ** 2).sum().backward()
    elif family == "md17":
        energy, forces = model(node_atom=case.t("z", dev), pos=pos.clone(), batch=case.t("batch", dev))
        (energy.sum() + (forces ** 2).sum()).backward()
    else:
        energy = model(oc20_data(case, dev, dtype))
        (energy ** 2).sum().backward()
    return energy, forces


def worst_grad(named: dict, ref: dict, n_min: int) -> float:
    """max over the reference gradients (at least ``n_min`` of them) of max|got - ref| / max|ref|, with max|ref| taken
    as at least 1e-12.  Every parameter the reference has a gradient for must have one here."""
    assert len(ref) >= n_min
    worst = 0.0
    for k, r in ref.items():
        got = named[k]
        assert got is not None, k
        worst = max(worst, float((got.detach().double().cpu() - r.double()).abs().max() / r.abs().max().clamp_min(1e-12)))
    return worst
