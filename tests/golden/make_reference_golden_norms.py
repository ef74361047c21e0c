"""Golden vectors from the reference's OWN norm and model files -> ``tests/golden/reference_norms_small.npz``:

  * ``mod/<case>/*`` - ``nets/graph_norm.py`` (``EquivariantGraphNorm``), ``nets/instance_norm.py``
    (``EquivariantInstanceNorm``) and ``nets/fast_layer_norm.py`` (``EquivariantLayerNormFast``) on one ragged batch
    of four graphs (5, 1, 7 and 4 nodes; the 0e channels of the 4-node graph are all equal, so only eps keeps its scale
    finite).  The irreps carry two 0e entries and a 0o entry.  Graph and instance norm: both normalisations, affine on
    and off, ``reduce`` 'mean' and 'max'; fast layer norm: both normalisations (the reference's torch statement needs
    the affine parameters).  Stored: input, output, and the gradients of ``sum(out * gy)`` for the input and every
    parameter;
  * ``qm9_<norm>/*``, ``md17_<norm>/*`` for ``norm_layer`` in graph / instance / fast_layer -
    ``nets/graph_attention_transformer.py`` and ``nets/graph_attention_transformer_md17.py``, small L2 configurations:
    the ``state_dict``, the energies (QM9: three molecules, one of them a lone atom; MD17: two molecules), the MD17
    forces (a derivative through the norms, which the force loss differentiates once more) and the names
    ``no_weight_decay()`` returns.

Same method and stand-ins as ``make_reference_golden_l4.py``, plus ``torch_geometric.nn.global_mean_pool`` /
``global_max_pool`` (segment mean and maximum over ``batch``, ``batch.max() + 1`` segments).  Everything runs in float64.

Run in the build container only: ``python tests/golden/make_reference_golden_norms.py``.
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

IRREPS = "6x0e+4x1e+3x0o+2x2e+4x0e"
SIZES = [5, 1, 7, 4]
QM9 = dict(irreps_in="5x0e", irreps_node_embedding="8x0e+4x1e+4x2e", num_layers=2, irreps_node_attr="1x0e",
           irreps_sh="1x0e+1x1e+1x2e", max_radius=5.0, number_of_basis=8, fc_neurons=[8, 8], irreps_feature="16x0e",
           irreps_head="4x0e+4x1e+4x2e", num_heads=2, irreps_pre_attn=None, rescale_degree=False, nonlinear_message=True,
           irreps_mlp_mid="12x0e+4x1e+4x2e", norm_layer="graph", alpha_drop=0.0, proj_drop=0.0, out_drop=0.0,
           drop_path_rate=0.0)
MD17 = dict(QM9, irreps_in="64x0e", basis_type="exp")
NORMS = ("graph", "instance", "fast_layer")


def _pools():
    def global_mean_pool(x, batch):
        G_ = int(batch.max()) + 1
        count = torch.zeros(G_, dtype=x.dtype).index_add_(0, batch, torch.ones(batch.shape[0], dtype=x.dtype))
        total = x.new_zeros((G_,) + tuple(x.shape[1:])).index_add(0, batch, x)
        return total / count.clamp(min=1).view((-1,) + (1,) * (x.dim() - 1))

    def global_max_pool(x, batch):
        G_ = int(batch.max()) + 1
        idx = batch.view((-1,) + (1,) * (x.dim() - 1)).expand_as(x)
        return x.new_zeros((G_,) + tuple(x.shape[1:])).scatter_reduce(0, idx, x, "amax", include_self=False)

    tgnn = sys.modules["torch_geometric.nn"]
    tgnn.global_mean_pool, tgnn.global_max_pool = global_mean_pool, global_max_pool


def _module_cases(out):
    gn = G._reference_module("graph_norm").EquivariantGraphNorm
    inn = G._reference_module("instance_norm").EquivariantInstanceNorm
    fln = G._reference_module("fast_layer_norm").EquivariantLayerNormFast
    gen = torch.Generator().manual_seed(1701)
    batch = torch.repeat_interleave(torch.arange(len(SIZES)), torch.tensor(SIZES))
    cases = [(kind, norm, affine, reduce) for kind in ("graph", "instance") for norm in ("component", "norm")
             for affine in (True, False) for reduce in ("mean", "max")]
    cases += [("fast_layer", norm, True, None) for norm in ("component", "norm")]
    for kind, norm, affine, reduce in cases:
        if kind == "fast_layer":
            m = fln(IRREPS, eps=1e-5, affine=affine, normalization=norm)
        else:
            m = {"graph": gn, "instance": inn}[kind](IRREPS, eps=1e-5, affine=affine, reduce=reduce, normalization=norm)
        m = m.double()
        with torch.no_grad():
            for p in m.parameters():
                p.copy_(G._f32(1.0 + 0.3 * torch.randn(p.shape, generator=gen, dtype=torch.float64)))
        x = G._f32(torch.randn(sum(SIZES), m.irreps.dim, generator=gen, dtype=torch.float64))
        x[13:17, 0:6] = 0.75                  # graph 3: its first 0e entry is constant
        x[13:17, 31:35] = -1.25               # and so is the second
        x.requires_grad_(True)
        gy = G._f32(torch.randn(x.shape, generator=gen, dtype=torch.float64))
        y = m(x, batch=batch)
        (y * gy).sum().backward()
        name = f"mod/{kind}_{norm}_{'affine' if affine else 'plain'}" + (f"_{reduce}" if reduce else "")
        out[f"{name}/x"], out[f"{name}/y"], out[f"{name}/gy"] = x.detach().numpy(), y.detach().numpy(), gy.numpy()
        out[f"{name}/gx"] = x.grad.numpy()
        for k, p in m.named_parameters():
            out[f"{name}/state/{k}"] = p.detach().float().numpy()
            out[f"{name}/grad/{k}"] = p.grad.numpy()
        out[f"{name}/batch"] = batch.numpy()
        print(f"{name}: |y| {float(y.detach().abs().max()):.3f}")


def _store(out, prefix, model, cfg, **arrays):
    """``GL._store`` without the parameter gradients (the energies and forces pin the models)."""
    GL._store(out, prefix, model, cfg, **arrays)
    for k in [k for k in out if k.startswith(f"{prefix}/grad/")]:
        del out[k]


def _models(out):
    gat = G._reference_module("graph_attention_transformer")
    md = G._reference_module("graph_attention_transformer_md17")
    for seed, norm in enumerate(NORMS):
        cfg = dict(QM9, norm_layer=norm)
        torch.manual_seed(81 + seed)
        model = gat.GraphAttentionTransformer(**cfg)
        gen = torch.Generator().manual_seed(8101 + seed)
        GL._move_off_init(model, gen)
        torch.set_default_dtype(torch.float64)
        model = model.double().eval()
        n_atoms = [8, 1, 6]
        batch = torch.repeat_interleave(torch.arange(3), torch.tensor(n_atoms))
        pos = G._f32(2.0 * torch.randn(sum(n_atoms), 3, generator=gen, dtype=torch.float64))
        pos[8] += 30.0                        # the lone atom has no neighbour
        z = torch.tensor([6, 1, 1, 8, 7, 1, 9, 6, 8, 6, 8, 1, 1, 7, 1])
        energy = model(f_in=None, pos=pos, batch=batch, node_atom=z)
        torch.set_default_dtype(torch.float32)
        _store(out, f"qm9_{norm}", model, cfg, pos=pos.float(), batch=batch, z=z, energy=energy,
               no_weight_decay=sorted(model.no_weight_decay()))
        print(f"qm9_{norm}: energy {energy.flatten().tolist()}")

        cfg = dict(MD17, norm_layer=norm)
        torch.manual_seed(91 + seed)
        model = md.GraphAttentionTransformerMD17(**cfg)
        gen = torch.Generator().manual_seed(9101 + seed)
        GL._move_off_init(model, gen)
        torch.set_default_dtype(torch.float64)
        model = model.double().eval()
        z = torch.tensor([6, 6, 8, 1, 1, 1, 6, 8, 1, 1, 1])
        batch = torch.repeat_interleave(torch.arange(2), torch.tensor([6, 5]))
        pos = G._f32(1.8 * torch.randn(11, 3, generator=gen, dtype=torch.float64))
        energy, forces = model(node_atom=z, pos=pos.clone(), batch=batch)
        torch.set_default_dtype(torch.float32)
        _store(out, f"md17_{norm}", model, cfg, pos=pos.float(), batch=batch, z=z, energy=energy, forces=forces,
               no_weight_decay=sorted(model.no_weight_decay()))
        print(f"md17_{norm}: energy {energy.flatten().tolist()}")


def main():
    if not os.path.isdir(G.REF):
        raise SystemExit(f"{G.REF} is not here: this generator runs in the build container only")
    G._stub_e3nn()
    G._stub_third_party()
    _pools()
    out: dict = {}
    _module_cases(out)
    _models(out)
    path = os.path.join(HERE, "reference_norms_small.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
