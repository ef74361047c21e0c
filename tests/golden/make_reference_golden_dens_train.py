"""Golden vectors of the DeNS input corruption, from the reference trainer's OWN function ->
``tests/golden/reference_dens_noise.npz``.

``add_masked_gaussian_noise_to_pos`` (``main_md17_dens.py:514-547``) is taken out of the reference's ``main_md17_dens.py``
with ``ast`` when this script runs (the file's imports - timm, ocpmodels, torch_geometric - are not installed, so the
module itself cannot be imported); nothing of it is stored.  It runs on CPU float32 inputs, with torch's global generator
seeded before each case, for ``corrupt_ratio`` in (None, 0.25) and ``prob`` in (0, 0.25, 1).  The fixture holds the
inputs, the seed of each case and what the function produced: both masks, the noise, the noised positions and the force
encoding input.

Run in the build container only: ``python tests/golden/make_reference_golden_dens_train.py``.
"""
from __future__ import annotations

import ast
import os
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
TRAINER = "/root/reference/main_md17_dens.py"
STD = 0.05
CASES = [(None, 0.0), (None, 0.25), (None, 1.0), (0.25, 0.0), (0.25, 0.25), (0.25, 1.0)]


def _reference_function(name: str):
    with open(TRAINER) as f:
        tree = ast.parse(f.read(), TRAINER)
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == name)
    namespace = {"torch": torch}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), TRAINER, "exec"), namespace)
    return namespace[name]


def case_name(corrupt_ratio, prob) -> str:
    return f"cr{'none' if corrupt_ratio is None else corrupt_ratio}_p{prob}"


def main():
    if not os.path.isfile(TRAINER):
        raise SystemExit(f"{TRAINER} is not here: this generator runs in the build container only")
    noise_fn = _reference_function("add_masked_gaussian_noise_to_pos")
    gen = torch.Generator().manual_seed(2718)
    n_graphs, per = 12, 21                                   # twelve aspirin-sized structures
    batch = torch.arange(n_graphs).repeat_interleave(per)
    pos = 1.5 * torch.randn(n_graphs * per, 3, generator=gen)
    dy = torch.randn(n_graphs * per, 3, generator=gen)
    out = {"pos": pos.numpy(), "dy": dy.numpy(), "batch": batch.numpy(), "std": np.asarray(STD)}
    for i, (corrupt_ratio, prob) in enumerate(CASES):
        seed = 100 + i
        data = types.SimpleNamespace(pos=pos.clone(), dy=dy.clone(), batch=batch.clone())
        torch.manual_seed(seed)
        noise_fn(data, std=STD, prob=prob, corrupt_ratio=corrupt_ratio)
        name = case_name(corrupt_ratio, prob)
        out.update({f"{name}/seed": np.asarray(seed), f"{name}/pos": data.pos.numpy(), f"{name}/noise_vec": data.noise_vec.numpy(),
                    f"{name}/noise_mask": data.noise_mask.numpy(), f"{name}/denoising_pos_mask": data.denoising_pos_mask.numpy(),
                    f"{name}/force": data.force.numpy()})
        print(f"  {name}: {int(data.noise_mask.sum())} of {data.noise_mask.numel()} atoms noised, "
              f"{int(data.denoising_pos_mask.view(n_graphs, per)[:, 0].sum())} of {n_graphs} structures drawn")
    path = os.path.join(HERE, "reference_dens_noise.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
