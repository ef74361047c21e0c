"""Spherical Bessel radial basis with polynomial envelope (the Bessel-basis QM9 / MD17 configurations).

The reference builds ``RadialBasis(num_basis, cutoff=max_radius, rbf={'name': 'spherical_bessel'})`` from ocpmodels 0.0.3
(``ocpmodels/models/gemnet/layers/radial_basis.py``; nets/graph_attention_transformer.py:785-787, ..._md17.py:178-180,
equiformer_md17_dens.py:122-124).  ocpmodels is not a dependency: this module restates its formulas, module structure and
parameter names (``envelope`` without parameters, ``rbf.frequencies``, so ``rbf.rbf.frequencies`` inside the models) from
that version.  They are not executed from it, and no ocpmodels checkpoint has been loaded to confirm the key names.
The arithmetic is ``ops.bessel_rbf_torch`` (CPU, float64) and the ``ops.BesselRbf`` kernels (CUDA float32).
"""
from __future__ import annotations

import math

import torch

from .. import ops


class PolynomialEnvelope(torch.nn.Module):
    """``1 + a x^p + b x^(p+1) + c x^(p+2)`` for ``x < 1``, else 0, with a = -(p+1)(p+2)/2, b = p(p+2), c = -p(p+1)/2;
    no parameters."""

    def __init__(self, exponent: int = 5):
        super().__init__()
        self.p = exponent


class SphericalBesselBasis(torch.nn.Module):
    """``sqrt(2 / cutoff^3) sin(f_k x) / x`` on scaled distances ``x``; ``frequencies`` start at ``pi * [1, ..., B]``."""

    def __init__(self, num_radial: int, cutoff: float):
        super().__init__()
        self.norm_const = math.sqrt(2 / cutoff ** 3)
        self.frequencies = torch.nn.Parameter(math.pi * torch.arange(1, num_radial + 1, dtype=torch.float32))


class RadialBasis(torch.nn.Module):
    """``forward(d) -> [E, num_radial]`` = envelope(d / cutoff) * basis(d / cutoff).  ``d = 0`` gives NaN, as in the
    reference (``0 / 0``); the neighbour lists this package builds have no zero-length edge.  Only the configuration the
    reference uses is implemented: the spherical Bessel basis with the default envelope (polynomial, exponent 5)."""

    def __init__(self, num_radial: int, cutoff: float, rbf: dict = {"name": "gaussian"},
                 envelope: dict = {"name": "polynomial", "exponent": 5}, scale_basis: bool = False):
        super().__init__()
        if rbf.get("name") != "spherical_bessel":
            raise ValueError(f"RadialBasis: only rbf 'spherical_bessel' is implemented, got {rbf!r}")
        if envelope.get("name") != "polynomial" or envelope.get("exponent") != 5 or scale_basis:
            raise ValueError("RadialBasis: only the polynomial envelope of exponent 5 without scale_basis is implemented")
        self.cutoff = cutoff
        self.inv_cutoff = 1 / cutoff
        self.envelope = PolynomialEnvelope(5)
        self.rbf = SphericalBesselBasis(num_radial, cutoff)

    def forward(self, d):
        return ops.bessel_rbf(d, self.rbf.frequencies, self.cutoff)
