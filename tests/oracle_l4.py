"""ORACLE extension (test infrastructure, never on the product path): e3nn 0.4.4's real spherical harmonics of degree 4,
restated from e3nn's generated closed forms (``e3nn/o3/_spherical_harmonics.py``, ``sh_4_*``), beside the degrees 0..3
of ``oracle.e3nn_ref._sh_norm``.

e3nn writes each ``sh_4_m`` ('component' normalisation) as a bilinear form in the unit vector and the 'component'
``sh_3_*``; here the result is divided by ``sqrt(9)`` to the 'norm' values ``_sh_norm`` returns.  Like the rest of the
oracle this shares no code with ``equiformer_b200``: ``tests/test_lmax4.py`` checks it independently of that package's
recurrence (equivariance under the Wigner D matrices, 'component' normalisation over the sphere) and then against
``o3/sh.py``.

``installed()`` routes ``oracle.e3nn_ref.spherical_harmonics`` through :func:`sh_norm`, so every degree-generic part of
the oracle (``oracle.equiformer_ref``, the e3nn stand-ins of ``tests/golden/make_reference_golden.py``) runs at l = 4.
"""
from __future__ import annotations

import contextlib
import math

import torch

from oracle import e3nn_ref as e3

_sh_norm_0_3 = e3._sh_norm


def sh_norm(l: int, x, y, z):
    """'norm'-normalised real SH of degree l <= 4 (``oracle.e3nn_ref._sh_norm`` for l <= 3)."""
    if l != 4:
        return _sh_norm_0_3(l, x, y, z)
    s0, s1, s2, s3, s4, s5, s6 = (_sh_norm_0_3(3, x, y, z) * math.sqrt(7.0)).unbind(-1)    # e3nn's sh_3_* ('component')
    r = math.sqrt
    sh4 = torch.stack([
        (3 / 4) * r(2) * (s0 * z + s6 * x),
        (3 / 4) * s0 * y + (3 / 8) * r(6) * s1 * z + (3 / 8) * r(6) * s5 * x,
        -(3 / 56) * r(14) * s0 * z + (3 / 14) * r(21) * s1 * y + (3 / 56) * r(210) * s2 * z + (3 / 56) * r(210) * s4 * x
        + (3 / 56) * r(14) * s6 * x,
        -(3 / 56) * r(42) * s1 * z + (3 / 28) * r(105) * s2 * y + (3 / 28) * r(70) * s3 * x + (3 / 56) * r(42) * s5 * x,
        -(3 / 28) * r(42) * s2 * x + (3 / 7) * r(7) * s3 * y - (3 / 28) * r(42) * s4 * z,
        -(3 / 56) * r(42) * s1 * x + (3 / 28) * r(70) * s3 * z + (3 / 28) * r(105) * s4 * y - (3 / 56) * r(42) * s5 * z,
        -(3 / 56) * r(14) * s0 * x - (3 / 56) * r(210) * s2 * x + (3 / 56) * r(210) * s4 * z + (3 / 14) * r(21) * s5 * y
        - (3 / 56) * r(14) * s6 * z,
        -(3 / 8) * r(6) * s1 * x + (3 / 8) * r(6) * s5 * z + (3 / 4) * s6 * y,
        (3 / 4) * r(2) * (s6 * z - s0 * x)], dim=-1)
    return sh4 / 3.0


@contextlib.contextmanager
def installed():
    """Within the block, ``oracle.e3nn_ref.spherical_harmonics`` (and everything built on it) accepts l = 4."""
    e3._sh_norm = sh_norm
    try:
        yield
    finally:
        e3._sh_norm = _sh_norm_0_3
