"""Per-graph equivariant normalisation without mean shift (drop-in for ``EquivariantInstanceNorm``,
``nets/instance_norm.py:9-134``): :class:`EquivariantGraphNorm` with the 0e mean subtracted as it is.  ``state_dict``
keys ``affine_weight`` / ``affine_bias``."""
from __future__ import annotations

from .graph_norm import EquivariantGraphNorm


class EquivariantInstanceNorm(EquivariantGraphNorm):
    _mean_shift = False
