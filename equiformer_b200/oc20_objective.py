"""The IS2RS auxiliary objective of the OC20 ``*_aux_*`` configurations, as plain torch.

The model side is ``GraphAttentionTransformerOC20(use_auxiliary_task=True)``, which returns ``(energy, aux)``.  These
are the trainer-side pieces those configurations depend on, restated from the reference trainer (``oc20/trainer/``;
line numbers cite its files) and from ocpmodels' ``L2MAELoss``:

* ``relaxation_target`` - what ``aux`` regresses: the displacement to the relaxed structure over the positions' std;
* ``masked_l2mae``      - the auxiliary loss over the atoms that move (``tag > 0``);
* ``auxiliary_task_weight`` - its weight, decayed linearly to 1 over training (``auxiliary_task_weight: 15.0``);
* ``interpolate_init_relaxed_pos`` - the input augmentation of ``use_interpolate_init_relaxed_pos: True``.

A training step is then ``l1(energy, energy_target) + w * masked_l2mae(aux, relaxation_target(...), tags)``.  None of
these functions synchronises with the host, so the loss can be captured in a CUDA graph together with the model.
"""
from __future__ import annotations

from typing import Optional

import torch

# base_trainer_v2.py:82-84
_INTERPOLATE_THRESHOLD = 0.5
_MIN_INTERPOLATE_FACTOR = 0.0
_GAUSSIAN_NOISE_STD = 0.3


def relaxation_target(pos: torch.Tensor, pos_relaxed: torch.Tensor, positions_std) -> torch.Tensor:
    """``(pos_relaxed - pos) / positions_std`` (energy_trainer_v2.py:426-432: the positions normalizer has mean 0, and
    the shipped configurations set one std for all three components)."""
    return (pos_relaxed - pos) / positions_std


def masked_l2mae(pred: torch.Tensor, target: torch.Tensor, tags: torch.Tensor) -> torch.Tensor:
    """Mean over the atoms with ``tag > 0`` of ``||pred - target||_2`` (energy_trainer_v2.py:434-438 with ocpmodels'
    ``L2MAELoss``, which is the mean of the row norms of the selected atoms).

    Written as ``sum(mask * d) / max(sum(mask), 1)`` instead of selecting rows by a boolean index, so the result needs no
    host synchronisation; a batch without any moving atom gives 0."""
    mask = (tags > 0).to(pred.dtype)
    d = (pred - target).norm(p=2, dim=-1)
    return (mask * d).sum() / mask.sum().clamp(min=1.0)


def auxiliary_task_weight(step, total_steps, weight: float = 15.0) -> float:
    """Linear decay of the auxiliary loss weight from ``weight`` at step 0 to 1 at ``total_steps`` and after
    (energy_trainer_v2.py:462-470); a weight at or below 1 stays constant."""
    weight_range = max(0.0, weight - 1.0)
    return weight - weight_range * min(1.0, float(step) / total_steps)


def interpolate_init_relaxed_pos(pos: torch.Tensor, pos_relaxed: torch.Tensor, batch: torch.Tensor, tags: torch.Tensor,
                                 n_frames: int, generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """Random structures between the initial and the relaxed positions (base_trainer_v2.py:81-126).  Returns new positions;
    ``pos`` is not modified.

    * Each frame is interpolated with probability 0.5 (:88-91); other frames come back unchanged.
    * In an interpolated frame every atom draws its own factor ``f ~ U(0, 1)`` (:93-95) and moves to
      ``f * pos + (1 - f) * pos_relaxed + noise`` (:116-118).
    * The noise is i.i.d. ``N(0, 0.3^2)`` per component.  The reference first builds a noise of random direction and
      normal length, then overwrites it with this draw (:108); this keeps what the reference actually does.
    * Only atoms with ``tag > 0`` move (:114-120).

    ``n_frames`` is the number of frames in ``batch`` (passed in, so no ``batch.max()`` host read is needed).  Draws come
    from ``generator`` when one is given (it must live on ``pos``'s device), so a seeded generator repeats the result."""
    n, dtype, dev = pos.shape[0], pos.dtype, pos.device
    threshold = (torch.rand((n_frames, 1), dtype=dtype, device=dev, generator=generator)
                 + (1.0 - _INTERPOLATE_THRESHOLD)).floor_()                         # 1: interpolate, 0: keep the frame
    threshold = threshold.index_select(0, batch)
    factor = torch.empty((n, 1), dtype=dtype, device=dev).uniform_(_MIN_INTERPOLATE_FACTOR, 1.0, generator=generator)
    noise = torch.empty((n, 3), dtype=dtype, device=dev).normal_(0.0, _GAUSSIAN_NOISE_STD, generator=generator)
    new_pos = (pos * factor + (1.0 - factor) * pos_relaxed + noise) * threshold + pos * (1.0 - threshold)
    return torch.where((tags > 0).unsqueeze(-1), new_pos, pos)
