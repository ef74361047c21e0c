"""The DeNS (denoising non-equilibrium structures) objective of the MD17 ``equiformer_dens`` configurations, as plain torch.

The model side is ``Equiformer_MD17_DeNS``, whose ``forward_edges`` returns ``(energy, dy)``: forces of the clean atoms
and the predicted position noise of the corrupted ones.  These are the trainer-side pieces those configurations depend
on, restated from the reference trainer ``main_md17_dens.py`` (line numbers cite that file):

* ``add_masked_gaussian_noise`` - the input corruption (``add_masked_gaussian_noise_to_pos``, :514-547);
* ``dens_loss``                 - energy + force + denoising loss with ``L2MAELoss`` (:389-403);
* ``denoising_pos_weight``      - the weight of the denoising term, optionally decayed linearly to 0 (:372-377).

None of these functions synchronises with the host, so the loss can be captured in a CUDA graph together with the model.
The trainer also parses ``--use-uncorrupted-force-encoding`` but never reads it: the forces of uncorrupted atoms are never
encoded, so nothing here restates that flag.
"""
from __future__ import annotations

from typing import Optional

import torch


def add_masked_gaussian_noise(pos: torch.Tensor, dy: torch.Tensor, batch: torch.Tensor, n_graphs: int, std: float,
                              prob: float, corrupt_ratio: Optional[float] = None,
                              generator: Optional[torch.Generator] = None):
    """Corrupt the positions of a random subset of structures (and, with ``corrupt_ratio``, of a random subset of their
    atoms) with ``N(0, std^2)`` noise.  Returns ``(pos_noised, noise_vec, noise_mask, denoising_pos_mask, force_enc)``:

    * ``denoising_pos_mask`` ``[N]`` bool - the atom's structure was drawn for denoising (probability ``prob``);
    * ``noise_mask`` ``[N]`` bool - the atom is corrupted (``denoising_pos_mask``, and with ``corrupt_ratio`` also drawn
      with that probability);
    * ``noise_vec`` ``[N, 3]`` - the noise drawn for every atom, the denoising target of the corrupted ones;
    * ``pos_noised`` - ``pos + noise_vec`` on corrupted atoms, ``pos`` elsewhere (``pos`` is not modified);
    * ``force_enc`` - ``dy`` on corrupted atoms and ``dy * 0`` elsewhere, the input of the model's force encoding.

    The draws are the reference's, in its order and dtype: ``rand(n_graphs)``, then ``rand(N)`` when ``corrupt_ratio`` is
    set, then ``normal_`` over ``[N, 3]``; so a generator seeded as the reference's global one gives the same result.
    ``n_graphs`` is passed in (no ``batch.max()`` host read); draws come from ``generator`` when one is given (it must
    live on ``pos``'s device)."""
    n, dtype, dev = pos.shape[0], pos.dtype, pos.device
    denoising_pos_mask = (torch.rand(n_graphs, dtype=dtype, device=dev, generator=generator) < prob).index_select(0, batch)
    noise_mask = denoising_pos_mask
    if corrupt_ratio is not None:
        noise_mask = noise_mask & (torch.rand(n, dtype=dtype, device=dev, generator=generator) < corrupt_ratio)
    force_enc = dy * noise_mask.to(dy.dtype).unsqueeze(-1)          # the reference zeroes the other rows by `*= 0`
    noise_vec = torch.zeros_like(pos).normal_(mean=0.0, std=std, generator=generator)
    pos_noised = torch.where(noise_mask.unsqueeze(-1), pos + noise_vec, pos)
    return pos_noised, noise_vec, noise_mask, denoising_pos_mask, force_enc


def _masked_l2mae(pred: torch.Tensor, target: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """Mean of the row norms ``||pred - target||_2`` over the rows of weight 1 (``L2MAELoss`` on the selected rows), as a
    weighted sum over the count; 0 when no row is selected."""
    d = (pred - target).norm(p=2, dim=-1)
    return (weight * d).sum() / weight.sum().clamp(min=1.0)


def dens_loss(pred_y: torch.Tensor, pred_dy: torch.Tensor, y: torch.Tensor, dy: torch.Tensor, noise_vec: torch.Tensor,
              noise_mask: torch.Tensor, task_mean, task_std, std: float, w_e, w_f, w_dn,
              atom_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``w_e * L_e + w_f * L_f + w_dn * L_dn`` (:389-403), each term an ``L2MAELoss``:

    * ``L_e``  - energies ``pred_y`` ``[G, 1]`` against ``(y - task_mean) / task_std``;
    * ``L_f``  - ``pred_dy`` of the atoms NOT in ``noise_mask`` against ``dy / task_std``;
    * ``L_dn`` - ``pred_dy`` of the atoms in ``noise_mask`` against ``noise_vec / std``.

    The masked means are masked sums over counts, so nothing selects rows by a boolean index; where the reference skips a
    term whose selection is empty (its mean is NaN), that term is 0 here.  ``atom_weight`` ``[N]`` (0 or 1) drops atoms
    from both atom terms - the padding atoms of a bucketed batch.  ``w_dn`` may be a device tensor (one element), so a
    decaying weight changes no captured graph."""
    dtype = pred_dy.dtype
    noised = noise_mask.to(dtype)
    clean = 1.0 - noised
    if atom_weight is not None:
        noised, clean = noised * atom_weight, clean * atom_weight
    loss_e = (pred_y - (y - task_mean) / task_std).norm(p=2, dim=-1).mean()
    loss_f = _masked_l2mae(pred_dy, dy / task_std, clean)
    loss_dn = _masked_l2mae(pred_dy, noise_vec / std, noised)
    if isinstance(w_dn, torch.Tensor):
        w_dn = w_dn.reshape(())
    return w_e * loss_e + w_f * loss_f + w_dn * loss_dn


def denoising_pos_weight(epoch, epochs, weight: float, linear_decay: bool) -> float:
    """The denoising loss weight of an epoch (:372-377): ``weight``, or with ``linear_decay`` decayed linearly from
    ``weight`` at epoch 0 to 0 at ``epochs`` and after."""
    if linear_decay:
        return weight * (1 - min(1.0, (epoch + 0.0) / epochs))
    return weight
