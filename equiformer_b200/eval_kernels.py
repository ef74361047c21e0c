"""Launchers of ``libeqf_b200_eval.so`` (``include/eqf_b200_eval.h``): one batch's metric terms added to a float64
accumulator on the device, and a torch statement of the same terms.

The accumulator is a float64 tensor of slots; each launcher adds to the slots it is handed (a contiguous slice of
``EQF_EVAL_GRAPH_SLOTS``, ``EQF_EVAL_ATOM_SLOTS`` or ``EQF_EVAL_BATCH_SLOTS`` elements):

* graph level: ``sum |e|``, ``sum e^2``, ``#{|e| < threshold}``, ``sum |pred - (y - mean) / std|`` and the graph count,
  with ``e = pred * std + mean - y`` over the first ``n_graphs`` rows;
* atom level: ``sum |pred_dy * std - dy|`` over components, ``sum ||pred_dy - dy / std||_2`` over atoms and the atom
  count, over the first ``n_atoms`` rows, ``n_atoms`` a device scalar;
* batch level: one batch's loss (a device scalar, or None) and the batch count.

The kernels are the only implementation the evaluation passes use.  The ``*_torch`` functions state the same terms in
torch with the same arguments (without the scratch): they are the tests' reference and the accumulator of the CPU tests.

:func:`predict_is2re_raw` launches the one kernel of ``libeqf_b200_predict.so`` (``include/eqf_b200_predict.h``): the
de-normalised energies and, optionally, predicted positions of a predict pass, stated in torch by
:func:`predict_is2re_torch`.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import _lib
from .ops import _kernel, _stream


def _check(rc: int, what: str) -> None:
    _lib.check(rc, what, _lib.load_eval())


def _flat(t: torch.Tensor, name: str, dtype, n: Optional[int] = None, at_least: bool = False) -> int:
    """Pointer of a contiguous buffer of ``dtype`` with ``n`` (or, ``at_least``, n or more) elements; the device is
    checked by :func:`_on_cuda` once every argument has passed."""
    if t.dtype != dtype:
        raise _lib.EqfError(f"{name} must be {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise _lib.EqfError(f"{name} must be contiguous")
    if n is not None and (t.numel() < n if at_least else t.numel() != n):
        raise _lib.EqfError(f"{name} has {t.numel()} elements, expected {'at least ' if at_least else ''}{n}")
    return t.data_ptr()


def _on_cuda(**tensors) -> None:
    """Every buffer on the accumulator's CUDA device; anything else raises."""
    dev = tensors["acc"].device
    for name, t in tensors.items():
        if t is not None and (not t.is_cuda or t.device != dev):
            raise _lib.EqfError(f"{name} lives on {t.device}: the metric kernels are CUDA-only (sm_90a) and take every "
                                f"buffer on the accumulator's device ({dev})")


def new_scratch(device) -> tuple:
    """The ``(partials, tickets)`` scratch of the graph and atom launchers: float64 ``[EQF_EVAL_SCRATCH]`` and a zeroed
    int32 counter.  Launches on one stream may share it."""
    return (torch.zeros(_lib.EQF_EVAL_SCRATCH, dtype=torch.float64, device=device),
            torch.zeros(1, dtype=torch.int32, device=device))


def eval_graph_raw(pred: torch.Tensor, y: torch.Tensor, n_graphs: int, mean: float, std: float, threshold: float,
                   acc: torch.Tensor, scratch: tuple) -> None:
    """Add the graph-level terms of rows ``< n_graphs`` of ``pred`` (float32, normalised, ``n_graphs`` or more rows of
    one element: padded outputs may follow) and ``y`` (float32 ``[n_graphs]``) to ``acc`` (float64 ``[5]``)."""
    n = int(n_graphs)
    partials, tickets = scratch
    args = (_flat(pred, "pred", torch.float32, n, at_least=True), _flat(y, "y", torch.float32, n), n, float(mean),
            float(std), float(threshold), _flat(partials, "partials", torch.float64, _lib.EQF_EVAL_SCRATCH),
            _flat(tickets, "tickets", torch.int32, 1), _flat(acc, "acc", torch.float64, _lib.EQF_EVAL_GRAPH_SLOTS))
    _on_cuda(pred=pred, y=y, partials=partials, tickets=tickets, acc=acc)
    with torch.cuda.device(acc.device), _kernel("eval_graph", 8 * n):
        rc = _lib.load_eval().eqf_eval_graph(*args, _stream())
    _check(rc, "eqf_eval_graph")


def eval_atom_raw(pred_dy: torch.Tensor, dy: torch.Tensor, n_atoms: torch.Tensor, std: float, acc: torch.Tensor,
                  scratch: tuple) -> None:
    """Add the atom-level terms of rows ``< n_atoms`` of ``pred_dy`` and ``dy`` (float32 ``[rows, 3]``; later rows are
    padding) to ``acc`` (float64 ``[3]``).  ``n_atoms`` is an int64 device scalar, read by the kernel."""
    rows = pred_dy.shape[0] if pred_dy.dim() == 2 else -1
    if pred_dy.dim() != 2 or pred_dy.shape[1] != 3 or tuple(dy.shape) != tuple(pred_dy.shape):
        raise _lib.EqfError(f"pred_dy and dy must both be [rows, 3], got {tuple(pred_dy.shape)} and {tuple(dy.shape)}")
    partials, tickets = scratch
    args = (_flat(pred_dy, "pred_dy", torch.float32), _flat(dy, "dy", torch.float32), rows,
            _flat(n_atoms, "n_atoms", torch.int64, 1), float(std),
            _flat(partials, "partials", torch.float64, _lib.EQF_EVAL_SCRATCH), _flat(tickets, "tickets", torch.int32, 1),
            _flat(acc, "acc", torch.float64, _lib.EQF_EVAL_ATOM_SLOTS))
    _on_cuda(pred_dy=pred_dy, dy=dy, n_atoms=n_atoms, partials=partials, tickets=tickets, acc=acc)
    with torch.cuda.device(acc.device), _kernel("eval_atom", 24 * rows):
        rc = _lib.load_eval().eqf_eval_atom(*args, _stream())
    _check(rc, "eqf_eval_atom")


def eval_batch_raw(loss: Optional[torch.Tensor], acc: torch.Tensor) -> None:
    """Add one batch's ``loss`` (a float32 device scalar, or None to count the batch only) to ``acc`` (float64 ``[2]``)."""
    args = (_flat(loss, "loss", torch.float32, 1) if loss is not None else None,
            _flat(acc, "acc", torch.float64, _lib.EQF_EVAL_BATCH_SLOTS))
    _on_cuda(loss=loss, acc=acc)
    with torch.cuda.device(acc.device), _kernel("eval_batch", 20):
        rc = _lib.load_eval().eqf_eval_batch(*args, _stream())
    _check(rc, "eqf_eval_batch")


# ------------------------------------------------------------------------------------------------ torch statement
def eval_graph_torch(pred, y, n_graphs: int, mean: float, std: float, threshold: float, acc: torch.Tensor) -> None:
    """:func:`eval_graph_raw` in torch: the terms in the inputs' dtype, summed in float64."""
    n = int(n_graphs)
    p, t = pred.reshape(-1)[:n], y.reshape(-1)[:n]
    e = p * std + mean - t
    ae = e.abs()
    terms = [ae.double().sum(), (e * e).double().sum(), (ae < threshold).double().sum(),
             (p - (t - mean) / std).abs().double().sum(), torch.tensor(float(n), dtype=torch.float64)]
    acc += torch.stack([x.to(acc.device) for x in terms])


def eval_atom_torch(pred_dy, dy, n_atoms, std: float, acc: torch.Tensor) -> None:
    """:func:`eval_atom_raw` in torch (``n_atoms`` an int or a one-element tensor)."""
    n = max(0, min(int(n_atoms), pred_dy.shape[0]))
    p, t = pred_dy[:n], dy[:n]
    terms = [(p * std - t).abs().double().sum(), (p - t / std).norm(p=2, dim=-1).double().sum(),
             torch.tensor(float(n), dtype=torch.float64)]
    acc += torch.stack([x.to(acc.device) for x in terms])


def eval_batch_torch(loss, acc: torch.Tensor) -> None:
    """:func:`eval_batch_raw` in torch."""
    l = torch.zeros((), dtype=torch.float64) if loss is None else loss.detach().reshape(()).double().cpu()
    acc += torch.stack([l, torch.tensor(1.0, dtype=torch.float64)]).to(acc.device)


# ------------------------------------------------------------------------------------------------ predictions
def predict_is2re_raw(energy: torch.Tensor, n_graphs: int, mean: float, std: float, energy_out: torch.Tensor,
                      pos: Optional[torch.Tensor] = None, delta: Optional[torch.Tensor] = None,
                      tags: Optional[torch.Tensor] = None, pos_std: float = 1.0,
                      pos_out: Optional[torch.Tensor] = None) -> None:
    """Write ``energy[:n_graphs] * std + mean`` into ``energy_out`` (float32, ``n_graphs`` or more rows of one element
    each) and, when ``delta`` is given, ``pos + (delta * pos_std + 0)`` on the rows with ``tags > 0`` and ``pos`` on the
    others into ``pos_out`` (``pos``, ``delta``, ``pos_out`` float32 ``[rows, 3]``, ``tags`` int64 ``[rows]``).  Rows past
    ``n_graphs`` of ``energy_out`` are left as they are."""
    n = int(n_graphs)
    with_pos = delta is not None
    if with_pos != (pos is not None) or with_pos != (tags is not None) or with_pos != (pos_out is not None):
        raise _lib.EqfError("pos, delta, tags and pos_out are given together or not at all")
    rows = 0
    if with_pos:
        rows = pos.shape[0] if pos.dim() == 2 else -1
        for name, t in (("pos", pos), ("delta", delta), ("pos_out", pos_out)):
            if t.dim() != 2 or t.shape[1] != 3 or t.shape[0] != rows:
                raise _lib.EqfError(f"pos, delta and pos_out must all be [rows, 3], got {name} {tuple(t.shape)}")
    args = (_flat(energy, "energy", torch.float32, n, at_least=True), n, float(mean), float(std),
            _flat(pos, "pos", torch.float32) if with_pos else None,
            _flat(delta, "delta", torch.float32) if with_pos else None,
            _flat(tags, "tags", torch.int64, rows) if with_pos else None, rows, float(pos_std),
            _flat(energy_out, "energy_out", torch.float32, n, at_least=True),
            _flat(pos_out, "pos_out", torch.float32) if with_pos else None)
    dev = energy_out.device
    for name, t in (("energy", energy), ("energy_out", energy_out), ("pos", pos), ("delta", delta), ("tags", tags),
                    ("pos_out", pos_out)):
        if t is not None and (not t.is_cuda or t.device != dev):
            raise _lib.EqfError(f"{name} lives on {t.device}: the prediction kernel is CUDA-only (sm_90a) and takes every "
                                f"buffer on energy_out's device ({dev})")
    lib = _lib.load_predict()
    with torch.cuda.device(dev), _kernel("predict_is2re", 8 * n + 32 * rows):
        rc = lib.eqf_predict_is2re(*args, _stream())
    _lib.check(rc, "eqf_predict_is2re", lib)


def predict_is2re_torch(energy, n_graphs: int, mean: float, std: float, pos=None, delta=None, tags=None,
                        pos_std: float = 1.0):
    """:func:`predict_is2re_raw` in torch, in the reference's operations: ``Normalizer.denorm`` (``tensor * std + mean``)
    of the energy, the positions normaliser's ``denorm`` (mean 0) of ``delta`` and ``pred_pos[mask] + delta_pos[mask]``
    over ``tags > 0`` (``energy_trainer_v2.predict``).  Returns the energies ``[n_graphs]`` and the positions (or None)."""
    e = energy.reshape(-1)[:int(n_graphs)] * std + mean
    if delta is None:
        return e, None
    p = pos.clone()
    m = tags > 0
    p[m] = p[m] + (delta * pos_std + 0.0)[m]
    return e, p
