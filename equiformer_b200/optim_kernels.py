"""Launchers of ``libeqf_b200_optim.so`` (``include/eqf_b200_optim.h``): gradient clipping, AdamW and the model EMA.

The optimiser kernels have a library of their own, next to ``libeqf_b200.so``; these are its only callers.  The optimiser
built on them is ``parallel.CapturableFlatAdamW``.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from . import _lib
from .ops import _kernel, _stream


def _check(rc: int, what: str) -> None:
    _lib.check(rc, what, _lib.load_optim())


def _flat(t: torch.Tensor, name: str, n: Optional[int] = None, dtype=torch.float32) -> int:
    """Device pointer of a contiguous CUDA buffer of ``dtype`` (and ``n`` elements); anything else raises."""
    if t.dtype != dtype:
        raise _lib.EqfError(f"{name} must be {dtype}, got {t.dtype}")
    if not t.is_cuda:
        raise _lib.EqfError(f"{name} lives on {t.device}: the optimiser kernels are CUDA-only (sm_90a)")
    if not t.is_contiguous():
        raise _lib.EqfError(f"{name} must be contiguous")
    if n is not None and t.numel() != n:
        raise _lib.EqfError(f"{name} has {t.numel()} elements, expected {n}")
    return t.data_ptr()


def flat_sqnorm_raw(g: torch.Tensor, max_norm: float, partials: torch.Tensor, tickets: torch.Tensor, norm: torch.Tensor,
                    coef: torch.Tensor) -> None:
    """``norm`` = ||g||, ``coef`` = min(1, max_norm / (norm + 1e-6)), both written on the device.  ``partials``: float64
    ``[EQF_OPTIM_MAX_CTAS]`` scratch; ``tickets``: int32 ``[1]`` counter, zero before the first call and after every call."""
    n = g.numel()
    args = (_flat(g, "gradient"), n, float(max_norm), _flat(partials, "partials", _lib.EQF_OPTIM_MAX_CTAS, torch.float64),
            _flat(tickets, "tickets", 1, torch.int32), _flat(norm, "norm", 1), _flat(coef, "coef", 1))
    with torch.cuda.device(g.device), _kernel("flat_sqnorm", 4 * n):
        rc = _lib.load_optim().eqf_flat_sqnorm(*args, _stream())
    _check(rc, "eqf_flat_sqnorm")


def flat_adamw_raw(g, p, m, v, decay, ema, coef, lr, step, betas, eps: float, ema_decay: Optional[float],
                   tickets, schedule=None) -> None:
    """One AdamW step on the flat buffers ``g, p, m, v`` (``decay``: per-element weight decay), in place: ``g *= coef``,
    ``step += 1``, and ``ema`` (or None) moved toward the new ``p`` by ``1 - ema_decay``.  ``coef`` / ``lr`` are float32
    ``[1]`` and ``step`` int64 ``[1]`` device tensors, ``tickets`` an int32 ``[1]`` counter as in :func:`flat_sqnorm_raw`;
    nothing is read from the host.  With a ``schedule`` (``lr_schedule.LrSchedule``) the rate is the schedule's at the
    step count before the step, and ``lr`` is left holding the next step's rate (``eqf_flat_adamw_scheduled``)."""
    n = p.numel()
    ptrs = [_flat(t, name, n) for t, name in ((g, "gradient"), (p, "parameters"), (m, "m"), (v, "v"), (decay, "decay"))]
    e = _flat(ema, "ema", n) if ema is not None else None
    args = (*ptrs, e, n, _flat(coef, "coef", 1), _flat(lr, "lr", 1), _flat(step, "step", 1, torch.int64),
            float(betas[0]), float(betas[1]), float(eps), float(ema_decay if ema is not None else 0.0),
            _flat(tickets, "tickets", 1, torch.int32))
    with torch.cuda.device(p.device), _kernel("flat_adamw", 4 * n * (10 if ema is None else 12)):
        if schedule is None:
            rc = _lib.load_optim().eqf_flat_adamw(*args, _stream())
        else:
            rc = _lib.load_optim().eqf_flat_adamw_scheduled(*args, ctypes.byref(schedule.descriptor), _stream())
    _check(rc, "eqf_flat_adamw_scheduled" if schedule is not None else "eqf_flat_adamw")
