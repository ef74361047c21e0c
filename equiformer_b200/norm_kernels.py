"""Launchers of ``libeqf_b200_norm.so`` (``include/eqf_b200_norm.h``): the per-graph equivariant norms.

The norms have a library of their own, next to ``libeqf_b200.so``; these are its only callers.  The autograd family
built on them is ``ops.SegmentNorm``.
"""
from __future__ import annotations

import ctypes
from typing import Sequence

import torch

from . import _lib
from .ops import _kernel, _require_cuda, _require_index, _stream


class SegNormLayout:
    """Static description of a per-graph norm: ``entries`` = (mul, 2l+1, is 0e) per irreps entry, in e3nn order."""

    def __init__(self, entries: Sequence[tuple], eps: float, component: bool):
        self.entries, self.eps, self.component = tuple((int(m), int(d), bool(s)) for m, d, s in entries), float(eps), bool(component)
        self.n_w = sum(m for m, _, _ in self.entries)
        self.n_s = sum(m for m, _, s in self.entries if s)
        self.c = None                        # more entries than the kernels take: the torch statement serves
        if len(self.entries) > _lib.EQF_NORM_MAX_ENTRIES:
            return
        c = _lib.EqfSegNormLayout()
        c.n_entries, c.n_w, c.n_s, c.component, c.eps = len(self.entries), self.n_w, self.n_s, int(component), self.eps
        iw = i_s = 0
        for k, (m, d, s) in enumerate(self.entries):
            c.mul[k], c.d[k], c.is_scalar[k], c.w_off[k] = m, d, int(s), iw
            c.s_off[k] = i_s if s else -1
            iw += m
            i_s += m if s else 0
        self.c = c


def _ptr_array(ts: Sequence[torch.Tensor]):
    arr = (ctypes.c_void_p * _lib.EQF_NORM_MAX_ENTRIES)()
    for i, t in enumerate(ts):
        arr[i] = t.data_ptr()
    return arr


def _check(rc: int, what: str) -> None:
    _lib.check(rc, what, _lib.load_norm())


def graph_ptr_raw(batch: torch.Tensor, n_graphs: int) -> torch.Tensor:
    """``ptr[g]`` = first node of graph g, ``g = 0 .. n_graphs``, from an ascending ``batch`` (no host read)."""
    batch = _require_index(batch, "norm batch")
    ptr = torch.empty(n_graphs + 1, device=batch.device, dtype=torch.int64)
    with torch.cuda.device(batch.device), _kernel("norm_graph_ptr", 8 * (batch.numel() + n_graphs + 1)):
        rc = _lib.load_norm().eqf_norm_graph_ptr(batch.data_ptr(), batch.numel(), n_graphs, ptr.data_ptr(), _stream())
    _check(rc, "eqf_norm_graph_ptr")
    return ptr


def norm_fwd_raw(lay: SegNormLayout, xs, graph_ptr, n_graphs: int, shift, w, b):
    """Planar blocks ``xs`` -> (blocks y, mean ``[G, n_s]``, rstd ``[G, n_w]``); ``shift`` None for the instance norm."""
    xs = [_require_cuda(x, "norm block") for x in xs]
    dev = xs[0].device
    ys = [torch.empty_like(x) for x in xs]
    mean = torch.empty((n_graphs, lay.n_s), device=dev, dtype=torch.float32)
    rstd = torch.empty((n_graphs, lay.n_w), device=dev, dtype=torch.float32)
    with torch.cuda.device(dev), _kernel("norm_fwd", 12 * sum(x.numel() for x in xs)):
        rc = _lib.load_norm().eqf_norm_fwd(ctypes.byref(lay.c), _ptr_array(xs), graph_ptr.data_ptr(), n_graphs,
                                           shift.data_ptr() if shift is not None else None, w.data_ptr(),
                                           b.data_ptr() if b is not None and b.numel() else None, _ptr_array(ys),
                                           mean.data_ptr(), rstd.data_ptr(), _stream())
    _check(rc, "eqf_norm_fwd")
    return ys, mean, rstd


def norm_bwd_raw(lay: SegNormLayout, xs, gys, graph_ptr, n_graphs: int, shift, w, mean, rstd):
    """-> (gx blocks, d w ``[n_w]``, d b ``[n_s]``, d shift ``[len(shift)]`` or None)."""
    gys = [_require_cuda(g, "norm gy block") for g in gys]
    dev = xs[0].device
    gxs = [torch.empty_like(x) for x in xs]
    cols = lay.n_w + 2 * lay.n_s
    part = torch.empty((n_graphs, cols), device=dev, dtype=torch.float32)
    sums = torch.empty(cols, device=dev, dtype=torch.float32)
    lib = _lib.load_norm()
    with torch.cuda.device(dev), _kernel("norm_bwd", 16 * sum(x.numel() for x in xs)):
        rc = lib.eqf_norm_bwd(ctypes.byref(lay.c), _ptr_array(xs), _ptr_array(gys), graph_ptr.data_ptr(), n_graphs,
                              shift.data_ptr() if shift is not None else None, w.data_ptr(), mean.data_ptr(),
                              rstd.data_ptr(), _ptr_array(gxs), part.data_ptr(), _stream())
    _check(rc, "eqf_norm_bwd")
    with torch.cuda.device(dev), _kernel("norm_param_reduce", 4 * part.numel()):
        rc = lib.eqf_norm_param_reduce(part.data_ptr(), n_graphs, cols, sums.data_ptr(), _stream())
    _check(rc, "eqf_norm_param_reduce")
    gw, gb, gs = sums[:lay.n_w], sums[lay.n_w:lay.n_w + lay.n_s], sums[lay.n_w + lay.n_s:]
    gshift = None
    if shift is not None:
        # every 0e entry reads shift[0 : mul] (nets/graph_norm.py:90 keeps its offset at 0)
        gshift = torch.zeros_like(shift)
        off = 0
        for m, _d, s in lay.entries:
            if s:
                gshift[:m] += gs[off:off + m]
                off += m
    return gxs, gw, gb, gshift
