"""Autograd operators over the sm_90a edge kernels (``libeqf_b200.so``).

Two closed families (every derivative of a member is another member, so ``create_graph=True`` -
the MD17 force path, ``nets/graph_attention_transformer_md17.py:318-325`` - works to any order):

* depth-wise tensor product: ``DtpOut`` / ``DtpGradX`` / ``DtpGradW`` / ``DtpGradY`` are the four
  partial derivatives of ``S(x, y, w, g)`` (see ``csrc/eqf_dtp.cu``);
* attention aggregation: ``AttnAggregate`` / ``EdgeDot`` / ``EdgeScale`` are the three partial
  derivatives of ``T(alpha, V, G)`` (see ``csrc/eqf_attn.cu``); ``SegSoftmax`` has a kernel forward
  and a backward written with differentiable ops on the small ``[E, H]`` tensors.

All operands are planar blocks ``[rows, 2l+1, mul]`` (see ``plan.py``).  Tensors must be CUDA fp32;
anything else raises - there is no CPU implementation on the product path.
"""
from __future__ import annotations

import contextlib
import ctypes
import os
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib
from .plan import DtpPlan

# ----------------------------------------------------------------------------- helpers


def _require_cuda(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise _lib.EqfError(
            f"{name} lives on {t.device}: the equiformer_b200 edge kernels are CUDA-only (sm_90a); "
            "there is no CPU fallback on the product path")
    if t.dtype != torch.float32:
        raise _lib.EqfError(f"{name} must be float32 (the reference trains in fp32), got {t.dtype}")
    return t.contiguous()


def _require_index(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise _lib.EqfError(f"{name} lives on {t.device}: CUDA index tensor required")
    if t.dtype != torch.int64:
        t = t.to(torch.int64)
    return t.contiguous()


def _stream() -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr_array(ts: Sequence[torch.Tensor]):
    arr = (ctypes.c_void_p * _lib.EQF_MAX_BLOCKS)()
    for i, t in enumerate(ts):
        arr[i] = t.data_ptr()
    return arr


def _operands(plan: DtpPlan, xs, y, w, gs, w_shared: bool, gather=None, w_offset=None) -> _lib.EqfEdgeOperands:
    """``gather = (src, dst, x2s)``: x rows are ``xs[b][src[e]] (+ x2s[b][dst[e]])`` instead of ``xs[b][e]``;
    ``w_offset`` ``[W]``: the kernels read ``w[e] + w_offset`` (plan-specialised kernels only)."""
    op = _lib.EqfEdgeOperands()
    if w_offset is not None:
        w_offset = _require_cuda(w_offset, "w_offset")
        if w_shared or tuple(w_offset.shape) != (plan.weight_numel,):
            raise ValueError("w_offset must be [weight_numel] and needs per-edge weights")
        op.w_offset = w_offset.data_ptr()
    if xs is not None:
        for i, t in enumerate(xs):
            op.x[i] = t.data_ptr()
    if gather is not None:
        src, dst, x2s = gather
        op.src = src.data_ptr()
        if x2s is not None:
            op.dst = dst.data_ptr()
            for i, t in enumerate(x2s):
                op.x2[i] = t.data_ptr()
    if gs is not None:
        for i, t in enumerate(gs):
            op.g[i] = t.data_ptr()
    op.y = y.data_ptr()
    op.w = w.data_ptr() if w is not None else None
    op.w_shared = 1 if w_shared else 0
    return op


def _check_blocks(plan: DtpPlan, xs, E: int, what: str):
    if len(xs) != len(plan.in1_blocks):
        raise ValueError(f"{what}: expected {len(plan.in1_blocks)} in1 blocks, got {len(xs)}")
    out = []
    for t, (l, mul) in zip(xs, plan.in1_blocks):
        t = _require_cuda(t, what)
        if tuple(t.shape) != (E, 2 * l + 1, mul):
            raise ValueError(f"{what}: block shape {tuple(t.shape)} != {(E, 2 * l + 1, mul)}")
        out.append(t)
    return out


def _check_groups(plan: DtpPlan, gs, E: int, what: str):
    if len(gs) != len(plan.out_groups):
        raise ValueError(f"{what}: expected {len(plan.out_groups)} output groups, got {len(gs)}")
    out = []
    for t, (l, _p, mul) in zip(gs, plan.out_groups):
        t = _require_cuda(t, what)
        if tuple(t.shape) != (E, 2 * l + 1, mul):
            raise ValueError(f"{what}: group shape {tuple(t.shape)} != {(E, 2 * l + 1, mul)}")
        out.append(t)
    return out


def _check_yw(plan: DtpPlan, y, w, E: Optional[int] = None):
    y = _require_cuda(y, "edge_attr")
    if y.dim() != 2 or y.shape[1] != plan.d_y:
        raise ValueError(f"edge_attr must be [E, {plan.d_y}], got {tuple(y.shape)}")
    E = y.shape[0]
    shared = None
    if w is not None:
        w = _require_cuda(w, "weight")
        if w.dim() == 1:
            shared = True
            if w.shape[0] != plan.weight_numel:
                raise ValueError(f"shared weight must be [{plan.weight_numel}], got {tuple(w.shape)}")
        else:
            shared = False
            if tuple(w.shape) != (E, plan.weight_numel):
                raise ValueError(f"per-edge weight must be [{E}, {plan.weight_numel}], got {tuple(w.shape)}")
    return y, w, E, shared


# ----------------------------------------------------------------------------- launch accounting


class KernelProfile:
    """Optional per-launch accounting used by ``bench.py``: launch count and CUDA-event timing per kernel name.

    ``records`` holds ``(name, algorithmic_bytes, start_event, end_event, flops)`` for every launch of one of *our*
    kernels while the profile is installed (events are recorded on the launching stream, around the launch only);
    ``flops`` = useful multiply-adds x 2 of a contraction kernel (0 for streaming kernels).
    """

    def __init__(self, time_events: bool = True, presleep_cycles: int = 0):
        self.time_events = time_events
        # GPU-side delay queued before each timed launch so that the host has enqueued start-event, kernel and end-event
        # before the GPU reaches them: in a host-bound eager pass the event pair would otherwise include launch gaps.
        self.presleep_cycles = presleep_cycles
        self.launches = 0
        self.records = []

    def summary(self):
        out = {}
        for name, nbytes, s, e, flops in self.records:
            ms = s.elapsed_time(e)
            d = out.setdefault(name, {"launches": 0, "ms": 0.0, "bytes": 0, "flops": 0})
            d["launches"] += 1
            d["ms"] += ms
            d["bytes"] += nbytes
            d["flops"] += flops
        return out


PROFILE: Optional[KernelProfile] = None


@contextlib.contextmanager
def _kernel(name: str, nbytes: int, flops: int = 0):
    prof = PROFILE
    if prof is None:
        yield
        return
    prof.launches += 1
    if not prof.time_events:
        yield
        return
    s = torch.cuda.Event(enable_timing=True)
    e = torch.cuda.Event(enable_timing=True)
    if prof.presleep_cycles:
        torch.cuda._sleep(prof.presleep_cycles)
    s.record()
    yield
    e.record()
    prof.records.append((name, nbytes, s, e, flops))


def _dtp_bytes(plan: DtpPlan, E: int, shared: bool, kind: str) -> int:
    d_in, d_out, w = plan.irreps_in1.dim, plan.irreps_out.dim, (0 if shared else plan.weight_numel)
    per_edge = {"forward": d_in + plan.d_y + w + d_out,
                "grad_x": d_out + plan.d_y + w + d_in,
                "grad_w": d_out + plan.d_y + d_in + w,
                "grad_y": d_out + d_in + w + 2 * plan.d_y,
                "grad_xw": d_out + d_in + plan.d_y + w + d_in + w}[kind]
    return 4 * per_edge * E


def _attn_bytes(lay: "HeadLayout", rows_edge: int, rows_node: int, kind: str) -> int:
    dv = sum(d * c for d, c in zip(lay.ds, lay.Cs))
    h = lay.n_heads
    per = {"aggregate": rows_edge * (dv + h) + rows_node * dv,
           "edge_dot": rows_edge * (2 * dv + h),
           "edge_scale": rows_edge * (2 * dv + h)}[kind]
    return 4 * per


# ----------------------------------------------------------------------------- raw kernel calls


def _check_gather(plan: DtpPlan, xs, gather, E: int, what: str):
    """Validate gathered operands; returns (xs, gather) with contiguous CUDA tensors."""
    if gather is None:
        return _check_blocks(plan, xs, E, what), None
    src, dst, x2s = gather
    n_rows = xs[0].shape[0]
    xs = _check_blocks(plan, xs, n_rows, what)
    src = _require_index(src, "edge_src")
    if src.numel() != E:
        raise ValueError(f"{what}: gather index has {src.numel()} entries for {E} edges")
    if x2s is not None:
        x2s = _check_blocks(plan, x2s, x2s[0].shape[0], what)
        dst = _require_index(dst, "edge_dst")
    return xs, (src, dst, x2s)


def dtp_forward_raw(plan: DtpPlan, xs, y, w, gather=None, w_offset=None) -> List[torch.Tensor]:
    y, w, E, shared = _check_yw(plan, y, w)
    xs, gather = _check_gather(plan, xs, gather, E, "dtp_forward x")
    outs = [torch.empty((E, 2 * l + 1, mul), device=y.device, dtype=torch.float32) for l, _p, mul in plan.out_groups]
    op = _operands(plan, xs, y, w, None, shared, gather, w_offset)
    with torch.cuda.device(y.device), _kernel("dtp_forward", _dtp_bytes(plan, E, shared, "forward")):
        rc = _lib.load().eqf_dtp_forward(plan.handle, ctypes.byref(op), E, _ptr_array(outs), _stream())
    _lib.check(rc, "eqf_dtp_forward")
    return outs


def dtp_grad_x_raw(plan: DtpPlan, gs, y, w) -> List[torch.Tensor]:
    y, w, E, shared = _check_yw(plan, y, w)
    gs = _check_groups(plan, gs, E, "dtp_grad_x g")
    gxs = [torch.empty((E, 2 * l + 1, mul), device=y.device, dtype=torch.float32) for l, mul in plan.in1_blocks]
    op = _operands(plan, None, y, w, gs, shared)
    with torch.cuda.device(y.device), _kernel("dtp_grad_x", _dtp_bytes(plan, E, shared, "grad_x")):
        rc = _lib.load().eqf_dtp_grad_x(plan.handle, ctypes.byref(op), E, _ptr_array(gxs), _stream())
    _lib.check(rc, "eqf_dtp_grad_x")
    return gxs


def _gw_buffer(plan: DtpPlan, E: int, shared: bool, device) -> torch.Tensor:
    if shared:
        # upper bound on the CTAs of whichever kernel generation runs; rows a launch does not write must read as zero
        rows = _lib.load().eqf_plan_partial_rows(plan.handle, E)
        return torch.zeros((max(rows, 1), plan.weight_numel), device=device, dtype=torch.float32)
    return torch.empty((E, plan.weight_numel), device=device, dtype=torch.float32)


def dtp_grad_w_raw(plan: DtpPlan, xs, y, gs, shared: bool) -> torch.Tensor:
    y, _, E, _ = _check_yw(plan, y, None)
    xs = _check_blocks(plan, xs, E, "dtp_grad_w x")
    gs = _check_groups(plan, gs, E, "dtp_grad_w g")
    if E == 0:
        return torch.zeros((plan.weight_numel,) if shared else (0, plan.weight_numel), device=y.device)
    gw = _gw_buffer(plan, E, shared, y.device)
    op = _operands(plan, xs, y, None, gs, shared)
    with torch.cuda.device(y.device), _kernel("dtp_grad_w", _dtp_bytes(plan, E, shared, "grad_w")):
        rc = _lib.load().eqf_dtp_grad_w(plan.handle, ctypes.byref(op), E, ctypes.c_void_p(gw.data_ptr()), _stream())
    _lib.check(rc, "eqf_dtp_grad_w")
    return _colsum(gw) if shared else gw


def dtp_grad_y_raw(plan: DtpPlan, xs, w, gs, y_like) -> torch.Tensor:
    y, w, E, shared = _check_yw(plan, y_like, w)
    xs = _check_blocks(plan, xs, E, "dtp_grad_y x")
    gs = _check_groups(plan, gs, E, "dtp_grad_y g")
    gy = torch.empty((E, plan.d_y), device=y.device, dtype=torch.float32)
    op = _operands(plan, xs, y, w, gs, shared)
    with torch.cuda.device(y.device), _kernel("dtp_grad_y", _dtp_bytes(plan, E, shared, "grad_y")):
        rc = _lib.load().eqf_dtp_grad_y(plan.handle, ctypes.byref(op), E, ctypes.c_void_p(gy.data_ptr()), _stream())
    _lib.check(rc, "eqf_dtp_grad_y")
    return gy


def dtp_grad_xw_raw(plan: DtpPlan, xs, y, w, gs, gather=None, w_offset=None) -> Tuple[List[torch.Tensor], torch.Tensor]:
    y, w, E, shared = _check_yw(plan, y, w)
    xs, gather = _check_gather(plan, xs, gather, E, "dtp_grad_xw x")
    gs = _check_groups(plan, gs, E, "dtp_grad_xw g")
    gxs = [torch.empty((E, 2 * l + 1, mul), device=y.device, dtype=torch.float32) for l, mul in plan.in1_blocks]
    if E == 0:
        return gxs, torch.zeros_like(w)
    gw = _gw_buffer(plan, E, shared, y.device)
    op = _operands(plan, xs, y, w, gs, shared, gather, w_offset)
    with torch.cuda.device(y.device), _kernel("dtp_grad_xw", _dtp_bytes(plan, E, shared, "grad_xw")):
        rc = _lib.load().eqf_dtp_grad_xw(plan.handle, ctypes.byref(op), E, _ptr_array(gxs),
                                         ctypes.c_void_p(gw.data_ptr()), _stream())
    _lib.check(rc, "eqf_dtp_grad_xw")
    return gxs, (_colsum(gw) if shared else gw)


# ----------------------------------------------------------------------------- DTP autograd family


def _fill(gs, likes):
    return [g if g is not None else torch.zeros_like(t) for g, t in zip(gs, likes)]


class DtpOut(torch.autograd.Function):
    """fs = dS/dg (x, y, w): the tensor product itself.  apply(plan, y, w, *xs) -> tuple(groups)."""

    @staticmethod
    def forward(ctx, plan: DtpPlan, y, w, *xs):
        ctx.plan = plan
        outs = dtp_forward_raw(plan, xs, y, w)
        ctx.save_for_backward(y, w, *xs)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *gs):
        plan = ctx.plan
        y, w, *xs = ctx.saved_tensors
        nb = len(xs)
        E = y.shape[0]
        gs = [g if g is not None else torch.zeros((E, 2 * l + 1, m), device=y.device)
              for g, (l, _p, m) in zip(gs, plan.out_groups)]
        need_y, need_w = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        need_x = any(ctx.needs_input_grad[3:3 + nb])
        gy = gw = None
        gxs = [None] * nb
        if torch.is_grad_enabled():  # create_graph=True: stay inside the differentiable family
            if need_x:
                gxs = list(DtpGradX.apply(plan, y, w, *gs))
            if need_w:
                gw = DtpGradW.apply(plan, y, w.dim() == 1, *xs, *gs)
            if need_y:
                gy = DtpGradY.apply(plan, y, w, *xs, *gs)
        else:
            gs = [g.contiguous() for g in gs]
            if need_x and need_w:
                gxs, gw = dtp_grad_xw_raw(plan, xs, y, w, gs)
            elif need_x:
                gxs = dtp_grad_x_raw(plan, gs, y, w)
            elif need_w:
                gw = dtp_grad_w_raw(plan, xs, y, gs, w.dim() == 1)
            if need_y:
                gy = dtp_grad_y_raw(plan, xs, w, gs, y)
        return (None, gy, gw, *gxs)


class DtpGradX(torch.autograd.Function):
    """gxs = dS/dx (g, y, w).  apply(plan, y, w, *gs) -> tuple(in1 blocks)."""

    @staticmethod
    def forward(ctx, plan: DtpPlan, y, w, *gs):
        ctx.plan = plan
        outs = dtp_grad_x_raw(plan, gs, y, w)
        ctx.save_for_backward(y, w, *gs)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *cxs):  # cotangents shaped like xs
        plan = ctx.plan
        y, w, *gs = ctx.saved_tensors
        E = y.shape[0]
        cxs = [c if c is not None else torch.zeros((E, 2 * l + 1, m), device=y.device)
               for c, (l, m) in zip(cxs, plan.in1_blocks)]
        need_y, need_w = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        need_g = any(ctx.needs_input_grad[3:])
        gy = gw = None
        ggs = [None] * len(gs)
        if need_g:
            ggs = list(DtpOut.apply(plan, y, w, *cxs))
        if need_w:
            gw = DtpGradW.apply(plan, y, w.dim() == 1, *cxs, *gs)
        if need_y:
            gy = DtpGradY.apply(plan, y, w, *cxs, *gs)
        return (None, gy, gw, *ggs)


class DtpGradW(torch.autograd.Function):
    """gw = dS/dw (x, y, g).  apply(plan, y, shared, *xs, *gs) -> [E, W] or [W]."""

    @staticmethod
    def forward(ctx, plan: DtpPlan, y, shared: bool, *xg):
        nb = len(plan.in1_blocks)
        xs, gs = xg[:nb], xg[nb:]
        ctx.plan, ctx.shared = plan, shared
        out = dtp_grad_w_raw(plan, xs, y, gs, shared)
        ctx.save_for_backward(y, *xg)
        return out

    @staticmethod
    def backward(ctx, cw):
        plan = ctx.plan
        y, *xg = ctx.saved_tensors
        nb = len(plan.in1_blocks)
        xs, gs = xg[:nb], xg[nb:]
        need_y = ctx.needs_input_grad[1]
        need_x = any(ctx.needs_input_grad[3:3 + nb])
        need_g = any(ctx.needs_input_grad[3 + nb:])
        cw = cw.contiguous()
        gy = None
        gxs = [None] * nb
        ggs = [None] * len(gs)
        if need_x:
            gxs = list(DtpGradX.apply(plan, y, cw, *gs))
        if need_g:
            ggs = list(DtpOut.apply(plan, y, cw, *xs))
        if need_y:
            gy = DtpGradY.apply(plan, y, cw, *xs, *gs)
        return (None, gy, None, *gxs, *ggs)


class DtpGradY(torch.autograd.Function):
    """gy = dS/dy (x, w, g).  apply(plan, y_like, w, *xs, *gs) -> [E, d_y] (y only fixes the shape)."""

    @staticmethod
    def forward(ctx, plan: DtpPlan, y_like, w, *xg):
        nb = len(plan.in1_blocks)
        xs, gs = xg[:nb], xg[nb:]
        ctx.plan = plan
        out = dtp_grad_y_raw(plan, xs, w, gs, y_like)
        ctx.save_for_backward(w, *xg)
        return out

    @staticmethod
    def backward(ctx, cy):
        plan = ctx.plan
        w, *xg = ctx.saved_tensors
        nb = len(plan.in1_blocks)
        xs, gs = xg[:nb], xg[nb:]
        need_w = ctx.needs_input_grad[2]
        need_x = any(ctx.needs_input_grad[3:3 + nb])
        need_g = any(ctx.needs_input_grad[3 + nb:])
        cy = cy.contiguous()
        gw = None
        gxs = [None] * nb
        ggs = [None] * len(gs)
        if need_x:
            gxs = list(DtpGradX.apply(plan, cy, w, *gs))
        if need_g:
            ggs = list(DtpOut.apply(plan, cy, w, *xs))
        if need_w:
            gw = DtpGradW.apply(plan, cy, w.dim() == 1, *xs, *gs)
        return (None, None, gw, *gxs, *ggs)


class DtpOutGathered(torch.autograd.Function):
    """DTP whose in1 operand is gathered inside the kernel: ``x_e = A[src_e] (+ B[dst_e])`` (ref :487 fused into :491).

    apply(plan, graph, n_b, y, w, *As, *Bs) with ``n_b`` = 0 (no B tables) or len(As).  First-order backward is two
    kernels (grad_xw with the same gather, then segment sums to the node tables by dst and - through the CSC - by src);
    under ``create_graph`` the backward re-expresses itself with the differentiable primitives instead.
    """

    @staticmethod
    def forward(ctx, plan: DtpPlan, graph: "Graph", n_b: int, y, w, *AB):
        nb = len(plan.in1_blocks)
        As, Bs = AB[:nb], (AB[nb:] if n_b else None)
        ctx.plan, ctx.graph, ctx.n_b = plan, graph, n_b
        outs = dtp_forward_raw(plan, As, y, w, gather=(graph.src, graph.dst, Bs))
        ctx.save_for_backward(y, w, *AB)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *gs):
        plan, graph, n_b = ctx.plan, ctx.graph, ctx.n_b
        y, w, *AB = ctx.saved_tensors
        nb = len(plan.in1_blocks)
        As, Bs = AB[:nb], (AB[nb:] if n_b else None)
        E = y.shape[0]
        gs = [g if g is not None else torch.zeros((E, 2 * l + 1, m), device=y.device)
              for g, (l, _p, m) in zip(gs, plan.out_groups)]
        need_y, need_w = ctx.needs_input_grad[3], ctx.needs_input_grad[4]
        need_x = any(ctx.needs_input_grad[5:])
        if torch.is_grad_enabled():   # higher-order: differentiable composition of the primitive family
            xs = [a.index_select(0, graph.src) for a in As]
            if Bs is not None:
                xs = [x + b.index_select(0, graph.dst) for x, b in zip(xs, Bs)]
            gy = DtpGradY.apply(plan, y, w, *xs, *gs) if need_y else None
            gw = DtpGradW.apply(plan, y, w.dim() == 1, *xs, *gs) if need_w else None
            gA = [None] * nb
            gB = [None] * nb
            if need_x:
                gxs = DtpGradX.apply(plan, y, w, *gs)
                gA = [torch.zeros_like(a).index_add(0, graph.src, g) for a, g in zip(As, gxs)]
                if Bs is not None:
                    gB = [torch.zeros_like(b).index_add(0, graph.dst, g) for b, g in zip(Bs, gxs)]
            return (None, None, None, gy, gw, *gA, *(gB if Bs is not None else []))
        gs = [g.contiguous() for g in gs]
        gather = (graph.src, graph.dst, Bs)
        gy = gw = None
        gA = [None] * nb
        gB = [None] * nb
        if need_x or need_w:
            gxs, gw_full = dtp_grad_xw_raw(plan, As, y, w, gs, gather=gather)
            gw = gw_full if need_w else None
            if need_x:
                lay = HeadLayout([2 * l + 1 for l, _ in plan.in1_blocks], [m for _, m in plan.in1_blocks], 1)
                gA = attn_aggregate_raw(lay, None, gxs, graph, by_src=True)
                if Bs is not None:
                    gB = attn_aggregate_raw(lay, None, gxs, graph)
        if need_y:
            xs = [a.index_select(0, graph.src) for a in As]
            if Bs is not None:
                xs = [x + b.index_select(0, graph.dst) for x, b in zip(xs, Bs)]
            gy = dtp_grad_y_raw(plan, xs, w, gs, y)
        return (None, None, None, gy, gw, *gA, *(gB if Bs is not None else []))


class DtpOutGatheredOffset(torch.autograd.Function):
    """:class:`DtpOutGathered` with per-edge weights ``w + offset`` where the ``[W]`` offset is added inside the kernels'
    weight load (the radial ``offset`` of ref radial_func.py:45-49 never takes its own pass over ``[E, W]``).

    apply(plan, graph, n_b, y, w, offset, *As, *Bs)."""

    @staticmethod
    def forward(ctx, plan: DtpPlan, graph: "Graph", n_b: int, y, w, offset, *AB):
        nb = len(plan.in1_blocks)
        As, Bs = AB[:nb], (AB[nb:] if n_b else None)
        ctx.plan, ctx.graph, ctx.n_b = plan, graph, n_b
        outs = dtp_forward_raw(plan, As, y, w, gather=(graph.src, graph.dst, Bs), w_offset=offset)
        ctx.save_for_backward(y, w, offset, *AB)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *gs):
        plan, graph, n_b = ctx.plan, ctx.graph, ctx.n_b
        y, w, offset, *AB = ctx.saved_tensors
        nb = len(plan.in1_blocks)
        As, Bs = AB[:nb], (AB[nb:] if n_b else None)
        E = y.shape[0]
        gs = [g if g is not None else torch.zeros((E, 2 * l + 1, m), device=y.device)
              for g, (l, _p, m) in zip(gs, plan.out_groups)]
        need_y, need_w, need_off = ctx.needs_input_grad[3:6]
        need_x = any(ctx.needs_input_grad[6:])
        if torch.is_grad_enabled() or need_y:    # higher order / forces: the differentiable family on w + offset
            fn = lambda yy, ww, oo, *ab: DtpOutGathered.apply(plan, graph, n_b, yy, ww + oo, *ab)
            grads = _higher_order_grads(fn, (y, w, offset, *AB), gs)
            return (None, None, None, *grads)
        gs = [g.contiguous() for g in gs]
        gw = goff = None
        gA = [None] * nb
        gB = [None] * nb
        if need_x or need_w or need_off:
            gxs, gw = dtp_grad_xw_raw(plan, As, y, w, gs, gather=(graph.src, graph.dst, Bs), w_offset=offset)
            if need_off:
                goff = colsum_raw(gw)
            if need_x:
                lay = HeadLayout([2 * l + 1 for l, _ in plan.in1_blocks], [m for _, m in plan.in1_blocks], 1)
                gA = attn_aggregate_raw(lay, None, gxs, graph, by_src=True)
                if Bs is not None:
                    gB = attn_aggregate_raw(lay, None, gxs, graph)
        return (None, None, None, None, gw if need_w else None, goff, *gA, *(gB if Bs is not None else []))


def depthwise_tensor_product_gathered(plan: DtpPlan, graph: "Graph", As, Bs, y, w, w_offset=None):
    """``DTP(A[src] (+ B[dst]), y; w (+ w_offset))`` with the gather done inside the kernel.  ``Bs`` may be None."""
    AB = (*As, *(Bs if Bs is not None else ()))
    n_b = 0 if Bs is None else len(Bs)
    if w_offset is not None:
        if plan.generated and w.dim() == 2 and fused_ok(y):
            return list(DtpOutGatheredOffset.apply(plan, graph, n_b, y, w, w_offset, *AB))
        w = w + w_offset
    return list(DtpOutGathered.apply(plan, graph, n_b, y, w, *AB))


# ----------------------------------------------------------------------------- K1: DTP fused into the per-degree linear

# EQF_FUSED: "1" fused forward everywhere, "0" the round-1 pipeline (DTP -> [E, 3136] in HBM -> GEMMs), "auto" (default) by
# size.  The fused forward keeps the [E, 3136] products out of HBM and out of the saved activations - what lets large
# periodic cells (E ~ 5e5) train at all - but its producer warps are latency bound (gathers + per-k-tile handshakes), so
# below _FUSED_MIN_EDGES the unfused pipeline is kept.
_FUSED_MODE = os.environ.get("EQF_FUSED", "auto")
_FUSED = _FUSED_MODE != "0"
_FUSED_MIN_EDGES = int(os.environ.get("EQF_FUSED_MIN_EDGES", "200000"))
_FUSED_SPLIT = {}


def dtp_linear_supported(plan: DtpPlan) -> bool:
    """True when every output group of ``plan`` can run through ``eqf_dtp_linear_fwd`` (multiplicities % 32 == 0, the
    tile's coupling blocks fit shared memory)."""
    ok = getattr(plan, "_fused_ok", None)
    if ok is None:
        lib = _lib.load()
        ok = all(lib.eqf_dtp_linear_supported(plan.handle, g) == 1 for g in range(len(plan.out_groups)))
        plan._fused_ok = ok
    return ok


def dtp_linear_ok(plan: DtpPlan, y: torch.Tensor, w: torch.Tensor) -> bool:
    """Policy: the fused kernel carries first-order training / inference on CUDA; when the edge harmonics need a
    gradient (MD17 forces, ``create_graph``) the closed differentiable family of the unfused kernels is used."""
    if not _FUSED or (_FUSED_MODE == "auto" and y.shape[0] < _FUSED_MIN_EDGES and not FUSED_ON_ANY_DEVICE):
        return False
    return (fused_ok(y) and not (torch.is_grad_enabled() and y.requires_grad)
            and y.shape[0] > 0 and dtp_linear_supported(plan))


def dtp_linear_fwd_raw(plan: DtpPlan, group: int, xs, y, w, Wt: torch.Tensor, gather=None, w_offset=None) -> torch.Tensor:
    """``C[e, k, :] = DTP_group(x, y; w)[e, k, :] @ Wt`` with the tensor product produced on chip as the A operand of the
    wgmma GEMM (``eqf_dtp_linear_fwd``): ``[E, 2 l3 + 1, N]``.  ``Wt`` is ``[K_group, N]``."""
    y, w, E, shared = _check_yw(plan, y, w)
    xs, gather = _check_gather(plan, xs, gather, E, "dtp_linear x")
    l3, _p, K = plan.out_groups[group]
    Wt = _require_cuda(Wt, "dtp_linear weight")
    if Wt.dim() != 2 or Wt.shape[0] != K:
        raise ValueError(f"dtp_linear: weight must be [{K}, N], got {tuple(Wt.shape)}")
    N = Wt.shape[1]
    d3 = 2 * l3 + 1
    C = torch.empty((E, d3, N), device=y.device, dtype=torch.float32)
    need = 2 * N * K
    split = _FUSED_SPLIT.get(y.device)
    if split is None or split.numel() < need:
        split = torch.empty(max(need, 1 << 20), device=y.device, dtype=torch.float32)
        _FUSED_SPLIT[y.device] = split
    op = _operands(plan, xs, y, w, None, shared, gather, w_offset)
    d_in = sum((2 * l + 1) * m for l, m in plan.in1_blocks)
    nbytes = 4 * (E * (d_in + plan.d_y + (0 if shared else K) + d3 * N) + K * N)
    with torch.cuda.device(y.device), _kernel("dtp_linear_fwd", nbytes, 2 * E * d3 * K * N):
        rc = _lib.load().eqf_dtp_linear_fwd(plan.handle, ctypes.byref(op), E, group, Wt.data_ptr(), N, Wt.stride(0),
                                            C.data_ptr(), N, split.data_ptr(), _stream())
    _lib.check(rc, "eqf_dtp_linear_fwd")
    return C


# widest linear that is fused: the fused kernel's column tiles are 64 wide (its consumers hold the accumulator in
# registers), and a wider linear would recompute the product once per tile, so its group is written to HBM once
# (eqf_dtp_group_forward) and read by the wgmma GEMM.  On the stress workload (H100) fusing the 128-column linears as
# well measured about 1 % slower per step.
_FUSED_MAX_N = int(os.environ.get("EQF_FUSED_MAX_N", "64"))


def dtp_group_forward_raw(plan: DtpPlan, group: int, xs, y, w, gather=None, w_offset=None) -> torch.Tensor:
    """One output group of the depth-wise product, ``[E, 2 l3 + 1, K]`` (``eqf_dtp_group_forward``)."""
    y, w, E, shared = _check_yw(plan, y, w)
    xs, gather = _check_gather(plan, xs, gather, E, "dtp_group_forward x")
    l3, _p, K = plan.out_groups[group]
    out = torch.empty((E, 2 * l3 + 1, K), device=y.device, dtype=torch.float32)
    op = _operands(plan, xs, y, w, None, shared, gather, w_offset)
    d_in = sum((2 * l + 1) * m for l, m in plan.in1_blocks)
    nbytes = 4 * E * (d_in + plan.d_y + (0 if shared else K) + (2 * l3 + 1) * K)
    with torch.cuda.device(y.device), _kernel("dtp_group_forward", nbytes):
        rc = _lib.load().eqf_dtp_group_forward(plan.handle, ctypes.byref(op), E, group, out.data_ptr(), _stream())
    _lib.check(rc, "eqf_dtp_group_forward")
    return out


def _dtp_linear_unfused(plan: DtpPlan, graph, n_b: int, y, w, offset, AB, Ws):
    """The same map from differentiable primitives (higher-order path, and the statement the fused kernel is tested
    against): DTP family + one GEMM per output group."""
    nb = len(plan.in1_blocks)
    As, Bs = AB[:nb], (AB[nb:] if n_b else None)
    if graph is not None:
        f = depthwise_tensor_product_gathered(plan, graph, As, Bs, y, w, offset)
    else:
        f = depthwise_tensor_product(plan, As, y, w if offset is None else w + offset)
    E = y.shape[0]
    return [matmul_f32(fg.reshape(E * fg.shape[1], fg.shape[2]), W).view(E, fg.shape[1], -1) for fg, W in zip(f, Ws)]


class DtpLinear(torch.autograd.Function):
    """K1 (ref nets/graph_attention_transformer.py:487-496): every output group of a depth-wise tensor product times its
    channel-mixing matrix, the ``[E, sum K]`` product never leaving the chip.

    apply(plan, graph_or_None, n_b, y, w, offset_or_None, *As, *Bs, *Ws) -> one ``[E, 2 l + 1, N_g]`` tensor per group.
    ``graph`` given: the in1 operand is ``A[src] (+ B[dst])``; None: ``As`` are per-edge blocks.  Backward (first order)
    recomputes the tensor product for the weight gradients, then runs the data-gradient GEMMs and the DTP backward;
    under ``create_graph`` it re-expresses itself with the differentiable primitives."""

    @staticmethod
    def forward(ctx, plan: DtpPlan, graph, n_b: int, y, w, offset, *rest):
        nb, ng = len(plan.in1_blocks), len(plan.out_groups)
        n_ab = nb + (nb if n_b else 0)
        AB, Ws = rest[:n_ab], rest[n_ab:]
        if len(Ws) != ng:
            raise ValueError(f"DtpLinear: expected {ng} weight matrices, got {len(Ws)}")
        As, Bs = AB[:nb], (AB[nb:] if n_b else None)
        gather = (graph.src, graph.dst, Bs) if graph is not None else None
        outs = []
        for g in range(ng):
            if Ws[g].shape[1] <= _FUSED_MAX_N:
                outs.append(dtp_linear_fwd_raw(plan, g, As, y, w, Ws[g], gather=gather, w_offset=offset))
            else:
                fg = dtp_group_forward_raw(plan, g, As, y, w, gather=gather, w_offset=offset)
                E, d = fg.shape[0], fg.shape[1]
                outs.append(gemm_raw(0, fg.reshape(E * d, fg.shape[2]), Ws[g].contiguous()).view(E, d, -1))
        ctx.plan, ctx.graph, ctx.n_b, ctx.n_ab, ctx.has_off = plan, graph, n_b, n_ab, offset is not None
        ctx.save_for_backward(y, w, *([offset] if offset is not None else []), *rest)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *dCs):
        plan, graph, n_b, n_ab = ctx.plan, ctx.graph, ctx.n_b, ctx.n_ab
        y, w, *saved = ctx.saved_tensors
        offset = saved.pop(0) if ctx.has_off else None
        AB, Ws = saved[:n_ab], saved[n_ab:]
        nb, ng = len(plan.in1_blocks), len(plan.out_groups)
        As, Bs = AB[:nb], (AB[nb:] if n_b else None)
        E = y.shape[0]
        dCs = [g if g is not None else torch.zeros((E, 2 * l + 1, W.shape[1]), device=y.device)
               for g, (l, _p, _k), W in zip(dCs, plan.out_groups, Ws)]
        need = ctx.needs_input_grad
        need_y, need_w, need_off = need[3], need[4], need[5]
        need_x = any(need[6:6 + n_ab])
        need_W = need[6 + n_ab:]
        if torch.is_grad_enabled() or need_y:
            fn = lambda yy, ww, oo, *r: tuple(_dtp_linear_unfused(plan, graph, n_b, yy, ww, oo, r[:n_ab], r[n_ab:]))
            grads = _higher_order_grads(fn, (y, w, offset, *AB, *Ws), dCs)
            return (None, None, None, *grads)
        gather = (graph.src, graph.dst, Bs) if graph is not None else None
        shared = w.dim() == 1
        f = dtp_forward_raw(plan, As, y, w, gather=gather, w_offset=offset)        # recomputed, not saved
        gWs, dfs = [], []
        for g in range(ng):
            d, K = f[g].shape[1], f[g].shape[2]
            dC2 = dCs[g].contiguous().reshape(E * d, -1)
            gWs.append(gemm_raw(2, f[g].reshape(E * d, K), dC2) if need_W[g] else None)
            dfs.append(gemm_raw(1, dC2, Ws[g]).view(E, d, K) if (need_x or need_w or need_off) else None)
        del f
        gw = goff = None
        gA = [None] * nb
        gB = [None] * nb
        if need_x or need_w or need_off:
            gxs, gw_full = dtp_grad_xw_raw(plan, As, y, w, dfs, gather=gather, w_offset=offset)
            gw = gw_full if need_w else None
            if need_off:
                goff = colsum_raw(gw_full)
            if need_x:
                if graph is None:
                    gA = gxs
                else:
                    lay = HeadLayout([2 * l + 1 for l, _ in plan.in1_blocks], [m for _, m in plan.in1_blocks], 1)
                    gA = attn_aggregate_raw(lay, None, gxs, graph, by_src=True)
                    if Bs is not None:
                        gB = attn_aggregate_raw(lay, None, gxs, graph)
        return (None, None, None, None, gw, goff, *gA, *(gB if Bs is not None else []), *gWs)


def dtp_linear(plan: DtpPlan, graph, As, Bs, y, w, w_offset, Ws):
    """Fused ``[DTP(A[src] (+ B[dst]), y; w (+ w_offset)) @ W_g for every output group g]`` (see :class:`DtpLinear`)."""
    AB = (*As, *(Bs if Bs is not None else ()))
    n_b = 0 if Bs is None else len(Bs)
    return list(DtpLinear.apply(plan, graph, n_b, y, w, w_offset, *AB, *Ws))


def depthwise_tensor_product(plan: DtpPlan, xs: Sequence[torch.Tensor], y: torch.Tensor, w: torch.Tensor):
    """Planar DTP: ``xs`` per in1 block ``[E, 2l+1, mul]`` -> list per output group ``[E, 2l+1, K]``."""
    return list(DtpOut.apply(plan, y, w, *xs))


# ----------------------------------------------------------------------------- attention family


class HeadLayout:
    """Planar value layout: groups ``[rows, d[g], C[g]]``; head h owns channels ``[h*C/H, (h+1)*C/H)``."""

    def __init__(self, ds: Sequence[int], Cs: Sequence[int], n_heads: int):
        if len(ds) != len(Cs) or not ds:
            raise ValueError("bad head layout")
        if len(ds) > _lib.EQF_MAX_BLOCKS or n_heads > _lib.EQF_MAX_HEADS:
            raise NotImplementedError("head layout exceeds kernel limits")
        for c in Cs:
            if c % n_heads:
                raise ValueError("channels per group must be divisible by the number of heads")
        self.ds, self.Cs, self.n_heads = tuple(ds), tuple(Cs), int(n_heads)
        c = _lib.EqfHeadLayout()
        c.n_groups = len(ds)
        c.n_heads = n_heads
        for i, (d, C) in enumerate(zip(ds, Cs)):
            c.d[i], c.C[i] = d, C
        self.c = c

    def check(self, ts, rows: int, what: str):
        if len(ts) != len(self.ds):
            raise ValueError(f"{what}: expected {len(self.ds)} groups")
        out = []
        for t, d, C in zip(ts, self.ds, self.Cs):
            t = _require_cuda(t, what)
            if tuple(t.shape) != (rows, d, C):
                raise ValueError(f"{what}: group shape {tuple(t.shape)} != {(rows, d, C)}")
            out.append(t)
        return out


class Graph:
    """Destination-sorted edge list + CSR ``row_ptr`` (built once per forward, shared by all layers)."""

    def __init__(self, edge_src: torch.Tensor, edge_dst: torch.Tensor, n_nodes: int, check_sorted: bool = True):
        self.n_nodes = int(n_nodes)
        self.perm = None
        edge_src = _require_index(edge_src, "edge_src")
        edge_dst = _require_index(edge_dst, "edge_dst")
        if check_sorted and edge_dst.numel() > 1 and bool((edge_dst[1:] < edge_dst[:-1]).any()):
            self.perm = torch.sort(edge_dst, stable=True).indices
            edge_src, edge_dst = edge_src[self.perm], edge_dst[self.perm]
        self.src, self.dst = edge_src, edge_dst
        self.n_edges = int(edge_dst.numel())
        counts = torch.bincount(edge_dst, minlength=self.n_nodes)
        self.row_ptr = torch.zeros(self.n_nodes + 1, dtype=torch.int64, device=edge_dst.device)
        torch.cumsum(counts, 0, out=self.row_ptr[1:])

    def sort_edges(self, t: torch.Tensor) -> torch.Tensor:
        return t if self.perm is None else t.index_select(0, self.perm)

    def build_csc(self) -> None:
        """Source-sorted view of the same edge list: ``src_perm`` (segment position -> edge id) and ``src_row_ptr``."""
        self._src_perm = torch.sort(self.src, stable=True).indices
        # counts by scatter-add (torch.bincount synchronises with the host; this has to be capturable in a CUDA graph)
        counts = torch.zeros(self.n_nodes, dtype=torch.int64, device=self.src.device)
        counts.index_add_(0, self.src, torch.ones_like(self.src))
        self._src_row_ptr = torch.zeros(self.n_nodes + 1, dtype=torch.int64, device=self.src.device)
        torch.cumsum(counts, 0, out=self._src_row_ptr[1:])

    @property
    def src_perm(self) -> torch.Tensor:
        if getattr(self, "_src_perm", None) is None:
            self.build_csc()
        return self._src_perm

    @property
    def src_row_ptr(self) -> torch.Tensor:
        if getattr(self, "_src_row_ptr", None) is None:
            self.build_csc()
        return self._src_row_ptr


def seg_softmax_raw(z: torch.Tensor, graph: Graph) -> torch.Tensor:
    z = _require_cuda(z, "attention logits")
    if z.dim() != 2 or z.shape[0] != graph.n_edges:
        raise ValueError("logits must be [E, H]")
    alpha = torch.empty_like(z)
    with torch.cuda.device(z.device), _kernel("seg_softmax", 8 * z.numel()):
        rc = _lib.load().eqf_seg_softmax(z.data_ptr(), graph.row_ptr.data_ptr(), graph.n_nodes, z.shape[1],
                                         alpha.data_ptr(), _stream())
    _lib.check(rc, "eqf_seg_softmax")
    return alpha


def seg_softmax_bwd_raw(alpha: torch.Tensor, ga: torch.Tensor, graph: Graph) -> torch.Tensor:
    ga = _require_cuda(ga, "softmax cotangent").contiguous()
    gz = torch.empty_like(alpha)
    with torch.cuda.device(alpha.device), _kernel("seg_softmax_bwd", 12 * alpha.numel()):
        rc = _lib.load().eqf_seg_softmax_bwd(alpha.data_ptr(), ga.data_ptr(), graph.row_ptr.data_ptr(), graph.n_nodes,
                                             alpha.shape[1], gz.data_ptr(), _stream())
    _lib.check(rc, "eqf_seg_softmax_bwd")
    return gz


def attn_aggregate_raw(lay: HeadLayout, alpha, Vs, graph: Graph, by_src: bool = False) -> List[torch.Tensor]:
    """Segment reduction over destination segments (default) or, with ``by_src``, over source segments via the CSC."""
    Vs = lay.check(Vs, graph.n_edges, "aggregate V")
    if alpha is not None:
        alpha = _require_cuda(alpha, "alpha")
        if tuple(alpha.shape) != (graph.n_edges, lay.n_heads):
            raise ValueError("alpha must be [E, H]")
    dev = Vs[0].device
    outs = [torch.empty((graph.n_nodes, d, C), device=dev, dtype=torch.float32) for d, C in zip(lay.ds, lay.Cs)]
    if by_src:
        row_ptr, perm = graph.src_row_ptr, graph.src_perm
    else:
        row_ptr, perm = graph.row_ptr, None
    with torch.cuda.device(dev), _kernel("attn_aggregate", _attn_bytes(lay, graph.n_edges, graph.n_nodes, "aggregate")):
        rc = _lib.load().eqf_attn_aggregate(ctypes.byref(lay.c), alpha.data_ptr() if alpha is not None else None,
                                            _ptr_array(Vs), row_ptr.data_ptr(),
                                            perm.data_ptr() if perm is not None else None, graph.n_nodes,
                                            _ptr_array(outs), _stream())
    _lib.check(rc, "eqf_attn_aggregate")
    return outs


def attn_edge_dot_raw(lay: HeadLayout, Vs, Gs, graph: Graph) -> torch.Tensor:
    Vs = lay.check(Vs, graph.n_edges, "edge_dot V")
    Gs = lay.check(Gs, graph.n_nodes, "edge_dot G")
    out = torch.empty((graph.n_edges, lay.n_heads), device=Vs[0].device, dtype=torch.float32)
    with torch.cuda.device(out.device), _kernel("attn_edge_dot", _attn_bytes(lay, graph.n_edges, graph.n_nodes, "edge_dot")):
        rc = _lib.load().eqf_attn_edge_dot(ctypes.byref(lay.c), _ptr_array(Vs), _ptr_array(Gs),
                                           graph.dst.data_ptr(), graph.n_edges, out.data_ptr(), _stream())
    _lib.check(rc, "eqf_attn_edge_dot")
    return out


def attn_edge_scale_raw(lay: HeadLayout, alpha, Gs, graph: Graph) -> List[torch.Tensor]:
    Gs = lay.check(Gs, graph.n_nodes, "edge_scale G")
    if alpha is not None:
        alpha = _require_cuda(alpha, "alpha")
    dev = Gs[0].device
    outs = [torch.empty((graph.n_edges, d, C), device=dev, dtype=torch.float32) for d, C in zip(lay.ds, lay.Cs)]
    with torch.cuda.device(dev), _kernel("attn_edge_scale", _attn_bytes(lay, graph.n_edges, graph.n_nodes, "edge_scale")):
        rc = _lib.load().eqf_attn_edge_scale(ctypes.byref(lay.c), alpha.data_ptr() if alpha is not None else None,
                                             _ptr_array(Gs), graph.dst.data_ptr(), graph.n_edges,
                                             _ptr_array(outs), _stream())
    _lib.check(rc, "eqf_attn_edge_scale")
    return outs


class SegSoftmax(torch.autograd.Function):
    """alpha = softmax of z over each destination segment (PyG semantics, +1e-16 in the denominator)."""

    @staticmethod
    def forward(ctx, z, graph: Graph):
        alpha = seg_softmax_raw(z, graph)
        ctx.graph = graph
        ctx.save_for_backward(alpha)
        return alpha

    @staticmethod
    def backward(ctx, ga):
        (alpha,) = ctx.saved_tensors
        g = ctx.graph
        # d alpha_e / d z_f = alpha_e (delta_ef - alpha_f) inside a segment (the 1e-16 is below fp32 resolution
        # of any non-empty segment sum, which is >= 1).  First order: one kernel; under create_graph the small [E, H]
        # tensors go through differentiable torch ops.
        if not torch.is_grad_enabled() and fused_ok(alpha):
            return seg_softmax_bwd_raw(alpha, ga, g), None
        t = alpha * ga
        s = torch.zeros((g.n_nodes, alpha.shape[1]), device=alpha.device, dtype=alpha.dtype).index_add(0, g.dst, t)
        return t - alpha * s.index_select(0, g.dst), None


class AttnAggregate(torch.autograd.Function):
    """outs[g][t] = sum_{e->t} alpha[e, head] V[g][e].  apply(lay, graph, alpha_or_None, *Vs)."""

    @staticmethod
    def forward(ctx, lay: HeadLayout, graph: Graph, alpha, *Vs):
        ctx.lay, ctx.graph = lay, graph
        ctx.has_alpha = alpha is not None
        outs = attn_aggregate_raw(lay, alpha, Vs, graph)
        if ctx.has_alpha:
            ctx.save_for_backward(alpha, *Vs)
        else:
            ctx.save_for_backward(*Vs)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *Gs):
        lay, graph = ctx.lay, ctx.graph
        saved = ctx.saved_tensors
        alpha, Vs = (saved[0], saved[1:]) if ctx.has_alpha else (None, saved)
        Gs = [G.contiguous() if G is not None else torch.zeros((graph.n_nodes, d, C), device=Vs[0].device)
              for G, d, C in zip(Gs, lay.ds, lay.Cs)]
        ga = None
        gVs = [None] * len(Vs)
        if ctx.has_alpha and ctx.needs_input_grad[2]:
            ga = EdgeDot.apply(lay, graph, *Vs, *Gs)
        if any(ctx.needs_input_grad[3:]):
            gVs = list(EdgeScale.apply(lay, graph, alpha, *Gs))
        return (None, None, ga, *gVs)


class EdgeDot(torch.autograd.Function):
    """galpha[e,h] = sum_{j in h} V[e,j] G[dst e, j].  apply(lay, graph, *Vs, *Gs)."""

    @staticmethod
    def forward(ctx, lay: HeadLayout, graph: Graph, *VG):
        n = len(lay.ds)
        ctx.lay, ctx.graph = lay, graph
        out = attn_edge_dot_raw(lay, VG[:n], VG[n:], graph)
        ctx.save_for_backward(*VG)
        return out

    @staticmethod
    def backward(ctx, ca):
        lay, graph = ctx.lay, ctx.graph
        n = len(lay.ds)
        VG = ctx.saved_tensors
        Vs, Gs = VG[:n], VG[n:]
        ca = ca.contiguous()
        gVs = [None] * n
        gGs = [None] * n
        if any(ctx.needs_input_grad[2:2 + n]):
            gVs = list(EdgeScale.apply(lay, graph, ca, *Gs))
        if any(ctx.needs_input_grad[2 + n:]):
            gGs = list(AttnAggregate.apply(lay, graph, ca, *Vs))
        return (None, None, *gVs, *gGs)


class EdgeScale(torch.autograd.Function):
    """outs[g][e] = alpha[e, head] G[g][dst e]  (alpha None: plain gather).  apply(lay, graph, alpha, *Gs)."""

    @staticmethod
    def forward(ctx, lay: HeadLayout, graph: Graph, alpha, *Gs):
        ctx.lay, ctx.graph = lay, graph
        ctx.has_alpha = alpha is not None
        outs = attn_edge_scale_raw(lay, alpha, Gs, graph)
        if ctx.has_alpha:
            ctx.save_for_backward(alpha, *Gs)
        else:
            ctx.save_for_backward(*Gs)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *cVs):
        lay, graph = ctx.lay, ctx.graph
        saved = ctx.saved_tensors
        alpha, Gs = (saved[0], saved[1:]) if ctx.has_alpha else (None, saved)
        cVs = [c.contiguous() if c is not None else torch.zeros((graph.n_edges, d, C), device=Gs[0].device)
               for c, d, C in zip(cVs, lay.ds, lay.Cs)]
        ga = None
        gGs = [None] * len(Gs)
        if ctx.has_alpha and ctx.needs_input_grad[2]:
            ga = EdgeDot.apply(lay, graph, *cVs, *Gs)
        if any(ctx.needs_input_grad[3:]):
            gGs = list(AttnAggregate.apply(lay, graph, alpha, *cVs))
        return (None, None, ga, *gGs)


def softmax_aggregate_raw(lay: HeadLayout, z: torch.Tensor, Vs, graph: Graph):
    """(outs, alpha): segment softmax of ``z`` and the alpha-weighted segment sums of ``Vs`` in one kernel."""
    Vs = lay.check(Vs, graph.n_edges, "softmax_aggregate V")
    z = _require_cuda(z, "attention logits")
    if tuple(z.shape) != (graph.n_edges, lay.n_heads):
        raise ValueError("logits must be [E, H]")
    dev = z.device
    outs = [torch.empty((graph.n_nodes, d, C), device=dev, dtype=torch.float32) for d, C in zip(lay.ds, lay.Cs)]
    alpha = torch.empty_like(z)
    nbytes = _attn_bytes(lay, graph.n_edges, graph.n_nodes, "aggregate") + 4 * z.numel()
    with torch.cuda.device(dev), _kernel("softmax_aggregate", nbytes):
        rc = _lib.load().eqf_attn_softmax_aggregate(ctypes.byref(lay.c), z.data_ptr(), _ptr_array(Vs), graph.row_ptr.data_ptr(),
                                                    graph.n_nodes, _ptr_array(outs), alpha.data_ptr(), _stream())
    _lib.check(rc, "eqf_attn_softmax_aggregate")
    return outs, alpha


def softmax_aggregate_ok(lay: HeadLayout, z: torch.Tensor) -> bool:
    # float4 lanes: every group's channels PER HEAD must be a multiple of 4 (a lane's four channels belong to one head)
    return (fused_ok(z) and lay.ds[0] == 1 and all((c // lay.n_heads) % 4 == 0 for c in lay.Cs) and z.shape[0] > 0)


class SoftmaxAggregate(torch.autograd.Function):
    """K2 (ref :508-513): ``outs[g][t] = sum_{e->t} softmax_t(z)[e, head] V[g][e]`` - softmax and aggregation in one launch.
    apply(lay, graph, z, *Vs).  Backward: EdgeDot / EdgeScale / segment-softmax backward on the saved alpha; under
    ``create_graph`` the softmax is rebuilt differentiably and the closed families take over."""

    @staticmethod
    def forward(ctx, lay: HeadLayout, graph: Graph, z, *Vs):
        outs, alpha = softmax_aggregate_raw(lay, z, Vs, graph)
        ctx.lay, ctx.graph = lay, graph
        ctx.save_for_backward(z, alpha, *Vs)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *Gs):
        lay, graph = ctx.lay, ctx.graph
        z, alpha, *Vs = ctx.saved_tensors
        Gs = [G.contiguous() if G is not None else torch.zeros((graph.n_nodes, d, C), device=z.device)
              for G, d, C in zip(Gs, lay.ds, lay.Cs)]
        need_z, need_V = ctx.needs_input_grad[2], any(ctx.needs_input_grad[3:])
        if torch.is_grad_enabled():
            fn = lambda zz, *vv: tuple(AttnAggregate.apply(lay, graph, SegSoftmax.apply(zz, graph), *vv))
            grads = _higher_order_grads(fn, (z, *Vs), Gs)
            return (None, None, *grads)
        gz = None
        gVs = [None] * len(Vs)
        if need_z:
            gz = seg_softmax_bwd_raw(alpha, attn_edge_dot_raw(lay, Vs, Gs, graph), graph)
        if need_V:
            gVs = attn_edge_scale_raw(lay, alpha, Gs, graph)
        return (None, None, gz, *gVs)


def attention_aggregate(lay: HeadLayout, graph: Graph, alpha: Optional[torch.Tensor], Vs: Sequence[torch.Tensor]):
    return list(AttnAggregate.apply(lay, graph, alpha, *Vs))


def segment_softmax(z: torch.Tensor, graph: Graph) -> torch.Tensor:
    return SegSoftmax.apply(z, graph)


# ----------------------------------------------------------------------------- fp32-accurate tensor-core GEMM

_GEMM_MODE = None


def gemm_backend() -> str:
    """Which kernel carries the fp32-accurate edge-level products:

    * ``'tf32x3'`` (default) - the hand-written wgmma 3xTF32 kernels of ``libeqf_b200.so`` (``eqf_gemm_tf32x3*``);
    * ``'torch'`` - cuBLAS SGEMM everywhere (``EQF_GEMM=torch``)."""
    global _GEMM_MODE
    if _GEMM_MODE is None:
        want = os.environ.get("EQF_GEMM", "tf32x3")
        if want not in ("tf32x3", "torch"):
            raise ValueError(f"EQF_GEMM={want!r}: expected 'tf32x3' or 'torch'")
        _GEMM_MODE = want
    return _GEMM_MODE


def gemm_backend_forced() -> bool:
    """EQF_GEMM_FORCE=1: every aligned product goes to the hand-written 3xTF32 kernels, whatever its size (tests)."""
    return os.environ.get("EQF_GEMM_FORCE", "0") == "1"


def _gemm_operand(t: torch.Tensor):
    """Row-major 2-D operand with 16-byte aligned rows: returns (tensor, leading dimension)."""
    if t.stride(1) != 1 or t.stride(0) % 4 != 0 or t.stride(0) < t.shape[1]:
        t = t.contiguous()
    if t.data_ptr() % 16 != 0:      # e.g. a view at an odd offset of a flat parameter buffer: TMA needs 16-byte rows
        t = t.clone(memory_format=torch.contiguous_format)
    return t, t.stride(0)


# reduction length from which the weight gradient runs as the sliced 3xTF32 launch (node-level products of 2 324 atoms x
# (2l+1) rows included)
_WGRAD_MIN_K = int(os.environ.get("EQF_WGRAD_MIN_K", "2048"))
# rows from which forward / data-gradient products leave the small-product kernel for the 3xTF32 kernels; EQF_GEMM_MIN_M=1 sends the small
# reference-run fixtures (tests/golden/reference_model_*.npz) through the hand-written kernels as well
_GEMM_MIN_M = int(os.environ.get("EQF_GEMM_MIN_M", "16384"))
# ... or this many flops (EQF_GEMM_MIN_FLOP; off by default): the 3xTF32 route costs a weight-split + GEMM launch pair
# per degree where the grouped small-product kernel takes all degrees - and, in the backward, data and weight gradients -
# in one launch.
_GEMM_MIN_FLOP = float(os.environ.get("EQF_GEMM_MIN_FLOP", "inf"))


def _use_tensor_cores(M: int, N: int, K: int) -> bool:
    """Forward / data-gradient product [M, K] x [K, N]: the wgmma 3xTF32 kernels (True) or the small-product kernel."""
    return M >= _GEMM_MIN_M or (M >= 1024 and 2.0 * M * N * K >= _GEMM_MIN_FLOP)


def gemm_raw(mode: int, A: torch.Tensor, B: torch.Tensor) -> torch.Tensor:
    """mode 0: A[M,K] B[K,N]; mode 1: A[M,K] B[N,K]^T; mode 2: A[K,M]^T B[K,N]  ->  C[M,N] (fp32 accurate)."""
    if mode == 0:
        (M, K), N = A.shape, B.shape[1]
        ok = B.shape[0] == K
    elif mode == 1:
        (M, K), N = A.shape, B.shape[0]
        ok = B.shape[1] == K
    else:
        (K, M), N = A.shape, B.shape[1]
        ok = B.shape[0] == K
    if not ok:
        raise ValueError(f"gemm mode {mode}: incompatible shapes {tuple(A.shape)} {tuple(B.shape)}")
    aligned = all(v % 4 == 0 for v in (A.shape[1], B.shape[1], N)) and min(M, N, K) > 0
    fast = A.is_cuda and A.dtype == torch.float32 and aligned
    backend = gemm_backend() if fast else "torch"
    forced = fast and gemm_backend_forced()
    # policy: the tensor-core kernels take the tall edge-level products (forward / data gradient from _GEMM_MIN_M rows,
    # weight gradient from _WGRAD_MIN_K reduction rows); below that the exact-fp32 small-product kernel
    if backend == "tf32x3":
        if mode != 2 and (forced or _use_tensor_cores(M, N, K)):
            return gemm_tf32x3_raw(A, B, b_is_kn=(mode == 0))
        if mode == 2 and (forced or K >= _WGRAD_MIN_K):
            return gemm_tf32x3_wgrad_raw(A, B)
    if fast and backend != "torch" and _SMALL_OWN:
        # small products (the whole MD17 regime, node-level leftovers): the exact-fp32 CUDA-core kernel, not cuBLAS
        split = mode == 2 and K >= 1024 and not _DETERMINISTIC   # long reduction, small output: split across CTAs, atomic adds
        C = (torch.zeros if split else torch.empty)((M, N), device=A.device, dtype=torch.float32)
        grouped_gemm_raw([(mode, A, B, C, 1.0, split)])
        return C
    if mode == 0:
        return A @ B
    return A @ B.t() if mode == 1 else A.t() @ B


_GEMM_SHAPE_NAMES = os.environ.get("EQF_PROFILE_GEMM_SHAPES", "0") == "1"


def _gemm_name(base: str, mode: int, M: int, N: int, K: int) -> str:
    """Kernel name for the bench's per-kernel table; with EQF_PROFILE_GEMM_SHAPES=1 one row per (mode, shape)."""
    return f"{base}[m{mode} {M}x{N}x{K}]" if _GEMM_SHAPE_NAMES else base


# EQF_DETERMINISTIC=1: weight gradients through per-slice partials + a fixed-order column sum (bitwise reproducible)
# instead of atomic adds whose summation order varies between runs
_DETERMINISTIC = os.environ.get("EQF_DETERMINISTIC", "0") == "1"
_TF32X3_SPLIT = {}


def gemm_tf32x3_raw(A: torch.Tensor, Bt: torch.Tensor, b_is_kn: bool = False) -> torch.Tensor:
    """``A[M, K] @ Bt[N, K]^T`` - or ``A @ B`` with ``B[K, N]`` when ``b_is_kn`` - through the hand-written wgmma
    3xTF32 kernels (``eqf_gemm_tf32x3``)."""
    A = _require_cuda(A, "gemm A")
    Bt = _require_cuda(Bt, "gemm B")
    M, K = A.shape
    N = Bt.shape[1] if b_is_kn else Bt.shape[0]
    if (Bt.shape[0] if b_is_kn else Bt.shape[1]) != K:
        raise ValueError(f"gemm_tf32x3: incompatible shapes {tuple(A.shape)} {tuple(Bt.shape)}")
    A, lda = _gemm_operand(A)
    if Bt.stride(1) != 1 or (not b_is_kn and Bt.stride(0) != K):
        Bt = Bt.contiguous()
    C = torch.empty((M, N), device=A.device, dtype=torch.float32)
    need = 2 * N * K
    split = _TF32X3_SPLIT.get(A.device)
    if split is None or split.numel() < need:
        split = torch.empty(max(need, 1 << 20), device=A.device, dtype=torch.float32)
        _TF32X3_SPLIT[A.device] = split
    with torch.cuda.device(A.device), _kernel(_gemm_name("gemm_tf32x3", 1, M, N, K), 4 * (A.numel() + Bt.numel() + C.numel()),
                                              2 * M * N * K):
        rc = _lib.load().eqf_gemm_tf32x3(A.data_ptr(), Bt.data_ptr(), C.data_ptr(), M, N, K, lda, Bt.stride(0), N,
                                         1 if b_is_kn else 0, split.data_ptr(), _stream())
    _lib.check(rc, "eqf_gemm_tf32x3")
    return C


def gemm_tf32x3_wgrad_raw(A: torch.Tensor, G: torch.Tensor) -> torch.Tensor:
    """``A[R, K1]^T @ G[R, N]`` (weight gradient) through the hand-written wgmma 3xTF32 kernel: per-slice partial
    products (one CTA per row slice and output tile) + one deterministic column sum over the slices."""
    A = _require_cuda(A, "wgrad A")
    G = _require_cuda(G, "wgrad G")
    (R, K1), N = A.shape, G.shape[1]
    if G.shape[0] != R:
        raise ValueError(f"gemm_tf32x3_wgrad: incompatible shapes {tuple(A.shape)} {tuple(G.shape)}")
    A, lda = _gemm_operand(A)
    G, ldg = _gemm_operand(G)
    lib = _lib.load()
    if not _DETERMINISTIC:      # slices add into W through atomic adds: one launch, no partial buffer / column sum
        W = torch.empty((K1, N), device=A.device, dtype=torch.float32)
        with torch.cuda.device(A.device), _kernel(_gemm_name("gemm_tf32x3_wgrad", 2, K1, N, R), 4 * (A.numel() + G.numel() + W.numel()),
                                                  2 * R * K1 * N):
            rc = lib.eqf_gemm_tf32x3_wgrad_accumulate(A.data_ptr(), G.data_ptr(), W.data_ptr(), R, K1, N, lda, ldg, _stream())
        _lib.check(rc, "eqf_gemm_tf32x3_wgrad_accumulate")
        return W
    slices = int(lib.eqf_gemm_tf32x3_wgrad_slices(R, K1, N))
    part = torch.empty((max(slices, 1), K1, N), device=A.device, dtype=torch.float32)
    with torch.cuda.device(A.device), _kernel("gemm_tf32x3_wgrad", 4 * (A.numel() + G.numel() + 2 * part.numel()), 2 * R * K1 * N):
        rc = lib.eqf_gemm_tf32x3_wgrad(A.data_ptr(), G.data_ptr(), part.data_ptr(), R, K1, N, lda, ldg, _stream())
    _lib.check(rc, "eqf_gemm_tf32x3_wgrad")
    if slices == 1:
        return part[0]
    return colsum_raw(part.view(slices, K1 * N)).view(K1, N)


class Gemm(torch.autograd.Function):
    """C = op(A) op(B) for the three layouts of :func:`gemm_raw`; closed under differentiation."""

    @staticmethod
    def forward(ctx, mode: int, A, B):
        ctx.mode = mode
        ctx.save_for_backward(A, B)
        return gemm_raw(mode, A, B)

    @staticmethod
    def backward(ctx, dC):
        A, B = ctx.saved_tensors
        mode = ctx.mode
        dA = dB = None
        if mode == 0:      # C = A B
            if ctx.needs_input_grad[1]:
                dA = Gemm.apply(1, dC, B)
            if ctx.needs_input_grad[2]:
                dB = Gemm.apply(2, A, dC)
        elif mode == 1:    # C = A B^T
            if ctx.needs_input_grad[1]:
                dA = Gemm.apply(0, dC, B)
            if ctx.needs_input_grad[2]:
                dB = Gemm.apply(2, dC, A)
        else:              # C = A^T B
            if ctx.needs_input_grad[1]:
                dA = Gemm.apply(1, B, dC)
            if ctx.needs_input_grad[2]:
                dB = Gemm.apply(0, A, dC)
        return None, dA, dB


def matmul_f32(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """``x[M,K] @ w[K,N]`` through the fp32-accurate tensor-core GEMM on CUDA (plain matmul elsewhere)."""
    if x.is_cuda and x.dtype == torch.float32:
        return Gemm.apply(0, x, w)
    return x @ w


def linear_f32(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``F.linear``: ``x @ weight^T + bias`` with ``weight`` stored ``[out, in]`` like ``nn.Linear``."""
    if x.is_cuda and x.dtype == torch.float32 and x.dim() == 2:
        out = Gemm.apply(1, x, weight)
        return out if bias is None else add_bias(out, bias)
    return torch.nn.functional.linear(x, weight, bias)


# ----------------------------------------------------------------------------- grouped small products
# All degrees of a node-level linear in one launch of the exact-fp32 CUDA-core kernel (csrc/eqf_gemm_small.cu): forward,
# data gradients and weight gradients (the two gradient sets share a launch in a first-order backward).  Round 1 sent each
# of these 30-80 MFLOP products to cuBLAS separately (~180 SIMT SGEMM launches per QM9 step).
_GROUPED = os.environ.get("EQF_GROUPED_GEMM", "1") != "0"
# EQF_SMALL_GEMM=cublas hands single small products (below the tensor-core thresholds) back to torch / cuBLAS (A/B switch)
_SMALL_OWN = os.environ.get("EQF_SMALL_GEMM", "own") != "cublas"


class LinearSpec:
    """Paths of a scalar-in2 'uvw' product on planar blocks: ``(i_in, i_out, w_off, mul_in, mul_out, c)`` per path,
    ``W_p = w[w_off : w_off + mul_in * mul_out].view(mul_in, mul_out)``, ``out[i_out] = c * x[i_in] @ W_p``."""

    def __init__(self, paths, w_numel: int):
        self.paths = tuple(paths)
        self.w_numel = int(w_numel)

    def aligned(self) -> bool:
        outs = [p[1] for p in self.paths]
        return (0 < len(self.paths) <= _lib.EQF_GROUP_MAX and len(set(outs)) == len(outs)
                and all(p[3] % 4 == 0 and p[4] % 4 == 0 and p[2] % 4 == 0 for p in self.paths))


def grouped_gemm_raw(problems) -> None:
    """``problems``: ``(mode, A, B, C, alpha, accumulate)`` with 2-D fp32 CUDA tensors (C written / added in place)."""
    lib = _lib.load()
    table = (_lib.EqfGemmProblem * len(problems))()
    nbytes = flops = 0
    keep = []
    for q, (mode, A, B, C, alpha, acc) in zip(table, problems):
        A, lda = _gemm_operand(A)
        B, ldb = _gemm_operand(B)
        keep += [A, B]
        if mode == 0:
            (M, K), N = A.shape, B.shape[1]
        elif mode == 1:
            (M, K), N = A.shape, B.shape[0]
        else:
            (K, M), N = A.shape, B.shape[1]
        if tuple(C.shape) != (M, N) or C.stride(1) != 1:
            raise ValueError(f"grouped gemm: output {tuple(C.shape)} does not match {(M, N)}")
        q.A, q.B, q.C = A.data_ptr(), B.data_ptr(), C.data_ptr()
        q.M, q.N, q.K, q.lda, q.ldb, q.ldc = M, N, K, lda, ldb, C.stride(0)
        q.mode, q.accumulate, q.alpha = mode, 1 if acc else 0, float(alpha)
        nbytes += 4 * (A.numel() + B.numel() + C.numel())
        flops += 2 * M * N * K
    dev = problems[0][1].device
    with torch.cuda.device(dev), _kernel("gemm_grouped", nbytes, flops):
        rc = lib.eqf_gemm_grouped(table, len(problems), _stream())
    _lib.check(rc, "eqf_gemm_grouped")


def _lin_w(spec: LinearSpec, w: torch.Tensor, p):
    return w.narrow(0, p[2], p[3] * p[4]).view(p[3], p[4])


def _lin_rows(t: torch.Tensor) -> torch.Tensor:
    return t.reshape(t.shape[0] * t.shape[1], t.shape[2])


def _lin_fwd_problems(spec, w, xs, outs):
    return [(0, _lin_rows(x), _lin_w(spec, w, p), _lin_rows(o), p[5], False) for p, x, o in zip(spec.paths, xs, outs)]


def _lin_dgrad_problems(spec, w, gs, dxs):
    return [(1, _lin_rows(g), _lin_w(spec, w, p), _lin_rows(dx), p[5], False) for p, g, dx in zip(spec.paths, gs, dxs)]


def _lin_wgrad_problems(spec, xs, gs, gw):
    return [(2, _lin_rows(x), _lin_rows(g), _lin_w(spec, gw, p), p[5], True) for p, x, g in zip(spec.paths, xs, gs)]


def _launch_grouped(problems):
    for i in range(0, len(problems), _lib.EQF_GROUP_MAX):
        grouped_gemm_raw(problems[i:i + _lib.EQF_GROUP_MAX])


class PlanarLinearFwd(torch.autograd.Function):
    """``outs[p] = c_p * xs[p] @ W_p`` for every path of the spec (``xs`` in path order); one launch."""

    @staticmethod
    def forward(ctx, spec: LinearSpec, w, *xs):
        ctx.spec = spec
        ctx.save_for_backward(w, *xs)
        w = w.detach()
        outs = [x.new_empty((x.shape[0], x.shape[1], p[4])) for p, x in zip(spec.paths, xs)]
        _launch_grouped(_lin_fwd_problems(spec, w, [x.detach() for x in xs], outs))
        return tuple(outs)

    @staticmethod
    def backward(ctx, *gs):
        spec = ctx.spec
        w, *xs = ctx.saved_tensors
        gs = [g if g is not None else torch.zeros((x.shape[0], x.shape[1], p[4]), device=x.device, dtype=x.dtype)
              for g, p, x in zip(gs, spec.paths, xs)]
        need_w = ctx.needs_input_grad[1]
        need_x = any(ctx.needs_input_grad[2:])
        if torch.is_grad_enabled():          # create_graph: stay inside the closed family
            gw = PlanarLinearWgrad.apply(spec, *xs, *gs) if need_w else None
            dxs = PlanarLinearDgrad.apply(spec, w, *gs) if need_x else [None] * len(xs)
            return (None, gw, *dxs)
        gs = [g.contiguous() for g in gs]
        problems, gw, dxs = [], None, [None] * len(xs)
        if need_x:
            dxs = [torch.empty_like(x) for x in xs]
            problems += _lin_dgrad_problems(spec, w, gs, dxs)
        if need_w:
            gw = torch.zeros_like(w)
            problems += _lin_wgrad_problems(spec, xs, gs, gw)
        if problems:
            _launch_grouped(problems)
        return (None, gw, *dxs)


class PlanarLinearDgrad(torch.autograd.Function):
    """``dxs[p] = c_p * gs[p] @ W_p^T``."""

    @staticmethod
    def forward(ctx, spec: LinearSpec, w, *gs):
        ctx.spec = spec
        ctx.save_for_backward(w, *gs)
        gs = [g.detach().contiguous() for g in gs]
        dxs = [g.new_empty((g.shape[0], g.shape[1], p[3])) for p, g in zip(spec.paths, gs)]
        _launch_grouped(_lin_dgrad_problems(spec, w.detach(), gs, dxs))
        return tuple(dxs)

    @staticmethod
    def backward(ctx, *ddx):
        spec = ctx.spec
        w, *gs = ctx.saved_tensors
        ddx = [d if d is not None else torch.zeros((g.shape[0], g.shape[1], p[3]), device=g.device, dtype=g.dtype)
               for d, p, g in zip(ddx, spec.paths, gs)]
        gw = PlanarLinearWgrad.apply(spec, *ddx, *gs) if ctx.needs_input_grad[1] else None
        ggs = PlanarLinearFwd.apply(spec, w, *ddx) if any(ctx.needs_input_grad[2:]) else [None] * len(gs)
        return (None, gw, *ggs)


class PlanarLinearWgrad(torch.autograd.Function):
    """flat ``gw`` with ``gw_p = c_p * xs[p]^T @ gs[p]`` (reduction over rows split across CTAs, fp32 atomic adds)."""

    @staticmethod
    def forward(ctx, spec: LinearSpec, *ts):
        n = len(spec.paths)
        xs, gs = ts[:n], ts[n:]
        ctx.spec = spec
        ctx.save_for_backward(*ts)
        gw = torch.zeros(spec.w_numel, device=xs[0].device, dtype=xs[0].dtype)
        _launch_grouped(_lin_wgrad_problems(spec, [x.detach().contiguous() for x in xs], [g.detach().contiguous() for g in gs], gw))
        return gw

    @staticmethod
    def backward(ctx, ggw):
        spec = ctx.spec
        n = len(spec.paths)
        ts = ctx.saved_tensors
        xs, gs = ts[:n], ts[n:]
        ggw = ggw.contiguous()
        dxs = PlanarLinearDgrad.apply(spec, ggw, *gs) if any(ctx.needs_input_grad[1:1 + n]) else [None] * n
        dgs = PlanarLinearFwd.apply(spec, ggw, *xs) if any(ctx.needs_input_grad[1 + n:]) else [None] * n
        return (None, *dxs, *dgs)


def planar_linear_grouped_ok(spec: LinearSpec, w: torch.Tensor, xs) -> bool:
    """All paths in one launch of the small-product kernel: CUDA fp32, aligned channels, every product below the row count
    from which the tensor-core kernels take over.  ``EQF_DETERMINISTIC=1`` keeps the per-degree route (the grouped weight
    gradients meet in ``gw`` through fp32 atomics, whose order is not fixed)."""
    if not (_GROUPED and not _DETERMINISTIC and w.is_cuda and w.dtype == torch.float32 and w.dim() == 1 and w.is_contiguous()
            and w.data_ptr() % 16 == 0 and spec.aligned() and gemm_backend() != "torch"):
        return False
    return all(x.is_cuda and x.dtype == torch.float32 and x.dim() == 3 and x.shape[2] == p[3]
               and not _use_tensor_cores(x.shape[0] * x.shape[1], max(p[3], p[4]), min(p[3], p[4])) for p, x in zip(spec.paths, xs))


def planar_linear_grouped(spec: LinearSpec, w: torch.Tensor, xs):
    """``[c_p * xs[p] @ W_p]`` in path order (autograd: the closed family above)."""
    return list(PlanarLinearFwd.apply(spec, w, *[x.contiguous() for x in xs]))


# ----------------------------------------------------------------------------- column sums / bias adds
_COLSUM_COUNTERS = {}


def colsum_raw(x: torch.Tensor) -> torch.Tensor:
    """``x.sum(0)`` of a 2-D fp32 CUDA tensor (unit column stride) through ``eqf_colsum`` (deterministic)."""
    x = _require_cuda(x, "colsum x")
    if x.dim() != 2:
        raise ValueError("colsum expects a 2-D tensor")
    if x.stride(1) != 1 and x.shape[1] > 1:
        x = x.contiguous()
    rows, cols = x.shape
    ld = x.stride(0) if rows > 1 else max(cols, 1)
    lib = _lib.load()
    if ld < cols or -(-cols // 32) > _lib.EQF_COLSUM_COUNTERS:
        return x.sum(0)
    out = torch.empty(cols, device=x.device, dtype=torch.float32)
    if cols == 0:
        return out
    counters = _COLSUM_COUNTERS.get(x.device)
    if counters is None:
        counters = torch.zeros(_lib.EQF_COLSUM_COUNTERS, device=x.device, dtype=torch.int32)
        _COLSUM_COUNTERS[x.device] = counters
    part = torch.empty(max(int(lib.eqf_colsum_scratch_floats(rows, cols)), 1), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device), _kernel("colsum", 4 * x.numel()):
        rc = lib.eqf_colsum(x.data_ptr(), rows, cols, ld, out.data_ptr(), part.data_ptr(), counters.data_ptr(), _stream())
    _lib.check(rc, "eqf_colsum")
    return out


def _colsum(x: torch.Tensor) -> torch.Tensor:
    """Column sum of kernel partials: the CUDA kernel on fp32 device tensors, ``sum(0)`` for the CPU test stand-ins."""
    return colsum_raw(x) if fused_ok(x) else x.sum(0)


class ColSum(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.rows = x.shape[0]
        return colsum_raw(x)

    @staticmethod
    def backward(ctx, g):
        return g.unsqueeze(0).expand(ctx.rows, -1)


class AddBias(torch.autograd.Function):
    """``x + b`` with ``b`` broadcast along the last dimension; the bias gradient is one ``eqf_colsum`` launch instead
    of autograd's generic broadcast reduction (ref: bias adds of tensor_product_rescale.py:120-134, radial offset)."""

    @staticmethod
    def forward(ctx, x, b):
        return x + b

    @staticmethod
    def backward(ctx, g):
        gb = None
        if ctx.needs_input_grad[1]:
            g2 = g.reshape(-1, g.shape[-1])
            gb = ColSum.apply(g2 if g2.stride(-1) == 1 else g2.contiguous())
        return g, gb


def add_bias(x: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    if fused_ok(x) and b.dim() == 1 and b.shape[0] == x.shape[-1] and x.numel() > 0:
        return AddBias.apply(x, b)
    return x + b


# ----------------------------------------------------------------------------- fused pointwise ops


def _higher_order_grads(fn, inputs, grad_outputs):
    """Backward of a fused op under ``create_graph``: rebuild the op from differentiable torch ops on the saved inputs
    and differentiate that (slow path, used only for second-order training such as MD17 force losses)."""
    with torch.enable_grad():
        # differentiate with respect to fresh views: one input may be an ancestor of another in the outer graph (the
        # edge harmonics feed the node tables), and the partial derivative asked for here must not follow that route
        inputs = [t.view_as(t) if (isinstance(t, torch.Tensor) and t.requires_grad) else t for t in inputs]
        outs = fn(*inputs)
        outs = outs if isinstance(outs, (tuple, list)) else (outs,)
        pairs = [(o, g) for o, g in zip(outs, grad_outputs) if g is not None and o.requires_grad]
        need = [t for t in inputs if isinstance(t, torch.Tensor) and t.requires_grad]
        grads = torch.autograd.grad([o for o, _ in pairs], need, [g for _, g in pairs], create_graph=True,
                                    allow_unused=True)
    it = iter(grads)
    return [next(it) if (isinstance(t, torch.Tensor) and t.requires_grad) else None for t in inputs]


def ln_silu_torch(x, gamma, beta, eps, bias=None):
    if bias is not None:
        x = x + bias
    return torch.nn.functional.silu(torch.nn.functional.layer_norm(x, x.shape[-1:], gamma, beta, eps))


def ln_silu_fwd_raw(x, gamma, beta, eps, bias=None):
    x = _require_cuda(x, "ln_silu x")
    R, C = x.shape
    y = torch.empty_like(x)
    mean = torch.empty(R, device=x.device, dtype=torch.float32)
    rstd = torch.empty(R, device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device), _kernel("ln_silu_fwd", 8 * x.numel()):
        rc = _lib.load().eqf_ln_silu_fwd(x.data_ptr(), bias.data_ptr() if bias is not None else None, gamma.data_ptr(),
                                         beta.data_ptr(), eps, R, C, y.data_ptr(), mean.data_ptr(), rstd.data_ptr(), _stream())
    _lib.check(rc, "eqf_ln_silu_fwd")
    return y, mean, rstd


def ln_silu_bwd_raw(x, gamma, beta, mean, rstd, gy, bias=None):
    """Returns (gx, dgamma, dbeta, dbias); dbias (= column sums of gx) is None when there is no bias."""
    gy = _require_cuda(gy, "ln_silu gy")
    R, C = x.shape
    rows = _lib.load().eqf_pointwise_rows(R)
    gx = torch.empty_like(x)
    part = torch.empty((rows, 3 * C), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device), _kernel("ln_silu_bwd", 12 * x.numel()):
        rc = _lib.load().eqf_ln_silu_bwd(x.data_ptr(), bias.data_ptr() if bias is not None else None, gamma.data_ptr(),
                                         beta.data_ptr(), mean.data_ptr(), rstd.data_ptr(), gy.data_ptr(), R, C,
                                         gx.data_ptr(), part.data_ptr(), _stream())
    _lib.check(rc, "eqf_ln_silu_bwd")
    sums = colsum_raw(part)                      # one reduction for the three parameter gradients
    return gx, sums[:C], sums[C:2 * C], (sums[2 * C:] if bias is not None else None)


class LnSilu(torch.autograd.Function):
    """``silu(layer_norm(x + bias))`` on ``[rows, C]`` (Linear bias + LayerNorm + SiLU of RadialProfile's hidden layers,
    ref radial_func.py:24-35); ``bias`` may be None."""

    @staticmethod
    def forward(ctx, x, bias, gamma, beta, eps: float):
        y, mean, rstd = ln_silu_fwd_raw(x, gamma, beta, eps, bias)
        ctx.eps, ctx.has_bias = eps, bias is not None
        ctx.save_for_backward(x, gamma, beta, mean, rstd, *([bias] if bias is not None else []))
        return y

    @staticmethod
    def backward(ctx, gy):
        x, gamma, beta, mean, rstd, *rest = ctx.saved_tensors
        bias = rest[0] if ctx.has_bias else None
        if torch.is_grad_enabled():
            if bias is None:
                gx, gg, gb = _higher_order_grads(lambda a, b, c: ln_silu_torch(a, b, c, ctx.eps), (x, gamma, beta), (gy,))
                return gx, None, gg, gb, None
            gx, gbias, gg, gb = _higher_order_grads(lambda a, p, b, c: ln_silu_torch(a, b, c, ctx.eps, p),
                                                    (x, bias, gamma, beta), (gy,))
            return gx, gbias, gg, gb, None
        gx, gg, gb, gbias = ln_silu_bwd_raw(x, gamma, beta, mean, rstd, gy.contiguous(), bias)
        return gx, gbias, gg, gb, None


FUSED_ON_ANY_DEVICE = False   # tests/_emulation.py flips this so the fused Functions are exercised on CPU stand-ins


def fused_ok(t: torch.Tensor) -> bool:
    return FUSED_ON_ANY_DEVICE or (t.is_cuda and t.dtype == torch.float32)


def ln_silu(x, gamma, beta, eps: float = 1e-5, bias=None):
    """``silu(LayerNorm(x + bias))``: the bias of the preceding Linear rides along (no separate add / bias-gradient pass)."""
    if fused_ok(x) and x.dim() == 2 and x.shape[1] <= 256:
        return LnSilu.apply(x.contiguous(), bias, gamma, beta, eps)
    return ln_silu_torch(x, gamma, beta, eps, bias)


class NormLayout:
    """Static description of an ``EquivariantLayerNormV2`` ('component', affine) for ``eqf_eln_fwd/bwd``."""

    def __init__(self, entries: Sequence[tuple], eps: float):
        # entries: (mul, dim, is_scalar) per irreps entry, in e3nn order
        if len(entries) > _lib.EQF_MAX_BLOCKS:
            raise NotImplementedError("norm layout exceeds kernel limits")
        self.entries, self.eps = tuple(entries), float(eps)
        self.dim = sum(m * d for m, d, _ in entries)
        self.n_w = sum(m for m, _, _ in entries)
        self.n_b = sum(m for m, _, sc in entries if sc)
        c = _lib.EqfNormLayout()
        c.n_entries, c.eps = len(entries), float(eps)
        for i, (m, d, sc) in enumerate(entries):
            c.mul[i], c.d[i], c.is_scalar[i] = m, d, int(bool(sc))
        self.c = c


def eln_torch(lay: NormLayout, x, w, b):
    """Differentiable torch statement of the fused equivariant LayerNorm (ref nets/layer_norm.py:104-152)."""
    out, off, iw, ib = [], 0, 0, 0
    for mul, d, scalar in lay.entries:
        f = x.narrow(1, off, mul * d).reshape(-1, mul, d)
        off += mul * d
        if scalar:
            f = f - f.mean(dim=1, keepdim=True)
        scale = (f.pow(2).mean(-1).mean(dim=1, keepdim=True) + lay.eps).pow(-0.5) * w[None, iw:iw + mul]
        iw += mul
        f = f * scale.unsqueeze(-1)
        if scalar:
            f = f + b[ib:ib + mul].reshape(mul, 1)
            ib += mul
        out.append(f.reshape(-1, mul * d))
    return torch.cat(out, dim=-1)


def eln_fwd_raw(lay: NormLayout, x, w, b):
    x = _require_cuda(x, "eln x")
    N = x.shape[0]
    y = torch.empty_like(x)
    rstd = torch.empty((N, len(lay.entries)), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device), _kernel("eln_fwd", 8 * x.numel()):
        rc = _lib.load().eqf_eln_fwd(ctypes.byref(lay.c), x.data_ptr(), w.data_ptr(), b.data_ptr(), N, y.data_ptr(),
                                     rstd.data_ptr(), _stream())
    _lib.check(rc, "eqf_eln_fwd")
    return y, rstd


def eln_bwd_raw(lay: NormLayout, x, w, rstd, gy):
    gy = _require_cuda(gy, "eln gy")
    N = x.shape[0]
    rows = _lib.load().eqf_eln_rows(ctypes.byref(lay.c), N)
    gx = torch.empty_like(x)
    part = torch.empty((rows, lay.n_w + lay.n_b), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device), _kernel("eln_bwd", 12 * x.numel()):
        rc = _lib.load().eqf_eln_bwd(ctypes.byref(lay.c), x.data_ptr(), w.data_ptr(), rstd.data_ptr(), gy.data_ptr(), N,
                                     gx.data_ptr(), part.data_ptr(), _stream())
    _lib.check(rc, "eqf_eln_bwd")
    sums = colsum_raw(part)
    return gx, sums[:lay.n_w], sums[lay.n_w:]


class EquivLayerNorm(torch.autograd.Function):
    """Fused ``EquivariantLayerNormV2`` forward/backward on e3nn-layout node rows."""

    @staticmethod
    def forward(ctx, lay: NormLayout, x, w, b):
        y, rstd = eln_fwd_raw(lay, x, w, b)
        ctx.lay = lay
        ctx.save_for_backward(x, w, b, rstd)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, w, b, rstd = ctx.saved_tensors
        if torch.is_grad_enabled():
            gx, gw, gb = _higher_order_grads(lambda a, c, e: eln_torch(ctx.lay, a, c, e), (x, w, b), (gy,))
            return None, gx, gw, gb
        gx, gw, gb = eln_bwd_raw(ctx.lay, x, w, rstd, gy.contiguous())
        return None, gx, gw, gb


def equivariant_layer_norm(lay: NormLayout, x, w, b):
    if fused_ok(x) and x.dim() == 2 and x.shape[0] > 0:
        return EquivLayerNorm.apply(lay, x.contiguous(), w, b)
    return eln_torch(lay, x, w, b)


def _planar_dims(lay: NormLayout):
    return tuple((m, d) for m, d, _ in lay.entries)


def eln_planar_torch(lay: NormLayout, xs, w, b):
    """Torch statement of the planar LayerNorm: through the e3nn-layout one (higher-order path, CPU stand-in)."""
    dims = _planar_dims(lay)
    return list(_to_planar_impl(eln_torch(lay, _from_planar_impl(xs), w, b), dims))


def eln_planar_fwd_raw(lay: NormLayout, xs, w, b):
    xs = [_require_cuda(x, "eln block").contiguous() for x in xs]
    N = xs[0].shape[0]
    ys = [torch.empty_like(x) for x in xs]
    rstd = torch.empty((N, len(lay.entries)), device=xs[0].device, dtype=torch.float32)
    with torch.cuda.device(xs[0].device), _kernel("eln_fwd", 8 * sum(x.numel() for x in xs)):
        rc = _lib.load().eqf_eln_fwd_planar(ctypes.byref(lay.c), _ptr_array(xs), w.data_ptr(), b.data_ptr(), N,
                                            _ptr_array(ys), rstd.data_ptr(), _stream())
    _lib.check(rc, "eqf_eln_fwd_planar")
    return ys, rstd


def eln_planar_bwd_raw(lay: NormLayout, xs, w, rstd, gys):
    gys = [_require_cuda(g, "eln gy block").contiguous() for g in gys]
    N = xs[0].shape[0]
    rows = _lib.load().eqf_eln_rows(ctypes.byref(lay.c), N)
    gxs = [torch.empty_like(x) for x in xs]
    part = torch.empty((rows, lay.n_w + lay.n_b), device=xs[0].device, dtype=torch.float32)
    with torch.cuda.device(xs[0].device), _kernel("eln_bwd", 12 * sum(x.numel() for x in xs)):
        rc = _lib.load().eqf_eln_bwd_planar(ctypes.byref(lay.c), _ptr_array(xs), w.data_ptr(), rstd.data_ptr(),
                                            _ptr_array(gys), N, _ptr_array(gxs), part.data_ptr(), _stream())
    _lib.check(rc, "eqf_eln_bwd_planar")
    sums = colsum_raw(part)
    return gxs, sums[:lay.n_w], sums[lay.n_w:]


class EquivLayerNormPlanar(torch.autograd.Function):
    """``EquivariantLayerNormV2`` on planar blocks (one packed ``[N, 2l+1, mul]`` tensor per entry) - the transformer
    blocks keep the node features in the layout the GEMM and tensor-product kernels read.  apply(lay, w, b, *xs)."""

    @staticmethod
    def forward(ctx, lay: NormLayout, w, b, *xs):
        xs = [x.contiguous() for x in xs]
        ys, rstd = eln_planar_fwd_raw(lay, xs, w, b)
        ctx.lay = lay
        ctx.save_for_backward(w, b, rstd, *xs)
        return tuple(ys)

    @staticmethod
    def backward(ctx, *gys):
        w, b, rstd, *xs = ctx.saved_tensors
        gys = [g if g is not None else torch.zeros_like(x) for g, x in zip(gys, xs)]
        if torch.is_grad_enabled():
            fn = lambda ww, bb, *blocks: tuple(eln_planar_torch(ctx.lay, list(blocks), ww, bb))
            grads = _higher_order_grads(fn, (w, b, *xs), gys)
            return (None, *grads)
        gxs, gw, gb = eln_planar_bwd_raw(ctx.lay, xs, w, rstd, gys)
        return (None, gw, gb, *gxs)


def equivariant_layer_norm_planar(lay: NormLayout, xs, w, b):
    if fused_ok(xs[0]) and xs[0].shape[0] > 0:
        return list(EquivLayerNormPlanar.apply(lay, w, b, *xs))
    return eln_planar_torch(lay, list(xs), w, b)


def gaussian_rbf_torch(dist, mean, std, weight, bias, cutoff: float):
    """Torch statement of GaussianRadialBasisLayer.forward (ref nets/gaussian_rbf.py:5-40, truncated pi included)."""
    x = weight * (dist / cutoff).unsqueeze(-1) + bias
    s = std.abs() + 1e-5
    z = (x - mean) / s
    return torch.exp(-0.5 * z * z) / (((2 * 3.14159) ** 0.5) * s)


def rbf_fwd_raw(dist, mean, std, weight, bias, cutoff: float):
    dist = _require_cuda(dist, "rbf dist").contiguous()
    E = dist.shape[0]
    out = torch.empty((E, 128), device=dist.device, dtype=torch.float32)
    with torch.cuda.device(dist.device), _kernel("rbf_fwd", 4 * (E + out.numel())):
        rc = _lib.load().eqf_rbf_fwd(dist.data_ptr(), mean.data_ptr(), std.data_ptr(), weight.data_ptr(), bias.data_ptr(),
                                     float(cutoff), E, out.data_ptr(), _stream())
    _lib.check(rc, "eqf_rbf_fwd")
    return out


def rbf_bwd_raw(dist, mean, std, weight, bias, cutoff: float, g):
    g = _require_cuda(g, "rbf g").contiguous()
    E = dist.shape[0]
    rows = _lib.load().eqf_pointwise_rows(E)
    g_dist = torch.empty(E, device=dist.device, dtype=torch.float32)
    part = torch.empty((rows, 258), device=dist.device, dtype=torch.float32)
    with torch.cuda.device(dist.device), _kernel("rbf_bwd", 4 * (2 * E + g.numel())):
        rc = _lib.load().eqf_rbf_bwd(dist.data_ptr(), mean.data_ptr(), std.data_ptr(), weight.data_ptr(), bias.data_ptr(),
                                     float(cutoff), g.data_ptr(), E, g_dist.data_ptr(), part.data_ptr(), _stream())
    _lib.check(rc, "eqf_rbf_bwd")
    sums = colsum_raw(part)
    return g_dist, sums[:128], sums[128:256], sums[256:257], sums[257:258]


class GaussianRbf(torch.autograd.Function):
    """Fused Gaussian radial basis (forward one kernel, backward one kernel + one column sum)."""

    @staticmethod
    def forward(ctx, dist, mean, std, weight, bias, cutoff: float):
        ctx.cutoff = cutoff
        ctx.save_for_backward(dist, mean, std, weight, bias)
        return rbf_fwd_raw(dist, mean, std, weight, bias, cutoff)

    @staticmethod
    def backward(ctx, g):
        dist, mean, std, weight, bias = ctx.saved_tensors
        if torch.is_grad_enabled():
            fn = lambda d, m, s, w, b: gaussian_rbf_torch(d, m, s, w, b, ctx.cutoff)
            grads = _higher_order_grads(fn, (dist, mean, std, weight, bias), (g,))
            return (*grads, None)
        gd, gm, gs, gw, gb = rbf_bwd_raw(dist, mean, std, weight, bias, ctx.cutoff, g)
        return gd, gm.view_as(mean), gs.view_as(std), gw.view_as(weight), gb.view_as(bias), None


def gaussian_rbf(dist, mean, std, weight, bias, cutoff: float):
    if fused_ok(dist) and dist.dim() == 1 and mean.numel() == 128 and dist.shape[0] > 0:
        return GaussianRbf.apply(dist.contiguous(), mean, std, weight, bias, float(cutoff))
    return gaussian_rbf_torch(dist, mean, std, weight, bias, cutoff)


# ----------------------------------------------------------------------------- edge geometry / exp-normal basis


def edge_geometry_torch(pos, src, dst, lmax: int, offsets=None):
    """Torch statement of the fused edge-geometry kernel (ref :866-870): (edge_vec, length, harmonics 0..lmax)."""
    from .o3.sh import spherical_harmonics
    vec = pos.index_select(0, src) - pos.index_select(0, dst)
    if offsets is not None:
        vec = vec + offsets
    return vec, vec.norm(dim=1), spherical_harmonics(list(range(lmax + 1)), vec, True, "component")


def _sh_couplings(device):
    from .o3.sh import _coupling_tensor
    return _coupling_tensor(1, torch.float32, device).contiguous(), _coupling_tensor(2, torch.float32, device).contiguous()


class EdgeGeometry(torch.autograd.Function):
    """(edge_vec, length, sh) of ``pos[src] - pos[dst] (+ offsets)`` in one kernel; backward = one kernel + two segment sums
    to the positions (destination-sorted CSR and its CSC).  apply(pos, graph, lmax, offsets_or_None)."""

    @staticmethod
    def forward(ctx, pos, graph: "Graph", lmax: int, offsets):
        pos = _require_cuda(pos, "pos")
        E = graph.n_edges
        a1, a2 = _sh_couplings(pos.device)
        vec = torch.empty((E, 3), device=pos.device, dtype=torch.float32)
        length = torch.empty(E, device=pos.device, dtype=torch.float32)
        sh = torch.empty((E, (lmax + 1) ** 2), device=pos.device, dtype=torch.float32)
        with torch.cuda.device(pos.device), _kernel("edge_geom_fwd", 4 * E * (6 + 4 + (lmax + 1) ** 2)):
            rc = _lib.load().eqf_edge_geom_fwd(pos.data_ptr(), graph.src.data_ptr(), graph.dst.data_ptr(),
                                               offsets.data_ptr() if offsets is not None else None, a1.data_ptr(), a2.data_ptr(),
                                               E, lmax, vec.data_ptr(), length.data_ptr(), sh.data_ptr(), _stream())
        _lib.check(rc, "eqf_edge_geom_fwd")
        ctx.graph, ctx.lmax, ctx.has_off = graph, lmax, offsets is not None
        ctx.save_for_backward(pos, vec, *([offsets] if offsets is not None else []))
        return vec, length, sh

    @staticmethod
    def backward(ctx, g_vec_out, g_len, g_sh):
        graph, lmax = ctx.graph, ctx.lmax
        pos, vec, *rest = ctx.saved_tensors
        offsets = rest[0] if ctx.has_off else None
        if torch.is_grad_enabled():        # second order (MD17 force training): differentiate the torch statement
            fn = lambda p, o: edge_geometry_torch(p, graph.src, graph.dst, lmax, o)
            gp, go = _higher_order_grads(fn, (pos, offsets), (g_vec_out, g_len, g_sh))
            return gp, None, None, go
        E = graph.n_edges
        a1, a2 = _sh_couplings(pos.device)
        gv = torch.empty((E, 3), device=pos.device, dtype=torch.float32)
        gs = g_sh.contiguous() if g_sh is not None else None
        gl = g_len.contiguous() if g_len is not None else None
        with torch.cuda.device(pos.device), _kernel("edge_geom_bwd", 4 * E * (6 + (lmax + 1) ** 2)):
            rc = _lib.load().eqf_edge_geom_bwd(vec.data_ptr(), a1.data_ptr(), a2.data_ptr(), E, lmax,
                                               gs.data_ptr() if gs is not None else None,
                                               gl.data_ptr() if gl is not None else None, gv.data_ptr(), _stream())
        _lib.check(rc, "eqf_edge_geom_bwd")
        if g_vec_out is not None:
            gv = gv + g_vec_out
        lay = HeadLayout([1], [3], 1)
        gsrc = attn_aggregate_raw(lay, None, [gv.view(E, 1, 3)], graph, by_src=True)[0].view(-1, 3)
        gdst = attn_aggregate_raw(lay, None, [gv.view(E, 1, 3)], graph)[0].view(-1, 3)
        return gsrc - gdst, None, None, (gv if offsets is not None and ctx.needs_input_grad[3] else None)


def edge_geometry(pos, graph: "Graph", lmax: int, offsets=None):
    """(edge_vec [E, 3], length [E], sh [E, (lmax + 1)^2]) - fused kernel on CUDA fp32, torch statement otherwise."""
    if pos.is_cuda and pos.dtype == torch.float32 and lmax <= 3 and graph.n_edges > 0:
        return EdgeGeometry.apply(pos, graph, lmax, offsets)
    return edge_geometry_torch(pos, graph.src, graph.dst, lmax, offsets)


def expnorm_torch(dist, means, betas, alpha: float, cutoff_upper: float):
    """Torch statement of ExpNormalSmearing.forward with CosineCutoff(0, cutoff_upper) (ref nets/expnorm_rbf.py:11-33, 73-78)."""
    d = dist.unsqueeze(-1)
    cut = 0.5 * (torch.cos(d * (3.141592653589793 / cutoff_upper)) + 1.0) * (d < cutoff_upper).to(d.dtype)
    return cut * torch.exp(-betas * (torch.exp(-alpha * d) - means) ** 2)


class ExpNormalRbf(torch.autograd.Function):
    """Exp-normal radial basis on ``[E]`` distances -> ``[E, B]`` (fixed means / betas); one kernel each way."""

    @staticmethod
    def forward(ctx, dist, means, betas, alpha: float, hi: float):
        dist = _require_cuda(dist, "expnorm dist")
        E, B = dist.shape[0], means.numel()
        out = torch.empty((E, B), device=dist.device, dtype=torch.float32)
        with torch.cuda.device(dist.device), _kernel("expnorm_fwd", 4 * (E + E * B)):
            rc = _lib.load().eqf_expnorm_fwd(dist.data_ptr(), means.data_ptr(), betas.data_ptr(), alpha, hi, E, B,
                                             out.data_ptr(), _stream())
        _lib.check(rc, "eqf_expnorm_fwd")
        ctx.alpha, ctx.hi = alpha, hi
        ctx.save_for_backward(dist, means, betas)
        return out

    @staticmethod
    def backward(ctx, g):
        dist, means, betas = ctx.saved_tensors
        if torch.is_grad_enabled() or ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            fn = lambda d, m, b: expnorm_torch(d, m, b, ctx.alpha, ctx.hi)
            gd, gm, gb = _higher_order_grads(fn, (dist, means, betas), (g,))
            return gd, gm, gb, None, None
        E, B = g.shape
        gd = torch.empty(E, device=g.device, dtype=torch.float32)
        g = g.contiguous()
        with torch.cuda.device(g.device), _kernel("expnorm_bwd", 4 * (2 * E + E * B)):
            rc = _lib.load().eqf_expnorm_bwd(dist.data_ptr(), means.data_ptr(), betas.data_ptr(), ctx.alpha, ctx.hi, E, B,
                                             g.data_ptr(), gd.data_ptr(), _stream())
        _lib.check(rc, "eqf_expnorm_bwd")
        return gd, None, None, None, None


def expnorm_rbf(dist, means, betas, alpha: float, cutoff_upper: float):
    if dist.is_cuda and dist.dtype == torch.float32 and dist.dim() == 1 and dist.shape[0] > 0:
        return ExpNormalRbf.apply(dist.contiguous(), means.contiguous(), betas.contiguous(), float(alpha), float(cutoff_upper))
    return expnorm_torch(dist, means, betas, alpha, cutoff_upper)


class GateLayout:
    """Static description of the fused gate + logits op (see ``eqf_gate_logits_fwd`` in include/eqf_b200.h)."""

    def __init__(self, n_alpha: int, n_scalars: int, n_heads: int, ds: Sequence[int], Cs: Sequence[int],
                 c_silu: float, c_sigmoid: float, c_slr: float, slope: float):
        if len(ds) > _lib.EQF_MAX_BLOCKS or n_heads > _lib.EQF_MAX_HEADS or n_alpha % n_heads:
            raise NotImplementedError("gate layout exceeds kernel limits")
        self.n_alpha, self.n_scalars, self.n_heads = n_alpha, n_scalars, n_heads
        self.ds, self.Cs = tuple(ds), tuple(Cs)
        self.c_silu, self.c_sigmoid, self.c_slr, self.slope = c_silu, c_sigmoid, c_slr, slope
        c = _lib.EqfGateLayout()
        c.n_gated, c.n_alpha, c.n_scalars, c.n_heads = len(ds), n_alpha, n_scalars, n_heads
        for i, (d, C) in enumerate(zip(ds, Cs)):
            c.d[i], c.C[i] = d, C
        c.c_silu, c.c_sigmoid, c.c_slr, c.slr_slope = c_silu, c_sigmoid, c_slr, slope
        self.c = c

    @property
    def width(self) -> int:
        return self.n_alpha + self.n_scalars + sum(self.Cs)


def gate_logits_torch(lay: GateLayout, t0, bias, alpha_dot, *gated):
    """Differentiable torch statement of the fused op (higher-order path and the CPU test stand-in)."""
    t = t0 if bias is None else t0 + bias
    E, H, A0, S = t.shape[0], lay.n_heads, lay.n_alpha, lay.n_scalars
    if A0 > 0:
        a = t[:, :A0].reshape(E, H, A0 // H)
        slr = 0.5 * (1 + lay.slope) * a + 0.5 * (1 - lay.slope) * a * (2 * torch.sigmoid(a) - 1)
        z = (lay.c_slr * slr * alpha_dot.reshape(1, H, A0 // H)).sum(-1)
    else:                                   # gate-only layout (node-level FFN): no logits
        z = t.new_zeros((E, H))
    v0 = lay.c_silu * torch.nn.functional.silu(t[:, A0:A0 + S])
    gates = lay.c_sigmoid * torch.sigmoid(t[:, A0 + S:])
    outs, off = [], 0
    for g, C in zip(gated, lay.Cs):
        outs.append(g * gates[:, off:off + C].unsqueeze(1))
        off += C
    return (z, v0, *outs)


def gate_logits_fwd_raw(lay: GateLayout, t0, bias, alpha_dot, gated):
    t0 = _require_cuda(t0, "gate t0")
    E = t0.shape[0]
    if t0.shape[1] != lay.width:
        raise ValueError(f"gate input must be [E, {lay.width}]")
    gated = [_require_cuda(g, "gated block") for g in gated]
    z = torch.empty((E, lay.n_heads), device=t0.device, dtype=torch.float32)
    v0 = torch.empty((E, lay.n_scalars), device=t0.device, dtype=torch.float32)
    vout = [torch.empty_like(g) for g in gated]
    nbytes = 4 * (t0.numel() + 2 * sum(g.numel() for g in gated) + v0.numel() + z.numel())
    with torch.cuda.device(t0.device), _kernel("gate_logits_fwd", nbytes):
        rc = _lib.load().eqf_gate_logits_fwd(ctypes.byref(lay.c), t0.data_ptr(),
                                             bias.data_ptr() if bias is not None else None, _ptr_array(gated),
                                             alpha_dot.data_ptr(), E, z.data_ptr(), v0.data_ptr(), _ptr_array(vout),
                                             _stream())
    _lib.check(rc, "eqf_gate_logits_fwd")
    return z, v0, vout


def gate_logits_bwd_raw(lay: GateLayout, t0, bias, alpha_dot, gated, gz, gv0, gvout):
    E = t0.shape[0]
    gz, gv0 = _require_cuda(gz, "gz"), _require_cuda(gv0, "gv0")
    gvout = [_require_cuda(g, "gvout") for g in gvout]
    rows = _lib.load().eqf_pointwise_rows(E)
    gt0 = torch.empty_like(t0)
    ggated = [torch.empty_like(g) for g in gated]
    gdot = torch.empty((rows, max(lay.n_alpha, 1)), device=t0.device, dtype=torch.float32)
    nbytes = 4 * (2 * t0.numel() + 3 * sum(g.numel() for g in gated) + gv0.numel() + gz.numel())
    with torch.cuda.device(t0.device), _kernel("gate_logits_bwd", nbytes):
        rc = _lib.load().eqf_gate_logits_bwd(ctypes.byref(lay.c), t0.data_ptr(),
                                             bias.data_ptr() if bias is not None else None, _ptr_array(gated),
                                             alpha_dot.data_ptr(), gz.data_ptr(), gv0.data_ptr(), _ptr_array(gvout), E,
                                             gt0.data_ptr(), _ptr_array(ggated), gdot.data_ptr(), _stream())
    _lib.check(rc, "eqf_gate_logits_bwd")
    return gt0, ggated, (colsum_raw(gdot) if lay.n_alpha > 0 else None)


def gate_only_layout(gate, lin_out_irreps) -> Optional[GateLayout]:
    """Layout for ``bias + Gate`` without logits (FFN), or None when the Gate is not in the canonical form
    ``[(scalars + gates) x 0e | gated entries]`` the kernel reads."""
    try:
        scal, gates, gated = gate.irreps_scalars, gate.irreps_gates, gate.irreps_gated
        canonical = (len(scal) == 1 and lin_out_irreps[0].ir.is_scalar()
                     and lin_out_irreps[0].mul == scal.dim + gates.dim
                     and [m for m, _ in lin_out_irreps[1:]] == [m for m, _ in gated]
                     and len(gated) <= _lib.EQF_MAX_BLOCKS)
        if not canonical:
            return None
        return GateLayout(0, scal.dim, 1, [ir.dim for _, ir in gated], [m for m, _ in gated],
                          gate.act_scalars.acts[0].cst, gate.act_gates.acts[0].cst, 1.0, 0.2)
    except (AttributeError, IndexError, NotImplementedError):
        return None


_GATE_DUMMY = {}


def gate_fused(lay: GateLayout, t0, bias, gated):
    """``Gate(bias + [t0 | gated])`` in one kernel (gate-only use of :class:`GateLogits`): returns (scalars, *gated)."""
    dummy = _GATE_DUMMY.get(t0.device)
    if dummy is None:
        dummy = torch.zeros(1, 1, device=t0.device, dtype=t0.dtype)
        _GATE_DUMMY[t0.device] = dummy
    _z, v0, *vs = GateLogits.apply(lay, t0, bias, dummy, *gated)
    return (v0, *vs)


class GateLogits(torch.autograd.Function):
    """(z, v0, *vout) = fused bias + Gate + attention logits (ref :492-495, :506-507).  apply(lay, t0, bias, alpha_dot, *gated)."""

    @staticmethod
    def forward(ctx, lay: GateLayout, t0, bias, alpha_dot, *gated):
        ctx.lay = lay
        ctx.has_bias = bias is not None
        alpha_dot = alpha_dot.contiguous()
        z, v0, vout = gate_logits_fwd_raw(lay, t0, bias, alpha_dot, gated)
        ctx.save_for_backward(t0, alpha_dot, *gated, *([bias] if bias is not None else []))
        return (z, v0, *vout)

    @staticmethod
    def backward(ctx, gz, gv0, *gvout):
        lay = ctx.lay
        saved = ctx.saved_tensors
        n = len(lay.ds)
        t0, alpha_dot, gated = saved[0], saved[1], saved[2:2 + n]
        bias = saved[2 + n] if ctx.has_bias else None
        zeros = lambda like: torch.zeros_like(like)
        gz = gz if gz is not None else t0.new_zeros((t0.shape[0], lay.n_heads))
        gv0 = gv0 if gv0 is not None else t0.new_zeros((t0.shape[0], lay.n_scalars))
        gvout = [g if g is not None else zeros(b) for g, b in zip(gvout, gated)]
        if torch.is_grad_enabled():
            ins = (t0, bias, alpha_dot, *gated)
            fn = lambda t, b, ad, *gs: gate_logits_torch(lay, t, b, ad, *gs)
            grads = _higher_order_grads(fn, ins, (gz, gv0, *gvout))
            return (None, *grads)
        gt0, ggated, gdot = gate_logits_bwd_raw(lay, t0, bias, alpha_dot, gated, gz.contiguous(), gv0.contiguous(),
                                                [g.contiguous() for g in gvout])
        gbias = _colsum(gt0) if bias is not None else None
        return (None, gt0, gbias, gdot.view_as(alpha_dot) if lay.n_alpha > 0 else None, *ggated)


# ----------------------------------------------------------------------------- layout conversion


def _to_planar_impl(x: torch.Tensor, dims) -> List[torch.Tensor]:
    out, off, R = [], 0, x.shape[0]
    for mul, d in dims:
        blk = x.narrow(1, off, mul * d).reshape(R, mul, d)
        out.append(blk.transpose(1, 2).contiguous() if d > 1 else blk.reshape(R, 1, mul).contiguous())
        off += mul * d
    return out


def _from_planar_impl(blocks: Sequence[torch.Tensor]) -> torch.Tensor:
    R = blocks[0].shape[0]
    return torch.cat([b.transpose(1, 2).reshape(R, -1) for b in blocks], dim=1)


class _ToPlanar(torch.autograd.Function):
    """Layout change with a hand-written transpose: the backward is ONE concatenation instead of autograd's
    zero-fill + slice-copy + add per entry (launch-count hygiene on the node path)."""

    @staticmethod
    def forward(ctx, x, dims):
        ctx.dims = dims
        return tuple(_to_planar_impl(x, dims))

    @staticmethod
    def backward(ctx, *gs):
        R = next(g for g in gs if g is not None).shape[0]
        ref = next(g for g in gs if g is not None)
        gs = [g if g is not None else ref.new_zeros((R, d, mul)) for g, (mul, d) in zip(gs, ctx.dims)]
        return _FromPlanar.apply(ctx.dims, *gs), None


class _FromPlanar(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dims, *blocks):
        ctx.dims = dims
        return _from_planar_impl(blocks)

    @staticmethod
    def backward(ctx, g):
        return (None, *_ToPlanar.apply(g, ctx.dims))


def to_planar(x: torch.Tensor, irreps) -> List[torch.Tensor]:
    """e3nn row layout ``[R, sum mul*(2l+1)]`` -> one ``[R, 2l+1, mul]`` block per irreps entry."""
    dims = tuple((mul, ir.dim) for mul, ir in irreps)
    if not x.requires_grad:
        return _to_planar_impl(x, dims)
    return list(_ToPlanar.apply(x, dims))


def from_planar(blocks: Sequence[torch.Tensor]) -> torch.Tensor:
    """Inverse of :func:`to_planar` (entries concatenated in order)."""
    if not any(b.requires_grad for b in blocks):
        return _from_planar_impl(blocks)
    dims = tuple((b.shape[2], b.shape[1]) for b in blocks)
    return _FromPlanar.apply(dims, *blocks)


class _SplitFlat(torch.autograd.Function):
    """Views of consecutive chunks of a flat parameter; backward = one ``cat`` (instead of zero-fill + copy + add per
    chunk, which is what autograd does for ``narrow``)."""

    @staticmethod
    def forward(ctx, w, sizes):
        ctx.sizes = sizes
        out, off = [], 0
        for n in sizes:
            out.append(w.narrow(0, off, n))
            off += n
        return tuple(out)

    @staticmethod
    def backward(ctx, *gs):
        ref = next(g for g in gs if g is not None)
        parts = [g.reshape(-1) if g is not None else ref.new_zeros(n) for g, n in zip(gs, ctx.sizes)]
        return torch.cat(parts), None


class _SplitColumns(torch.autograd.Function):
    """Contiguous column blocks of ``[R, sum(sizes)]``; the backward is ONE concatenation (autograd's per-slice backward
    would zero-fill and copy a full-width buffer per block)."""

    @staticmethod
    def forward(ctx, x, sizes):
        ctx.sizes = sizes
        ctx.rows = x.shape[0]
        return tuple(c.contiguous() for c in x.split(list(sizes), dim=1))

    @staticmethod
    def backward(ctx, *gs):
        ref = next(g for g in gs if g is not None)
        gs = [g if g is not None else ref.new_zeros((ctx.rows, n)) for g, n in zip(gs, ctx.sizes)]
        return torch.cat(gs, dim=1), None


def split_columns(x: torch.Tensor, sizes: Sequence[int]) -> List[torch.Tensor]:
    return list(_SplitColumns.apply(x, tuple(int(n) for n in sizes)))


def split_flat(w: torch.Tensor, sizes: Sequence[int]) -> List[torch.Tensor]:
    if not w.requires_grad or w.dim() != 1:
        out, off = [], 0
        for n in sizes:
            out.append(w.narrow(-1, off, n))
            off += n
        return out
    return list(_SplitFlat.apply(w, tuple(sizes)))
