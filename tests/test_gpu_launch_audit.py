"""Every kernel launch of the trained steps, re-evaluated in float64 from that launch's own float32 inputs.

The per-kernel tests run on ``randn`` inputs at chosen shapes and the model tests compare end results at 1e-4 (energies)
and 1e-3 (gradients); a kernel that is wrong by 1e-4 in one output group, one head or the last partial tile of one call
passes both.  Here one eager forward + backward of each workload runs with every leaf ``*_raw`` wrapper of
``equiformer_b200.ops`` (the functions that call the library) wrapped.  Per call the wrapper

1. snapshots the inputs (in-place outputs such as the ``C`` of an accumulating grouped product included),
2. runs the real kernel and synchronises,
3. checks that the inputs are bit-for-bit unchanged and every output is finite,
4. evaluates the float64 statement of the call on the GPU from the snapshot and compares elementwise,
5. frees everything: nothing is kept across calls but counters.

Criteria (``CRITERIA``, one row per entry point):

* multilinear calls (tensor products, GEMMs, aggregations, column sums): the componentwise first-order rounding bound
  ``|out - ref| <= tau * u * sqrt(K) * ref_abs`` with ``u = 2^-24``, ``K`` the reduction length of that output (per
  output group, per data-gradient block and for the weight gradient of a tensor-product call; per problem of a grouped
  launch, whose forward, data- and weight-gradient products also have a tau each) and ``ref_abs`` the same float64
  statement on the absolute values of every operand (coupling coefficients included).  Unlike the
  max-normalised error of the rest of the suite this also binds small entries (l = 3 blocks, cancelling sums), and an
  entry whose ``ref_abs`` is 0 (a zero-in-degree node) must be exactly 0.  The ratio printed per entry point is
  ``max |out - ref| / (u sqrt(K) ref_abs)``; next to it, the ratio a single-pass TF32 evaluation of the same call would
  reach (operands rounded to TF32, statement in float64), which every ``tau`` must stay below;
* nonlinear calls (softmax family, LayerNorm + SiLU, equivariant LayerNorm, gate / logits, radial bases, edge
  geometry): error over the largest magnitude of each output, with the suite's 2e-5 (forward) / 5e-5 (backward); the
  node rows of the softmax-aggregate family at nodes without incoming edges must be exactly 0 (the Bessel workload
  carries an isolated atom so that they occur).

Launch coverage goes through the loaded library itself: every ``eqf_*`` symbol called while a workload runs is recorded
with whether an audited wrapper was active, so a compute launch outside one fails the workload by name, whichever
route it took.  The workloads run once per module (fixture ``audited``); ``test_every_compute_entry_point_was_audited``
asks that every compute symbol of
``_lib.SIGNATURES`` was launched inside an audited wrapper or sits in ``NOT_AUDITED`` with its reason.  The CPU test at
the end checks the same statically: every compute call of ``ops.py`` / ``graph.py`` sits inside a wrapped function.
"""
from __future__ import annotations

import ast
import gc
import math
import os
import time

import numpy as np
import pytest
import torch

from tests import _emulation as emu

U = 2.0 ** -24
TOL_FWD, TOL_BWD = 2e-5, 5e-5

# entry point -> (kind, tau, worst ratio measured on an H100 SXM 80 GB at 700 W over all workloads of this file).
# kind "lin": componentwise bound, tau in units of u sqrt(K) (ratio measured / tau >= 4x headroom);
# kind "fwd" / "bwd": max-normalised error against TOL_FWD / TOL_BWD (measured worst error next to it).
CRITERIA = {
    "dtp_forward_raw": ("lin", 7, 1.66),
    "dtp_group_forward_raw": ("lin", 6.5, 1.52),
    "dtp_linear_fwd_raw": ("lin", 3, 0.72),
    "dtp_grad_x_raw": ("lin", 2.5, 0.61),
    "dtp_grad_w_raw": ("lin", 2, 0.452),
    "dtp_grad_y_raw": ("lin", 0.25, 0.0544),
    "dtp_grad_xw_raw": ("lin", 5, 1.21),
    "gemm_tf32x3_raw": ("lin", 10, 2.37),
    "gemm_tf32x3_wgrad_raw": ("lin", 0.9, 0.212),
    "grouped_gemm_raw": ("lin", {0: 12, 1: 12, 2: 16}, {0: 2.82, 1: 2.84, 2: 3.93}),   # per mode: forward, dgrad, wgrad
    "colsum_raw": ("lin", 1.5, 0.308),
    "attn_aggregate_raw": ("lin", 5, 1.03),
    "attn_edge_dot_raw": ("lin", 1, 0.228),
    "attn_edge_scale_raw": ("lin", 8, 2.0),
    "seg_softmax_raw": ("fwd", TOL_FWD, 1.33e-07),
    "seg_softmax_bwd_raw": ("bwd", TOL_BWD, 1.55e-07),
    "softmax_aggregate_raw": ("fwd", TOL_FWD, 4.06e-07),
    "dot_softmax_aggregate_raw": ("fwd", TOL_FWD, 3.35e-07),
    "dot_softmax_aggregate_bwd_raw": ("bwd", TOL_BWD, 4.93e-07),
    "mlp_softmax_aggregate_raw": ("fwd", TOL_FWD, 3.73e-07),
    "mlp_softmax_aggregate_bwd_raw": ("bwd", TOL_BWD, 1.87e-07),
    "ln_silu_fwd_raw": ("fwd", TOL_FWD, 9.4e-07),
    "ln_silu_bwd_raw": ("bwd", TOL_BWD, 3.05e-07),
    "eln_fwd_raw": ("fwd", TOL_FWD, 1.78e-07),
    "eln_bwd_raw": ("bwd", TOL_BWD, 1.99e-07),
    "eln_planar_fwd_raw": ("fwd", TOL_FWD, 1.74e-07),
    "eln_planar_bwd_raw": ("bwd", TOL_BWD, 1.75e-07),
    "gate_logits_fwd_raw": ("fwd", TOL_FWD, 2.08e-07),
    "gate_logits_bwd_raw": ("bwd", TOL_BWD, 2.42e-07),
    "rbf_fwd_raw": ("fwd", TOL_FWD, 2.8e-06),
    "rbf_bwd_raw": ("bwd", TOL_BWD, 5.26e-06),
    "bessel_fwd_raw": ("fwd", TOL_FWD, 4.63e-07),
    "bessel_bwd_raw": ("bwd", TOL_BWD, 1.21e-05),
    "edge_geom_fwd_raw": ("fwd", TOL_FWD, 4.62e-07),
    "edge_geom_bwd_raw": ("bwd", TOL_BWD, 6.99e-08),
    "expnorm_fwd_raw": ("fwd", TOL_FWD, 4.37e-07),
    "expnorm_bwd_raw": ("bwd", TOL_BWD, 1.08e-05),
}

# library symbols that launch no computation: plan set-up and introspection, launch-geometry and scratch-size queries
NON_COMPUTE = {"eqf_version", "eqf_last_error", "eqf_device_sm_count", "eqf_plan_create", "eqf_plan_destroy", "eqf_plan_info",
               "eqf_plan_partial_rows", "eqf_dtp_linear_supported", "eqf_fused_set_timeline", "eqf_attn_mlp_rows",
               "eqf_pointwise_rows", "eqf_eln_rows", "eqf_gemm_tf32x3_wgrad_slices", "eqf_colsum_scratch_floats"}
# compute symbols the audit does not re-evaluate, with the reason
NOT_AUDITED = {
    "eqf_radius_graph_count": "neighbour lists: integer outputs, tested bit for bit against the torch brute force "
                              "(test_gpu_kernels.py, test_neighbour_list_pbc.py)",
    "eqf_radius_graph_fill": "as eqf_radius_graph_count",
    "eqf_radius_graph_pbc_count": "as eqf_radius_graph_count, and against a float64 brute force",
    "eqf_radius_graph_pbc_fill": "as eqf_radius_graph_pbc_count",
    "eqf_gemm_tf32x3_wgrad": "per-slice weight gradient, reached only with EQF_DETERMINISTIC=1 (tested in "
                             "test_gpu_kernels.py); the default step runs eqf_gemm_tf32x3_wgrad_accumulate",
}
# nonlinear entry points whose node-level outputs are sums over each node's incoming edges
NODE_SEGMENT_SUMS = {"softmax_aggregate_raw", "dot_softmax_aggregate_raw", "dot_softmax_aggregate_bwd_raw",
                     "mlp_softmax_aggregate_raw"}
# functions outside the audited wrappers that may call the library's compute symbols (neighbour lists, see NOT_AUDITED)
UNWRAPPED_CALLERS = {"_radius_graph_cuda", "radius_graph_pbc"}


# ------------------------------------------------------------------------------------------------ tensor plumbing
def _map(fn, obj):
    """``fn`` on every tensor of a nested list / tuple / dict structure (other objects pass through)."""
    if isinstance(obj, torch.Tensor):
        return fn(obj)
    if isinstance(obj, (list, tuple)):
        return type(obj)(_map(fn, o) for o in obj)
    if isinstance(obj, dict):
        return {k: _map(fn, v) for k, v in obj.items()}
    return obj


def _tensors(obj):
    if isinstance(obj, torch.Tensor):
        return [obj]
    if isinstance(obj, (list, tuple)):
        return [t for o in obj for t in _tensors(o)]
    if isinstance(obj, dict):
        return [t for v in obj.values() for t in _tensors(v)]
    return []


def _flat_outputs(obj):
    """Outputs in order, ``None`` kept (a missing optional output)."""
    if obj is None or isinstance(obj, torch.Tensor):
        return [obj]
    return [t for o in obj for t in _flat_outputs(o)]


def _f64(t):
    return t.double() if t.is_floating_point() else t


def _abs64(t):
    return t.double().abs() if t.is_floating_point() else t


def _tf32_64(t):
    """float32 rounded to TF32 (10 explicit mantissa bits, round to nearest), then float64."""
    if t.dtype != torch.float32:
        return _f64(t)
    i = t.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32).double().view(t.shape)


def _largest_operand(args):
    """max(1, largest |operand|) of a call, for the underflow allowance ``K * 2^-126 * max(1, largest operand)`` of the
    componentwise bound: the tensor cores flush subnormal operands and products to zero, so a sum of K such terms may
    come back as 0 (seen in the MD17 double backward, where whole weight-gradient entries are sums of subnormal
    products).  That allowance is far below any rounding error of a normal-range entry."""
    return max([1.0] + [float(t.abs().max()) for t in _tensors(args) if t.is_floating_point() and t.numel()])


class _AbsPlan:
    """A DTP plan whose coupling coefficients are replaced by their absolute values (for ``ref_abs``)."""

    def __init__(self, plan):
        self._plan = plan
        self.cg64 = np.abs(plan.cg64)

    def __getattr__(self, name):
        return getattr(self._plan, name)


def _describe(args):
    parts = []
    for t in _tensors(args):
        parts.append(f"{tuple(t.shape)}{'' if t.is_contiguous() else ' strides ' + str(t.stride())}")
    return ", ".join(parts[:12]) + (" ..." if len(parts) > 12 else "")


# ------------------------------------------------------------------------------------------------ float64 statements
def _vjp(fn, inputs, cotangents):
    """Gradients of ``fn(*inputs)`` (float64) for the float tensors of ``inputs`` that are not None."""
    with torch.enable_grad():
        ins = [t.detach().requires_grad_(True) if isinstance(t, torch.Tensor) and t.is_floating_point() else t for t in inputs]
        outs = fn(*ins)
        outs = outs if isinstance(outs, (tuple, list)) else (outs,)
        pairs = [(o, g) for o, g in zip(outs, cotangents) if g is not None and o.requires_grad]
        need = [t for t in ins if isinstance(t, torch.Tensor) and t.requires_grad]
        grads = torch.autograd.grad([o for o, _ in pairs], need, [g for _, g in pairs], allow_unused=True)
    it = iter(grads)
    return [next(it) if isinstance(t, torch.Tensor) and t.requires_grad else None for t in ins]


def _dtp_ks(plan, kind, E=1, shared=False):
    """Reduction length (terms per output element) of each output of a DTP call of ``plan``: one per output group
    (forward), one per in1 block (data gradient), one for the weight gradient (times E when the weights are shared and
    the gradient sums over edges) and one for the harmonics gradient."""
    d = lambda l: 2 * l + 1
    if kind == "forward":
        per = [0] * len(plan.out_groups)
        for p in plan.paths:
            per[p.out_group] = max(per[p.out_group], d(p.l1) * d(p.l2))
        return per
    if kind == "grad_x":
        per = [0] * len(plan.in1_blocks)
        for p in plan.paths:
            per[p.in1_block] += d(p.l2) * d(p.l3)
        return per
    if kind == "grad_w":
        return [max(d(p.l1) * d(p.l2) * d(p.l3) for p in plan.paths) * (E if shared else 1)]
    per = {}
    for p in plan.paths:
        per[p.in2_off] = per.get(p.in2_off, 0) + d(p.l1) * d(p.l3) * p.mul
    return [max(per.values())]


def _gemm_ref(conv, args, kw):
    A, Bt = conv(args[0]), conv(args[1])
    kn = kw.get("b_is_kn", args[2] if len(args) > 2 else False)
    return [A @ (Bt if kn else Bt.t())]


def _grouped_ref(conv, args, kw):
    outs = []
    for mode, A, B, C, alpha, acc in args[0]:
        A, B = conv(A), conv(B)
        val = (abs(alpha) if conv is _abs64 else alpha) * (A @ B if mode == 0 else A @ B.t() if mode == 1 else A.t() @ B)
        outs.append(conv(C) + val if acc else val)
    return outs


def _degree(graph, by_src=False):
    idx = graph.src if by_src else graph.dst
    return int(torch.bincount(idx, minlength=graph.n_nodes).max()) if idx.numel() else 1


def _lin_ref(name, args, kw, conv, plan_of):
    """(references, reduction lengths), one of each per output, of a multilinear entry point; operands converted by
    ``conv``, the plan mapped by ``plan_of``."""
    a = _map(conv, args)
    k = _map(conv, kw)
    if name.startswith("dtp_"):
        plan = args[0]
        fn = getattr(emu, name)
        out = fn(plan_of(plan), *a[1:], **k)
        if name == "dtp_forward_raw":
            Ks = _dtp_ks(plan, "forward")
        elif name == "dtp_group_forward_raw":
            Ks = [_dtp_ks(plan, "forward")[args[1]]]
        elif name == "dtp_linear_fwd_raw":
            Ks = [_dtp_ks(plan, "forward")[args[1]] * plan.out_groups[args[1]][2]]
        elif name == "dtp_grad_x_raw":
            Ks = _dtp_ks(plan, "grad_x")
        elif name == "dtp_grad_w_raw":
            Ks = _dtp_ks(plan, "grad_w", args[2].shape[0], args[4])
        elif name == "dtp_grad_y_raw":
            Ks = _dtp_ks(plan, "grad_y")
        else:                                   # (gxs, gw): each data-gradient block and the weight gradient on their own K
            Ks = _dtp_ks(plan, "grad_x") + _dtp_ks(plan, "grad_w", args[2].shape[0], args[3].dim() == 1)
        return _flat_outputs(out), Ks
    if name == "gemm_tf32x3_raw":
        return _gemm_ref(conv, args, kw), [args[0].shape[1]]
    if name == "gemm_tf32x3_wgrad_raw":
        return [a[0].t() @ a[1]], [args[0].shape[0]]
    if name == "grouped_gemm_raw":             # one K per problem: a launch mixes data and weight gradients
        Ks = [(A.shape[0] if m == 2 else A.shape[1]) + (1 if acc else 0) for m, A, B, C, al, acc in args[0]]
        return _grouped_ref(conv, args, kw), Ks
    if name == "colsum_raw":
        return [a[0].sum(0)], [args[0].shape[0]]
    lay = args[0]
    if name == "attn_aggregate_raw":
        by_src = k.get("by_src", a[4] if len(a) > 4 else False)
        outs = emu.attn_aggregate_raw(*a, **k)
        return outs, [_degree(args[3], by_src)] * len(outs)
    if name == "attn_edge_dot_raw":
        return [emu.attn_edge_dot_raw(*a, **k)], [sum(d * c // lay.n_heads for d, c in zip(lay.ds, lay.Cs))]
    if name == "attn_edge_scale_raw":
        outs = emu.attn_edge_scale_raw(*a, **k)
        return outs, [1] * len(outs)
    raise KeyError(name)


def _oracle_bessel(dist, freq, cutoff):
    from tests import oracle_bessel
    return oracle_bessel.bessel_rbf({"m.rbf.frequencies": freq}, "m", dist, cutoff)


def _nonlin_ref(name, args, kw):
    """float64 references of a nonlinear entry point, one per output (None: output not compared)."""
    from equiformer_b200 import ops
    a = _map(_f64, args)
    k = _map(_f64, kw)
    if name in ("seg_softmax_raw", "seg_softmax_bwd_raw", "softmax_aggregate_raw", "dot_softmax_aggregate_raw",
                "dot_softmax_aggregate_bwd_raw", "mlp_softmax_aggregate_raw", "mlp_softmax_aggregate_bwd_raw"):
        return _flat_outputs(getattr(emu, name)(*a, **k))
    if name == "ln_silu_fwd_raw":
        return _flat_outputs(emu.ln_silu_fwd_raw(*a, **k))
    if name == "ln_silu_bwd_raw":
        x, gamma, beta, _mean, _rstd, gy = a[:6]
        bias = a[6] if len(a) > 6 else k.get("bias")
        # the model's LayerNorm eps (radial_func.py); the launch receives rstd, not eps
        gx, gbias, gg, gb = _vjp(lambda xx, pp, g1, b1: ops.ln_silu_torch(xx, g1, b1, 1e-5, pp), (x, bias, gamma, beta), (gy,))
        return [gx, gg, gb, gbias]
    if name == "eln_fwd_raw":
        lay, x, w, b = a
        return [ops.eln_torch(lay, x, w, b), None]
    if name == "eln_bwd_raw":
        lay, x, w, _rstd, gy = a
        b = x.new_zeros(lay.n_b)
        gx, gw, gb = _vjp(lambda xx, ww, bb: ops.eln_torch(lay, xx, ww, bb), (x, w, b), (gy,))
        return [gx, gw, gb]
    if name == "eln_planar_fwd_raw":
        lay, xs, w, b = a
        return [*ops.eln_planar_torch(lay, list(xs), w, b), None]
    if name == "eln_planar_bwd_raw":
        lay, xs, w, _rstd, gys = a
        b = xs[0].new_zeros(lay.n_b)
        g = _vjp(lambda ww, bb, *blocks: tuple(ops.eln_planar_torch(lay, list(blocks), ww, bb)), (w, b, *xs), list(gys))
        return [*g[2:], g[0], g[1]]
    if name == "gate_logits_fwd_raw":
        lay, t0, bias, alpha_dot, gated = a
        z, v0, *vout = ops.gate_logits_torch(lay, t0, bias, alpha_dot, *gated)
        return [z if lay.n_alpha > 0 else None, v0, *vout]
    if name == "gate_logits_bwd_raw":
        lay, t0, bias, alpha_dot, gated, gz, gv0, gvout = a
        g = _vjp(lambda t, ad, *gs: ops.gate_logits_torch(lay, t, bias, ad, *gs), (t0, alpha_dot, *gated), (gz, gv0, *gvout))
        return [g[0], *g[2:], g[1].reshape(-1) if lay.n_alpha > 0 else None]
    if name == "rbf_fwd_raw":
        return [ops.gaussian_rbf_torch(*a)]
    if name == "rbf_bwd_raw":
        return list(emu.rbf_bwd_raw(*a))
    if name == "bessel_fwd_raw":
        return [_oracle_bessel(*a)]
    if name == "bessel_bwd_raw":
        dist, freq, cutoff, g, need_dist = a
        gd, gf = _vjp(lambda d, f: _oracle_bessel(d, f, cutoff), (dist, freq), (g,))
        return [gd if need_dist else None, gf]
    if name == "edge_geom_fwd_raw":
        pos, graph, lmax, offsets = a
        return list(ops.edge_geometry_torch(pos, graph.src, graph.dst, lmax, offsets))
    if name == "edge_geom_bwd_raw":
        vec, lmax, g_sh, g_len = a
        from equiformer_b200.o3.sh import spherical_harmonics
        fn = lambda v: (spherical_harmonics(list(range(lmax + 1)), v, True, "component"), v.norm(dim=1))
        return [_vjp(fn, (vec,), (g_sh, g_len))[0]]
    if name == "expnorm_fwd_raw":
        return [ops.expnorm_torch(*a)]
    if name == "expnorm_bwd_raw":
        dist, means, betas, alpha, hi, g = a
        return [_vjp(lambda d: ops.expnorm_torch(d, means, betas, alpha, hi), (dist,), (g,))[0]]
    raise KeyError(name)


# ------------------------------------------------------------------------------------------------ the audit
class _Stat:
    def __init__(self):
        self.calls, self.worst, self.tf32, self.empty_rows = 0, 0.0, 0.0, 0
        self.by_mode = {}          # grouped products: mode -> [worst ratio, worst TF32 ratio]


class Audit:
    """Wraps the leaf wrappers of ``ops`` and the loaded library for one workload; collects failures and statistics."""

    def __init__(self, workload: str):
        self.workload = workload
        self.depth = 0
        self.index = 0
        self.stats = {}
        self.failures = []
        self.symbols = {}              # symbol -> launches inside an audited wrapper
        self.unaudited = {}            # compute symbol -> launches outside any audited wrapper

    def install(self, monkeypatch, inner=None):
        """``inner``: entry point -> function(real) -> replacement, applied under the audit (seeded faults)."""
        from equiformer_b200 import _lib, ops
        for name in CRITERIA:
            real = getattr(ops, name)
            if inner and name in inner:
                real = inner[name](real)
            monkeypatch.setattr(ops, name, self._wrap(name, real))
        monkeypatch.setattr(_lib, "_lib", _LibRecorder(_lib.load(), self))

    def _wrap(self, name, real):
        def audited(*args, **kw):
            if self.depth:                       # a wrapper called from an audited one: its result is checked there
                return real(*args, **kw)
            snap = _map(lambda t: t.detach().clone(), (args, kw))
            self.depth += 1
            try:
                out = real(*args, **kw)
            finally:
                self.depth -= 1
            torch.cuda.synchronize()
            self._check(name, args, kw, snap, out)
            del snap
            return out
        return audited

    def _fail(self, name, msg):
        self.failures.append(f"{self.workload}: {name} call {self.index}: {msg}")

    def _check(self, name, args, kw, snap, out):
        self.index += 1
        kind, tau, _measured = CRITERIA[name]
        s_args, s_kw = snap
        mutated = set()
        if name == "grouped_gemm_raw":            # C is written in place: the output, not an input
            mutated = {id(p[3]) for p in args[0]}
            outs = [p[3] for p in args[0]]
        else:
            outs = _flat_outputs(out)
        for t, s in zip(_tensors((args, kw)), _tensors((s_args, s_kw))):
            if id(t) not in mutated and not torch.equal(t, s):
                self._fail(name, f"modified an input of shape {tuple(t.shape)}")
        shapes = _describe(s_args)
        st = self.stats.setdefault(name, _Stat())
        st.calls += 1
        with torch.no_grad():
            if kind == "lin":
                ident = lambda p: p
                refs, Ks = _lin_ref(name, s_args, s_kw, _f64, ident)
                absr, _ = _lin_ref(name, s_args, s_kw, _abs64, _AbsPlan)
                tf32, _ = _lin_ref(name, s_args, s_kw, _tf32_64, ident)
                assert len(refs) == len(outs) == len(Ks), (name, len(refs), len(outs), len(Ks))
                big = _largest_operand(s_args)
                # grouped launches mix forward, data- and weight-gradient products: each mode has its own tau
                modes = [p[0] for p in s_args[0]] if name == "grouped_gemm_raw" else [None] * len(outs)
                for i, (o, r, ra, rt, K, mode) in enumerate(zip(outs, refs, absr, tf32, Ks, modes)):
                    t_i = tau[mode] if isinstance(tau, dict) else tau
                    sub = st.by_mode.setdefault(mode, [0.0, 0.0])
                    scale = U * math.sqrt(max(K, 1))
                    floor = K * 2.0 ** -126 * big
                    if not bool(torch.isfinite(o).all()):
                        self._fail(name, f"output {i} {tuple(o.shape)} is not finite ({shapes})")
                        continue
                    err = (o.double() - r).abs()
                    bound = ra * scale + floor
                    ratio = torch.where(ra > 0, err / bound,
                                        torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err)))
                    tr = ((rt - r).abs() / bound).where(ra > 0, torch.zeros_like(err))
                    worst = float(ratio.max()) if ratio.numel() else 0.0
                    t32 = float(tr.max()) if tr.numel() else 0.0
                    st.worst, st.tf32 = max(st.worst, worst), max(st.tf32, t32)
                    sub[0], sub[1] = max(sub[0], worst), max(sub[1], t32)
                    if worst > t_i:
                        at = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
                        what = f"output {i} (mode {mode})" if mode is not None else f"output {i}"
                        self._fail(name, f"{what} {tuple(o.shape)}: ratio {worst:.3g} > tau {t_i} (K = {K}) at "
                                         f"row {at[0]}, index {tuple(int(x) for x in at[1:])}: got {float(o[at]):.9g}, "
                                         f"float64 {float(r[at]):.9g}, |terms| {float(ra[at]):.3g}; inputs {shapes}")
                del refs, absr, tf32
            else:
                refs = _nonlin_ref(name, s_args, s_kw)
                assert len(refs) == len(outs), (name, len(refs), len(outs))
                if name in NODE_SEGMENT_SUMS:
                    self._check_empty_segments(name, s_args, outs, shapes, st)
                for i, (o, r) in enumerate(zip(outs, refs)):
                    if r is None or o is None:
                        continue
                    if not bool(torch.isfinite(o).all()):
                        self._fail(name, f"output {i} {tuple(o.shape)} is not finite ({shapes})")
                        continue
                    d = (o.double() - r).abs()
                    err = float(d.max()) / max(float(r.abs().max()), 1e-30) if d.numel() else 0.0
                    st.worst = max(st.worst, err)
                    if err > tau:
                        at = np.unravel_index(int(d.argmax()), tuple(d.shape))
                        self._fail(name, f"output {i} {tuple(o.shape)}: error {err:.3g} of the largest magnitude > {tau} "
                                         f"at row {at[0]}, index {tuple(int(x) for x in at[1:])}: got {float(o[at]):.9g}, "
                                         f"float64 {float(r[at]):.9g}; inputs {shapes}")
                del refs

    def _check_empty_segments(self, name, args, outs, shapes, st):
        """Node rows of the softmax-aggregate family are sums over the node's incoming edges: a node without any must
        come back exactly 0, not merely within the tolerance of the largest entry."""
        from equiformer_b200 import ops
        graph = next(a for a in args if isinstance(a, ops.Graph))
        empty = torch.bincount(graph.dst, minlength=graph.n_nodes) == 0
        if not bool(empty.any()):
            return
        for i, o in enumerate(outs):
            if o is None or o.shape[0] != graph.n_nodes or graph.n_nodes == graph.n_edges:
                continue
            st.empty_rows += int(empty.sum())
            bad = (o[empty].reshape(int(empty.sum()), -1) != 0).any(1)
            if bool(bad.any()):
                row = int(empty.nonzero()[int(bad.nonzero()[0])])
                self._fail(name, f"output {i} {tuple(o.shape)}: node {row} has no incoming edge but a non-zero row; "
                                 f"inputs {shapes}")

    def report(self):
        print(f"\n[audit] {self.workload}: {self.index} audited calls")
        for name in sorted(self.stats):
            st = self.stats[name]
            kind, tau, _ = CRITERIA[name]
            extra = f"  tf32 {st.tf32:9.3g}  tau {tau}" if kind == "lin" else f"  tol {tau}"
            if st.empty_rows:
                extra += f"  ({st.empty_rows} rows of nodes without incoming edges exactly 0)"
            print(f"[audit]   {name:32s} {st.calls:5d} calls  worst {st.worst:9.3g}{extra}")
            for mode in sorted(m for m in st.by_mode if m is not None):
                w, t = st.by_mode[mode]
                print(f"[audit]     mode {mode}: worst {w:9.3g}  tf32 {t:9.3g}  tau {tau[mode]}")


class _LibRecorder:
    """The loaded library with every ``eqf_*`` call recorded (symbol, inside an audited wrapper or not)."""

    def __init__(self, lib, audit: Audit):
        self._lib, self._audit = lib, audit

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("eqf_") or name in NON_COMPUTE:
            return fn
        audit = self._audit

        def call(*args):
            if audit.depth:
                audit.symbols[name] = audit.symbols.get(name, 0) + 1
            else:
                audit.unaudited[name] = audit.unaudited.get(name, 0) + 1
            return fn(*args)
        return call


# ------------------------------------------------------------------------------------------------ workloads
def _bench():
    import bench
    return bench


def _l1(out, tgt):
    return (out - tgt).abs().mean()


def _l2mae(pred, tgt):
    return (pred - tgt).norm(p=2, dim=-1).mean()


def _pbc_graph(d):
    from equiformer_b200.graph import radius_graph_pbc
    edge, offs, _ = radius_graph_pbc(d["pos"], d["batch"], d["cell"], 5.0, 500)
    src, dst = edge[0], edge[1]
    offsets = torch.bmm(offs.to(d["pos"].dtype).view(-1, 1, 3), d["cell"].index_select(0, d["batch"].index_select(0, dst))).view(-1, 3)
    return src, dst, d["pos"].index_select(0, src) - d["pos"].index_select(0, dst) + offsets


def _bench_step(wl, dev, n_graphs=None, alpha_drop=0.0):
    """One eager forward + backward of bench.py's step for ``wl`` (its ``forward_loss``, restated)."""
    b = _bench()
    model = b.build_model(wl, dev, alpha_drop)
    d = {k: v.to(dev) for k, v in b.make_inputs(wl, seed=0, n_graphs=n_graphs).items()}

    def run():
        model.zero_grad(set_to_none=True)
        if wl == "qm9":
            loss = _l1(model(f_in=None, pos=d["pos"], batch=d["batch"], node_atom=d["z"], n_graphs=d["target"].shape[0]),
                       d["target"])
        elif wl == "md17_l3":
            energy, forces = model(node_atom=d["z"], pos=d["pos"], batch=d["batch"])
            loss = 1.0 * _l2mae(energy, d["target"]) + 100.0 * _l2mae(forces, d["ftarget"])
        else:
            src, dst, edge_vec = _pbc_graph(d)
            if wl == "oc20_l1":
                out = model.forward_edges(edge_vec, d["batch"], d["z"], d["tags"], src, dst, n_graphs=d["target"].shape[0])
            else:
                out = model.forward_edges(d["pos"], d["batch"], d["z"], src, dst, n_graphs=1, edges_sorted=True,
                                          edge_vec=edge_vec)
            loss = _l1(out, d["target"])
        loss.backward()
        return loss.detach(), {k: p.grad for k, p in model.named_parameters()}
    return run


def _oc20_variant_step(kind, dev):
    from tests.test_oc20_aux import _frames
    torch.manual_seed(0)
    if kind == "e3":
        from tests.test_oc20_e3 import _full_model
        model = _full_model(num_layers=2)
    elif kind == "dp":
        from equiformer_b200.nets.dp_attention_transformer_oc20 import OC20_DP_L1_256, DotProductAttentionTransformerOC20
        model = DotProductAttentionTransformerOC20(None, None, 1, **dict(OC20_DP_L1_256, num_layers=2))
    else:
        from equiformer_b200.nets.graph_attention_transformer_oc20 import OC20_L1_256, GraphAttentionTransformerOC20
        model = GraphAttentionTransformerOC20(None, None, 1, **dict(OC20_L1_256, num_layers=2))
    model = model.to(dev).train()                      # attention dropout at the configurations' 0.2: masked kernels
    pos, batch, z, tags, src, dst, edge_vec = _frames(dev, seed=3)
    target = torch.randn(4, 1, generator=torch.Generator().manual_seed(7)).to(dev)

    def run():
        loss = _l1(model.forward_edges(edge_vec, batch, z, tags, src, dst, n_graphs=4), target)
        loss.backward()
        return loss.detach(), None
    return run


def _bessel_step(dev):
    from equiformer_b200.nets import model_entrypoint
    from equiformer_b200.synthetic import qm9_like_batch
    torch.manual_seed(0)
    model = model_entrypoint("graph_attention_transformer_nonlinear_bessel_l2")(irreps_in="5x0e", radius=5.0, num_basis=8)
    model = model.to(dev).train()
    pos, batch, z = qm9_like_batch(64, seed=0)
    # a 65th molecule of one atom, far from the rest: a node without incoming edges, whose aggregated rows must be 0
    pos = torch.cat([pos, torch.full((1, 3), 1.0e3)])
    batch = torch.cat([batch, torch.tensor([64])])
    z = torch.cat([z, z[:1]])
    pos, batch, z = (t.to(dev) for t in (pos, batch, z))
    target = torch.randn(65, 1, generator=torch.Generator().manual_seed(1)).to(dev)

    def run():
        loss = _l1(model(f_in=None, pos=pos, batch=batch, node_atom=z, n_graphs=65), target)
        loss.backward()
        return loss.detach(), None
    return run


def _dens_step(dev):
    from equiformer_b200.graphs import DensTrainStep
    from tests.test_md17_dens_train import STD, TASK_MEAN, TASK_STD, _conformers, _trainer
    model, bucket, _opt = _trainer("MD17_DENS_L2", dev)
    step = DensTrainStep(model, bucket, capture=False, task_mean=TASK_MEAN, task_std=TASK_STD, std=STD, prob=0.25,
                         corrupt_ratio=0.25, w_e=1.0, w_f=80.0)
    pos, batch, z, y, dy = _conformers(8, 0, dev)
    w_dn = torch.tensor([5.0], device=dev)

    def run():
        gen = torch.Generator(device=dev).manual_seed(100)
        return step(pos, batch, z, y, dy, 8, w_dn, generator=gen).detach(), None
    return run


# workload -> (builder(dev) -> step, lower the fused-forward threshold so that K1 and the group forward run)
WORKLOADS = {
    "qm9": (lambda dev: _bench_step("qm9", dev), False),
    "md17_l3": (lambda dev: _bench_step("md17_l3", dev), False),
    "oc20_l1": (lambda dev: _bench_step("oc20_l1", dev), False),
    # 2 000 atoms instead of 5 000: an eager step plus per-call snapshots and float64 references must fit a shared card
    "stress_2k": (lambda dev: _bench_step("stress", dev, n_graphs=2000), True),
    "oc20_e3": (lambda dev: _oc20_variant_step("e3", dev), True),
    "oc20_dp": (lambda dev: _oc20_variant_step("dp", dev), False),
    "oc20_linear": (lambda dev: _oc20_variant_step("linear", dev), False),
    "qm9_bessel": (_bessel_step, False),
    "md17_dens": (_dens_step, False),
}

def _release():
    gc.collect()
    torch.cuda.empty_cache()


def _run_audited(wl, dev, monkeypatch, inner=None):
    from equiformer_b200 import ops
    build, low_fused = WORKLOADS[wl]
    if low_fused:
        monkeypatch.setattr(ops, "_FUSED_MIN_EDGES", 1)
    step = build(dev)
    audit = Audit(wl)
    audit.install(monkeypatch, inner)
    try:
        loss, grads = step()
        torch.cuda.synchronize()
    finally:
        monkeypatch.undo()
    return audit, loss, grads, step


@pytest.fixture(scope="module")
def audited(cuda_device):
    """Every workload once under the audit: workload -> (audit, loss) or the exception it raised."""
    runs = {}
    for wl in WORKLOADS:
        torch.cuda.reset_peak_memory_stats()
        t0 = time.time()
        try:
            with pytest.MonkeyPatch.context() as mp:
                audit, loss, _grads, _step = _run_audited(wl, cuda_device, mp)
            audit.report()
            print(f"[audit] {wl}: {time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
            runs[wl] = (audit, float(loss))
        except Exception as exc:             # reported by that workload's test, the others still run
            runs[wl] = exc
        finally:
            _release()
    return runs


@pytest.mark.gpu
@pytest.mark.parametrize("wl", list(WORKLOADS))
def test_every_launch_matches_its_float64_statement(audited, wl):
    run = audited[wl]
    if isinstance(run, Exception):
        raise run
    audit, loss = run
    assert math.isfinite(loss)
    stray = {s: n for s, n in audit.unaudited.items() if s not in NOT_AUDITED}
    assert not stray, f"{wl}: compute launches outside any audited wrapper: {stray}"
    assert not audit.failures, "\n".join(audit.failures[:20])
    if wl in ("stress_2k", "oc20_e3"):
        assert audit.stats.get("dtp_linear_fwd_raw") and audit.stats.get("dtp_group_forward_raw"), wl
    if wl == "qm9_bessel":
        assert audit.stats["softmax_aggregate_raw"].empty_rows > 0, "the isolated atom's rows were not checked"


@pytest.mark.gpu
def test_every_compute_entry_point_was_audited(audited):
    """Over the workloads: each compute symbol of the library ran inside an audited wrapper, or is in NOT_AUDITED;
    each multilinear tau lies below what a single-pass TF32 evaluation reaches on the same calls."""
    from equiformer_b200 import _lib
    seen, worst, by_mode = {}, {}, {}
    for wl, run in audited.items():
        assert not isinstance(run, Exception), f"{wl} did not run: {run!r}"
        audit, _loss = run
        for sym, n in audit.symbols.items():
            seen[sym] = seen.get(sym, 0) + n
        for name, st in audit.stats.items():
            w, t = worst.get(name, (0.0, 0.0))
            worst[name] = (max(w, st.worst), max(t, st.tf32))
            for mode, (wm, tm) in st.by_mode.items():
                if mode is not None:
                    a, b = by_mode.get(mode, (0.0, 0.0))
                    by_mode[mode] = (max(a, wm), max(b, tm))
    compute = set(_lib.SIGNATURES) - NON_COMPUTE
    missing = sorted(s for s in compute if s not in seen and s not in NOT_AUDITED)
    assert not missing, f"compute entry points no workload reached: {missing}"
    print("\n[audit] worst over all workloads (entry point: ratio / error, TF32 ratio)")
    for name in sorted(worst):
        kind, tau, _ = CRITERIA[name]
        w, t = worst[name]
        print(f"[audit]   {name:32s} {w:9.3g}  {t:9.3g}")
        if kind == "lin" and not isinstance(tau, dict):
            assert tau < t, f"{name}: tau {tau} would accept a single-pass TF32 product (TF32 ratio {t:.3g})"
    for mode in sorted(by_mode):
        w, t = by_mode[mode]
        tau = CRITERIA["grouped_gemm_raw"][1][mode]
        print(f"[audit]   grouped_gemm_raw mode {mode}          {w:9.3g}  {t:9.3g}")
        assert tau < t, f"grouped_gemm_raw mode {mode}: tau {tau} would accept a single-pass TF32 product ({t:.3g})"


# ------------------------------------------------------------------------------------------------ the audit has teeth
def _once(fn, call=1):
    """Apply ``fn`` to the outputs of the ``call``-th call only."""
    def make(real):
        state = {"n": 0}

        def faulty(*args, **kw):
            out = real(*args, **kw)
            state["n"] += 1
            if state["n"] == call:
                fn(out)
            return out
        return faulty
    return make


def _scale_dtp_group(outs):
    outs[-1][..., -32:] *= 1.0 + 1e-4


def _tf32_operands(real):
    def single_pass(A, Bt, b_is_kn=False):
        return real(_tf32_64(A).float(), _tf32_64(Bt).float(), b_is_kn=b_is_kn)
    return single_pass


def _drop_last_edge(out):
    gxs, _gw = out
    gxs[0][-1].zero_()


def _scale_head(out):
    outs, _alpha = out
    C = outs[0].shape[2]
    outs[0][..., : C // 4] *= 1.0 + 1e-4          # head 0 of the 4 heads of the QM9 model


def _scale_mixed_dgrad(real):
    """The first grouped launch that holds data- and weight-gradient products together (a first-order planar-linear
    backward): its first data-gradient output scaled by 1 + 1e-4."""
    state = {"done": False}

    def faulty(problems):
        real(problems)
        modes = {p[0] for p in problems}
        if not state["done"] and {1, 2} <= modes:
            state["done"] = True
            next(p for p in problems if p[0] == 1)[3].mul_(1.0 + 1e-4)
    return faulty


FAULTS = {
    # the second call, block 0's first product: the first is the edge-degree embedding, whose input has zero l >= 1
    # blocks, so the last channels of its output groups are exactly 0 and a scaling cannot show
    "dtp_forward_group_scaled": ("dtp_forward_raw", _once(_scale_dtp_group, call=2)),
    "gemm_single_pass_tf32": ("gemm_tf32x3_raw", _tf32_operands),
    "dtp_grad_xw_last_edge_dropped": ("dtp_grad_xw_raw", _once(_drop_last_edge)),
    "softmax_aggregate_head_scaled": ("softmax_aggregate_raw", _once(_scale_head)),
    "grouped_dgrad_of_mixed_launch_scaled": ("grouped_gemm_raw", _scale_mixed_dgrad),
}


@pytest.fixture(scope="module")
def qm9_clean(cuda_device):
    """Loss and gradients of the unaudited, fault-free QM9 step (to tell whether the end-to-end tolerances would see a
    seeded fault)."""
    loss, grads = _bench_step("qm9", cuda_device)()
    out = float(loss), {k: g.detach().clone() for k, g in grads.items() if g is not None}
    _release()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("fault", list(FAULTS))
def test_seeded_fault_is_caught_and_named(cuda_device, monkeypatch, qm9_clean, fault):
    entry, make = FAULTS[fault]
    try:
        audit, loss, grads, _ = _run_audited("qm9", cuda_device, monkeypatch, inner={entry: make})
        named = [f for f in audit.failures if f.startswith(f"qm9: {entry} ")]
        assert named, f"{fault}: the audit did not flag {entry}: {audit.failures[:3]}"
        others = [f for f in audit.failures if not f.startswith(f"qm9: {entry} ")]
        assert not others, f"{fault}: flagged other entry points too: {others[:3]}"
        clean_loss, clean_grads = qm9_clean
        e_loss = abs(float(loss) - clean_loss) / abs(clean_loss)
        e_grad = max(float((grads[k] - g).abs().max() / g.abs().max().clamp_min(1e-12)) for k, g in clean_grads.items())
        print(f"\n[fault] {fault}: {len(named)} flagged call(s), first: {named[0][:200]}")
        print(f"[fault] {fault}: end to end, loss off by {e_loss:.2e} (tolerance 1e-4), worst parameter gradient off by "
              f"{e_grad:.2e} of its largest entry (tolerance 1e-3): "
              f"{'caught' if e_loss > 1e-4 or e_grad > 1e-3 else 'not caught'} by the model tests")
    finally:
        _release()


# ------------------------------------------------------------------------------------------------ static coverage (CPU)
def _compute_calls(path):
    """(enclosing top-level function, symbol) of every ``.eqf_*`` compute call in a source file."""
    tree = ast.parse(open(path).read())
    found = []
    for top in tree.body:
        nodes = [top] if isinstance(top, (ast.FunctionDef, ast.ClassDef)) else []
        for node in nodes:
            for sub in ast.walk(node):
                if (isinstance(sub, ast.Call) and isinstance(sub.func, ast.Attribute) and sub.func.attr.startswith("eqf_")
                        and sub.func.attr not in NON_COMPUTE):
                    found.append((node.name, sub.func.attr))
        if not nodes:
            for sub in ast.walk(top):
                if isinstance(sub, ast.Attribute) and sub.attr.startswith("eqf_") and sub.attr not in NON_COMPUTE:
                    found.append(("<module>", sub.attr))
    return found


def test_every_compute_call_sits_in_an_audited_wrapper():
    """A kernel launched from anywhere but a function of CRITERIA would run unaudited: every compute call of the
    library in ops.py / graph.py sits in one (or is a neighbour-list launch, see NOT_AUDITED), and every function
    CRITERIA names exists and launches something."""
    from equiformer_b200 import _lib, ops
    pkg = os.path.dirname(os.path.abspath(ops.__file__))
    calls = _compute_calls(os.path.join(pkg, "ops.py")) + _compute_calls(os.path.join(pkg, "graph.py"))
    assert calls
    stray = [(fn, sym) for fn, sym in calls if fn not in CRITERIA and not (fn in UNWRAPPED_CALLERS and sym in NOT_AUDITED)]
    assert not stray, f"compute calls outside the audited wrappers: {stray}"
    assert all(sym in _lib.SIGNATURES for _fn, sym in calls)
    callers = {fn for fn, _sym in calls}
    assert set(CRITERIA) <= callers, sorted(set(CRITERIA) - callers)
