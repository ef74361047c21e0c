"""-m gpu: the edge and row kernels past their grid caps, where every warp or CTA runs more than one pass of its
grid-stride loop, against fp64 references.

Almost every kernel is launched with a capped grid and walks its edges or rows in a grid-stride loop; the per-kernel
suite (test_gpu_kernels.py) stays below the caps, so each warp runs one pass there.  Here every case is sized from the
launch formula of the kernel it exercises (``*_pass`` below, one per launcher), with C = the edges or rows one pass
covers and G = the edges a warp takes per step:

* E = 2 C: every warp runs exactly two full passes;
* E = 2 C + C / 3 + G - 1: only some warps run a third pass, and it ends in a partial edge group.

That covers the later passes, the partial last pass and the accumulators carried across passes (the shared-weight
gradient of the tensor product, the per-CTA partial sums of the LayerNorm + SiLU and gate backward kernels).  Per-edge
outputs are compared chunk by chunk with the fp64 table walk of tests/_emulation.py (run on the GPU in float64); the
error is the worst difference over the largest reference magnitude across all chunks, as ``rel_err`` in the rest of
the suite, with the suite's tolerances.  A failure names the worst edge and the pass it belongs to.
"""
from __future__ import annotations

import math

import pytest
import torch

from tests import _emulation as emu
from tests.helpers import rel_err
from tests.test_gpu_kernels import GATE_LOGITS_CFGS, GATE_ONLY_CFGS

pytestmark = pytest.mark.gpu
TOL = 2e-5          # single kernel vs fp64, as test_gpu_kernels.py
TOL_BWD = 5e-5      # row-kernel backward (parameter gradients are sums over all rows), as test_gpu_kernels.py
CHUNK = 8192        # edges per fp64 reference evaluation

DTP_PLANS = {
    "qm9_l2": ("128x0e+64x1e+32x2e", "1x0e+1x1e+1x2e"),
    "md17_l3": ("128x0e+64x1e+64x2e+32x3e", "1x0e+1x1e+1x2e+1x3e"),
    "oc20_l1": ("256x0e+128x1e", "1x0e+1x1e"),
    "e3_l2": ("128x0e+32x0o+32x1e+32x1o+16x2e+16x2o", "1x0e+1x1o+1x2e"),     # generic float4 kernels
    "odd_mul": ("6x0e+3x1e+2x2e", "1x0e+1x1e+1x2e"),                          # generic scalar kernels
}
GENERATED = ("qm9_l2", "md17_l3", "oc20_l1")
SIZES = ("two_passes", "partial_third_pass")


@pytest.fixture(autouse=True)
def _release_cached_memory():
    """The cases allocate up to a few GB each: print the peak, hand the cached blocks back to the card's other users."""
    if torch.cuda.is_available():
        torch.cuda.reset_peak_memory_stats()
    yield
    if torch.cuda.is_available():
        print(f"[memory] peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ pass sizes
def _sms() -> int:
    from equiformer_b200 import _lib
    return _lib.load().eqf_device_sm_count()


def _gen_dtp_pass(plan):
    """Generated DTP forward / backward / grad_y (codegen.py ``grid_for_edges``): min(ceil(ceil(E / G) / 8), 8 SMs)
    CTAs of 8 warps, each warp G edges per step; G as ``codegen.generate`` computes it."""
    from equiformer_b200 import codegen
    G = max(codegen._Block(b, l, mul).epw for b, (l, mul) in enumerate(plan.in1_blocks))
    return 8 * _sms() * 8 * G, G


def _generic_dtp_pass(plan):
    """Generic scalar / float4 DTP kernels (eqf_dtp.cu ``grid_for``, eqf_dtp_vec.cu ``vgrid_bwd``): min(ceil(E / te),
    8 SMs) CTAs, one tile of te edges per CTA step."""
    te = plan.info()["tile_edges"]
    return 8 * _sms() * te, te


def _group_forward_pass():
    """``eqf_dtp_group_forward`` (eqf_fused.cu): min(ceil(E / 32), 8 SMs) CTAs of 32 edges per step."""
    return 32 * 8 * _sms(), 32


# eqf_pointwise.cu ``pointwise_grid``: min(ceil(rows / 8), 132 * 8) CTAs of 8 warps (132 is a literal there); one row
# per warp step, two for the 64-wide LayerNorm + SiLU kernels (half a warp per row)
_POINTWISE_CTAS = 132 * 8


def _pointwise_pass(rows_per_warp=1):
    return 8 * _POINTWISE_CTAS * rows_per_warp, rows_per_warp


def _edge_scale_pass(vec: bool, max_rowlen: int):
    """``eqf_attn_edge_scale`` (eqf_attn.cu): float4 kernel min(ceil(E / 8), 132 * 16) CTAs of 8 warps, one edge per
    warp step; scalar kernel min(ceil(E * rowlen / 256), 132 * 32) CTAs, one element per thread step."""
    if vec:
        return 8 * 132 * 16, 1
    return 132 * 32 * 256 // max_rowlen, 1


def _size(C: int, G: int, which: str) -> int:
    return 2 * C if which == "two_passes" else 2 * C + C // 3 + G - 1


def _report(what: str, n: int, C: int):
    print(f"[passes] {what}: {n} edges/rows, {C} per pass -> {math.ceil(n / C)} passes ({n / C:.3f})")


# ------------------------------------------------------------------------------------------------ chunked comparison
class _Worst:
    """Largest |kernel - reference| over the largest |reference|, accumulated over edge chunks; remembers the edge."""

    def __init__(self, what: str, per_pass: int):
        self.what, self.per_pass = what, per_pass
        self.diff, self.scale, self.at = 0.0, 0.0, -1

    def add(self, out, ref, e0: int):
        d = (out.double() - ref).abs().reshape(ref.shape[0], -1).amax(1)
        i = int(d.argmax())
        if float(d[i]) > self.diff:
            self.diff, self.at = float(d[i]), e0 + i
        self.scale = max(self.scale, float(ref.abs().max()))

    def check(self, tol=TOL):
        err = self.diff / max(self.scale, 1e-30)
        assert err < tol, (f"{self.what}: error {err:.3e} of the largest magnitude, worst at edge {self.at} "
                           f"(pass {self.at // self.per_pass}, edge {self.at % self.per_pass} of that pass)")


def _compare_chunked(outs, ref_fn, E: int, what: str, per_pass: int, tol=TOL):
    """``ref_fn(a, b)`` -> fp64 references of edges [a, b) for every tensor of ``outs``."""
    worst = [_Worst(f"{what}[{k}]", per_pass) for k in range(len(outs))]
    for a in range(0, E, CHUNK):
        b = min(E, a + CHUNK)
        for k, ref in enumerate(ref_fn(a, b)):
            worst[k].add(outs[k][a:b], ref, a)
    for w in worst:
        w.check(tol)


def _plan(name):
    from equiformer_b200 import codegen
    plan = codegen.plan_for(*DTP_PLANS[name])
    assert plan.generated == (name in GENERATED), name
    return plan


def _randn(gen, *shape):
    return torch.randn(*shape, generator=gen, device=gen.device)


def _rows(ts, a, b):
    return [t[a:b].double() for t in ts]


# ------------------------------------------------------------------------------------------------ DTP family
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("name", list(DTP_PLANS))
def test_dtp_family_multipass(cuda_device, name, shared, size):
    """forward, grad_x, grad_y, grad_w and grad_xw past the cap of the kernels that run the plan (generated for the
    shipped configurations, generic float4 for the E(3) plan, scalar for odd multiplicities); the shared-weight
    gradients are sums over all passes of every warp."""
    from equiformer_b200 import _lib, ops
    plan = _plan(name)
    C, G = _gen_dtp_pass(plan) if plan.generated else _generic_dtp_pass(plan)
    E = _size(C, G, size)
    _report(f"dtp {name} {'shared' if shared else 'per-edge'} w", E, C)
    gen = torch.Generator(device=cuda_device).manual_seed(E + len(name) + shared)
    xs = [_randn(gen, E, 2 * l + 1, mul) for l, mul in plan.in1_blocks]
    y = _randn(gen, E, plan.d_y)
    w = _randn(gen, plan.weight_numel) if shared else _randn(gen, E, plan.weight_numel)
    w_at = (lambda a, b: w.double()) if shared else (lambda a, b: w[a:b].double())

    out = ops.dtp_forward_raw(plan, xs, y, w)
    if not plan.generated:      # the generic kernels' grid (= the partial-row count of the shared-weight gradient) is full
        assert _lib.load().eqf_plan_partial_rows(plan.handle, E) == 8 * _sms()
    _compare_chunked(out, lambda a, b: emu.dtp_forward_raw(plan, _rows(xs, a, b), y[a:b].double(), w_at(a, b)),
                     E, "forward", C)
    del out
    gs = [_randn(gen, E, 2 * l + 1, mul) for l, _p, mul in plan.out_groups]
    gx_ref = lambda a, b: emu.dtp_grad_x_raw(plan, _rows(gs, a, b), y[a:b].double(), w_at(a, b))
    gx = ops.dtp_grad_x_raw(plan, gs, y, w)
    _compare_chunked(gx, gx_ref, E, "grad_x", C)
    del gx
    gy = ops.dtp_grad_y_raw(plan, xs, w, gs, y)
    _compare_chunked([gy], lambda a, b: [emu.dtp_grad_y_raw(plan, _rows(xs, a, b), w_at(a, b), _rows(gs, a, b),
                                                            y[a:b].double())], E, "grad_y", C)
    del gy
    gw_ref = lambda a, b: emu.dtp_grad_w_raw(plan, _rows(xs, a, b), y[a:b].double(), _rows(gs, a, b), shared)
    gw_shared_ref = sum(gw_ref(a, min(E, a + CHUNK)) for a in range(0, E, CHUNK)) if shared else None
    gx, gw = ops.dtp_grad_xw_raw(plan, xs, y, w, gs)
    _compare_chunked(gx, gx_ref, E, "grad_xw x", C)
    if shared:
        assert rel_err(gw, gw_shared_ref) < TOL, ("grad_xw shared w", rel_err(gw, gw_shared_ref))
    else:
        _compare_chunked([gw], lambda a, b: [gw_ref(a, b)], E, "grad_xw w", C)
    del gx, gw, w
    # the weight gradient alone: no generated variant, so the scalar kernel runs for every plan
    Cw, _ = _generic_dtp_pass(plan)
    gw = ops.dtp_grad_w_raw(plan, xs, y, gs, shared)
    if shared:
        assert rel_err(gw, gw_shared_ref) < TOL, ("grad_w shared", rel_err(gw, gw_shared_ref))
    else:
        _compare_chunked([gw], lambda a, b: [gw_ref(a, b)], E, "grad_w", Cw)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("name", GENERATED)
def test_dtp_grad_w_scalar_kernel_multipass(cuda_device, name, shared, size):
    """``dtp_grad_w`` has no generated variant (it is what ``DtpGradW`` runs under ``create_graph``, the MD17 forces):
    the scalar kernel sized from its own cap, te edges per tile."""
    from equiformer_b200 import _lib, ops
    plan = _plan(name)
    C, G = _generic_dtp_pass(plan)
    E = _size(C, G, size)
    _report(f"dtp_grad_w {name} {'shared' if shared else 'per-edge'}", E, C)
    gen = torch.Generator(device=cuda_device).manual_seed(E + 5 * shared)
    xs = [_randn(gen, E, 2 * l + 1, mul) for l, mul in plan.in1_blocks]
    y = _randn(gen, E, plan.d_y)
    gs = [_randn(gen, E, 2 * l + 1, mul) for l, _p, mul in plan.out_groups]
    gw = ops.dtp_grad_w_raw(plan, xs, y, gs, shared)
    ref = lambda a, b: emu.dtp_grad_w_raw(plan, _rows(xs, a, b), y[a:b].double(), _rows(gs, a, b), shared)
    if shared:
        total = sum(ref(a, min(E, a + CHUNK)) for a in range(0, E, CHUNK))
        assert rel_err(gw, total) < TOL, rel_err(gw, total)
    else:
        _compare_chunked([gw], lambda a, b: [ref(a, b)], E, "grad_w", C)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("name", GENERATED)
def test_dtp_gathered_offset_multipass(cuda_device, name, size):
    """Generated forward and grad_xw with the node tables gathered in the kernel (x = A[src] + B[dst]) and the radial
    offset added to the per-edge weights, past the cap."""
    from equiformer_b200 import ops
    plan = _plan(name)
    C, G = _gen_dtp_pass(plan)
    E = _size(C, G, size)
    _report(f"dtp gathered + offset {name}", E, C)
    n_nodes = E // 16
    gen = torch.Generator(device=cuda_device).manual_seed(E + 11)
    As = [_randn(gen, n_nodes, 2 * l + 1, mul) for l, mul in plan.in1_blocks]
    Bs = [_randn(gen, n_nodes, 2 * l + 1, mul) for l, mul in plan.in1_blocks]
    src = torch.randint(0, n_nodes, (E,), generator=gen, device=cuda_device)
    dst = torch.sort(torch.randint(0, n_nodes, (E,), generator=gen, device=cuda_device)).values
    y = _randn(gen, E, plan.d_y)
    w = _randn(gen, E, plan.weight_numel)
    off = _randn(gen, plan.weight_numel)
    gather = (src, dst, Bs)
    x_at = lambda a, b: [A.double()[src[a:b]] + B.double()[dst[a:b]] for A, B in zip(As, Bs)]
    w_at = lambda a, b: w[a:b].double() + off.double()

    out = ops.dtp_forward_raw(plan, As, y, w, gather=gather, w_offset=off)
    _compare_chunked(out, lambda a, b: emu.dtp_forward_raw(plan, x_at(a, b), y[a:b].double(), w_at(a, b)),
                     E, "gathered forward", C)
    del out
    gs = [_randn(gen, E, 2 * l + 1, mul) for l, _p, mul in plan.out_groups]
    gx, gw = ops.dtp_grad_xw_raw(plan, As, y, w, gs, gather=gather, w_offset=off)
    _compare_chunked(gx, lambda a, b: emu.dtp_grad_x_raw(plan, _rows(gs, a, b), y[a:b].double(), w_at(a, b)),
                     E, "gathered grad_xw x", C)
    _compare_chunked([gw], lambda a, b: [emu.dtp_grad_w_raw(plan, x_at(a, b), y[a:b].double(), _rows(gs, a, b), False)],
                     E, "gathered grad_xw w", C)


# ------------------------------------------------------------------------------------------------ fused-kernel producer
@pytest.mark.parametrize("name,group,widths,shared", [("qm9_l2", 0, (352, 128), False), ("qm9_l2", 0, (352, 128), True),
                                                      ("md17_l3", 3, (32,), False)])
def test_fused_producer_multipass(cuda_device, name, group, widths, shared):
    """``dtp_group_forward`` past its cap, and ``dtp_linear_fwd`` (the same producer feeding the wgmma GEMM) at the
    same size: gathered node tables with the radial offset on per-edge weights, plain rows on shared weights."""
    from equiformer_b200 import ops
    plan = _plan(name)
    C, G = _group_forward_pass()
    E = _size(C, G, "partial_third_pass")
    _report(f"dtp_group_forward {name} group {group}", E, C)
    l3, _p, K = plan.out_groups[group]
    gen = torch.Generator(device=cuda_device).manual_seed(E + group + shared)
    rows = E if shared else E // 16
    xs = [_randn(gen, rows, 2 * l + 1, mul) for l, mul in plan.in1_blocks]
    y = _randn(gen, E, plan.d_y)
    if shared:
        w, off, gather = _randn(gen, plan.weight_numel), None, None
        x_at = lambda a, b: _rows(xs, a, b)
        w_at = lambda a, b: w.double()
    else:
        w, off = _randn(gen, E, plan.weight_numel), _randn(gen, plan.weight_numel)
        x2 = [_randn(gen, rows, 2 * l + 1, mul) for l, mul in plan.in1_blocks]
        src = torch.randint(0, rows, (E,), generator=gen, device=cuda_device)
        dst = torch.sort(torch.randint(0, rows, (E,), generator=gen, device=cuda_device)).values
        gather = (src, dst, x2)
        x_at = lambda a, b: [A.double()[src[a:b]] + B.double()[dst[a:b]] for A, B in zip(xs, x2)]
        w_at = lambda a, b: w[a:b].double() + off.double()
    Wts = [_randn(gen, K, N) / K ** 0.5 for N in widths]
    outs = [ops.dtp_group_forward_raw(plan, group, xs, y, w, gather=gather, w_offset=off)]
    outs += [ops.dtp_linear_fwd_raw(plan, group, xs, y, w, Wt, gather=gather, w_offset=off) for Wt in Wts]

    def ref(a, b):
        f = emu.dtp_forward_raw(plan, x_at(a, b), y[a:b].double(), w_at(a, b))[group]
        return [f] + [torch.einsum("eku,un->ekn", f, Wt.double()) for Wt in Wts]

    _compare_chunked(outs, ref, E, f"group {group} forward | linears {widths}", C)


# ------------------------------------------------------------------------------------------------ row kernels
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("C", [64, 48, 96, 256])      # 64: the half-warp fwd64 / bwd64 kernels; 2 / 4 / 8 columns per lane
def test_ln_silu_multipass(cuda_device, C, with_bias, size):
    """silu(LayerNorm(x + bias)) forward and backward past the row cap: gx and the parameter gradients, which are
    per-warp register sums over the passes, then per-CTA partial rows reduced by ``eqf_colsum``."""
    from equiformer_b200 import _lib, ops
    per_pass, G = _pointwise_pass(2 if C == 64 else 1)
    R = _size(per_pass, G, size)
    _report(f"ln_silu C={C}", R, per_pass)
    lib = _lib.load()
    assert lib.eqf_pointwise_rows(R) == _POINTWISE_CTAS                          # backward grid saturated
    assert lib.eqf_pointwise_rows((R + 1) // 2 if C == 64 else R) == _POINTWISE_CTAS   # forward grid saturated
    gen = torch.Generator(device=cuda_device).manual_seed(R + C + with_bias)
    x = _randn(gen, R, C) * 2 + 0.3
    gamma, beta = _randn(gen, C), _randn(gen, C)
    bias = _randn(gen, C) if with_bias else None
    gy = _randn(gen, R, C)
    assert x.data_ptr() % 16 == 0 and gy.data_ptr() % 16 == 0
    y, mean, rstd = ops.ln_silu_fwd_raw(x, gamma, beta, 1e-5, bias)
    ins = [t.double().requires_grad_(True) for t in (x, gamma, beta, *([bias] if with_bias else []))]
    ref = ops.ln_silu_torch(ins[0], ins[1], ins[2], 1e-5, ins[3] if with_bias else None)
    assert rel_err(y, ref) < TOL
    gx, gg, gb, gbias = ops.ln_silu_bwd_raw(x, gamma, beta, mean, rstd, gy, bias)
    rg = torch.autograd.grad(ref, ins, gy.double())
    for what, a, b in (("gx", gx, rg[0]), ("dgamma", gg, rg[1]), ("dbeta", gb, rg[2])):
        assert rel_err(a, b) < TOL_BWD, (what, rel_err(a, b))
    if with_bias:
        assert rel_err(gbias, rg[3]) < TOL_BWD, ("dbias", rel_err(gbias, rg[3]))


def _gate_layout(cfg):
    from equiformer_b200 import ops
    return ops.GateLayout(cfg["A0"], cfg["S"], cfg["H"], cfg["ds"], cfg["Cs"], 1.6791767923989418, 1.8467055342154763,
                          1.531320475574866, 0.2)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("cfg", GATE_LOGITS_CFGS)
def test_gate_logits_multipass(cuda_device, cfg, size):
    """bias + Gate + attention logits past the row cap (float4 and scalar kernels): the alpha_dot gradient is a per-warp
    sum over the passes (registers or shared atomics), then per-CTA partial rows; d bias = colsum of d t0."""
    from equiformer_b200 import _lib, ops
    lay = _gate_layout(cfg)
    C, G = _pointwise_pass()
    E = _size(C, G, size)
    _report(f"gate_logits A0={cfg['A0']} S={cfg['S']} H={cfg['H']}", E, C)
    assert _lib.load().eqf_pointwise_rows(E) == _POINTWISE_CTAS
    gen = torch.Generator(device=cuda_device).manual_seed(E + cfg["A0"] + cfg["S"])
    t0 = _randn(gen, E, lay.width)
    bias = _randn(gen, lay.width) * 0.3
    ad = _randn(gen, cfg["H"], cfg["A0"] // cfg["H"])
    gated = [_randn(gen, E, d_, c) for d_, c in zip(cfg["ds"], cfg["Cs"])]
    z, v0, vout = ops.gate_logits_fwd_raw(lay, t0, bias, ad, gated)
    ins = [t.double().requires_grad_(True) for t in (t0, bias, ad, *gated)]
    ref = ops.gate_logits_torch(lay, ins[0], ins[1], ins[2], *ins[3:])
    for k, (a, b) in enumerate(zip((z, v0, *vout), ref)):
        assert rel_err(a, b) < TOL, (k, rel_err(a, b))
    gouts = [_randn(gen, *r.shape) for r in ref]
    gt0, ggated, gdot = ops.gate_logits_bwd_raw(lay, t0, bias, ad, gated, gouts[0], gouts[1], gouts[2:])
    rg = torch.autograd.grad(ref, ins, [t.double() for t in gouts])
    assert rel_err(gt0, rg[0]) < TOL_BWD, ("dt0", rel_err(gt0, rg[0]))
    assert rel_err(ops.colsum_raw(gt0), rg[1]) < TOL_BWD, ("dbias", rel_err(ops.colsum_raw(gt0), rg[1]))
    assert rel_err(gdot.view_as(ad), rg[2]) < TOL_BWD, ("dalpha_dot", rel_err(gdot.view_as(ad), rg[2]))
    for a, b in zip(ggated, rg[3:]):
        assert rel_err(a, b) < TOL_BWD, ("dgated", rel_err(a, b))


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("cfg", GATE_ONLY_CFGS)
def test_gate_only_multipass(cuda_device, cfg, size):
    """Gate-only use of the fused gate kernel (FFN) through its autograd wrapper past the row cap."""
    from equiformer_b200 import ops
    lay = ops.GateLayout(0, cfg["S"], 1, cfg["ds"], cfg["Cs"], 1.6791767923989418, 1.8467055342154763, 1.0, 0.2)
    C, G = _pointwise_pass()
    N = _size(C, G, size)
    _report(f"gate_fused S={cfg['S']}", N, C)
    gen = torch.Generator(device=cuda_device).manual_seed(N + cfg["S"])
    t0 = _randn(gen, N, lay.width)
    bias = _randn(gen, lay.width) * 0.3
    gated = [_randn(gen, N, d_, c) for d_, c in zip(cfg["ds"], cfg["Cs"])]
    gouts = [_randn(gen, N, cfg["S"])] + [_randn(gen, *t.shape) for t in gated]
    leaves = [t.clone().requires_grad_(True) for t in (t0, bias, *gated)]
    outs = ops.gate_fused(lay, leaves[0], leaves[1], leaves[2:])
    ins = [t.double().requires_grad_(True) for t in (t0, bias, *gated)]
    _z, *ref = ops.gate_logits_torch(lay, ins[0], ins[1], None, *ins[2:])
    for a, b in zip(outs, ref):
        assert rel_err(a, b) < TOL
    grads = torch.autograd.grad(outs, leaves, gouts)
    rgrads = torch.autograd.grad(ref, ins, [t.double() for t in gouts])
    for k, (a, b) in enumerate(zip(grads, rgrads)):
        assert rel_err(a, b) < TOL_BWD, (k, rel_err(a, b))


# ------------------------------------------------------------------------------------------------ attention edge kernels
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("H,dims,chans", [(4, (1, 3, 5), (128, 64, 32)), (2, (1, 3), (6, 2))])   # float4 / scalar
def test_attn_edge_kernels_multipass(cuda_device, H, dims, chans, size):
    """``attn_edge_scale`` (gather, alpha, alpha x dropout mask) and ``attn_edge_dot`` past the edge-scale cap, against
    the fp64 statements of tests/_emulation.py."""
    from equiformer_b200 import ops
    lay = ops.HeadLayout(dims, chans, H)
    vec = all((d * c) % 4 == 0 and (c // H) % 4 == 0 for d, c in zip(dims, chans))
    C, G = _edge_scale_pass(vec, max(d * c for d, c in zip(dims, chans)))
    E = _size(C, G, size)
    _report(f"attn edge_scale {'float4' if vec else 'scalar'} H={H}", E, C)
    n_nodes = E // 20
    g = torch.Generator().manual_seed(E + H)
    dst = torch.sort(torch.randint(0, n_nodes, (E,), generator=g)).values
    src = torch.randint(0, n_nodes, (E,), generator=g)
    alpha = torch.rand(E, H, generator=g)
    keep = (torch.rand(E, H, generator=g) > 0.2).float() / 0.8
    Gs = [torch.randn(n_nodes, d, c, generator=g) for d, c in zip(dims, chans)]
    Vs = [torch.randn(E, d, c, generator=g) for d, c in zip(dims, chans)]
    dev = lambda t: t.to(cuda_device)
    graph = ops.Graph(dev(src), dev(dst), n_nodes)
    cpu_graph = type("G", (), {"dst": dst, "n_nodes": n_nodes, "n_edges": E})
    G64 = [t.double() for t in Gs]
    for what, al, kp, ref_alpha in (("gather", None, None, None), ("alpha", alpha, None, alpha.double()),
                                    ("alpha x keep", alpha, keep, alpha.double() * keep.double())):
        out = ops.attn_edge_scale_raw(lay, dev(al) if al is not None else None, [dev(t) for t in Gs], graph,
                                      keep=dev(kp) if kp is not None else None)
        for k, (a, b) in enumerate(zip(out, emu.attn_edge_scale_raw(lay, ref_alpha, G64, cpu_graph))):
            assert rel_err(a, b) < TOL, (what, k, rel_err(a, b))
        del out
    ga = ops.attn_edge_dot_raw(lay, [dev(v) for v in Vs], [dev(t) for t in Gs], graph)
    ref = emu.attn_edge_dot_raw(lay, [v.double() for v in Vs], G64, cpu_graph)
    assert rel_err(ga, ref) < TOL, rel_err(ga, ref)
