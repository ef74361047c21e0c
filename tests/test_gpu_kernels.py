"""-m gpu: every sm_90a kernel against the fp64 oracle (and the table-walking emulation) on seeded inputs.

Tolerance: fp32 kernels vs fp64 oracle, max-abs error relative to the output's max magnitude <= 2e-5 for a single
kernel (north_star: 1e-4 relative end to end).
"""
from __future__ import annotations

import pytest
import torch

from tests import _emulation as emu
from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
TOL = 2e-5

CONFIGS = {
    "qm9_l2": ("128x0e+64x1e+32x2e", "1x0e+1x1e+1x2e", "128x0e+64x1e+32x2e"),
    "md17_l3": ("128x0e+64x1e+64x2e+32x3e", "1x0e+1x1e+1x2e+1x3e", "128x0e+64x1e+64x2e+32x3e"),
    "oc20_l1": ("256x0e+128x1e", "1x0e+1x1e", "256x0e+128x1e"),
    "odd_mul": ("20x0e+12x1e+4x2e", "1x0e+1x1e+1x2e", "20x0e+12x1e+4x2e"),
    "e3_parity": ("32x0e+8x0o+8x1e+8x1o+4x2e+4x2o", "1x0e+1x1o+1x2e", "32x0e+8x0o+8x1e+8x1o+4x2e+4x2o"),
}


def _dtp(name):
    from equiformer_b200.nets.graph_attention_transformer import DepthwiseTensorProduct
    a, b, c = CONFIGS[name]
    return DepthwiseTensorProduct(a, b, c, internal_weights=False, bias=False)


def _inputs(plan, E, shared, seed=0, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(E, 2 * l + 1, mul, generator=g, dtype=dtype) for l, mul in plan.in1_blocks]
    y = torch.randn(E, plan.d_y, generator=g, dtype=dtype)
    w = torch.randn((plan.weight_numel,) if shared else (E, plan.weight_numel), generator=g, dtype=dtype)
    gs = [torch.randn(E, 2 * l + 1, mul, generator=g, dtype=dtype) for l, _p, mul in plan.out_groups]
    return xs, y, w, gs


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("E", [1, 37, 1000])
def test_dtp_family_vs_emulation(cuda_device, name, shared, E):
    """forward / grad_x / grad_w / grad_y / grad_xw kernels == fp64 table walk (ragged tile: E not a multiple of 8)."""
    from equiformer_b200 import ops
    plan = _dtp(name).tp.plan
    xs, y, w, gs = _inputs(plan, E, shared)
    f = lambda t: t.float().to(cuda_device)
    xs_d, y_d, w_d, gs_d = [f(t) for t in xs], f(y), f(w), [f(t) for t in gs]
    # references are computed from the fp32-rounded inputs, in fp64
    r = lambda t: t.float().double()
    xs_r, y_r, w_r, gs_r = [r(t) for t in xs], r(y), r(w), [r(t) for t in gs]

    out = ops.dtp_forward_raw(plan, xs_d, y_d, w_d)
    ref = emu.dtp_forward_raw(plan, xs_r, y_r, w_r)
    for a, b in zip(out, ref):
        assert rel_err(a, b) < TOL
    gx = ops.dtp_grad_x_raw(plan, gs_d, y_d, w_d)
    for a, b in zip(gx, emu.dtp_grad_x_raw(plan, gs_r, y_r, w_r)):
        assert rel_err(a, b) < TOL
    gw = ops.dtp_grad_w_raw(plan, xs_d, y_d, gs_d, shared)
    assert rel_err(gw, emu.dtp_grad_w_raw(plan, xs_r, y_r, gs_r, shared)) < TOL
    gy = ops.dtp_grad_y_raw(plan, xs_d, w_d, gs_d, y_d)
    assert rel_err(gy, emu.dtp_grad_y_raw(plan, xs_r, w_r, gs_r, y_r)) < TOL
    gx2, gw2 = ops.dtp_grad_xw_raw(plan, xs_d, y_d, w_d, gs_d)
    for a, b in zip(gx2, gx):
        assert rel_err(a, b) < TOL
    assert rel_err(gw2, gw) < TOL


@pytest.mark.parametrize("name", ["qm9_l2", "md17_l3", "oc20_l1"])
def test_dtp_e3nn_layout_vs_oracle(cuda_device, name):
    """TensorProductRescale.forward(x, y, weight) in e3nn layout == oracle per-instruction einsum (ref tensor_product_rescale.py:139-141)."""
    from oracle import e3nn_ref as e3
    from oracle import equiformer_ref as R
    dtp = _dtp(name)
    a, b, c = CONFIGS[name]
    E = 257
    g = torch.Generator().manual_seed(1)
    x = torch.randn(E, dtp.irreps_in1.dim, generator=g)
    y = torch.randn(E, dtp.irreps_in2.dim, generator=g)
    w = torch.randn(E, dtp.tp.weight_numel, generator=g)
    out = dtp.to(cuda_device)(x.to(cuda_device), y.to(cuda_device), w.to(cuda_device))
    irr_out, ins = R.dtp_instructions(e3.parse_irreps(a), e3.parse_irreps(b), e3.parse_irreps(c))
    ref = e3.tensor_product(x.double(), y.double(), w.double(), e3.parse_irreps(a), e3.parse_irreps(b), irr_out, ins, False)
    assert str(dtp.irreps_out) == "+".join(f"{m}x{l}{'e' if p == 1 else 'o'}" for m, l, p in irr_out)
    assert rel_err(out, ref) < TOL


def test_dtp_empty_and_errors(cuda_device):
    from equiformer_b200 import _lib, ops
    plan = _dtp("qm9_l2").tp.plan
    xs, y, w, gs = _inputs(plan, 0, False, dtype=torch.float32)
    out = ops.dtp_forward_raw(plan, [t.to(cuda_device) for t in xs], y.to(cuda_device), w.to(cuda_device))
    assert [tuple(o.shape) for o in out] == [(0, 1, 224), (0, 3, 384), (0, 5, 352)]
    xs, y, w, gs = _inputs(plan, 4, False, dtype=torch.float32)
    with pytest.raises(_lib.EqfError):  # CPU tensors must fail loudly - no fallback
        ops.dtp_forward_raw(plan, xs, y, w)
    with pytest.raises(ValueError):
        ops.dtp_forward_raw(plan, [t.to(cuda_device) for t in xs[:-1]], y.to(cuda_device), w.to(cuda_device))


def _graph(n_nodes, E, seed, device, with_empty=True):
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(seed)
    dst = torch.randint(0, n_nodes, (E,), generator=g)
    if with_empty and n_nodes > 2:
        dst[dst == 1] = 0  # node 1 has no incoming edge
    dst = torch.sort(dst).values
    src = torch.randint(0, n_nodes, (E,), generator=g)
    return ops.Graph(src.to(device), dst.to(device), n_nodes), src, dst


@pytest.mark.parametrize("H,dims,chans", [(4, (1, 3, 5), (128, 64, 32)), (8, (1, 3), (256, 128)), (1, (1, 3, 5), (20, 12, 4)),
                                          (4, (1, 3, 5, 7), (128, 64, 64, 32)), (2, (1, 3), (6, 2))])   # last: scalar kernels
def test_attention_family(cuda_device, H, dims, chans):
    """seg_softmax (PyG semantics, :508), aggregate (:512-513), edge_dot, edge_scale vs fp64 torch on ragged segments."""
    from equiformer_b200 import ops
    from oracle import equiformer_ref as R
    n_nodes, E = 61, 700
    graph, src, dst = _graph(n_nodes, E, 5, cuda_device)
    g = torch.Generator().manual_seed(7)
    z = torch.randn(E, H, generator=g) * 3
    Vs = [torch.randn(E, d, c, generator=g) for d, c in zip(dims, chans)]
    Gs = [torch.randn(n_nodes, d, c, generator=g) for d, c in zip(dims, chans)]
    lay = ops.HeadLayout(dims, chans, H)
    dev = lambda t: t.to(cuda_device)

    alpha = ops.seg_softmax_raw(dev(z), graph)
    alpha_ref = R.pyg_softmax(z.double(), dst, n_nodes)
    assert rel_err(alpha, alpha_ref) < TOL
    sums = torch.zeros(n_nodes, H, dtype=torch.float64).index_add_(0, dst, alpha.double().cpu())
    has = torch.bincount(dst, minlength=n_nodes) > 0
    assert torch.allclose(sums[has], torch.ones_like(sums[has]), atol=1e-5) and (sums[~has] == 0).all()

    cpu_graph = type("G", (), {"dst": dst, "n_nodes": n_nodes, "n_edges": E})
    a64 = alpha_ref
    out = ops.attn_aggregate_raw(lay, dev(a64.float()), [dev(v) for v in Vs], graph)
    ref = emu.attn_aggregate_raw(lay, a64.float().double(), [v.double() for v in Vs], cpu_graph)
    for a, b in zip(out, ref):
        assert rel_err(a, b) < TOL
    out = ops.attn_aggregate_raw(lay, None, [dev(v) for v in Vs], graph)       # plain segment sum
    for a, b in zip(out, emu.attn_aggregate_raw(lay, None, [v.double() for v in Vs], cpu_graph)):
        assert rel_err(a, b) < TOL
    ga = ops.attn_edge_dot_raw(lay, [dev(v) for v in Vs], [dev(t) for t in Gs], graph)
    assert rel_err(ga, emu.attn_edge_dot_raw(lay, [v.double() for v in Vs], [t.double() for t in Gs], cpu_graph)) < TOL
    sc = ops.attn_edge_scale_raw(lay, dev(a64.float()), [dev(t) for t in Gs], graph)
    for a, b in zip(sc, emu.attn_edge_scale_raw(lay, a64.float().double(), [t.double() for t in Gs], cpu_graph)):
        assert rel_err(a, b) < TOL
    # K2: softmax + aggregation in one kernel == the two-kernel result, and its autograd == the unfused composition
    if ops.softmax_aggregate_ok(lay, dev(z)):
        outs, alpha2 = ops.softmax_aggregate_raw(lay, dev(z), [dev(v) for v in Vs], graph)
        assert rel_err(alpha2, alpha_ref) < TOL
        for a, b in zip(outs, emu.attn_aggregate_raw(lay, a64, [v.double() for v in Vs], cpu_graph)):
            assert rel_err(a, b) < TOL
        zz = dev(z).requires_grad_(True)
        vv = [dev(v).requires_grad_(True) for v in Vs]
        cots = [dev(t) for t in Gs]
        g1 = torch.autograd.grad(ops.SoftmaxAggregate.apply(lay, graph, zz, *vv), [zz, *vv], cots)
        g2 = torch.autograd.grad(ops.AttnAggregate.apply(lay, graph, ops.SegSoftmax.apply(zz, graph), *vv), [zz, *vv], cots)
        for a, b in zip(g1, g2):
            assert rel_err(a, b) < 1e-5


def test_unsorted_edges_are_sorted_once(cuda_device):
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(0)
    dst = torch.randint(0, 9, (50,), generator=g)
    src = torch.randint(0, 9, (50,), generator=g)
    graph = ops.Graph(src.to(cuda_device), dst.to(cuda_device), 9)
    assert graph.perm is not None and bool((graph.dst[1:] >= graph.dst[:-1]).all())
    assert graph.row_ptr[-1].item() == 50


@pytest.mark.parametrize("M,N,K", [(36000, 352, 224), (108000, 64, 384), (180000, 32, 352), (2304, 128, 128), (36000, 960, 64),
                                   (1001 * 4, 480, 352), (12, 8, 4)])
def test_fast_fp32_gemm_all_layouts(cuda_device, M, N, K, monkeypatch):
    """Fast-fp32 GEMM entry point (gemm_raw) vs fp64 matmul: forward, data-grad and weight-grad layouts."""
    from equiformer_b200 import ops
    monkeypatch.setenv("EQF_GEMM_FORCE", "1")   # exercise the 3xTF32 kernels for every layout / size, not just the policy's picks
    g = torch.Generator().manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g)
    B = torch.randn(K, N, generator=g)
    dC = torch.randn(M, N, generator=g)
    d = lambda t: t.to(cuda_device)
    # fp32-level accuracy (fp32 accumulation error grows ~sqrt(reduction length)); single-pass TF32 would be ~1e-3
    tol = lambda red: 2e-6 * max(1.0, (red / 256) ** 0.5)
    assert rel_err(ops.gemm_raw(0, d(A), d(B)), A.double() @ B.double()) < tol(K)
    assert rel_err(ops.gemm_raw(1, d(dC), d(B)), dC.double() @ B.double().t()) < tol(N)   # dA = dC B^T
    assert rel_err(ops.gemm_raw(2, d(A), d(dC)), A.double().t() @ dC.double()) < tol(M)   # dB = A^T dC
    # strided A (a channel slice of a wider planar buffer, as sep_alpha reads the DTP output)
    wide = torch.randn(M, K + 8, generator=g)
    view = d(wide)[:, 4:4 + K]
    assert rel_err(ops.gemm_raw(0, view, d(B)), wide[:, 4:4 + K].double() @ B.double()) < tol(K)


@pytest.mark.parametrize("M,N,K", [(100, 16, 32), (1000, 48, 64), (3001, 72, 100), (36000, 224, 224), (36000, 352, 224),
                                   (36000, 960, 64), (108000, 384, 64), (33000, 128, 960), (129, 256, 16), (128, 272, 36)])
def test_tf32x3_tcgen05_gemm(cuda_device, M, N, K):
    """Hand-written wgmma 3xTF32 GEMM C = A Bt^T vs fp64: ragged rows, K tails, single and multiple column tiles,
    strided A.  Accuracy: a few 1e-6 of max|C| at K ~ 224, far from single-pass TF32's 1e-3."""
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g)
    Bt = torch.randn(N, K, generator=g)
    d = lambda t: t.to(cuda_device)
    tol = 6e-6 * max(1.0, (K / 256) ** 0.5)
    ref = A.double() @ Bt.double().t()
    out = ops.gemm_tf32x3_raw(d(A), d(Bt))
    assert out.shape == (M, N) and rel_err(out, ref) < tol
    wide = torch.randn(M, K + 8, generator=g)
    out = ops.gemm_tf32x3_raw(d(wide)[:, 4:4 + K], d(Bt))
    assert rel_err(out, wide[:, 4:4 + K].double() @ Bt.double().t()) < tol
    # exactly representable inputs (small integers) must give the exact product
    Ai = torch.randint(-8, 9, (M, K), generator=g).float()
    Bi = torch.randint(-8, 9, (N, K), generator=g).float()
    assert torch.equal(ops.gemm_tf32x3_raw(d(Ai), d(Bi)).cpu(), Ai @ Bi.t())
    # weight given as B[K, N] (forward layout): transposed while it is split
    assert rel_err(ops.gemm_tf32x3_raw(d(A), d(Bt).t().contiguous(), b_is_kn=True), ref) < tol


@pytest.mark.parametrize("R,K1,N", [(100, 32, 32), (1000, 64, 48), (3001, 100, 72), (36000, 224, 224), (36000, 224, 352),
                                    (36000, 64, 960), (2324, 128, 128), (11620, 32, 32), (108000, 384, 64), (17, 260, 40)])
@pytest.mark.parametrize("deterministic", ["1", "0"])
def test_tf32x3_tcgen05_weight_gradient(cuda_device, R, K1, N, deterministic, monkeypatch):
    """Hand-written wgmma 3xTF32 weight gradient W = A^T G (MN-major operands, per-slice register accumulators) vs fp64.
    The tensor-core accumulation truncates, so the error grows with the rows per slice (~1e-5 at 2 000 rows); single-pass
    TF32 would be 1e-3.  ``deterministic`` picks the reduction route every check of the case runs on: "1" per-slice
    partials + fixed-order column sum (bitwise reproducible), "0" atomic adds into W."""
    from equiformer_b200 import ops
    monkeypatch.setattr(ops, "_DETERMINISTIC", deterministic == "1")
    g = torch.Generator().manual_seed(R + K1 + N)
    A = torch.randn(R, K1, generator=g)
    G = torch.randn(R, N, generator=g)
    d = lambda t: t.to(cuda_device)
    out0 = ops.gemm_tf32x3_wgrad_raw(d(A), d(G))
    assert out0.shape == (K1, N) and rel_err(out0, A.double().t() @ G.double()) < 4e-5
    wide = torch.randn(R, K1 + 8, generator=g)
    out = ops.gemm_tf32x3_wgrad_raw(d(wide)[:, 4:4 + K1], d(G))
    assert rel_err(out, wide[:, 4:4 + K1].double().t() @ G.double()) < 4e-5
    Ai = torch.randint(-4, 5, (R, K1), generator=g).float()
    Gi = torch.randint(-4, 5, (R, N), generator=g).float()
    assert torch.equal(ops.gemm_tf32x3_wgrad_raw(d(Ai), d(Gi)).cpu(), Ai.t() @ Gi)
    if deterministic == "1":       # the fixed summation order gives the same bits on every call
        assert torch.equal(ops.gemm_tf32x3_wgrad_raw(d(A), d(G)), out0)


def test_gemm_autograd_closure(cuda_device):
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(0)
    A = torch.randn(64, 32, generator=g).to(cuda_device).requires_grad_(True)
    B = torch.randn(32, 16, generator=g).to(cuda_device).requires_grad_(True)
    out = ops.matmul_f32(A, B)
    (gA,) = torch.autograd.grad(out.pow(2).sum(), A, create_graph=True)
    gA.pow(2).sum().backward()
    A2 = A.detach().double().requires_grad_(True)
    B2 = B.detach().double().requires_grad_(True)
    (gA2,) = torch.autograd.grad((A2 @ B2).pow(2).sum(), A2, create_graph=True)
    gA2.pow(2).sum().backward()
    assert rel_err(A.grad, A2.grad) < 1e-5 and rel_err(B.grad, B2.grad) < 1e-5


def test_aggregate_hub_degrees(cuda_device):
    """Segment sums with in-/out-degrees 0, 1, 31, 32, 33 and 70, with and without weights and through the CSC
    permutation: pins the unrolled edge loop of the aggregation kernel at its even / odd / long-segment cases."""
    from equiformer_b200 import ops
    degrees = [0, 1, 31, 32, 33, 70, 3, 0, 5]
    n_nodes, H = len(degrees), 4
    dst = torch.repeat_interleave(torch.arange(n_nodes), torch.tensor(degrees))
    E = dst.numel()
    g = torch.Generator().manual_seed(5)
    hub_src = torch.repeat_interleave(torch.arange(n_nodes), torch.tensor(degrees[::-1]))[torch.randperm(E, generator=g)]
    dims, chans = (1, 3, 5), (128, 64, 32)
    lay = ops.HeadLayout(dims, chans, H)
    graph = ops.Graph(hub_src.to(cuda_device), dst.to(cuda_device), n_nodes)
    cpu_graph = type("G", (), {"dst": dst, "n_nodes": n_nodes, "n_edges": E})
    Vs = [torch.randn(E, d, c, generator=g) for d, c in zip(dims, chans)]
    alpha = torch.rand(E, H, generator=g)
    dev = lambda t: t.to(cuda_device)
    for al in (alpha, None):
        out = ops.attn_aggregate_raw(lay, None if al is None else dev(al), [dev(v) for v in Vs], graph)
        ref = emu.attn_aggregate_raw(lay, None if al is None else al.double(), [v.double() for v in Vs], cpu_graph)
        for a, b in zip(out, ref):
            assert rel_err(a, b) < TOL
    by_src = ops.attn_aggregate_raw(lay, None, [dev(v) for v in Vs], graph, by_src=True)     # through the CSC permutation
    for a, v in zip(by_src, Vs):
        exp = torch.zeros(n_nodes, *v.shape[1:], dtype=torch.float64).index_add_(0, hub_src, v.double())
        assert rel_err(a, exp) < TOL


@pytest.mark.parametrize("with_b", [True, False])
def test_dtp_gather_fused_and_csc_aggregate(cuda_device, with_b):
    """x = A[src] (+ B[dst]) gathered inside the kernels (ref :487 folded into :491) and the CSC segment sum."""
    from equiformer_b200 import ops
    plan = _dtp("qm9_l2").tp.plan
    n_nodes, E = 53, 611
    graph, src, dst = _graph(n_nodes, E, 11, cuda_device)
    g = torch.Generator().manual_seed(3)
    As = [torch.randn(n_nodes, 2 * l + 1, m, generator=g) for l, m in plan.in1_blocks]
    Bs = [torch.randn(n_nodes, 2 * l + 1, m, generator=g) for l, m in plan.in1_blocks] if with_b else None
    y = torch.randn(E, plan.d_y, generator=g)
    w = torch.randn(E, plan.weight_numel, generator=g)
    gs = [torch.randn(E, 2 * l + 1, m, generator=g) for l, _p, m in plan.out_groups]
    d = lambda t: t.to(cuda_device)
    dB = [d(t) for t in Bs] if with_b else None
    xs64 = [a.double()[src] + (b.double()[dst] if with_b else 0) for a, b in zip(As, Bs or As)]
    out = ops.dtp_forward_raw(plan, [d(t) for t in As], d(y), d(w), gather=(graph.src, graph.dst, dB))
    for a, b in zip(out, emu.dtp_forward_raw(plan, xs64, y.double(), w.double())):
        assert rel_err(a, b) < TOL
    gx, gw = ops.dtp_grad_xw_raw(plan, [d(t) for t in As], d(y), d(w), [d(t) for t in gs], gather=(graph.src, graph.dst, dB))
    gx_ref = emu.dtp_grad_x_raw(plan, [t.double() for t in gs], y.double(), w.double())
    for a, b in zip(gx, gx_ref):
        assert rel_err(a, b) < TOL
    assert rel_err(gw, emu.dtp_grad_w_raw(plan, xs64, y.double(), [t.double() for t in gs], False)) < TOL
    lay = ops.HeadLayout([2 * l + 1 for l, _ in plan.in1_blocks], [m for _, m in plan.in1_blocks], 1)
    by_src = ops.attn_aggregate_raw(lay, None, gx, graph, by_src=True)
    for a, ref in zip(by_src, gx_ref):
        exp = torch.zeros(n_nodes, *ref.shape[1:], dtype=torch.float64).index_add_(0, src, ref)
        assert rel_err(a, exp) < TOL


@pytest.mark.parametrize("cfg", ["qm9_l2", "md17_l3"])
def test_dtp_weight_offset_fused(cuda_device, cfg):
    """w[e] + offset added inside the generated kernels' weight load (radial offset, ref radial_func.py:45-49):
    forward and grad_xw vs the fp64 statement on w + offset; the autograd wrapper returns colsum(gw) for the offset."""
    from equiformer_b200 import ops
    plan = _dtp(cfg).tp.plan
    if not plan.generated:
        pytest.skip("no plan-specialised kernels for this configuration")
    n_nodes, E = 41, 523
    graph, src, dst = _graph(n_nodes, E, 5, cuda_device)
    g = torch.Generator().manual_seed(9)
    As = [torch.randn(n_nodes, 2 * l + 1, m, generator=g) for l, m in plan.in1_blocks]
    Bs = [torch.randn(n_nodes, 2 * l + 1, m, generator=g) for l, m in plan.in1_blocks]
    y = torch.randn(E, plan.d_y, generator=g)
    w = torch.randn(E, plan.weight_numel, generator=g)
    off = torch.randn(plan.weight_numel, generator=g)
    gs = [torch.randn(E, 2 * l + 1, m, generator=g) for l, _p, m in plan.out_groups]
    d = lambda t: t.to(cuda_device)
    xs64 = [a.double()[src] + b.double()[dst] for a, b in zip(As, Bs)]
    w64 = w.double() + off.double()
    gather = (graph.src, graph.dst, [d(t) for t in Bs])
    out = ops.dtp_forward_raw(plan, [d(t) for t in As], d(y), d(w), gather=gather, w_offset=d(off))
    for a, b in zip(out, emu.dtp_forward_raw(plan, xs64, y.double(), w64)):
        assert rel_err(a, b) < TOL
    gx, gw = ops.dtp_grad_xw_raw(plan, [d(t) for t in As], d(y), d(w), [d(t) for t in gs], gather=gather, w_offset=d(off))
    for a, b in zip(gx, emu.dtp_grad_x_raw(plan, [t.double() for t in gs], y.double(), w64)):
        assert rel_err(a, b) < TOL
    gw_ref = emu.dtp_grad_w_raw(plan, xs64, y.double(), [t.double() for t in gs], False)
    assert rel_err(gw, gw_ref) < TOL
    # autograd wrapper
    leaves = [d(t).requires_grad_(True) for t in (w, off, *As, *Bs)]
    outs = ops.depthwise_tensor_product_gathered(plan, graph, leaves[2:2 + len(As)], leaves[2 + len(As):], d(y), leaves[0], leaves[1])
    grads = torch.autograd.grad(outs, leaves, [d(t) for t in gs])
    assert rel_err(grads[0], gw_ref) < TOL and rel_err(grads[1], gw_ref.sum(0)) < 1e-5


@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("R,C", [(1, 64), (1000, 64), (4097, 96), (33, 256)])
def test_ln_silu_fused(cuda_device, R, C, with_bias):
    """silu(LayerNorm(x + bias)) forward and (gx, dgamma, dbeta, dbias) backward vs fp64 torch (RadialProfile hidden
    layers: the Linear's bias rides along in the LayerNorm kernel)."""
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(R + C)
    x = torch.randn(R, C, generator=g) * 2 + 0.3
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    bias = torch.randn(C, generator=g) if with_bias else None
    gy = torch.randn(R, C, generator=g)
    d = lambda t: t.to(cuda_device)
    db = d(bias) if with_bias else None
    y, mean, rstd = ops.ln_silu_fwd_raw(d(x), d(gamma), d(beta), 1e-5, db)
    xs = [t.double().requires_grad_(True) for t in (x, gamma, beta)]
    b64 = bias.double().requires_grad_(True) if with_bias else None
    ref = ops.ln_silu_torch(xs[0], xs[1], xs[2], 1e-5, b64)
    assert rel_err(y, ref) < TOL
    gx, gg, gb, gbias = ops.ln_silu_bwd_raw(d(x), d(gamma), d(beta), mean, rstd, d(gy), db)
    rx, rg, rb, *rest = torch.autograd.grad(ref, xs + ([b64] if with_bias else []), gy.double())
    assert rel_err(gx, rx) < 5e-5 and rel_err(gg, rg) < 5e-5 and rel_err(gb, rb) < 5e-5
    if with_bias:
        assert rel_err(gbias, rest[0]) < 5e-5
        # autograd wrapper
        leaves = [d(t).requires_grad_(True) for t in (x, bias, gamma, beta)]
        out = ops.ln_silu(leaves[0], leaves[2], leaves[3], 1e-5, bias=leaves[1])
        ax, abias, ag, ab = torch.autograd.grad(out, leaves, d(gy))
        assert rel_err(ax, rx) < 5e-5 and rel_err(abias, rest[0]) < 5e-5 and rel_err(ag, rg) < 5e-5 and rel_err(ab, rb) < 5e-5
    else:
        assert gbias is None


@pytest.mark.parametrize("rows,cols", [(1, 1), (7, 3), (32560, 64), (32560, 352), (32560, 960), (1184, 64), (197, 24576),
                                       (2324, 130), (100000, 5), (3, 86016)])
def test_colsum(cuda_device, rows, cols):
    """Column sums (bias / offset gradients, reduction of kernel partials) vs fp64, contiguous and row-strided input;
    repeated calls share the self-resetting tile counters."""
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(rows + cols)
    x = torch.randn(rows, cols, generator=g) + 0.1
    ref = x.double().sum(0)
    scale = ref.abs().max().clamp_min(1.0)
    for _ in range(3):
        out = ops.colsum_raw(x.to(cuda_device))
        assert ((out.cpu().double() - ref).abs().max() / scale) < 2e-6
    wide = torch.randn(rows, cols + 12, generator=g).to(cuda_device)
    view = wide[:, 4:4 + cols]
    out = ops.colsum_raw(view)
    ref = view.cpu().double().sum(0)
    assert ((out.cpu().double() - ref).abs().max() / ref.abs().max().clamp_min(1.0)) < 2e-6


def test_add_bias_autograd(cuda_device):
    from equiformer_b200 import ops
    x = torch.randn(5000, 3, 96, device=cuda_device, requires_grad=True)
    b = torch.randn(96, device=cuda_device, requires_grad=True)
    g = torch.randn(5000, 3, 96, device=cuda_device)
    gx, gb = torch.autograd.grad(ops.add_bias(x, b), (x, b), g)
    assert torch.equal(gx, g)
    assert rel_err(gb, g.double().sum((0, 1))) < 1e-6
    # second order: d/dg of <colsum(g), v> is v broadcast
    gg = g.clone().requires_grad_(True)
    (gb2,) = torch.autograd.grad(ops.add_bias(x, b), (b,), gg, create_graph=True)
    v = torch.randn(96, device=cuda_device)
    (back,) = torch.autograd.grad((gb2 * v).sum(), gg)
    assert torch.allclose(back, v.expand_as(back))


@pytest.mark.parametrize("entries", [[(128, 1, True), (64, 3, False), (32, 5, False)],
                                     [(128, 1, True), (64, 3, False), (64, 5, False), (32, 7, False)],
                                     [(256, 1, True), (128, 3, False)],
                                     [(8, 1, True), (8, 1, False), (5, 3, False)]])
@pytest.mark.parametrize("N", [1, 1461, 5000])
def test_equivariant_layer_norm_fused(cuda_device, entries, N):
    """EquivariantLayerNormV2 ('component', affine; ref nets/layer_norm.py:104-152) fused fwd / bwd vs fp64 torch."""
    from equiformer_b200 import ops
    lay = ops.NormLayout(entries, 1e-5)
    g = torch.Generator().manual_seed(N)
    x = torch.randn(N, lay.dim, generator=g) * 1.5 + 0.2
    w, b = torch.randn(lay.n_w, generator=g), torch.randn(lay.n_b, generator=g)
    gy = torch.randn(N, lay.dim, generator=g)
    d = lambda t: t.to(cuda_device)
    y, rstd = ops.eln_fwd_raw(lay, d(x), d(w), d(b))
    xs = [t.double().requires_grad_(True) for t in (x, w, b)]
    ref = ops.eln_torch(lay, *xs)
    assert rel_err(y, ref) < TOL
    gx, gw, gb = ops.eln_bwd_raw(lay, d(x), d(w), rstd, d(gy))
    rx, rw, rb = torch.autograd.grad(ref, xs, gy.double())
    assert rel_err(gx, rx) < 5e-5 and rel_err(gw, rw) < 5e-5 and rel_err(gb, rb) < 5e-5
    # through the module, autograd wiring included
    xd, wd, bd = (d(t).requires_grad_(True) for t in (x, w, b))
    out = ops.equivariant_layer_norm(lay, xd, wd, bd)
    ax, aw, ab = torch.autograd.grad(out, (xd, wd, bd), d(gy))
    assert rel_err(ax, rx) < 5e-5 and rel_err(aw, rw) < 5e-5 and rel_err(ab, rb) < 5e-5


@pytest.mark.parametrize("entries", [[(128, 1, True), (64, 3, False), (32, 5, False)], [(8, 1, True), (8, 1, False), (5, 3, False)]])
@pytest.mark.parametrize("N", [1, 2324])
def test_equivariant_layer_norm_planar(cuda_device, entries, N):
    """The planar variant (one packed [N, 2l+1, mul] block per entry) agrees with the e3nn-layout statement in fp64."""
    from equiformer_b200 import ops
    lay = ops.NormLayout(entries, 1e-5)
    g = torch.Generator().manual_seed(N + len(entries))
    xs = [torch.randn(N, d, m, generator=g) * 1.5 + 0.2 for m, d, _ in entries]
    gys = [torch.randn(N, d, m, generator=g) for m, d, _ in entries]
    w, b = torch.randn(lay.n_w, generator=g), torch.randn(lay.n_b, generator=g)
    d_ = lambda t: t.to(cuda_device)
    leaves64 = [t.double().requires_grad_(True) for t in (w, b, *xs)]
    ref = ops.eln_planar_torch(lay, leaves64[2:], leaves64[0], leaves64[1])
    rgrads = torch.autograd.grad(ref, leaves64, [t.double() for t in gys])
    leaves = [d_(t).requires_grad_(True) for t in (w, b, *xs)]
    out = ops.equivariant_layer_norm_planar(lay, leaves[2:], leaves[0], leaves[1])
    for a, r in zip(out, ref):
        assert rel_err(a, r) < TOL
    grads = torch.autograd.grad(out, leaves, [d_(t) for t in gys])
    for a, r in zip(grads, rgrads):
        assert rel_err(a, r) < 5e-5


@pytest.mark.parametrize("cfg", [dict(A0=128, S=128, H=4, ds=(3, 5), Cs=(64, 32)), dict(A0=256, S=256, H=8, ds=(3,), Cs=(128,)),
                                 dict(A0=128, S=128, H=4, ds=(3, 5, 7), Cs=(64, 64, 32)),
                                 dict(A0=16, S=16, H=4, ds=(3, 5), Cs=(8, 4)),       # tiny heads: one lane per head
                                 dict(A0=64, S=20, H=4, ds=(3,), Cs=(6,))])          # falls back to the scalar kernels
def test_gate_logits_fused(cuda_device, cfg):
    """bias + Gate + attention logits in one kernel (ref :492-495, :506-507) vs the fp64 torch statement, fwd and bwd."""
    from equiformer_b200 import ops
    lay = ops.GateLayout(cfg["A0"], cfg["S"], cfg["H"], cfg["ds"], cfg["Cs"], 1.6791767923989418, 1.8467055342154763,
                         1.531320475574866, 0.2)
    E = 777
    g = torch.Generator().manual_seed(1)
    t0 = torch.randn(E, lay.width, generator=g)
    bias = torch.randn(lay.width, generator=g) * 0.3
    ad = torch.randn(cfg["H"], cfg["A0"] // cfg["H"], generator=g)
    gated = [torch.randn(E, d_, c, generator=g) for d_, c in zip(cfg["ds"], cfg["Cs"])]
    d = lambda t: t.to(cuda_device)
    z, v0, vout = ops.gate_logits_fwd_raw(lay, d(t0), d(bias), d(ad), [d(t) for t in gated])
    ins = [t.double().requires_grad_(True) for t in (t0, bias, ad, *gated)]
    ref = ops.gate_logits_torch(lay, ins[0], ins[1], ins[2], *ins[3:])
    for a, b in zip((z, v0, *vout), ref):
        assert rel_err(a, b) < TOL
    gouts = [torch.randn(r.shape, generator=g) for r in ref]
    gt0, ggated, gdot = ops.gate_logits_bwd_raw(lay, d(t0), d(bias), d(ad), [d(t) for t in gated], d(gouts[0]), d(gouts[1]),
                                                [d(t) for t in gouts[2:]])
    rg = torch.autograd.grad(ref, ins, [t.double() for t in gouts])
    assert rel_err(gt0, rg[0]) < 5e-5 and rel_err(gt0.sum(0), rg[1]) < 5e-5
    assert rel_err(gdot.view_as(ad), rg[2]) < 5e-5
    for a, b in zip(ggated, rg[3:]):
        assert rel_err(a, b) < 5e-5


@pytest.mark.parametrize("cfg", [dict(S=384, ds=(3, 5), Cs=(192, 96)), dict(S=20, ds=(3,), Cs=(6,))])   # vec / scalar kernels
def test_gate_only_fused(cuda_device, cfg):
    """Gate-only use of the fused kernel (FFN: bias + SiLU on scalars + sigmoid gates on the rest, ref :128-154)."""
    from equiformer_b200 import ops
    lay = ops.GateLayout(0, cfg["S"], 1, cfg["ds"], cfg["Cs"], 1.6791767923989418, 1.8467055342154763, 1.0, 0.2)
    N = 2324
    g = torch.Generator().manual_seed(2)
    t0 = torch.randn(N, lay.width, generator=g)
    bias = torch.randn(lay.width, generator=g) * 0.3
    gated = [torch.randn(N, d_, c, generator=g) for d_, c in zip(cfg["ds"], cfg["Cs"])]
    gouts = [torch.randn(N, cfg["S"], generator=g)] + [torch.randn_like(t) for t in gated]
    d = lambda t: t.to(cuda_device)
    leaves = [d(t).requires_grad_(True) for t in (t0, bias, *gated)]
    outs = ops.gate_fused(lay, leaves[0], leaves[1], leaves[2:])
    ins = [t.double().requires_grad_(True) for t in (t0, bias, *gated)]
    _z, *ref = ops.gate_logits_torch(lay, ins[0], ins[1], None, *ins[2:])
    for a, b in zip(outs, ref):
        assert rel_err(a, b) < TOL
    grads = torch.autograd.grad(outs, leaves, [d(t) for t in gouts])
    rgrads = torch.autograd.grad(ref, ins, [t.double() for t in gouts])
    for a, b in zip(grads, rgrads):
        assert rel_err(a, b) < 5e-5


@pytest.mark.parametrize("n_graphs,cap,loop", [(1, 1000, False), (7, 1000, False), (7, 5, False), (3, 1000, True), (40, 12, False)])
def test_radius_graph_kernels_match_torch_statement(cuda_device, n_graphs, cap, loop):
    """Neighbour list (count / fill kernels) == the torch brute force, bit for bit: same edges, same order, same CSR."""
    from equiformer_b200.graph import radius_graph, radius_graph_csr, radius_graph_torch
    g = torch.Generator().manual_seed(n_graphs * 31 + cap)
    sizes = torch.randint(1, 30, (n_graphs,), generator=g)
    batch = torch.repeat_interleave(torch.arange(n_graphs), sizes)
    pos = torch.rand(int(sizes.sum()), 3, generator=g) * 4.0
    pos[0] = pos[-1] if n_graphs == 1 else pos[0]            # a coincident pair (d = 0) when both are in one graph
    p, b = pos.to(cuda_device), batch.to(cuda_device)
    for bb in (b, None):
        ref = radius_graph_torch(p, 2.5, bb, max_num_neighbors=cap, loop=loop)
        out, row_ptr = radius_graph_csr(p, 2.5, bb, max_num_neighbors=cap, loop=loop)
        assert torch.equal(out, ref)
        assert torch.equal(radius_graph(p, 2.5, bb, max_num_neighbors=cap, loop=loop), ref)
        counts = torch.bincount(ref[1], minlength=p.shape[0])
        assert torch.equal(row_ptr[1:], torch.cumsum(counts, 0)) and int(row_ptr[0]) == 0
    empty = radius_graph(p[:1], 2.5, None, max_num_neighbors=cap, loop=False)
    assert empty.shape == (2, 0)


@pytest.mark.parametrize("E", [1, 777, 32560])
def test_gaussian_rbf_fused(cuda_device, E):
    """GaussianRadialBasisLayer (ref nets/gaussian_rbf.py:5-40) fused forward / backward vs the fp64 torch statement."""
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(E)
    dist = torch.rand(E, generator=g) * 5.0
    mean = torch.rand(1, 128, generator=g)
    std = (torch.rand(1, 128, generator=g) * 0.99 + 0.01) * torch.where(torch.rand(1, 128, generator=g) < 0.1, -1.0, 1.0)
    weight, bias = torch.tensor([[1.3]]), torch.tensor([[-0.05]])
    gout = torch.randn(E, 128, generator=g)
    d = lambda t: t.to(cuda_device)
    leaves = [d(t).requires_grad_(True) for t in (dist, mean, std, weight, bias)]
    out = ops.gaussian_rbf(*leaves, 5.0)
    ins = [t.double().requires_grad_(True) for t in (dist, mean, std, weight, bias)]
    ref = ops.gaussian_rbf_torch(*ins, 5.0)
    assert rel_err(out, ref) < 2e-6
    grads = torch.autograd.grad(out, leaves, d(gout))
    rgrads = torch.autograd.grad(ref, ins, gout.double())
    for a, b in zip(grads, rgrads):
        assert rel_err(a, b) < 5e-5


def test_segment_softmax_backward_fused(cuda_device):
    """First-order backward of the segment softmax (one kernel) vs autograd through an fp64 per-segment softmax."""
    from equiformer_b200 import ops
    n_nodes, E, H = 37, 500, 4
    graph, src, dst = _graph(n_nodes, E, 21, cuda_device)
    g = torch.Generator().manual_seed(5)
    z = torch.randn(E, H, generator=g)
    ga = torch.randn(E, H, generator=g)
    zd = z.to(cuda_device).requires_grad_(True)
    alpha = ops.segment_softmax(zd, graph)
    (gz,) = torch.autograd.grad(alpha, zd, ga.to(cuda_device))
    z64 = z.double().requires_grad_(True)
    out = torch.zeros(E, H, dtype=torch.float64)
    for t in range(n_nodes):
        m = dst == t
        if m.any():
            out = out + torch.zeros(E, H, dtype=torch.float64).masked_scatter(m[:, None].expand(E, H), torch.softmax(z64[m], dim=0))
    (ref,) = torch.autograd.grad(out, z64, ga.double())
    assert rel_err(alpha, out) < TOL and rel_err(gz, ref) < 5e-5


# ------------------------------------------------------------------------------------------------ K1: fused DTP -> linear
FUSED_CASES = [("qm9_l2", False, True, 32560), ("qm9_l2", True, False, 32560), ("qm9_l2", False, True, 1000),
               ("qm9_l2", True, False, 37), ("qm9_l2", False, False, 1), ("md17_l3", False, True, 1700),
               ("md17_l3", True, False, 345), ("oc20_l1", False, True, 20011), ("oc20_l1", True, False, 4097)]


@pytest.mark.parametrize("name,shared,gather,E", FUSED_CASES)
def test_fused_dtp_linear_forward_vs_fp64(cuda_device, name, shared, gather, E):
    """``eqf_dtp_linear_fwd`` (tensor product produced on chip as the register A operand of the wgmma 3xTF32 GEMM) against
    the fp64 table walk followed by an fp64 matmul, every output group; output widths as the model uses them (wide 0e
    group in column tiles, 64 / 32 columns) plus one odd width; gathered per-edge weights with the radial offset folded
    in, and shared weights on per-edge blocks."""
    from equiformer_b200 import ops
    plan = _dtp(name).tp.plan
    assert ops.dtp_linear_supported(plan)
    g = torch.Generator().manual_seed(E + 7)
    n_nodes = max(E // 14, 2)
    rows = n_nodes if gather else E
    xs = [torch.randn(rows, 2 * l + 1, mul, generator=g) for l, mul in plan.in1_blocks]
    x2 = [torch.randn(rows, 2 * l + 1, mul, generator=g) for l, mul in plan.in1_blocks] if gather else None
    y = torch.randn(E, plan.d_y, generator=g)
    w = torch.randn((plan.weight_numel,) if shared else (E, plan.weight_numel), generator=g)
    off = None if shared else torch.randn(plan.weight_numel, generator=g)
    dst = torch.sort(torch.randint(0, n_nodes, (E,), generator=g)).values
    src = torch.randint(0, n_nodes, (E,), generator=g)
    widths = {0: [352, 128], 1: [64, 48], 2: [32], 3: [32]}
    f = lambda t: t.to(cuda_device)
    xs_d, y_d, w_d = [f(t) for t in xs], f(y), f(w)
    gat_d = (f(src), f(dst), [f(t) for t in x2]) if gather else None
    gat_r = (src, dst, [t.double() for t in x2]) if gather else None
    ref_f = emu.dtp_forward_raw(plan, [t.double() for t in xs], y.double(), w.double(), gat_r,
                                off.double() if off is not None else None)
    for gi, (l, _p, K) in enumerate(plan.out_groups):
        fg = ops.dtp_group_forward_raw(plan, gi, xs_d, y_d, w_d, gather=gat_d, w_offset=f(off) if off is not None else None)
        assert rel_err(fg, ref_f[gi]) < TOL, gi                 # the same producer writing one group to HBM
        for N in widths[l]:
            Wt = torch.randn(K, N, generator=g) / K ** 0.5
            out = ops.dtp_linear_fwd_raw(plan, gi, xs_d, y_d, w_d, f(Wt), gather=gat_d,
                                         w_offset=f(off) if off is not None else None)
            ref = torch.einsum("eku,un->ekn", ref_f[gi], Wt.double())
            assert out.shape == ref.shape
            assert rel_err(out, ref) < TOL, (gi, N, rel_err(out, ref))


def test_fused_dtp_linear_autograd_matches_unfused(cuda_device):
    """``ops.DtpLinear`` (forward fused, backward = recompute + GEMMs + DTP backward) against the unfused differentiable
    composition on the same inputs: outputs and every gradient (node tables, radial weights, offset, linear weights)."""
    from equiformer_b200 import ops
    plan = _dtp("qm9_l2").tp.plan
    E, n_nodes = 20000, 1500
    g = torch.Generator().manual_seed(3)
    dev = cuda_device
    dst = torch.sort(torch.randint(0, n_nodes, (E,), generator=g)).values.to(dev)
    src = torch.randint(0, n_nodes, (E,), generator=g).to(dev)
    graph = ops.Graph(src, dst, n_nodes)
    mk = lambda *s: torch.randn(*s, generator=g).to(dev).requires_grad_(True)
    As = [mk(n_nodes, 2 * l + 1, m) for l, m in plan.in1_blocks]
    Bs = [mk(n_nodes, 2 * l + 1, m) for l, m in plan.in1_blocks]
    y = torch.randn(E, plan.d_y, generator=g).to(dev)
    w, off = mk(E, plan.weight_numel), mk(plan.weight_numel)
    Ws = [(torch.randn(K, N, generator=g) / K ** 0.5).to(dev).requires_grad_(True)
          for (_l, _p, K), N in zip(plan.out_groups, (352, 64, 32))]
    cots = [torch.randn(E, 2 * l + 1, N, generator=g).to(dev) for (l, _p, _K), N in zip(plan.out_groups, (352, 64, 32))]
    leaves = [*As, *Bs, w, off, *Ws]
    outs = ops.dtp_linear(plan, graph, As, Bs, y, w, off, Ws)
    grads = torch.autograd.grad(outs, leaves, cots)
    ref_outs = ops._dtp_linear_unfused(plan, graph, len(Bs), y, w, off, (*As, *Bs), Ws)
    ref_grads = torch.autograd.grad(ref_outs, leaves, cots)
    for a, b in zip(outs, ref_outs):
        assert rel_err(a, b) < TOL
    for a, b in zip(grads, ref_grads):
        assert rel_err(a, b) < 5e-5


# ------------------------------------------------------------------------------------------------ edge-feature producers
@pytest.mark.parametrize("lmax", [1, 2, 3])
@pytest.mark.parametrize("with_offsets", [False, True])
def test_edge_geometry_kernel_vs_torch_statement(cuda_device, lmax, with_offsets):
    """``ops.EdgeGeometry`` (edge vector, length, harmonics up to l = 3 in one kernel; backward kernel + two segment sums to
    the positions) against the fp64 torch chain it replaces (ref :866-870), values and the gradient w.r.t. ``pos``."""
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(11 + lmax)
    n, E = 300, 4000
    pos = torch.randn(n, 3, generator=g) * 2.0
    dst = torch.sort(torch.randint(0, n, (E,), generator=g)).values
    src = torch.randint(0, n, (E,), generator=g)
    src = torch.where(src == dst, (src + 1) % n, src)
    off = torch.randn(E, 3, generator=g) * 0.3 if with_offsets else None
    graph = ops.Graph(src.to(cuda_device), dst.to(cuda_device), n)
    p = pos.to(cuda_device).requires_grad_(True)
    vec, length, sh = ops.edge_geometry(p, graph, lmax, off.to(cuda_device) if off is not None else None)
    p64 = pos.double().requires_grad_(True)
    rvec, rlen, rsh = ops.edge_geometry_torch(p64, src, dst, lmax, off.double() if off is not None else None)
    assert rel_err(vec, rvec) < 1e-6 and rel_err(length, rlen) < 1e-6 and rel_err(sh, rsh) < 5e-6
    cs, cl = torch.randn(E, (lmax + 1) ** 2, generator=g), torch.randn(E, generator=g)
    (gp,) = torch.autograd.grad([sh, length], [p], [cs.to(cuda_device), cl.to(cuda_device)])
    (rp,) = torch.autograd.grad([rsh, rlen], [p64], [cs.double(), cl.double()])
    assert rel_err(gp, rp) < 2e-5


def test_expnorm_rbf_kernel_vs_torch_statement(cuda_device):
    """``ops.ExpNormalRbf`` (ref nets/expnorm_rbf.py:73-78 with the cosine cutoff) values and d/d dist vs fp64 torch, and the
    module against the reference-run fixture's parameters."""
    from equiformer_b200 import ops
    from equiformer_b200.nets.expnorm_rbf import ExpNormalSmearing
    mod = ExpNormalSmearing(0.0, 5.0, 32, trainable=False)
    g = torch.Generator().manual_seed(3)
    d = torch.rand(5000, generator=g) * 6.0              # some beyond the cutoff
    dd = d.to(cuda_device).requires_grad_(True)
    out = ops.expnorm_rbf(dd, mod.means.to(cuda_device), mod.betas.to(cuda_device), mod.alpha, 5.0)
    d64 = d.double().requires_grad_(True)
    ref = ops.expnorm_torch(d64, mod.means.double(), mod.betas.double(), mod.alpha, 5.0)
    assert rel_err(out, ref) < 2e-6
    cot = torch.randn(5000, 32, generator=g)
    (gd,) = torch.autograd.grad(out, dd, cot.to(cuda_device))
    (rd,) = torch.autograd.grad(ref, d64, cot.double())
    assert rel_err(gd, rd) < 1e-5
    assert rel_err(mod.to(cuda_device)(d.to(cuda_device)), ref) < 2e-6


# ------------------------------------------------------------------------------------------------ grouped small products
def test_grouped_gemm_three_modes_vs_fp64(cuda_device):
    """``eqf_gemm_grouped``: the three operand layouts (forward, data gradient, split-reduction weight gradient) in one
    launch, ragged row counts, outputs narrower than a tile, reductions that are not multiples of the k-chunk."""
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(5)
    dev = cuda_device
    r = lambda *s: torch.randn(*s, generator=g)
    cases = [(0, r(2324 * 3, 64), r(64, 64), 0.5, False), (0, r(1001, 100), r(100, 32), 1.0, False),
             (1, r(2324 * 5, 32), r(36, 32), 0.25, False), (1, r(130, 128), r(128, 128), 1.0, False),
             (2, r(6972, 64), r(6972, 64), 2.0, True), (2, r(300, 128), r(300, 36), 1.0, True),
             (2, r(11620, 32), r(11620, 32), 1.0, True), (0, r(7, 4), r(4, 4), 1.0, False)]
    probs, refs = [], []
    for mode, A, B, alpha, acc in cases:
        Ad, Bd = A.double(), B.double()
        ref = alpha * (Ad @ Bd if mode == 0 else Ad @ Bd.t() if mode == 1 else Ad.t() @ Bd)
        C = torch.zeros(ref.shape, device=dev) if acc else torch.full(ref.shape, float("nan"), device=dev)
        probs.append((mode, A.to(dev), B.to(dev), C, alpha, acc))
        refs.append(ref)
    ops.grouped_gemm_raw(probs)
    for (mode, _A, _B, C, _a, _acc), ref in zip(probs, refs):
        assert rel_err(C, ref) < TOL, (mode, tuple(C.shape), rel_err(C, ref))


def test_planar_linear_grouped_matches_per_path_products(cuda_device, monkeypatch):
    """``LinearRS.planar`` through the grouped launch (forward, first-order gradients in one launch, the ``create_graph``
    family for the MD17 forces) against the per-degree products it replaces: outputs, gradients, second-order gradients."""
    from equiformer_b200 import ops
    from equiformer_b200.nets.tensor_product_rescale import LinearRS
    torch.manual_seed(0)
    lin = LinearRS("128x0e+64x1e+32x2e", "64x0e+64x1e+16x2e", bias=True).to(cuda_device)
    R = 777
    g = torch.Generator().manual_seed(1)
    xs0 = [torch.randn(R, 2 * l + 1, m, generator=g).to(cuda_device) for l, m in ((0, 128), (1, 64), (2, 32))]
    cots = [torch.randn(R, 2 * l + 1, m, generator=g).to(cuda_device) for l, m in ((0, 64), (1, 64), (2, 16))]

    def run(grouped):
        monkeypatch.setattr(ops, "_GROUPED", grouped)
        prof = ops.KernelProfile(time_events=False)
        xs = [x.clone().requires_grad_(True) for x in xs0]
        monkeypatch.setattr(ops, "PROFILE", prof)
        outs = lin.planar(xs)
        grads = torch.autograd.grad(outs, [*xs, lin.tp.weight], cots, create_graph=True)
        # a scalar of the first-order gradients, differentiated again (the shape of the MD17 force loss)
        s = sum((gr * gr).sum() for gr in grads)
        second = torch.autograd.grad(s, [*xs, lin.tp.weight])
        plain = torch.autograd.grad(lin.planar(xs), [*xs, lin.tp.weight], cots)      # first-order backward: one launch
        monkeypatch.setattr(ops, "PROFILE", None)
        return outs, [*grads, *plain], second, prof.launches

    o1, g1, s1, n1 = run(True)
    o0, g0, s0, _n0 = run(False)
    for a, b in zip([*o1, *g1, *s1], [*o0, *g0, *s0]):
        assert rel_err(a, b) < 5e-5, rel_err(a, b)
    assert n1 >= 3            # grouped launches were counted (forward, data gradients, weight gradients, second order)
