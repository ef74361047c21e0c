"""Equiformer at Lmax = 4: degree-4 harmonics, depth-wise products and forces on the sm_90a kernels.

CPU: the oracle's degree-4 harmonics (tests/oracle_l4.py) against the rotation matrices of the real Wigner 3j of
``o3/wigner.py``, their 'component' normalisation over the sphere and ``o3/sh.py``; the float64 oracle and the mirror (kernels
emulated in float64) against the reference's own model files at l = 4 (tests/golden/reference_model_l4_small.npz,
tests/golden/make_reference_golden_l4.py); the path table of a full ``0..4 x 0..4`` depth-wise product, which the
fused DTP -> linear kernel declines; degree-4 plans live in ``libeqf_b200_l4.so``, whose every kernel entry a GPU case
claims; an E(3) model at l = 4 still fails on the block limit.

-m gpu: the edge-geometry kernel at lmax 4 (forward, backward to positions) against float64 on short and axis-aligned
edges; every DTP entry point an l = 4 model reaches, under the launch audit's float64 bounds; the QM9 and MD17 l = 4
models against the fixture, eager and captured.
"""
from __future__ import annotations

import numpy as np
import pytest
import scipy.linalg
import torch

from oracle import e3nn_ref as e3
from oracle import equiformer_ref as R
from tests import oracle_l4
from tests.helpers import rel_err
from tests.reference_fixtures import load, mirror, oracle_config, run_mirror, run_oracle, worst_grad

FIXTURE = "reference_model_l4_small.npz"
SH4 = "1x0e+1x1e+1x2e+1x3e+1x4e"
FULL_IN1 = "32x0e+16x1e+16x2e+16x3e+16x4e"


@pytest.fixture
def oracle_at_l4():
    with oracle_l4.installed():
        yield


# ------------------------------------------------------------------------------------------------ oracle harmonics
def _generators(l: int) -> np.ndarray:
    """so(3) generators of degree l in e3nn's real basis, from the real Wigner 3j (l, 1, l) alone: ``G_a[i, j]``
    is proportional to ``w3j[i, a, j]``; the scale makes the Casimir ``sum_a G_a^2 = -l (l + 1)``, the sign makes
    ``[G_x, G_y]`` the same multiple of ``G_z`` as at l = 1, where ``exp(theta n . G)`` is checked to be the rotation."""
    from equiformer_b200.o3.wigner import wigner_3j_np
    w = wigner_3j_np(l, 1, l)
    G = np.stack([w[:, a, :] for a in range(3)])
    G *= np.sqrt(l * (l + 1) * (2 * l + 1) / -np.trace(sum(g @ g for g in G)))
    kappa = np.sum((G[0] @ G[1] - G[1] @ G[0]) * G[2]) / np.sum(G[2] * G[2])
    return G, kappa


def _wigner_D(l: int, axis: np.ndarray, angle: float) -> np.ndarray:
    G, kappa = _generators(l)
    G1, kappa1 = _generators(1)
    n = axis / np.linalg.norm(axis)
    sign1 = 1.0
    R = scipy.linalg.expm(angle * np.einsum("a,aij->ij", n, G1))
    K = np.array([[0, -n[2], n[1]], [n[2], 0, -n[0]], [-n[1], n[0], 0]])
    rot = scipy.linalg.expm(angle * K)                         # Rodrigues: rotation by `angle` about `n`
    if not np.allclose(R, rot, atol=1e-12):
        sign1 = -1.0
        assert np.allclose(scipy.linalg.expm(-angle * np.einsum("a,aij->ij", n, G1)), rot, atol=1e-12)
    sign = sign1 * np.sign(kappa * kappa1)                     # same structure constants as the l = 1 generators
    return scipy.linalg.expm(sign * angle * np.einsum("a,aij->ij", n, G)), rot


def test_oracle_degree4_harmonics_are_equivariant():
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(200, 3, generator=gen, dtype=torch.float64)
    for axis, angle in [(np.array([0.3, -1.2, 0.7]), 1.1), (np.array([1.0, 0.0, 0.0]), -2.4), (np.array([0.0, 1.0, 0.2]), 0.6)]:
        D, rot = _wigner_D(4, axis, angle)
        D1, _ = _wigner_D(1, axis, angle)
        assert np.allclose(D1, rot, atol=1e-12)
        with oracle_l4.installed():
            y = e3.spherical_harmonics([4], x, True, "component").numpy()
            y_rot = e3.spherical_harmonics([4], x @ torch.from_numpy(rot).T, True, "component").numpy()
        assert np.abs(y_rot - y @ D.T).max() < 1e-12


def test_oracle_degree4_harmonics_have_component_normalisation():
    """Sphere means by a quadrature exact for these degree-8 polynomials (Gauss-Legendre in the polar coordinate y, 20
    equal steps in the azimuth): every component has mean square 1 and the components are orthogonal, so the mean of
    |Y_4|^2 is 2l + 1 = 9."""
    t, wt = np.polynomial.legendre.leggauss(8)
    phi = 2 * np.pi * np.arange(20) / 20
    Y, P = np.meshgrid(t, phi, indexing="ij")
    s = np.sqrt(1 - Y ** 2)
    pts = torch.from_numpy(np.stack([s * np.sin(P), Y, s * np.cos(P)], -1).reshape(-1, 3))
    weights = torch.from_numpy(np.repeat(wt, 20) / (2 * 20))
    with oracle_l4.installed():
        y = e3.spherical_harmonics([4], pts, True, "component")
    gram = torch.einsum("n,ni,nj->ij", weights, y, y)
    assert float((gram - torch.eye(9, dtype=torch.float64)).abs().max()) < 1e-12
    assert abs(float(torch.einsum("n,ni,ni->", weights, y, y)) - 9.0) < 1e-12


def test_oracle_degree4_harmonics_equal_the_package_recurrence():
    from equiformer_b200.o3.sh import spherical_harmonics
    x = torch.randn(500, 3, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    with oracle_l4.installed():
        ref = e3.spherical_harmonics([0, 1, 2, 3, 4], x, True, "component")
    assert float((spherical_harmonics(SH4, x, True, "component") - ref).abs().max()) < 1e-12
    with pytest.raises(NotImplementedError):                 # outside the block the oracle stops at l = 3 as before
        e3.spherical_harmonics([4], x, True, "component")


# ------------------------------------------------------------------------------------------------ reference fixture
@pytest.mark.parametrize("kind", ["qm9", "md17"])
def test_oracle_matches_reference_l4_model_files(kind, oracle_at_l4):
    case = load(FIXTURE, kind)
    assert case.cfg["irreps_sh"] == SH4 and case.cfg["irreps_node_embedding"].endswith("4e")
    energy, forces, params = run_oracle(kind, case, oracle_config(kind, case.cfg))
    if forces is not None:
        assert rel_err(forces.detach(), case.t("forces")) < 1e-10
    assert rel_err(energy.detach(), case.t("energy")) < 1e-10
    assert worst_grad({k: v.grad for k, v in params.items()}, case.grads, 51) < 1e-10


def _mirror(kind, case):
    from equiformer_b200.nets.graph_attention_transformer import GraphAttentionTransformer
    from equiformer_b200.nets.graph_attention_transformer_md17 import GraphAttentionTransformerMD17
    return mirror({"qm9": GraphAttentionTransformer, "md17": GraphAttentionTransformerMD17}[kind], case.cfg, case.state)


@pytest.mark.parametrize("kind", ["qm9", "md17"])
def test_mirror_with_emulated_kernels_matches_reference_l4_model_files(kind):
    from tests._emulation import emulated_kernels
    case = load(FIXTURE, kind)
    model = _mirror(kind, case).double()
    with emulated_kernels():
        energy, forces = run_mirror(kind, model, case)
    assert rel_err(energy.detach(), case.t("energy")) < 1e-10
    if forces is not None:
        assert rel_err(forces.detach(), case.t("forces")) < 1e-10
    assert worst_grad({k: p.grad for k, p in model.named_parameters()}, case.grads, 51) < 1e-7


# ------------------------------------------------------------------------------------------------ plans and routes
def _full_plan():
    from equiformer_b200 import codegen
    return codegen.plan_for(FULL_IN1, SH4)


def test_full_degree4_depthwise_plan():
    """Every (l1, l2, l3) of ``0..4 x 0..4`` inside the triangle rule with l3 <= 4 is a path; the native plan accepts it
    and runs it on the table-walk kernels (no generated kernel, the float4 variant since every multiplicity is % 4)."""
    from equiformer_b200 import _lib, ops
    plan = _full_plan()
    want = sorted((l1, l2, l3) for l1 in range(5) for l2 in range(5) for l3 in range(abs(l1 - l2), min(l1 + l2, 4) + 1))
    assert sorted((p.l1, p.l2, p.l3) for p in plan.paths) == want
    assert [l for l, _p, _m in plan.out_groups] == [0, 1, 2, 3, 4]
    assert sum(1 for p in plan.paths if p.l3 == 2) == 16
    assert plan.max_degree == 4 and plan.lib is _lib.load_l4()
    info = plan.info()
    assert info["n_paths"] == len(want) and info["generated"] == 0 and info["vec_ok"] == 1
    # the fused DTP -> linear kernel holds one coupling row of <= 7 entries: degree-4 plans take the unfused route
    assert not ops.dtp_linear_supported(plan)


def test_degree4_plans_are_created_by_the_l4_library():
    """libeqf_b200.so refuses degree 4 as before; libeqf_b200_l4.so accepts it and refuses degree 5 (2l+1 = 11)."""
    import ctypes
    from equiformer_b200 import _lib
    h = ctypes.c_void_p()
    one = (ctypes.c_int32 * 1)
    cg = (ctypes.c_float * 121)()
    desc = (_lib.EqfPathDesc * 1)(_lib.EqfPathDesc(4, 0, 4, 8, 0, 0, 0, 0, 0, 0))
    main, l4 = _lib.load(), _lib.load_l4()
    assert main.eqf_plan_create(desc, 1, one(4), one(8), 1, one(4), one(8), 1, 1, 8, cg, 121, ctypes.byref(h)) == -3
    assert l4.eqf_plan_create(desc, 1, one(4), one(8), 1, one(4), one(8), 1, 1, 8, cg, 121, ctypes.byref(h)) == 0
    l4.eqf_plan_destroy(h)
    desc[0] = _lib.EqfPathDesc(5, 0, 5, 8, 0, 0, 0, 0, 0, 0)
    rc = l4.eqf_plan_create(desc, 1, one(5), one(8), 1, one(5), one(8), 1, 1, 8, cg, 121, ctypes.byref(h))
    assert rc == -3 and b"0..4" in l4.eqf_last_error()
    desc[0] = _lib.EqfPathDesc(1, 1, 3, 8, 0, 0, 0, 0, 0, 0)                       # (1,1,3) violates the triangle rule
    rc = l4.eqf_plan_create(desc, 1, one(1), one(8), 1, one(3), one(8), 1, 4, 8, cg, 121, ctypes.byref(h))
    assert rc < 0 and b"triangle" in l4.eqf_last_error()


# kernel entries of libeqf_b200_l4.so, each claimed by the GPU case that launches it (test_degree4_dtp_entry_points...)
L4_CLAIMS = {
    "vec": {"eqf::dtp_forward_vec_kernel<true>", "eqf::dtp_forward_vec_kernel<false>", "eqf::dtp_grad_x_vec_kernel<false>",
            "eqf::dtp_grad_x_vec_kernel<true>", "eqf::dtp_grad_w_kernel", "eqf::dtp_grad_y_kernel"},
    "scalar": {"eqf::dtp_forward_kernel", "eqf::dtp_grad_x_kernel<false>", "eqf::dtp_grad_x_kernel<true>",
               "eqf::dtp_grad_w_kernel", "eqf::dtp_grad_y_kernel"},
}
# multiplicities % 4 == 0 select the float4 kernels; 6 / 2 channels the scalar ones
PLANS = {"vec": FULL_IN1, "scalar": "6x0e+2x1e+2x2e+2x3e+2x4e"}


def test_l4_library_inventory_is_claimed():
    """Every kernel entry of the degree-4 library is claimed by a GPU case below, and every claim is in the binary."""
    from equiformer_b200 import _lib
    from tests.test_gpu_kernel_instances import inventory
    inv = inventory(_lib.L4_LIB_PATH)
    claimed = set().union(*L4_CLAIMS.values())
    assert inv == claimed, (sorted(inv - claimed), sorted(claimed - inv))


def test_lmax3_plans_keep_the_fused_route():
    from equiformer_b200 import codegen, ops
    assert ops.dtp_linear_supported(codegen.plan_for("32x0e+32x1e+32x2e+32x3e", "1x0e+1x1e+1x2e+1x3e"))


def test_e3_model_at_degree4_still_exceeds_the_block_limit():
    from equiformer_b200.nets.graph_attention_transformer import GraphAttentionTransformer
    irreps = "+".join(f"4x{l}{p}" for l in range(5) for p in "eo")
    with pytest.raises(NotImplementedError, match="exceeds kernel limits|too many"):
        GraphAttentionTransformer(irreps_in="5x0e", irreps_node_embedding=irreps, num_layers=1,
                                  irreps_sh="1x0e+1x1o+1x2e+1x3o+1x4e", irreps_feature="8x0e", irreps_head=irreps,
                                  num_heads=1, irreps_mlp_mid=irreps, fc_neurons=[8, 8], number_of_basis=8)


# ------------------------------------------------------------------------------------------------ GPU: edge geometry
@pytest.mark.gpu
def test_edge_geometry_kernel_at_lmax4(cuda_device):
    """Forward (vec, length, Y_0..Y_4) and the backward to positions against the float64 torch statement, on random,
    very short (1e-4 A) and axis-aligned edges (where the harmonics' polar terms are all zero or one)."""
    from equiformer_b200 import ops
    gen = torch.Generator().manual_seed(4)
    n = 40
    pos = torch.randn(n, 3, generator=gen) * 2.0
    pos[1] = pos[0] + torch.tensor([1e-4, -2e-4, 5e-5])
    pos[3] = pos[2] + torch.tensor([0.0, 1.3, 0.0])
    pos[5] = pos[4] + torch.tensor([-0.9, 0.0, 0.0])
    pos[7] = pos[6] + torch.tensor([0.0, 0.0, 2.1])
    src = torch.randint(0, n, (600,), generator=gen)
    dst = torch.randint(0, n, (600,), generator=gen)
    src = torch.cat([src, torch.tensor([1, 0, 3, 2, 5, 4, 7, 6])])
    dst = torch.cat([dst, torch.tensor([0, 1, 2, 3, 4, 5, 6, 7])])
    keep = src != dst
    src, dst = src[keep], dst[keep]
    order = torch.argsort(dst, stable=True)
    src, dst = src[order], dst[order]
    graph = ops.Graph(src.to(cuda_device), dst.to(cuda_device), n)
    p = pos.to(cuda_device).requires_grad_(True)
    vec, length, sh = ops.edge_geometry(p, graph, 4)
    assert sh.shape == (src.numel(), 25)
    p64 = pos.double().requires_grad_(True)
    rvec, rlen, rsh = ops.edge_geometry_torch(p64, graph.src.cpu(), graph.dst.cpu(), 4)
    assert rel_err(vec, rvec) < 1e-6 and rel_err(length, rlen) < 1e-6
    assert float((sh.detach().double().cpu() - rsh.detach()).abs().max()) < 2e-5 * 3
    g_sh = torch.randn(sh.shape, generator=gen)
    g_len = torch.randn(length.shape, generator=gen)
    (sh * g_sh.to(cuda_device)).sum().add((length * g_len.to(cuda_device)).sum()).backward()
    ((rsh * g_sh.double()).sum() + (rlen * g_len.double()).sum()).backward()
    assert rel_err(p.grad, p64.grad) < 5e-4


# ------------------------------------------------------------------------------------------------ GPU: DTP entry points
@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(PLANS))
def test_degree4_dtp_entry_points_under_the_launch_audit(cuda_device, monkeypatch, kind):
    """Per-edge and shared weights, the gathered forward and backward, grad_x, grad_w, grad_xw and grad_y of a full
    ``0..4 x 0..4`` plan: each call re-evaluated in float64 by the launch audit with its bounds unchanged, and the set of
    kernels launched equal to the claim of L4_CLAIMS."""
    from equiformer_b200 import codegen, ops
    from tests.test_gpu_kernel_instances import _launched
    from tests.test_gpu_launch_audit import Audit
    plan = codegen.plan_for(PLANS[kind], SH4)
    assert plan.info()["vec_ok"] == (kind == "vec")
    E, n = 3001, 211
    gen = torch.Generator(device=cuda_device).manual_seed(9)
    rnd = lambda *s: torch.randn(*s, generator=gen, device=cuda_device)
    xs = [rnd(E, 2 * l + 1, m) for l, m in plan.in1_blocks]
    As = [rnd(n, 2 * l + 1, m) for l, m in plan.in1_blocks]
    Bs = [rnd(n, 2 * l + 1, m) for l, m in plan.in1_blocks]
    gs = [rnd(E, 2 * l + 1, m) for l, _p, m in plan.out_groups]
    y = rnd(E, plan.d_y)
    w = rnd(E, plan.weight_numel)
    ws = rnd(plan.weight_numel)
    src = torch.randint(0, n, (E,), generator=gen, device=cuda_device)
    dst = torch.sort(torch.randint(0, n, (E,), generator=gen, device=cuda_device)).values

    def run(dev):
        for weights in (w, ws):
            ops.dtp_forward_raw(plan, xs, y, weights)
            ops.dtp_grad_x_raw(plan, gs, y, weights)
            ops.dtp_grad_w_raw(plan, xs, y, gs, weights.dim() == 1)
            ops.dtp_grad_xw_raw(plan, xs, y, weights, gs)
            ops.dtp_grad_y_raw(plan, xs, weights, gs, y)
        ops.dtp_forward_raw(plan, As, y, w, gather=(src, dst, Bs))
        ops.dtp_grad_xw_raw(plan, As, y, w, gs, gather=(src, dst, Bs))
        ops.dtp_forward_raw(plan, As, y, w, gather=(src, dst, None))

    audit = Audit(f"lmax4_dtp_{kind}")
    audit.install(monkeypatch)
    try:
        launched = _launched(run, cuda_device)
    finally:
        monkeypatch.undo()
    audit.report()
    assert not audit.unaudited, audit.unaudited
    assert not audit.failures, "\n".join(audit.failures[:20])
    assert audit.index >= 13
    # the shared-weight gradient's per-CTA partial rows are summed by the main library's column sum, as for every plan
    dtp = {k for k in launched if not k.startswith("eqf::colsum_kernel<")}
    assert launched - dtp and dtp == L4_CLAIMS[kind], (sorted(dtp - L4_CLAIMS[kind]), sorted(L4_CLAIMS[kind] - dtp))


# ------------------------------------------------------------------------------------------------ GPU: models
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["qm9", "md17"])
def test_cuda_l4_models_match_reference_model_files(cuda_device, kind):
    """The captured step (``GraphedForwardBackward`` for QM9, ``GraphedStep`` for MD17) against the fixture's loss, then
    the eager step: energy (and MD17 forces, through the double backward) and parameter gradients against the fixture,
    and the captured gradients against the eager ones.  The captured step runs first, as in the other capture tests."""
    from equiformer_b200 import ops
    from equiformer_b200.graphs import GraphedForwardBackward, GraphedStep
    from equiformer_b200.parallel import FlatGradAllReduce
    case = load(FIXTURE, kind)
    cfg = case.cfg
    model = _mirror(kind, case).to(cuda_device)
    assert not ops.dtp_linear_supported(model.blocks[0].ga.sep_act.dtp.tp.plan)
    pos, batch, z = case.t("pos", cuda_device), case.t("batch", cuda_device), case.t("z", cuda_device)
    bucket = FlatGradAllReduce(model.parameters())
    if kind == "qm9":
        gfb = GraphedForwardBackward(model, lambda out, tgt: ((out - tgt) ** 2).sum(), bucket, max_radius=cfg["max_radius"])
        target = torch.zeros(2, 1, device=cuda_device)
        for _ in range(2):
            loss = gfb(pos, batch, z, target).clone()
        assert gfb.captures == 1
    else:
        graph = ops.Graph(*R.radius_graph(pos, cfg["max_radius"], batch), pos.shape[0])

        def captured(pos, batch, z, src, dst, row_ptr):
            csr = ops.Graph.__new__(ops.Graph)
            csr.n_nodes, csr.n_edges, csr.perm = int(pos.shape[0]), int(src.numel()), None
            csr.src, csr.dst, csr.row_ptr = src, dst, row_ptr
            csr._src_perm = csr._src_row_ptr = None
            e, f = model.forward_edges(z, pos.detach().requires_grad_(True), batch, src, dst, graph=csr, n_graphs=1)
            return e.sum() + (f ** 2).sum()

        step = GraphedStep(captured, bucket)
        for _ in range(2):
            loss = step((int(pos.shape[0]), graph.n_edges), [pos, batch, z, graph.src, graph.dst, graph.row_ptr]).clone()
        assert step.captures == 1
    captured_grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
    energy_ref = case.t("energy")
    ref_loss = ((energy_ref ** 2).sum() if kind == "qm9" else energy_ref.sum() + (case.t("forces") ** 2).sum())
    assert abs(float(loss) - float(ref_loss)) <= 1e-4 * abs(float(ref_loss))
    assert worst_grad(captured_grads, case.grads, 51) < 1e-3

    bucket.zero_grad()
    energy, forces = run_mirror(kind, model, case, cuda_device, torch.float32)
    assert rel_err(energy, case.t("energy")) < 1e-4
    if forces is not None:
        assert rel_err(forces, case.t("forces")) < 1e-4
    assert worst_grad({k: p.grad for k, p in model.named_parameters()}, case.grads, 51) < 1e-3
    worst = max((rel_err(p.grad, captured_grads[k]), k) for k, p in model.named_parameters() if k in captured_grads)
    assert worst[0] < 1e-4, worst
