"""The spherical Bessel radial basis and the Bessel-basis configurations.

CPU: the torch statement (``ops.bessel_rbf_torch``) against scipy's spherical Bessel function j0 and the orthonormality of
the un-enveloped basis; the module, the oracle (tests/oracle_bessel.py) and the host mirrors of a small QM9 and a small
MD17 model against the reference's own model files run with the restated ocpmodels ``RadialBasis``
(tests/golden/make_reference_golden_bessel.py);
state-dict and no-weight-decay tables of the six registered Bessel configurations; ``BesselRbf`` gradcheck /
gradgradcheck through emulated kernel launches.

-m gpu: ``eqf_bessel_fwd / _bwd`` against float64 over basis sizes, edge counts and past the grid cap; the three GEMM
products of the stacked K = 8 first layer of the radial MLPs; the CUDA models against the fixture, eager and captured;
one captured QM9 training step against the eager step.
"""
from __future__ import annotations

import contextlib
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import equiformer_ref as R
from tests import oracle_bessel as OB
from tests.helpers import rel_err
from tests.reference_fixtures import GOLDEN, load, mirror, oracle_config, run_mirror, worst_grad

FIXTURE = "reference_model_bessel_small.npz"
SHAPES = os.path.join(GOLDEN, "reference_state_shapes_bessel.json")
TOL = 2e-5          # kernel vs fp64
TOL_FREQ = 5e-5     # frequency gradient: a sum over all edges
_POINTWISE_CTAS = 132 * 8   # eqf_pointwise.cu pointwise_grid: min(ceil(E / 8), 132 * 8) CTAs of 8 warps, one edge per warp


def _part(prefix):
    case = load(FIXTURE, prefix)
    assert "rbf.rbf.frequencies" in case.grads
    return case


def _envelope(x):
    return np.where(x < 1, 1 - 21 * x ** 5 + 35 * x ** 6 - 15 * x ** 7, 0.0)


# ------------------------------------------------------------------------------------------------ scipy anchors (CPU)

def test_torch_statement_is_the_enveloped_spherical_bessel_j0():
    """sqrt(2/c^3) sin(f x) / x = sqrt(2/c^3) f j0(f x): the torch statement against scipy's j0, independent of the
    restatement of ocpmodels the fixtures use; 128 functions so the argument reaches 128 pi."""
    from scipy.special import spherical_jn
    from equiformer_b200 import ops
    c = 5.0
    d = np.linspace(0.01, 5.5, 301)
    f = math.pi * np.arange(1, 129) + np.linspace(-0.2, 0.3, 128)
    x = d / c
    ref = _envelope(x)[:, None] * math.sqrt(2 / c ** 3) * f[None, :] * spherical_jn(0, f[None, :] * x[:, None])
    out = ops.bessel_rbf_torch(torch.from_numpy(d), torch.from_numpy(f), c)
    assert rel_err(out, torch.from_numpy(ref)) < 1e-12
    assert torch.all(out[d >= c] == 0)


def test_unenveloped_basis_is_orthonormal():
    """With f_k = pi k the functions sqrt(2/c^3) sin(f_k r/c) / (r/c) are orthonormal under int_0^c . r^2 dr."""
    from scipy.integrate import quad
    from scipy.special import spherical_jn
    c = 5.0
    phi = lambda k, r: math.sqrt(2 / c ** 3) * math.pi * k * spherical_jn(0, math.pi * k * r / c)
    for k in range(1, 9):
        for l in range(k, 9):
            val, _ = quad(lambda r: phi(k, r) * phi(l, r) * r * r, 0.0, c, limit=200)
            assert abs(val - (1.0 if k == l else 0.0)) < 1e-10, (k, l, val)


def test_zero_distance_gives_nan_as_the_reference():
    from equiformer_b200 import ops
    out = ops.bessel_rbf_torch(torch.tensor([0.0, 1.0], dtype=torch.float64), torch.tensor([math.pi, 2 * math.pi], dtype=torch.float64), 5.0)
    assert torch.isnan(out[0]).all() and torch.isfinite(out[1]).all()


# ------------------------------------------------------------------------------------------------ fixture (CPU)

def test_module_matches_reference_restatement():
    from equiformer_b200.nets.bessel_rbf import RadialBasis
    case = load(FIXTURE, "module")
    m = RadialBasis(128, 5.0, rbf={"name": "spherical_bessel"})
    assert [k for k, _ in m.named_parameters()] == ["rbf.frequencies"]
    assert torch.equal(m.rbf.frequencies.detach(), torch.tensor(np.pi * np.arange(1, 129, dtype=np.float32)))
    m.load_state_dict(case.state)
    out = m.double()(case.t("dist", dtype=torch.float64))
    assert rel_err(out, case.t("y")) < 1e-12
    p = {"m.rbf.frequencies": case.state["rbf.frequencies"].double()}
    assert rel_err(OB.bessel_rbf(p, "m", case.t("dist", dtype=torch.float64), 5.0), case.t("y")) < 1e-12


def test_oracle_qm9_bessel_model_matches_reference():
    p = _part("qm9")
    params = {k: v.double().requires_grad_(True) if v.is_floating_point() else v for k, v in p.state.items()}
    pos, batch, z = p.t("pos", dtype=torch.float64), p.t("batch"), p.t("z")
    ocfg = oracle_config("qm9", p.cfg, basis_type="bessel")
    energy = OB.model_forward_bessel(params, ocfg, pos, batch, z, n_graphs=2)
    assert rel_err(energy.detach(), p.t("energy")) < 1e-11
    (energy ** 2).sum().backward()
    assert worst_grad({k: v.grad for k, v in params.items()}, p.grads, 80) < 1e-8


def test_oracle_md17_bessel_model_matches_reference():
    p = _part("md17")
    params = {k: v.double().requires_grad_(True) if v.is_floating_point() else v for k, v in p.state.items()}
    pos, batch, z = p.t("pos", dtype=torch.float64), p.t("batch"), p.t("z")
    ocfg = oracle_config("md17", p.cfg, basis_type="bessel")
    e, f = OB.energy_and_forces_bessel(params, ocfg, pos, batch, z, 1, create_graph=True)
    assert rel_err(e.detach(), p.t("energy")) < 1e-11
    assert rel_err(f.detach(), p.t("forces")) < 1e-10
    (e.sum() + (f ** 2).sum()).backward()
    assert worst_grad({k: v.grad for k, v in params.items()}, p.grads, 80) < 1e-8


def _bessel_fwd_emulated(dist, freq, cutoff):
    from equiformer_b200 import ops
    return ops.bessel_rbf_torch(dist, freq, cutoff)


def _bessel_bwd_emulated(dist, freq, cutoff, g, need_dist):
    from equiformer_b200 import ops
    ins = [t.detach().requires_grad_(True) for t in (dist, freq)]
    with torch.enable_grad():
        out = ops.bessel_rbf_torch(ins[0], ins[1], cutoff)
    gd, gf = torch.autograd.grad(out, ins, g)
    return (gd if need_dist else None), gf


@contextlib.contextmanager
def _emulated():
    """tests/_emulation.py's stand-ins plus the two Bessel launches (restated in torch, as the others are)."""
    from equiformer_b200 import ops
    from tests._emulation import emulated_kernels
    saved = ops.bessel_fwd_raw, ops.bessel_bwd_raw
    try:
        ops.bessel_fwd_raw, ops.bessel_bwd_raw = _bessel_fwd_emulated, _bessel_bwd_emulated
        with emulated_kernels():
            yield
    finally:
        ops.bessel_fwd_raw, ops.bessel_bwd_raw = saved


def test_bessel_rbf_gradcheck_through_emulated_launch():
    """First order through the backward launch (grad mode off inside it), second order through the torch statement."""
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(5)
    d = (0.3 + 5.0 * torch.rand(13, generator=g, dtype=torch.float64)).requires_grad_(True)
    f = (math.pi * torch.arange(1, 9, dtype=torch.float64) + 0.1 * torch.randn(8, generator=g, dtype=torch.float64)).requires_grad_(True)
    with _emulated():
        fn = lambda dd, ff: ops.BesselRbf.apply(dd, ff, 5.0)
        assert torch.autograd.gradcheck(fn, (d, f))
        assert torch.autograd.gradgradcheck(fn, (d, f))
        out = ops.bessel_rbf(d, f, 5.0)
        assert out.grad_fn is not None and "BesselRbf" in type(out.grad_fn).__name__


def test_mirror_models_match_reference_on_host():
    """The mirrors' own wiring with the kernel launches emulated in float64: QM9 energies + gradients of sum(E^2); MD17
    energy, forces and gradients of the energy + force loss."""
    from equiformer_b200.nets.graph_attention_transformer import GraphAttentionTransformer
    from equiformer_b200.nets.graph_attention_transformer_md17 import GraphAttentionTransformerMD17
    p = _part("qm9")
    model = mirror(GraphAttentionTransformer, p.cfg, p.state).double()
    with _emulated():
        energy, _forces = run_mirror("qm9", model, p)
    assert rel_err(energy.detach(), p.t("energy")) < 1e-10
    assert worst_grad({k: q.grad for k, q in model.named_parameters()}, p.grads, 80) < 1e-7

    p = _part("md17")
    model = mirror(GraphAttentionTransformerMD17, p.cfg, p.state).double()
    with _emulated():
        e, f = run_mirror("md17", model, p)
    assert rel_err(e.detach(), p.t("energy")) < 1e-10
    assert rel_err(f.detach(), p.t("forces")) < 1e-9
    assert worst_grad({k: q.grad for k, q in model.named_parameters()}, p.grads, 80) < 1e-6


def _shape_table():
    with open(SHAPES) as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(_shape_table()))
def test_bessel_configurations_have_the_reference_parameters(name):
    """Each registered Bessel configuration constructs at its real size with the reference constructor's parameter and
    buffer names / shapes (``rbf.rbf.frequencies`` included) and the same ``no_weight_decay()`` set."""
    from equiformer_b200.nets import model_entrypoint
    ref = _shape_table()[name]
    model = model_entrypoint(name)(irreps_in="64x0e" if name.endswith("md17") else "5x0e", radius=5.0,
                                   num_basis=ref["num_basis"])
    mine = {k: list(v.shape) for k, v in model.state_dict().items() if not k.endswith("tp.output_mask")}
    assert mine == ref["state"]
    assert mine["rbf.rbf.frequencies"] == [ref["num_basis"]]
    assert sorted(model.no_weight_decay()) == ref["no_weight_decay"]
    assert "rbf.rbf.frequencies" in ref["no_weight_decay"]


def test_dens_and_dot_product_models_take_the_bessel_basis():
    from equiformer_b200.nets import equiformer_md17_dens as D
    from equiformer_b200.nets.dp_attention_transformer import DotProductAttentionTransformerMD17
    from equiformer_b200.nets.bessel_rbf import RadialBasis
    small = dict(irreps_node_embedding="16x0e+8x1e+4x2e", num_layers=1, number_of_basis=8, basis_type="bessel",
                 fc_neurons=[16, 16], irreps_head="8x0e+4x1e+2x2e", num_heads=2, irreps_mlp_mid="24x0e+12x1e+6x2e")
    for model in (D.Equiformer_MD17_DeNS(irreps_feature="32x0e+16x1e+8x2e", irreps_pre_attn="16x0e+8x1e+4x2e", **small),
                  DotProductAttentionTransformerMD17(irreps_feature="32x0e", **small)):
        assert isinstance(model.rbf, RadialBasis)
        assert "rbf.rbf.frequencies" in model.no_weight_decay()


# ------------------------------------------------------------------------------------------------ GPU

def _kernel_case(dev, E, B, seed):
    g = torch.Generator().manual_seed(seed)
    dist = 0.3 + 5.0 * torch.rand(E, generator=g)           # a few beyond the 5 A cutoff
    freq = math.pi * torch.arange(1, B + 1, dtype=torch.float32) + 0.1 * torch.randn(B, generator=g)
    gout = torch.randn(E, B, generator=g)
    return dist, freq, gout


def _fp64_reference(dist, freq, gout):
    from equiformer_b200 import ops
    d, f = dist.double().requires_grad_(True), freq.double().requires_grad_(True)
    out = ops.bessel_rbf_torch(d, f, 5.0)
    gd, gf = torch.autograd.grad(out, (d, f), gout.double())
    return out.detach(), gd, gf


def _check_kernels(dev, E, B, seed, need_dist):
    from equiformer_b200 import ops
    dist, freq, gout = _kernel_case(dev, E, B, seed)
    out = ops.bessel_fwd_raw(dist.to(dev), freq.to(dev), 5.0)
    gd, gf = ops.bessel_bwd_raw(dist.to(dev), freq.to(dev), 5.0, gout.to(dev), need_dist)
    ref_out, ref_gd, ref_gf = _fp64_reference(dist, freq, gout)
    assert rel_err(out.cpu(), ref_out) < TOL
    assert rel_err(gf.cpu(), ref_gf) < TOL_FREQ
    if need_dist:
        assert rel_err(gd.cpu(), ref_gd) < TOL
    else:
        assert gd is None


@pytest.mark.gpu
@pytest.mark.parametrize("B", [8, 32, 128])
@pytest.mark.parametrize("E", [1, 777, 32560])
@pytest.mark.parametrize("need_dist", [True, False])
def test_bessel_kernels_vs_fp64(cuda_device, E, B, need_dist):
    _check_kernels(cuda_device, E, B, E + B, need_dist)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["two_passes", "partial_third_pass"])
def test_bessel_kernels_past_the_grid_cap(cuda_device, which):
    """C = 8 warps x 1056 CTAs edges per pass; E = 2 C (two full passes) and 2 C + C / 3 (some warps run a third)."""
    C = 8 * _POINTWISE_CTAS
    E = 2 * C if which == "two_passes" else 2 * C + C // 3
    from equiformer_b200 import _lib
    assert _lib.load().eqf_pointwise_rows(E) == _POINTWISE_CTAS
    _check_kernels(cuda_device, E, 128, 11, True)


@pytest.mark.gpu
def test_bessel_kernels_reject_unsupported_sizes(cuda_device):
    from equiformer_b200 import _lib, ops
    d = torch.rand(10, device=cuda_device) + 1.0
    for B in (6, 132):
        with pytest.raises(_lib.EqfError):
            ops.bessel_rbf(d, torch.ones(B, device=cuda_device), 5.0)


@pytest.mark.gpu
@pytest.mark.parametrize("deterministic", [False, True])
def test_k8_first_layer_gemms(cuda_device, monkeypatch, deterministic):
    """The stacked first Linear of the 7 radial MLPs at num_basis = 8: [E, 8] x [8, 448] forward, the N = 8 data gradient
    and the weight gradients (K1 = 8 and K1 = 448 columns of A) through the wgmma kernels, at E = 32 560 vs fp64."""
    from equiformer_b200 import ops
    monkeypatch.setattr(ops, "_DETERMINISTIC", deterministic)
    E = 32560
    g = torch.Generator().manual_seed(8)
    X, W, G = torch.randn(E, 8, generator=g), torch.randn(448, 8, generator=g), torch.randn(E, 448, generator=g)
    d = lambda t: t.to(cuda_device)
    assert ops._use_tensor_cores(E, 448, 8) and E >= ops._WGRAD_MIN_K and ops.gemm_backend() == "tf32x3"
    assert rel_err(ops.gemm_raw(1, d(X), d(W)).cpu(), X.double() @ W.double().t()) < 1e-5
    assert rel_err(ops.gemm_raw(0, d(G), d(W)).cpu(), G.double() @ W.double()) < 1e-5
    assert rel_err(ops.gemm_raw(2, d(G), d(X)).cpu(), G.double().t() @ X.double()) < 4e-5
    assert rel_err(ops.gemm_raw(2, d(X), d(G)).cpu(), X.double().t() @ G.double()) < 4e-5


@pytest.mark.gpu
def test_cuda_qm9_bessel_model_matches_reference(cuda_device):
    """Energies and gradients of sum(E^2) through GraphedStep (capture + replay), then eager.  The captured step runs
    first, as in the other capture tests: its warm-up runs on a side stream, never on the default one."""
    from equiformer_b200 import ops
    from equiformer_b200.graphs import GraphedStep
    from equiformer_b200.nets.graph_attention_transformer import GraphAttentionTransformer
    from equiformer_b200.parallel import FlatGradAllReduce
    p = _part("qm9")
    model = mirror(GraphAttentionTransformer, p.cfg, p.state).to(cuda_device)
    pos, batch, z = (p.t(k, cuda_device) for k in ("pos", "batch", "z"))
    graph = ops.Graph(*R.radius_graph(pos, 5.0, batch), pos.shape[0])
    src, dst = graph.src, graph.dst
    bucket = FlatGradAllReduce(model.parameters())

    def captured(pos, batch, z, src, dst, row_ptr):
        csr = ops.Graph.__new__(ops.Graph)
        csr.n_nodes, csr.n_edges, csr.perm = int(batch.shape[0]), int(src.numel()), None
        csr.src, csr.dst, csr.row_ptr = src, dst, row_ptr
        csr._src_perm = csr._src_row_ptr = None
        e = model.forward_edges(pos, batch, z, src, dst, graph=csr, n_graphs=2)
        return (e ** 2).sum()

    step = GraphedStep(captured, bucket)
    for _ in range(2):
        loss = step((int(pos.shape[0]), int(src.numel())), [pos, batch, z, src, dst, graph.row_ptr]).clone()
    assert step.captures == 1
    assert rel_err(loss.cpu(), (p.t("energy") ** 2).sum()) < 1e-4
    assert worst_grad({k: q.grad for k, q in model.named_parameters()}, p.grads, 80) < 1e-3

    bucket.zero_grad()
    energy, _forces = run_mirror("qm9", model, p, cuda_device, torch.float32)
    assert rel_err(energy.detach().cpu(), p.t("energy")) < 5e-5
    assert worst_grad({k: q.grad for k, q in model.named_parameters()}, p.grads, 80) < 1e-3


@pytest.mark.gpu
def test_cuda_md17_bessel_model_matches_reference(cuda_device):
    """Energy, forces and gradients of the energy + force loss (double backward through the basis), captured, then
    eager."""
    from equiformer_b200 import ops
    from equiformer_b200.graphs import GraphedStep
    from equiformer_b200.nets.graph_attention_transformer_md17 import GraphAttentionTransformerMD17
    from equiformer_b200.parallel import FlatGradAllReduce
    p = _part("md17")
    model = mirror(GraphAttentionTransformerMD17, p.cfg, p.state).to(cuda_device)
    pos, batch, z = (p.t(k, cuda_device) for k in ("pos", "batch", "z"))
    graph = ops.Graph(*R.radius_graph(pos, 5.0, batch), pos.shape[0])
    bucket = FlatGradAllReduce(model.parameters())

    def captured(pos, batch, z, src, dst, row_ptr):
        csr = ops.Graph.__new__(ops.Graph)
        csr.n_nodes, csr.n_edges, csr.perm = int(batch.shape[0]), int(src.numel()), None
        csr.src, csr.dst, csr.row_ptr = src, dst, row_ptr
        csr._src_perm = csr._src_row_ptr = None
        ee, ff = model.forward_edges(z, pos.detach().requires_grad_(True), batch, src, dst, graph=csr, n_graphs=1)
        return ee.sum() + (ff ** 2).sum()

    step = GraphedStep(captured, bucket)
    for _ in range(2):
        loss = step((int(pos.shape[0]), graph.n_edges), [pos, batch, z, graph.src, graph.dst, graph.row_ptr]).clone()
    assert step.captures == 1
    ref_loss = float(p.t("energy").sum() + (p.t("forces") ** 2).sum())
    assert abs(float(loss) - ref_loss) / abs(ref_loss) < 1e-4
    assert worst_grad({k: q.grad for k, q in model.named_parameters()}, p.grads, 80) < 1e-3

    bucket.zero_grad()
    e, f = run_mirror("md17", model, p, cuda_device, torch.float32)
    assert rel_err(e.detach().cpu(), p.t("energy")) < 5e-5
    assert rel_err(f.detach().cpu(), p.t("forces")) < 2e-4
    assert worst_grad({k: q.grad for k, q in model.named_parameters()}, p.grads, 80) < 1e-3


@pytest.mark.gpu
def test_captured_qm9_bessel_training_step_matches_eager(cuda_device):
    """graph_attention_transformer_nonlinear_bessel_l2 at num_basis = 8 on 128 synthetic molecules (E ~ 32 k, so the
    K = 8 first layer runs on the wgmma kernels): the captured forward + L1 loss + backward gives the eager loss and
    gradients, the frequency gradient included."""
    from equiformer_b200.graphs import GraphedForwardBackward
    from equiformer_b200.nets import model_entrypoint
    from equiformer_b200.parallel import FlatGradAllReduce
    from equiformer_b200.synthetic import qm9_like_batch
    torch.manual_seed(0)
    model = model_entrypoint("graph_attention_transformer_nonlinear_bessel_l2")(irreps_in="5x0e", radius=5.0, num_basis=8)
    model = model.to(cuda_device).train()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    pos, batch, z = (t.to(cuda_device) for t in qm9_like_batch(128, seed=0))
    target = torch.randn(128, 1, generator=torch.Generator().manual_seed(1)).to(cuda_device)
    loss_fn = lambda out, tgt: (out - tgt).abs().mean()
    bucket = FlatGradAllReduce(model.parameters())
    gfb = GraphedForwardBackward(model, loss_fn, bucket, max_radius=5.0)
    for _ in range(2):
        loss_g = gfb(pos, batch, z, target).clone()
    grads_g = bucket.flat.clone()
    assert gfb.captures == 1
    bucket.zero_grad()
    loss_e = loss_fn(model(f_in=None, pos=pos, batch=batch, node_atom=z, n_graphs=128), target)
    loss_e.backward()
    assert rel_err(loss_g, loss_e.detach()) < 1e-5
    assert rel_err(grads_g, bucket.flat) < 1e-5
    gf = model.rbf.rbf.frequencies.grad
    assert gf is not None and float(gf.abs().max()) > 0
