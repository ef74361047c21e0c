"""Parity against vectors produced by the REFERENCE'S OWN CODE (tests/golden/reference_modules.npz).

``tests/golden/make_reference_golden.py`` imports five reference modules from /root/reference behind a stub e3nn (see its
docstring) and records inputs, ``state_dict`` and float64 outputs.  Here the fixture pins

* the oracle's restatements of those modules (CPU, float64, 1e-12),
* the host-side mirrors in ``equiformer_b200.nets`` loaded from the reference's ``state_dict`` (CPU, float64, 1e-12 -
  which also proves the parameter names and shapes are the reference's), and
* on a GPU, the same mirrors in float32 through the fused CUDA kernels (radial basis, LayerNorm+SiLU, equivariant
  layer norm) within the float32 tolerance written next to each check.
"""
from __future__ import annotations

import os

import numpy as np
import pytest
import torch

from oracle import e3nn_ref as e3
from oracle import equiformer_ref as R
from tests.helpers import assert_same_grad_presence, rel_err
from tests.reference_fixtures import (GOLDEN, dens_setup, load, load_state, mirror, oc20_data, oracle_config, run_mirror,
                                      run_oracle, worst_grad)

FIXTURE = "reference_modules.npz"
LN_CASES = ["qm9_l2", "md17_l3", "oc20_l1", "ffn_mid"]


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, FIXTURE))


def _state(prefix, dtype=torch.float64):
    return {k: v.to(dtype) for k, v in load(FIXTURE, prefix).state.items()}


def _t(gold, key, dtype=torch.float64):
    return torch.from_numpy(gold[key]).to(dtype)


def _params(prefix, name="m"):
    return {f"{name}.{k}": v for k, v in _state(prefix).items()}


# ------------------------------------------------------------------------------------------------ oracle (CPU, fp64)

def test_oracle_gaussian_rbf_matches_reference(gold):
    out = R.gaussian_rbf(_params("gaussian_rbf"), "m", _t(gold, "gaussian_rbf/dist"), float(gold["gaussian_rbf/cutoff"]))
    assert rel_err(out, _t(gold, "gaussian_rbf/y")) < 1e-12


def test_oracle_expnorm_rbf_matches_reference(gold):
    out = R.expnorm_rbf(_params("expnorm_rbf"), "m", _t(gold, "expnorm_rbf/dist"), float(gold["expnorm_rbf/cutoff"]))
    assert rel_err(out, _t(gold, "expnorm_rbf/y")) < 1e-12


@pytest.mark.parametrize("tag", ["qm9", "small"])
def test_oracle_radial_profile_matches_reference(gold, tag):
    out = R.radial_profile(_params(f"radial_profile_{tag}"), "m", _t(gold, f"radial_profile_{tag}/x"))
    assert rel_err(out, _t(gold, f"radial_profile_{tag}/y")) < 1e-12


@pytest.mark.parametrize("tag", LN_CASES)
def test_oracle_layer_norm_matches_reference(gold, tag):
    irreps = e3.parse_irreps(str(gold[f"layer_norm_{tag}/irreps"]))
    out = R.layer_norm_v2(_params(f"layer_norm_{tag}"), "m", irreps, _t(gold, f"layer_norm_{tag}/x"),
                          float(gold[f"layer_norm_{tag}/eps"]))
    assert rel_err(out, _t(gold, f"layer_norm_{tag}/y")) < 1e-12


# ------------------------------------------------------------------------------------ host-side mirrors (CPU, fp64)

def _mirror(kind, gold, tag=None):
    from equiformer_b200.nets import expnorm_rbf, gaussian_rbf, layer_norm, radial_func
    if kind == "gaussian_rbf":
        m, prefix = gaussian_rbf.GaussianRadialBasisLayer(int(gold["gaussian_rbf/num_basis"]), float(gold["gaussian_rbf/cutoff"])), kind
    elif kind == "expnorm_rbf":
        m, prefix = expnorm_rbf.ExpNormalSmearing(0.0, float(gold["expnorm_rbf/cutoff"]), int(gold["expnorm_rbf/num_rbf"]), False), kind
    elif kind == "radial_profile":
        prefix = f"radial_profile_{tag}"
        m = radial_func.RadialProfile([int(c) for c in gold[f"{prefix}/ch_list"]])
    else:
        prefix = f"layer_norm_{tag}"
        m = layer_norm.EquivariantLayerNormV2(str(gold[f"{prefix}/irreps"]), eps=float(gold[f"{prefix}/eps"]))
    missing = m.load_state_dict(_state(prefix, torch.float32), strict=True)      # the reference's own keys and shapes
    assert not missing.missing_keys and not missing.unexpected_keys
    return m, prefix


@pytest.mark.parametrize("kind,tag,x_key", [("gaussian_rbf", None, "dist"), ("expnorm_rbf", None, "dist"),
                                            ("radial_profile", "qm9", "x"), ("radial_profile", "small", "x")]
                         + [("layer_norm", t, "x") for t in LN_CASES])
def test_host_mirror_matches_reference_on_cpu(gold, kind, tag, x_key):
    m, prefix = _mirror(kind, gold, tag)
    out = m.double()(_t(gold, f"{prefix}/{x_key}"))
    assert rel_err(out, _t(gold, f"{prefix}/y")) < 1e-12


def test_activation_mirror_matches_reference_structure(gold):
    """fast_activation.py:15-87 run by the reference's code; the normalize2mom constants inside are ours in both."""
    from equiformer_b200.nets.fast_activation import Activation
    m = Activation(str(gold["activation/irreps"]), [torch.nn.SiLU(), torch.tanh])
    assert rel_err(m(_t(gold, "activation/x")), _t(gold, "activation/y")) < 1e-12


# ------------------------------------------------------------------------------------------- CUDA kernels (GPU, fp32)

@pytest.mark.gpu
@pytest.mark.parametrize("kind,tag,x_key,tol", [("gaussian_rbf", None, "dist", 1e-5), ("radial_profile", "qm9", "x", 1e-5),
                                                ("radial_profile", "small", "x", 1e-5)]
                         + [("layer_norm", t, "x", 5e-6) for t in LN_CASES])
def test_cuda_path_matches_reference(gold, cuda_device, kind, tag, x_key, tol):
    """The fused kernels (``rbf_fwd``, ``ln_silu_fwd`` + GEMM, ``eln_fwd``) behind the mirrored modules against the
    reference-generated float64 outputs; tolerance = float32 evaluation of a float64 fixture (relative to max|y|)."""
    m, prefix = _mirror(kind, gold, tag)
    m = m.to(cuda_device)
    x = _t(gold, f"{prefix}/{x_key}", torch.float32).to(cuda_device)
    with torch.no_grad():
        out = m(x)
    assert rel_err(out, _t(gold, f"{prefix}/y")) < tol


# ------------------------------------------------- the reference's model file end to end (reference_model_small.npz)

SMALL = "reference_model_small.npz"
MD17_SMALL = "reference_model_md17_small.npz"


def test_oracle_model_matches_reference_model_file():
    """``GraphAttentionTransformer.forward`` of the reference (its own files executed; e3nn / scatter / softmax /
    radius-graph calls served by the oracle's restatements - see the generator) vs ``oracle.model_forward`` fed the
    reference's ``state_dict``: pins instruction lists, irreps sorting, rescale and bias handling, head reshapes,
    attention wiring, residuals and scale factors of the restatement.  Both sides are float64."""
    case = load(SMALL)
    params = R.cast_params(case.state, torch.float64)
    pos, batch, z = case.t("pos", dtype=torch.float64), case.t("batch"), case.t("z")
    energy = R.model_forward(params, oracle_config("qm9", case.cfg), pos, batch, z, n_graphs=2)
    assert rel_err(energy, case.t("energy")) < 1e-11


def test_oracle_md17_model_matches_reference_model_file():
    """The same for ``nets/graph_attention_transformer_md17.py`` (Lmax = 3, exp-normal basis, forces = -dE/dpos by
    autograd through the reference's own forward) vs ``oracle.energy_and_forces``."""
    case = load(MD17_SMALL)
    params = R.cast_params(case.state, torch.float64)
    pos, batch, z = case.t("pos", dtype=torch.float64), case.t("batch"), case.t("z")
    energy, forces = R.energy_and_forces(params, oracle_config("md17", case.cfg), pos, batch, z, n_graphs=1)
    assert rel_err(energy, case.t("energy")) < 1e-11
    assert rel_err(forces, case.t("forces")) < 1e-10


def test_mirror_models_take_the_reference_state_dict():
    """Names and shapes of every parameter / buffer the reference's model files create (executed, not read) exist in the
    host-side mirrors: the drop-in property of the module API, checked on the CPU."""
    from equiformer_b200.nets.graph_attention_transformer import GraphAttentionTransformer
    from equiformer_b200.nets.graph_attention_transformer_md17 import GraphAttentionTransformerMD17
    for name, cls in ((SMALL, GraphAttentionTransformer), (MD17_SMALL, GraphAttentionTransformerMD17)):
        case = load(name)
        mirror(cls, case.cfg, case.state)


@pytest.mark.gpu
def test_cuda_model_matches_reference_model_file(cuda_device):
    """The CUDA path (generic plan kernels at these small channel counts) under the QM9 mirror, loaded with the
    reference's ``state_dict``, against the energy the reference's own model file produced; float32 vs a float64
    fixture, two blocks deep: 5e-5 of max|E|."""
    from equiformer_b200.nets.graph_attention_transformer import GraphAttentionTransformer
    case = load(SMALL)
    model = mirror(GraphAttentionTransformer, case.cfg, case.state).to(cuda_device)
    pos = case.t("pos", cuda_device)
    batch, z = case.t("batch", cuda_device), case.t("z", cuda_device)
    with torch.no_grad():
        energy = model(f_in=None, pos=pos, batch=batch, node_atom=z)
    assert rel_err(energy, case.t("energy")) < 5e-5


@pytest.mark.gpu
def test_cuda_md17_model_matches_reference_model_file(cuda_device):
    """Energy and forces (``-dE/dpos`` through the closed autograd families) of the MD17 mirror on CUDA against the
    reference's own MD17 model file: 5e-5 / 2e-4 relative to the largest component."""
    from equiformer_b200.nets.graph_attention_transformer_md17 import GraphAttentionTransformerMD17
    case = load(MD17_SMALL)
    model = mirror(GraphAttentionTransformerMD17, case.cfg, case.state).to(cuda_device)
    pos = case.t("pos", cuda_device)
    batch, z = case.t("batch", cuda_device), case.t("z", cuda_device)
    energy, forces = model(node_atom=z, pos=pos, batch=batch)
    assert rel_err(energy.detach(), case.t("energy")) < 5e-5
    assert rel_err(forces.detach(), case.t("forces")) < 2e-4


SHAPES = os.path.join(GOLDEN, "reference_state_shapes.json")


def _shape_table():
    import json
    with open(SHAPES) as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(_shape_table()))
def test_registered_models_have_the_reference_parameters(name):
    """Every registered configuration that runs without ocpmodels' Bessel basis, at its real size: the names and shapes
    of all parameters and buffers created by the reference's constructors (executed by the generator) against the
    mirror's ``state_dict`` - the drop-in contract for checkpoints, and the parameter counts of the paper
    (3.53 M for ``graph_attention_transformer_nonlinear_l2``)."""
    from equiformer_b200.nets import model_entrypoint
    ref = _shape_table()[name]
    model = model_entrypoint(name)(irreps_in="64x0e" if name.endswith("md17") else "5x0e", radius=5.0, num_basis=128)
    mine = {k: list(v.shape) for k, v in model.state_dict().items() if not k.endswith("tp.output_mask")}
    assert sorted(mine) == sorted(ref)
    assert mine == ref


HEADLINE = "reference_model_headline.npz"


def _closed_form_state(g, shapes):
    """state_dict as the generator set it: small tensors verbatim, large ones from the closed form"""
    from tests.helpers import closed_form_tensor
    state = {}
    for k, shape in shapes.items():
        if f"small/{k}" in g:
            state[k] = torch.from_numpy(g[f"small/{k}"])
        elif f"stat/{k}" in g:
            mean, std = (float(v) for v in g[f"stat/{k}"])
            state[k] = closed_form_tensor(k, shape, mean, std)
        else:
            state[k] = torch.zeros(shape)          # e3nn's empty `tp.weight` buffers of externally weighted products
            assert state[k].numel() == 0, k
    return state


def _headline_state():
    g = load(HEADLINE).arrays
    return g, _closed_form_state(g, _shape_table()["graph_attention_transformer_nonlinear_l2"])


def test_oracle_headline_model_matches_reference_model_file():
    """The headline configuration itself (``graph_attention_transformer_nonlinear_l2``, 6 blocks, 3.53 M parameters)
    run by the reference's own model file on 16 atoms vs ``oracle.model_forward`` with the same parameters."""
    g, state = _headline_state()
    params = R.cast_params(state, torch.float64)
    pos, batch, z = torch.from_numpy(g["pos"]).double(), torch.from_numpy(g["batch"]), torch.from_numpy(g["z"])
    energy = R.model_forward(params, R.Config(), pos, batch, z, n_graphs=2)
    assert rel_err(energy, torch.from_numpy(g["energy"])) < 1e-10


@pytest.mark.gpu
def test_cuda_headline_model_matches_reference_model_file(cuda_device):
    """The CUDA path of the headline configuration (generated ``qm9_l2`` kernels, wgmma GEMMs, planar-resident blocks)
    against the energies the reference's own model file returned for the same parameters.  Float32 through six blocks
    against a float64 fixture whose closed-form readout weights cancel to |E| ~ 0.07 while block outputs are ~3: the
    float32 CPU oracle is 1.6e-5 away from the fixture in absolute terms, the bound here is 3e-4."""
    from equiformer_b200.nets import model_entrypoint
    g, state = _headline_state()
    model = model_entrypoint("graph_attention_transformer_nonlinear_l2")(irreps_in="5x0e", radius=5.0, num_basis=128)
    model = load_state(model, state).eval().to(cuda_device)
    pos = torch.from_numpy(g["pos"]).to(cuda_device)
    batch, z = torch.from_numpy(g["batch"]).to(cuda_device), torch.from_numpy(g["z"]).to(cuda_device)
    with torch.no_grad():
        energy = model(f_in=None, pos=pos, batch=batch, node_atom=z)
    assert float((energy.double().cpu() - torch.from_numpy(g["energy"])).abs().max()) < 3e-4


@pytest.fixture
def tensor_core_gemms_everywhere():
    """Lower the row thresholds of the GEMM policy (``ops._GEMM_MIN_M`` / ``_WGRAD_MIN_K``) so that even the 16-atom reference-run fixtures go through the hand-written wgmma kernels instead
    of cuBLAS (VERDICT r1: at these sizes ``M = E (2l+1) << 16 384`` and every product used to be a cuBLAS call)."""
    from equiformer_b200 import ops
    old = ops._GEMM_MIN_M, ops._WGRAD_MIN_K
    ops._GEMM_MIN_M, ops._WGRAD_MIN_K = 1, 1
    yield
    ops._GEMM_MIN_M, ops._WGRAD_MIN_K = old


@pytest.mark.gpu
def test_cuda_headline_model_matches_reference_through_tcgen05_gemms(cuda_device, tensor_core_gemms_everywhere):
    """As ``test_cuda_headline_model_matches_reference_model_file`` with every aligned product on the wgmma 3xTF32
    kernels (forward + one backward pass; the gradients are checked against the oracle in the next test - this fixture's
    closed-form weights leave several gradients at rounding-noise level)."""
    from equiformer_b200 import ops
    from equiformer_b200.nets import model_entrypoint
    g, state = _headline_state()
    model = model_entrypoint("graph_attention_transformer_nonlinear_l2")(irreps_in="5x0e", radius=5.0, num_basis=128)
    model = load_state(model, state).eval().to(cuda_device)
    pos = torch.from_numpy(g["pos"]).to(cuda_device)
    batch, z = torch.from_numpy(g["batch"]).to(cuda_device), torch.from_numpy(g["z"]).to(cuda_device)
    prof = ops.KernelProfile(time_events=False)
    ops.PROFILE = prof
    try:
        energy = model(f_in=None, pos=pos, batch=batch, node_atom=z)
        energy.sum().backward()
    finally:
        ops.PROFILE = None
    assert float((energy.detach().double().cpu() - torch.from_numpy(g["energy"])).abs().max()) < 3e-4
    assert prof.summary() is not None and prof.launches > 300


@pytest.mark.gpu
def test_cuda_small_model_gradients_through_tcgen05_gemms_match_oracle(cuda_device, tensor_core_gemms_everywhere):
    """Every parameter gradient of the headline model on a five-molecule batch, all aligned products (forward, data and
    weight gradients, node level included) on the wgmma kernels, against the fp64 oracle - the same bound as the
    cuBLAS-policy run of tests/test_gpu_model.py."""
    from equiformer_b200.nets import model_entrypoint
    from tests.helpers import molecules
    torch.manual_seed(0)
    model = model_entrypoint("graph_attention_transformer_nonlinear_l2")(irreps_in="5x0e", radius=5.0, num_basis=128)
    model = model.to(cuda_device).eval()
    gen = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for p in model.parameters():
            p.add_(torch.randn(p.shape, generator=gen).to(p.device) * 0.05)
    pos, batch, z = molecules([9, 14, 5, 11, 7], seed=2)
    out = model(f_in=None, pos=pos.to(cuda_device), batch=batch.to(cuda_device), node_atom=z.to(cuda_device))
    out.sum().backward()
    params = {k: v.requires_grad_(v.is_floating_point() and v.numel() > 0)
              for k, v in R.cast_params(model.state_dict(), torch.float64).items()}
    ref = R.model_forward(params, R.Config(), pos.double(), batch, z, 5)
    ref.sum().backward()
    assert rel_err(out, ref) < 1e-4
    grads = {k: p.grad for k, p in model.named_parameters()}
    ref = {k: params[k].grad for k, g in grads.items() if assert_same_grad_presence(k, g, params[k].grad)}
    assert worst_grad(grads, ref, 1) < 1e-3


@pytest.mark.gpu
def test_cuda_md17_model_matches_reference_through_tcgen05_gemms(cuda_device, tensor_core_gemms_everywhere):
    """Energy and forces of the MD17 fixture (a double-backward-capable path) with the wgmma kernels forced on."""
    from equiformer_b200.nets.graph_attention_transformer_md17 import GraphAttentionTransformerMD17
    case = load(MD17_SMALL)
    model = mirror(GraphAttentionTransformerMD17, case.cfg, case.state).to(cuda_device)
    pos = case.t("pos", cuda_device)
    batch, z = case.t("batch", cuda_device), case.t("z", cuda_device)
    energy, forces = model(node_atom=z, pos=pos, batch=batch)
    assert rel_err(energy.detach(), case.t("energy")) < 5e-5
    assert rel_err(forces.detach(), case.t("forces")) < 2e-4


# --------------------------------- host logic of the mirrors (kernels emulated in float64 on the CPU) vs the reference

def test_mirror_host_logic_matches_reference_model_files():
    """The mirrors' own wiring (planar layouts, fused-op call sequence, autograd closure for the forces) with the raw
    kernel calls swapped for float64 torch walks (tests/_emulation.py), against the three reference-run model fixtures."""
    from equiformer_b200.nets import model_entrypoint
    from equiformer_b200.nets.graph_attention_transformer import GraphAttentionTransformer
    from equiformer_b200.nets.graph_attention_transformer_md17 import GraphAttentionTransformerMD17
    from tests._emulation import emulated_kernels

    case = load(SMALL)
    model = mirror(GraphAttentionTransformer, case.cfg, case.state).double()
    with emulated_kernels(), torch.no_grad():
        energy = model(f_in=None, pos=case.t("pos", dtype=torch.float64), batch=case.t("batch"), node_atom=case.t("z"))
    assert rel_err(energy, case.t("energy")) < 1e-10

    case = load(MD17_SMALL)
    model = mirror(GraphAttentionTransformerMD17, case.cfg, case.state).double()
    with emulated_kernels():
        energy, forces = model(node_atom=case.t("z"), pos=case.t("pos", dtype=torch.float64), batch=case.t("batch"))
    assert rel_err(energy.detach(), case.t("energy")) < 1e-10
    assert rel_err(forces.detach(), case.t("forces")) < 1e-9

    g, state = _headline_state()
    model = model_entrypoint("graph_attention_transformer_nonlinear_l2")(irreps_in="5x0e", radius=5.0, num_basis=128)
    model = load_state(model, state).eval().double()
    with emulated_kernels(), torch.no_grad():
        energy = model(f_in=None, pos=torch.from_numpy(g["pos"]).double(), batch=torch.from_numpy(g["batch"]),
                       node_atom=torch.from_numpy(g["z"]))
    assert rel_err(energy, torch.from_numpy(g["energy"])) < 1e-9


def test_drop_modules_draw_like_the_reference(gold):
    """DropPath / GraphDropPath / EquivariantDropout / EquivariantScalarsDropout in training mode (drop.py:31-106): with
    the same torch seed the mirrors must make the same draws in the same order and scale the same way - bit for bit."""
    from equiformer_b200.nets import drop
    x, batch = _t(gold, "drop/x", torch.float32), torch.from_numpy(gold["drop/batch"])
    for tag, module, args in (("drop_path", drop.DropPath(0.3), (x,)), ("graph_drop_path", drop.GraphDropPath(0.4), (x, batch)),
                              ("equivariant_dropout", drop.EquivariantDropout("128x0e+64x1e+32x2e", 0.25), (x,)),
                              ("scalars_dropout", drop.EquivariantScalarsDropout("128x0e+64x1e+32x2e", 0.25), (x,))):
        module.train()
        torch.manual_seed(321)
        assert torch.equal(module(*args), _t(gold, f"drop/{tag}", torch.float32)), tag


# ------------------------------------------------------------ one block at the OC20 IS2RE l1_256_nonlinear sizes

OC20_BLOCK = "reference_block_oc20_l1.npz"


def _oc20_block():
    import json
    block = load(OC20_BLOCK)
    g = block.arrays
    state = _closed_form_state(g, json.loads(str(g["shapes"])))
    inputs = {k: block.t(k) for k in ("x", "edge_src", "edge_dst", "edge_sh", "edge_scalars")}
    return g, state, block.cfg, inputs


def test_oracle_block_matches_reference_at_oc20_sizes():
    """``TransBlock`` (graph_attention_transformer.py:575-667) at the channel counts of the OC20 ``l1_256_nonlinear``
    configuration (256x0e+128x1e, 8 heads, Lmax = 1), run by the reference's code, vs ``oracle.trans_block``."""
    g, state, kw, t = _oc20_block()
    cfg = R.Config(irreps_node_embedding=kw["irreps_node_input"], irreps_sh=kw["irreps_edge_attr"], irreps_head=kw["irreps_head"],
                   irreps_mlp_mid=kw["irreps_mlp_mid"], num_heads=kw["num_heads"], nonlinear_message=kw["nonlinear_message"])
    params = {f"b.{k}": v for k, v in R.cast_params(state, torch.float64).items()}
    irreps = e3.parse_irreps(kw["irreps_node_input"])
    x = t["x"].double()
    out = R.trans_block(params, "b", cfg, irreps, irreps, x, torch.ones_like(x[:, :1]), t["edge_src"], t["edge_dst"],
                        t["edge_sh"].double(), t["edge_scalars"].double())
    assert rel_err(out, torch.from_numpy(g["y"])) < 1e-10


def test_mirror_block_host_logic_matches_reference_at_oc20_sizes():
    from equiformer_b200.nets.graph_attention_transformer import TransBlock
    from tests._emulation import emulated_kernels
    g, state, kw, t = _oc20_block()
    blk = mirror(TransBlock, kw, state).double()
    x = t["x"].double()
    with emulated_kernels(), torch.no_grad():
        out = blk(node_input=x, node_attr=torch.ones_like(x[:, :1]), edge_src=t["edge_src"], edge_dst=t["edge_dst"],
                  edge_attr=t["edge_sh"].double(), edge_scalars=t["edge_scalars"].double(),
                  batch=torch.zeros(x.shape[0], dtype=torch.long))
    assert rel_err(out, torch.from_numpy(g["y"])) < 1e-10


@pytest.mark.gpu
def test_cuda_block_matches_reference_at_oc20_sizes(cuda_device):
    """The CUDA path of one transformer block at the OC20 ``l1_256_nonlinear`` sizes (generated ``oc20_l1`` kernels,
    8 heads) against the reference-run fixture; float32 vs float64, same bound as the layer-level oracle test
    (tests/test_gpu_model.py::test_oc20_l1_layer_vs_oracle).  Written after the round-1 GPU budget ended."""
    from equiformer_b200.nets.graph_attention_transformer import TransBlock
    g, state, kw, t = _oc20_block()
    blk = mirror(TransBlock, kw, state).to(cuda_device)
    d = lambda v: v.to(cuda_device)
    x = d(t["x"])
    with torch.no_grad():
        out = blk(node_input=x, node_attr=torch.ones_like(x[:, :1]), edge_src=d(t["edge_src"]), edge_dst=d(t["edge_dst"]),
                  edge_attr=d(t["edge_sh"]), edge_scalars=d(t["edge_scalars"]),
                  batch=torch.zeros(x.shape[0], dtype=torch.long, device=cuda_device))
    assert rel_err(out, torch.from_numpy(g["y"])) < 1e-4


# --------------------------------------------------------------- backward: parameter gradients of the reference's models

def test_parameter_gradients_match_reference_qm9_small():
    """d(sum E^2)/d(parameters) from the reference's own backward through its own forward, vs autograd through the
    oracle and through the mirror (closed autograd families, kernels emulated)."""
    from equiformer_b200.nets.graph_attention_transformer import GraphAttentionTransformer
    from tests._emulation import emulated_kernels
    case = load(SMALL)
    _energy, _forces, params = run_oracle("qm9", case, oracle_config("qm9", case.cfg))
    assert worst_grad({k: v.grad for k, v in params.items()}, case.grads, 80) < 1e-8
    model = mirror(GraphAttentionTransformer, case.cfg, case.state).double()
    with emulated_kernels():
        run_mirror("qm9", model, case)
    assert worst_grad({k: p.grad for k, p in model.named_parameters()}, case.grads, 80) < 1e-7


def test_parameter_gradients_match_reference_md17_small():
    """The energy + force loss of MD17 training (a second derivative through the forward): parameter gradients from the
    reference's model file vs the oracle and the mirror."""
    from equiformer_b200.nets.graph_attention_transformer_md17 import GraphAttentionTransformerMD17
    from tests._emulation import emulated_kernels
    case = load(MD17_SMALL)
    _energy, _forces, params = run_oracle("md17", case, oracle_config("md17", case.cfg))
    assert worst_grad({k: v.grad for k, v in params.items()}, case.grads, 80) < 1e-8
    model = mirror(GraphAttentionTransformerMD17, case.cfg, case.state).double().train()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    with emulated_kernels():
        run_mirror("md17", model, case)
    assert worst_grad({k: p.grad for k, p in model.named_parameters()}, case.grads, 80) < 1e-6


# ------------------------------------------------------------------ dot-product attention variant (SURVEY.md 8f-4)

DP_SMALL = "reference_model_dp_small.npz"


def test_oracle_dot_product_attention_model_matches_reference_model_file():
    """``nets/dp_attention_transformer.py`` (DotProductAttention / DPTransBlock / DotProductAttentionTransformer) run by
    the reference's code vs the oracle's restatement: energies and parameter gradients of sum E^2."""
    case = load(DP_SMALL)
    energy, _forces, params = run_oracle("qm9", case, oracle_config("qm9", case.cfg, attention="dot_product"))
    assert rel_err(energy.detach(), case.t("energy")) < 1e-11
    assert worst_grad({k: v.grad for k, v in params.items()}, case.grads, 70) < 1e-8


def test_mirror_dot_product_attention_matches_reference_model_file():
    """The mirror of the dot-product variant (``ops.EdgeDot`` logits on the existing kernels; emulated here in float64)
    loaded with the reference's ``state_dict``: energies and parameter gradients against the reference-run fixture."""
    from equiformer_b200.nets.dp_attention_transformer import DotProductAttentionTransformer
    from tests._emulation import emulated_kernels
    case = load(DP_SMALL)
    model = mirror(DotProductAttentionTransformer, case.cfg, case.state).double()
    with emulated_kernels():
        energy, _forces = run_mirror("qm9", model, case)
    assert rel_err(energy.detach(), case.t("energy")) < 1e-10
    assert worst_grad({k: p.grad for k, p in model.named_parameters()}, case.grads, 70) < 1e-7


@pytest.mark.gpu
def test_cuda_dot_product_attention_matches_reference_model_file(cuda_device):
    """The dot-product variant on the CUDA kernels (float32) against the reference-run energies.  Written after the
    round-1 GPU budget ended."""
    from equiformer_b200.nets.dp_attention_transformer import DotProductAttentionTransformer
    case = load(DP_SMALL)
    model = mirror(DotProductAttentionTransformer, case.cfg, case.state).to(cuda_device)
    with torch.no_grad():
        energy = model(f_in=None, pos=case.t("pos", cuda_device, torch.float32), batch=case.t("batch", cuda_device),
                       node_atom=case.t("z", cuda_device))
    assert rel_err(energy, case.t("energy")) < 5e-5


def test_dot_product_md17_variant_matches_reference_model_file():
    """``nets/dp_attention_transformer_md17.py`` (Lmax = 3, exp-normal basis, forces by autograd) run by the reference's
    code: the oracle and the mirror (emulated kernels) against energy, forces and the gradients of the energy + force loss."""
    from equiformer_b200.nets.dp_attention_transformer import DotProductAttentionTransformerMD17
    from tests._emulation import emulated_kernels
    case = load("reference_model_dp_md17_small.npz")
    e, f, params = run_oracle("md17", case, oracle_config("md17", case.cfg, attention="dot_product"))
    assert rel_err(e.detach(), case.t("energy")) < 1e-11
    assert rel_err(f.detach(), case.t("forces")) < 1e-10
    assert worst_grad({k: v.grad for k, v in params.items()}, case.grads, 70) < 1e-8

    model = mirror(DotProductAttentionTransformerMD17, case.cfg, case.state).double().train()
    with emulated_kernels():
        e, f = run_mirror("md17", model, case)
    assert rel_err(e.detach(), case.t("energy")) < 1e-10
    assert rel_err(f.detach(), case.t("forces")) < 1e-9
    assert worst_grad({k: p.grad for k, p in model.named_parameters()}, case.grads, 70) < 1e-6


# --------------------------------------------------------------- the OC20 model file (periodic boundary conditions, tags)
OC20_SMALL = "reference_model_oc20_small.npz"


def test_oracle_oc20_model_matches_reference_model_file():
    """``nets/graph_attention_transformer_oc20.py`` run end to end (tests/golden/make_reference_golden_oc20.py: two
    triclinic periodic frames, tags, 84 atom types) vs ``oracle.model_forward_oc20``: energy and parameter gradients."""
    case = load(OC20_SMALL)
    ocfg = oracle_config("oc20", case.cfg)
    params = {k: v.requires_grad_(v.is_floating_point() and v.numel() > 0) for k, v in R.cast_params(case.state, torch.float64).items()}
    t = case.t
    edge = t("edge_index")
    energy = R.model_forward_oc20(params, ocfg, t("pos").double(), t("cell").double(), t("batch"), t("z"), t("tags"), 2,
                                  edge[0], edge[1], t("cell_offsets"))
    assert rel_err(energy, t("energy")) < 1e-10
    (energy * torch.tensor([[1.0], [-0.7]])).sum().backward()
    for k, ref in case.grads.items():
        assert rel_err(params[k].grad, ref) < 1e-6, k


def _oc20_mirror(case):
    from equiformer_b200.nets.graph_attention_transformer_oc20 import GraphAttentionTransformerOC20
    return mirror(GraphAttentionTransformerOC20, case.cfg, case.state, None, None, 1)


def test_mirror_oc20_model_matches_reference_model_file():
    """The OC20 mirror (own periodic neighbour list, kernels emulated in float64) loaded with the reference's
    ``state_dict``: same edge list as the fixture's, energy 1e-10, parameter gradients 1e-6."""
    from equiformer_b200.graph import radius_graph_pbc
    from tests._emulation import emulated_kernels
    case = load(OC20_SMALL)
    cfg = case.cfg
    model = _oc20_mirror(case).double()
    data = oc20_data(case)
    edge, offs, _d2 = radius_graph_pbc(data.pos.float(), data.batch, data.cell.float(), cfg["max_radius"], cfg["max_neighbors"])
    assert torch.equal(edge, case.t("edge_index")) and torch.equal(offs.long(), case.t("cell_offsets").long())
    with emulated_kernels():
        energy = model(data)
        (energy * torch.tensor([[1.0], [-0.7]], dtype=torch.float64)).sum().backward()
    assert rel_err(energy, case.t("energy")) < 1e-10
    for k, ref in case.grads.items():
        assert rel_err(model.get_parameter(k).grad, ref) < 1e-6, k


@pytest.mark.gpu
def test_cuda_oc20_model_matches_reference_model_file(cuda_device):
    """The OC20 mirror on CUDA (periodic neighbour-list kernels + the edge kernels) against the reference's own output."""
    from equiformer_b200.graph import radius_graph_pbc
    case = load(OC20_SMALL)
    cfg = case.cfg
    model = _oc20_mirror(case).to(cuda_device)
    data = oc20_data(case, cuda_device, torch.float32)
    edge, offs, _d2 = radius_graph_pbc(data.pos, data.batch, data.cell, cfg["max_radius"], cfg["max_neighbors"])
    assert torch.equal(edge.cpu(), case.t("edge_index"))
    assert torch.equal(offs.cpu().long(), case.t("cell_offsets").long())
    energy = model(data)
    (energy * torch.tensor([[1.0], [-0.7]], device=cuda_device)).sum().backward()
    assert rel_err(energy, case.t("energy")) < 1e-4
    worst = max(rel_err(model.get_parameter(k).grad, ref) for k, ref in case.grads.items())
    assert worst < 1e-3, worst


# --------------------------------------------------------------- the DeNS variant (nets/equiformer_md17_dens.py)
DENS_SMALL = "reference_model_dens_small.npz"


def test_mirror_dens_model_matches_reference_model_file():
    """``Equiformer_MD17_DeNS`` (force encoding + denoising head on) loaded with the reference's ``state_dict``, kernels
    emulated in float64: energies, the forces / predicted-noise output and the gradients of an energy + output loss."""
    from tests._emulation import emulated_kernels
    case, model, data = dens_setup(DENS_SMALL)
    with emulated_kernels():
        energy, dy = model(data)
        (energy.sum() + (dy ** 2).sum()).backward()
    assert rel_err(energy, case.t("energy")) < 1e-10
    assert rel_err(dy, case.t("dy")) < 1e-9
    for k, ref in case.grads.items():
        assert rel_err(model.get_parameter(k).grad, ref) < 1e-6, k


@pytest.mark.gpu
def test_cuda_dens_model_matches_reference_model_file(cuda_device):
    case, model, data = dens_setup(DENS_SMALL, cuda_device, torch.float32)
    energy, dy = model(data)
    (energy.sum() + (dy ** 2).sum()).backward()
    assert rel_err(energy, case.t("energy")) < 1e-4
    assert rel_err(dy, case.t("dy")) < 3e-4
    worst = max(rel_err(model.get_parameter(k).grad, ref) for k, ref in case.grads.items())
    assert worst < 2e-3, worst
