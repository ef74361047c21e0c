"""The OC20 E(3) configuration (``OC20_L1_256_E3_NONLINEAR``, l1_256_e3_nonlinear_g@2_local.yml), its generated
depth-wise product kernel (codegen tag ``oc20_l1_e3``) and the parity branch of every layer.

CPU: the configuration against its yml; the full-size ``state_dict`` / ``no_weight_decay()`` table and the small OC20,
QM9 and MD17 E(3) runs of the reference's model files (tests/golden/reference_model_e3_small.npz,
tests/golden/make_reference_golden_e3.py) against the oracle and the mirror (kernels emulated in float64); the committed
``csrc/gen/dtp_gen_oc20_l1_e3.cu`` against the plan every depth-wise product of the model resolves to; the fast-route
predicates of the full-size layer.

-m gpu: the generated forward, backward (grad_x + grad_w) and grad_y kernels of the E(3) plan against the fp64 table walk
of tests/_emulation.py below and past the grid cap, per-edge and shared weights, gathered operands with the radial
offset; a bitwise-repeatable backward; the CUDA OC20, QM9 and MD17 E(3) models against the fixture, captured and
eager; a full-size E(3) block against the float64 oracle; the graph-captured training step against the eager step with
attention dropout on.
"""
from __future__ import annotations

import json
import os
import re

import numpy as np
import pytest
import torch

from oracle import e3nn_ref as e3
from oracle import equiformer_ref as R
from tests import _emulation as emu
from tests.helpers import rel_err
from tests.reference_fixtures import GOLDEN, load, mirror, oracle_config, run_mirror, run_oracle, worst_grad

FIXTURE = "reference_model_e3_small.npz"
GEN_FILE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "equiformer_b200", "csrc", "gen",
                        "dtp_gen_oc20_l1_e3.cu")
E3_PLAN = ("256x0e+64x0o+64x1e+64x1o", "1x0e+1x1o")


# ------------------------------------------------------------------------------------------------ configuration, table
def test_oc20_e3_configuration_matches_the_yml():
    """The model block of oc20/configs/is2re/all/graph_attention_transformer/l1_256_e3_nonlinear_g@2_local.yml:5-31."""
    from equiformer_b200.nets.graph_attention_transformer_oc20 import OC20_L1_256_E3_NONLINEAR
    yml = dict(irreps_node_embedding="256x0e+64x0o+64x1e+64x1o", num_layers=6, irreps_node_attr="1x0e",
               use_node_attr=False, irreps_sh="1x0e+1x1o", max_radius=5.0, number_of_basis=128, fc_neurons=[64, 64],
               use_atom_edge_attr=False, irreps_atom_edge_attr="1x0e", irreps_feature="512x0e",
               irreps_head="32x0e+8x0o+8x1e+8x1o", num_heads=8, irreps_pre_attn="256x0e+64x0o+64x1e+64x1o",
               rescale_degree=False, nonlinear_message=True, irreps_mlp_mid="768x0e+192x0o+192x1e+192x1o",
               norm_layer="layer", alpha_drop=0.2, proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0, otf_graph=True,
               use_pbc=True, max_neighbors=500)
    assert OC20_L1_256_E3_NONLINEAR == yml


def _full_model(**over):
    from equiformer_b200.nets import model_entrypoint
    from equiformer_b200.nets.graph_attention_transformer_oc20 import OC20_L1_256_E3_NONLINEAR
    return model_entrypoint("graph_attention_transformer_oc20")(**dict(OC20_L1_256_E3_NONLINEAR, **over))


def test_full_size_state_dict_and_no_weight_decay_match_the_reference():
    g = np.load(os.path.join(GOLDEN, FIXTURE))
    model = _full_model()
    assert len(model.blocks) == 6 and all(b.ga.nonlinear_message for b in model.blocks)
    mine = {k: list(v.shape) for k, v in model.state_dict().items() if not k.endswith("tp.output_mask")}
    assert mine == json.loads(str(g["oc20_full/state"]))
    assert sorted(model.no_weight_decay()) == json.loads(str(g["oc20_full/no_weight_decay"]))
    assert sum(p.numel() for p in model.parameters()) == 8766851


def _model_plans(model):
    yield "edge_deg_embed.dw", model.edge_deg_embed.dw.tp.plan
    for i, b in enumerate(model.blocks):
        yield f"blocks.{i}.ga.sep_act", b.ga.sep_act.dtp.tp.plan
        yield f"blocks.{i}.ga.sep_value", b.ga.sep_value.dtp.tp.plan


def test_committed_generated_kernel_is_the_plan_of_every_depthwise_product():
    """The signature the committed file registers is ``plan_signature`` of the plan that the edge-degree embedding and
    both products of every block build, and the file is what the generator emits today: a drift in either would send
    the model back to the generic kernels without a word."""
    from equiformer_b200 import codegen
    assert ("oc20_l1_e3",) + E3_PLAN in codegen.KNOWN_CONFIGS
    with open(GEN_FILE) as f:
        text = f.read()
    sig = int(re.search(r"GeneratedKernels kernels = \{0x([0-9a-f]{16})ULL", text).group(1), 16)
    plan = codegen.plan_for(*E3_PLAN)
    assert codegen.supported(plan) and codegen.plan_signature(plan) == sig
    assert codegen.generate(plan, "oc20_l1_e3") == text
    model = _full_model()
    names = []
    for name, p in _model_plans(model):
        assert codegen.plan_signature(p) == sig, name
        names.append(name)
    assert len(names) == 1 + 2 * 6
    # the four output groups are separate even / odd groups at l = 0 and l = 1
    assert [(l, p, m) for l, p, m in plan.out_groups] == [(0, 1, 320), (0, -1, 128), (1, 1, 192), (1, -1, 384)]
    assert len(plan.paths) == 10 and {p.out_group for p in plan.paths} == {0, 1, 2, 3}


def test_fast_route_predicates_hold_at_full_size():
    from equiformer_b200 import ops
    model = _full_model()
    assert ops.dtp_linear_supported(model.edge_deg_embed.dw.tp.plan)
    assert model.edge_deg_embed._fuse_proj
    for i, b in enumerate(model.blocks):
        ga = b.ga
        assert ga._alpha_single_gemm and ga._gate_layout is not None and ga._fuse_act and ga._fuse_value, i
        assert b.norm_1.supports_planar and b.norm_2.supports_planar, i
        assert b.ffn._gate_layout is not None, i
    assert all(b.supports_planar for b in model.blocks[:-1])         # the last block projects to irreps_feature


# ------------------------------------------------------------------------------------------------ reference fixture
@pytest.mark.parametrize("kind", ["oc20", "qm9", "md17"])
def test_oracle_matches_reference_e3_model_files(kind):
    case = load(FIXTURE, kind)
    assert any(ir.endswith("o") for ir in case.cfg["irreps_node_embedding"].split("+"))
    energy, forces, params = run_oracle(kind, case, oracle_config(kind, case.cfg))
    if forces is not None:
        assert rel_err(forces.detach(), case.t("forces")) < 1e-10
    assert rel_err(energy.detach(), case.t("energy")) < 1e-10
    assert worst_grad({k: v.grad for k, v in params.items()}, case.grads, 51) < 1e-8


def _mirror(kind, case):
    from equiformer_b200.nets.graph_attention_transformer import GraphAttentionTransformer
    from equiformer_b200.nets.graph_attention_transformer_md17 import GraphAttentionTransformerMD17
    from equiformer_b200.nets.graph_attention_transformer_oc20 import GraphAttentionTransformerOC20
    if kind == "oc20":
        return mirror(GraphAttentionTransformerOC20, case.cfg, case.state, None, None, 1)
    return mirror({"qm9": GraphAttentionTransformer, "md17": GraphAttentionTransformerMD17}[kind], case.cfg, case.state)


@pytest.mark.parametrize("kind", ["oc20", "qm9", "md17"])
def test_mirror_with_emulated_kernels_matches_reference_e3_model_files(kind):
    from tests._emulation import emulated_kernels
    case = load(FIXTURE, kind)
    model = _mirror(kind, case).double()
    with emulated_kernels():
        energy, forces = run_mirror(kind, model, case)
    assert rel_err(energy.detach(), case.t("energy")) < 1e-10
    if forces is not None:
        assert rel_err(forces.detach(), case.t("forces")) < 1e-10
    assert worst_grad({k: p.grad for k, p in model.named_parameters()}, case.grads, 51) < 1e-7


# ------------------------------------------------------------------------------------------------ GPU: generated kernels
def _e3_plan():
    from equiformer_b200 import codegen
    plan = codegen.plan_for(*E3_PLAN)
    assert plan.generated and plan.info()["generated"] == 1
    return plan


@pytest.fixture
def _free_cached_memory():
    yield
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["below_cap", "two_passes", "partial_third_pass"])
@pytest.mark.parametrize("shared", [False, True])
def test_generated_e3_kernels_match_the_table_walk(cuda_device, _free_cached_memory, shared, size):
    """forward (all four output groups), grad_x, grad_y and grad_xw of the generated kernels against the fp64 table walk,
    with per-edge weights (sep_act, the edge-degree embedding) and shared weights (sep_value); below the cap every warp
    takes one step, past it the later and partial passes and the shared-weight sums carried across them."""
    from equiformer_b200 import ops
    from tests.test_gpu_multipass import CHUNK, TOL, _compare_chunked, _gen_dtp_pass, _randn, _report, _rows, _size
    plan = _e3_plan()
    C, G = _gen_dtp_pass(plan)
    E = 5003 if size == "below_cap" else _size(C, G, size)
    _report(f"dtp oc20_l1_e3 {'shared' if shared else 'per-edge'} w", E, C)
    gen = torch.Generator(device=cuda_device).manual_seed(E + shared)
    xs = [_randn(gen, E, 2 * l + 1, mul) for l, mul in plan.in1_blocks]
    y = _randn(gen, E, plan.d_y)
    w = _randn(gen, plan.weight_numel) if shared else _randn(gen, E, plan.weight_numel)
    w_at = (lambda a, b: w.double()) if shared else (lambda a, b: w[a:b].double())

    out = ops.dtp_forward_raw(plan, xs, y, w)
    assert [tuple(o.shape[1:]) for o in out] == [(1, 320), (1, 128), (3, 192), (3, 384)]
    _compare_chunked(out, lambda a, b: emu.dtp_forward_raw(plan, _rows(xs, a, b), y[a:b].double(), w_at(a, b)),
                     E, "forward", C)
    del out
    gs = [_randn(gen, E, 2 * l + 1, mul) for l, _p, mul in plan.out_groups]
    gx_ref = lambda a, b: emu.dtp_grad_x_raw(plan, _rows(gs, a, b), y[a:b].double(), w_at(a, b))
    _compare_chunked(ops.dtp_grad_x_raw(plan, gs, y, w), gx_ref, E, "grad_x", C)
    gy = ops.dtp_grad_y_raw(plan, xs, w, gs, y)
    _compare_chunked([gy], lambda a, b: [emu.dtp_grad_y_raw(plan, _rows(xs, a, b), w_at(a, b), _rows(gs, a, b),
                                                            y[a:b].double())], E, "grad_y", C)
    del gy
    gw_ref = lambda a, b: emu.dtp_grad_w_raw(plan, _rows(xs, a, b), y[a:b].double(), _rows(gs, a, b), shared)
    gx, gw = ops.dtp_grad_xw_raw(plan, xs, y, w, gs)
    _compare_chunked(gx, gx_ref, E, "grad_xw x", C)
    if shared:
        total = sum(gw_ref(a, min(E, a + CHUNK)) for a in range(0, E, CHUNK))
        assert rel_err(gw, total) < TOL, ("grad_xw shared w", rel_err(gw, total))
    else:
        _compare_chunked([gw], lambda a, b: [gw_ref(a, b)], E, "grad_xw w", C)


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["below_cap", "partial_third_pass"])
def test_generated_e3_kernels_gathered_with_offset(cuda_device, _free_cached_memory, size):
    """x = A[src] + B[dst] gathered in the kernel and the radial offset added to the per-edge weights (the route of
    sep_act and of the edge-degree embedding)."""
    from equiformer_b200 import ops
    from tests.test_gpu_multipass import _compare_chunked, _gen_dtp_pass, _randn, _rows, _size
    plan = _e3_plan()
    C, G = _gen_dtp_pass(plan)
    E = 4099 if size == "below_cap" else _size(C, G, size)
    n_nodes = max(E // 16, 7)
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


@pytest.mark.gpu
def test_generated_e3_backward_is_bitwise_repeatable(cuda_device):
    """Per-edge-weight backward (grad_x + grad_w: one writer per output element) and grad_y (per-warp shared-memory
    slots summed in a fixed order) give identical bits on every call.  The shared-weight gradient is left out: its
    warps add their partials into one shared-memory row with atomics, as in the other generated plans."""
    from equiformer_b200 import ops
    plan = _e3_plan()
    E = 40000
    gen = torch.Generator(device=cuda_device).manual_seed(3)
    xs = [torch.randn(E, 2 * l + 1, mul, generator=gen, device=cuda_device) for l, mul in plan.in1_blocks]
    y = torch.randn(E, plan.d_y, generator=gen, device=cuda_device)
    w = torch.randn(E, plan.weight_numel, generator=gen, device=cuda_device)
    gs = [torch.randn(E, 2 * l + 1, mul, generator=gen, device=cuda_device) for l, _p, mul in plan.out_groups]
    runs = []
    for _ in range(2):
        gx, gw = ops.dtp_grad_xw_raw(plan, xs, y, w, gs)
        runs.append([*gx, gw, ops.dtp_grad_y_raw(plan, xs, w, gs, y)])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ GPU: model level
def _csr(batch, src, dst, row_ptr):
    from equiformer_b200 import ops
    csr = ops.Graph.__new__(ops.Graph)
    csr.n_nodes, csr.n_edges, csr.perm = int(batch.shape[0]), int(src.numel()), None
    csr.src, csr.dst, csr.row_ptr = src, dst, row_ptr
    csr._src_perm = csr._src_row_ptr = None
    return csr


def _graph_inputs(kind, case, dev):
    """(graph, edge_vec for OC20) of the fixture's frames: the reference's periodic edge list for OC20, the oracle's
    radius graph otherwise."""
    from equiformer_b200 import ops
    t = lambda k: case.t(k, dev)
    pos, batch = t("pos"), t("batch")
    if kind == "oc20":
        edge = t("edge_index")
        vec = R.pbc_edge_vectors(pos, t("cell"), batch, edge[0], edge[1], t("cell_offsets"))
        return ops.Graph(edge[0], edge[1], pos.shape[0]), vec
    return ops.Graph(*R.radius_graph(pos, 5.0, batch), pos.shape[0]), None


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["oc20", "qm9", "md17"])
def test_cuda_e3_models_match_reference_model_files(cuda_device, kind):
    """The fixture's loss and parameter gradients through ``GraphedStep`` (capture + replay), then eager (energy, MD17
    forces, gradients).  The captured step runs first, as in the other capture tests."""
    from equiformer_b200.graphs import GraphedStep
    from equiformer_b200.parallel import FlatGradAllReduce
    case = load(FIXTURE, kind)
    model = _mirror(kind, case).to(cuda_device)
    t = lambda k: case.t(k, cuda_device)
    pos, batch, z = t("pos"), t("batch"), t("z")
    graph, edge_vec = _graph_inputs(kind, case, cuda_device)
    bucket = FlatGradAllReduce(model.parameters())
    n_graphs = 1 if kind == "md17" else 2

    def captured(pos, edge_vec, batch, z, tags, src, dst, row_ptr):
        csr = _csr(batch, src, dst, row_ptr)
        if kind == "oc20":
            e = model.forward_edges(edge_vec, batch, z, tags, src, dst, graph=csr, n_graphs=n_graphs)
            return (e ** 2).sum()
        if kind == "qm9":
            e = model.forward_edges(pos, batch, z, src, dst, graph=csr, n_graphs=n_graphs)
            return (e ** 2).sum()
        e, f = model.forward_edges(z, pos.detach().requires_grad_(True), batch, src, dst, graph=csr, n_graphs=n_graphs)
        return e.sum() + (f ** 2).sum()

    step = GraphedStep(captured, bucket)
    tags = t("tags") if kind == "oc20" else torch.zeros_like(z)
    vec = edge_vec if edge_vec is not None else torch.zeros(graph.n_edges, 3, device=cuda_device)
    for _ in range(2):
        loss = step((int(pos.shape[0]), graph.n_edges), [pos, vec, batch, z, tags, graph.src, graph.dst,
                                                          graph.row_ptr]).clone()
    assert step.captures == 1
    energy_ref = case.t("energy")
    ref_loss = energy_ref.sum() + (case.t("forces") ** 2).sum() if kind == "md17" else (energy_ref ** 2).sum()
    assert abs(float(loss) - float(ref_loss)) / abs(float(ref_loss)) < 1e-4
    assert worst_grad({k: q.grad for k, q in model.named_parameters()}, case.grads, 51) < 1e-3

    bucket.zero_grad()
    energy, forces = run_mirror(kind, model, case, cuda_device, torch.float32)
    assert rel_err(energy, case.t("energy")) < 5e-5
    if forces is not None:
        assert rel_err(forces, case.t("forces")) < 2e-4
    assert worst_grad({k: p.grad for k, p in model.named_parameters()}, case.grads, 51) < 1e-3


@pytest.mark.gpu
def test_full_size_e3_block_matches_the_oracle(cuda_device):
    """One full-size ``OC20_L1_256_E3_NONLINEAR`` block on 4 synthetic periodic frames, its depth-wise products on the
    generated kernels: output and parameter / input gradients against the float64 oracle on the same inputs."""
    from equiformer_b200 import ops
    from tests.test_oc20_aux import _frames
    torch.manual_seed(0)
    model = _full_model(num_layers=2).to(cuda_device).eval()
    blk = model.blocks[0]
    assert blk.supports_planar and blk.ga.sep_act.dtp.tp.plan.generated and blk.ga.sep_value.dtp.tp.plan.generated
    pos, batch, _z, _tags, src, dst, edge_vec = _frames(cuda_device, n_frames=4, seed=0)
    E, n = int(src.numel()), int(pos.shape[0])
    print(f"[full size] {n} atoms, {E} edges")
    g = torch.Generator().manual_seed(1)
    x = torch.randn(n, blk.irreps_node_input.dim, generator=g).to(cuda_device)
    sh = e3.spherical_harmonics([0, 1], edge_vec.double().cpu(), True, "component").float().to(cuda_device)
    rbf = torch.rand(E, 128, generator=g).to(cuda_device)
    G = torch.randn(n, blk.irreps_node_output.dim, generator=g).to(cuda_device)
    graph = ops.Graph(src, dst, n)
    xi = x.clone().requires_grad_(True)
    node_attr = torch.ones(n, 1, device=cuda_device)
    out = blk(xi, node_attr, src, dst, sh, rbf, batch, graph=graph)
    out.backward(G)

    params = {k: v.requires_grad_(v.is_floating_point() and v.numel() > 0)
              for k, v in R.cast_params(blk.state_dict(), torch.float64).items()}
    cfg = R.Config(irreps_node_embedding="256x0e+64x0o+64x1e+64x1o", irreps_sh="1x0e+1x1o",
                   irreps_head="32x0e+8x0o+8x1e+8x1o", irreps_mlp_mid="768x0e+192x0o+192x1e+192x1o", num_heads=8,
                   nonlinear_message=True)
    emb = e3.parse_irreps(cfg.irreps_node_embedding)
    cpu64 = lambda v: v.detach().cpu().double()
    x64 = cpu64(x).requires_grad_(True)
    prefixed = {f"blk.{k}": v for k, v in params.items()}
    ref = R.trans_block(prefixed, "blk", cfg, emb, emb, x64, torch.ones(n, 1, dtype=torch.float64), src.cpu(), dst.cpu(),
                        cpu64(sh), cpu64(rbf))
    (ref * cpu64(G)).sum().backward()
    assert rel_err(out, ref) < 1e-4
    assert rel_err(xi.grad, x64.grad) < 1e-4
    worst = max((rel_err(blk.get_parameter(k).grad, v.grad), k) for k, v in params.items() if v.grad is not None)
    assert worst[0] < 1e-3, worst


@pytest.mark.gpu
def test_graphed_e3_oc20_step_matches_eager(cuda_device):
    """2-block ``OC20_L1_256_E3_NONLINEAR`` (``alpha_drop=0.2``) through ``graphs.GraphedStep``: each replay's loss and
    gradients equal the eager step's from the same generator state, so the replay draws the same dropout masks."""
    from equiformer_b200.graphs import GraphedStep
    from equiformer_b200.parallel import FlatGradAllReduce
    from tests.test_oc20_aux import _frames
    torch.manual_seed(0)
    model = _full_model(num_layers=2).to(cuda_device).train()
    assert model.blocks[0].ga.alpha_dropout.p == 0.2
    assert model.edge_deg_embed.dw.tp.plan.generated
    bucket = FlatGradAllReduce(model.parameters())
    pos, batch, z, tags, src, dst, edge_vec = _frames(cuda_device, seed=3)
    target = torch.randn(4, 1, generator=torch.Generator().manual_seed(7)).to(cuda_device)
    n = int(pos.shape[0])
    row_ptr = torch.zeros(n + 1, dtype=torch.int64, device=cuda_device)
    torch.cumsum(torch.zeros(n, dtype=torch.int64, device=cuda_device).index_add_(0, dst, torch.ones_like(dst)), 0,
                 out=row_ptr[1:])

    def captured(edge_vec, target, batch, z, tags, src, dst, row_ptr):
        energy = model.forward_edges(edge_vec, batch, z, tags, src, dst, graph=_csr(batch, src, dst, row_ptr),
                                     n_graphs=target.shape[0])
        return (energy - target).abs().mean()

    step = GraphedStep(captured, bucket)
    key = (n, int(src.numel()), 4)
    inputs = [edge_vec, target, batch, z, tags, src, dst, row_ptr]
    step(key, inputs)
    assert step.captures == 1
    losses = []
    for _ in range(2):
        state = torch.cuda.get_rng_state()
        loss_g = step(key, inputs).clone()
        grads_g = bucket.flat.clone()
        after = torch.cuda.get_rng_state()
        torch.cuda.set_rng_state(state)
        bucket.zero_grad()
        loss_e = (model.forward_edges(edge_vec, batch, z, tags, src, dst, n_graphs=4) - target).abs().mean()
        loss_e.backward()
        assert rel_err(loss_g, loss_e.detach()) < 1e-5
        assert rel_err(grads_g, bucket.flat) < 1e-5
        assert torch.equal(torch.cuda.get_rng_state(), after)
        losses.append(float(loss_g))
    assert losses[0] != losses[1]
    assert step.captures == 1
