"""The linear-message graph attention (``GraphAttention`` with ``nonlinear_message=False``) on the fused kernels
``eqf_attn_mlp_softmax_aggregate`` / ``_bwd`` (``ops.MlpSoftmaxAggregate``), and the OC20 ``l1_256`` configuration.

CPU: ``OC20_L1_256`` against its yml; the full-size ``state_dict`` / ``no_weight_decay()`` table and the small QM9, MD17
and OC20 linear-message runs of the reference's model files (tests/golden/reference_model_linear_small.npz,
tests/golden/make_reference_golden_linear.py) against the oracle and the mirror (existing chain, kernels emulated in
float64); the host logic of ``MlpSoftmaxAggregate`` with float64 stand-ins for the two raw kernels: gradcheck, and its
``create_graph`` route against the chain it is rebuilt from.

-m gpu: the kernels against the chain (the ``alpha_act`` statement -> ``SegSoftmax`` -> ``* keep`` -> ``AttnAggregate``
on the contiguous value scalars) on the OC20 and QM9 / MD17 L2 head layouts, with and without the dropout mask,
including zero-in-degree nodes and node counts past the grid cap; bitwise-repeatable backward; double backward; the CUDA
models against the fixture; a full-size ``OC20_L1_256`` layer against the chain; the graph-captured training step
against the eager step with attention dropout on.
"""
from __future__ import annotations

import json
import os
import types

import numpy as np
import pytest
import torch

from tests import _emulation as emu
from tests.helpers import rel_err
from tests.reference_fixtures import GOLDEN, load, mirror, oracle_config, run_mirror, run_oracle, worst_grad

FIXTURE = "reference_model_linear_small.npz"
TOL = 2e-5                      # kernel vs the float32 chain

# head layouts: (H, A, value ds, value Cs) - the value scalars (R = A channels per head) lead
LAYOUTS = {"oc20_l1": (8, 32, (1, 3), (256, 128)),                 # 8 x (32x0e+16x1e), alpha 32 per head
           "qm9_md17_l2": (4, 32, (1, 3, 5), (128, 64, 32))}       # 4 x (32x0e+16x1e+8x2e)


# ------------------------------------------------------------------------------------------------ configuration, table
def test_oc20_l1_256_configuration_matches_the_yml():
    """The model block of oc20/configs/is2re/all/graph_attention_transformer/l1_256_g@2_local.yml:5-31, restated."""
    from equiformer_b200.nets.graph_attention_transformer_oc20 import OC20_L1_256
    yml = dict(irreps_node_embedding="256x0e+128x1e", num_layers=8, irreps_node_attr="1x0e", use_node_attr=False,
               irreps_sh="1x0e+1x1e", max_radius=5.0, number_of_basis=128, fc_neurons=[64, 64], use_atom_edge_attr=False,
               irreps_atom_edge_attr="1x0e", irreps_feature="512x0e", irreps_head="32x0e+16x1e", num_heads=8,
               irreps_pre_attn="256x0e+128x1e", rescale_degree=False, nonlinear_message=False,
               irreps_mlp_mid="768x0e+384x1e", norm_layer="layer", alpha_drop=0.2, proj_drop=0.0, out_drop=0.0,
               drop_path_rate=0.0, otf_graph=True, use_pbc=True, max_neighbors=500)
    assert OC20_L1_256 == yml


def test_full_size_state_dict_and_no_weight_decay_match_the_reference():
    from equiformer_b200.nets import model_entrypoint
    from equiformer_b200.nets.graph_attention_transformer_oc20 import OC20_L1_256
    g = np.load(os.path.join(GOLDEN, FIXTURE))
    model = model_entrypoint("graph_attention_transformer_oc20")(**OC20_L1_256)
    assert len(model.blocks) == 8 and all(not b.ga.nonlinear_message for b in model.blocks)
    assert all(b.ga._mlp_layout is not None for b in model.blocks)
    mine = {k: list(v.shape) for k, v in model.state_dict().items() if not k.endswith("tp.output_mask")}
    assert mine == json.loads(str(g["oc20_full/state"]))
    assert sorted(model.no_weight_decay()) == json.loads(str(g["oc20_full/no_weight_decay"]))


# ------------------------------------------------------------------------------------------------ reference fixture
def _mirror(kind, case):
    from equiformer_b200.nets.graph_attention_transformer import GraphAttentionTransformer
    from equiformer_b200.nets.graph_attention_transformer_md17 import GraphAttentionTransformerMD17
    from equiformer_b200.nets.graph_attention_transformer_oc20 import GraphAttentionTransformerOC20
    if kind == "oc20":
        return mirror(GraphAttentionTransformerOC20, case.cfg, case.state, None, None, 1)
    return mirror({"qm9": GraphAttentionTransformer, "md17": GraphAttentionTransformerMD17}[kind], case.cfg, case.state)


@pytest.mark.parametrize("kind", ["qm9", "md17", "oc20"])
def test_oracle_matches_reference_linear_message_model_files(kind):
    case = load(FIXTURE, kind)
    energy, forces, params = run_oracle(kind, case, oracle_config(kind, case.cfg))
    if forces is not None:
        assert rel_err(forces.detach(), case.t("forces")) < 1e-10
    assert rel_err(energy.detach(), case.t("energy")) < 1e-10
    assert worst_grad({k: v.grad for k, v in params.items()}, case.grads, 51) < 1e-8


@pytest.mark.parametrize("kind", ["qm9", "md17", "oc20"])
def test_mirror_with_emulated_kernels_matches_reference_linear_message_model_files(kind):
    """float64 CPU stand-ins: the predicate of the fused kernel is false, so the existing chain runs."""
    from tests._emulation import emulated_kernels
    case = load(FIXTURE, kind)
    model = _mirror(kind, case).double()
    with emulated_kernels():
        energy, forces = run_mirror(kind, model, case)
    assert rel_err(energy.detach(), case.t("energy")) < 1e-10
    if forces is not None:
        assert rel_err(forces.detach(), case.t("forces")) < 1e-10
    assert worst_grad({k: p.grad for k, p in model.named_parameters()}, case.grads, 51) < 1e-7


# ------------------------------------------------------------------------------------------------ host logic (float64)
@pytest.fixture
def stand_ins(monkeypatch):
    from equiformer_b200 import ops
    monkeypatch.setattr(ops, "mlp_softmax_aggregate_raw", emu.mlp_softmax_aggregate_raw)
    monkeypatch.setattr(ops, "mlp_softmax_aggregate_bwd_raw", emu.mlp_softmax_aggregate_bwd_raw)
    with emu.emulated_kernels():
        yield ops


def _small_case(ops, dtype=torch.float64, seed=0):
    g = torch.Generator().manual_seed(seed)
    H, A = 2, 4
    lay = ops.MlpAttnLayout(ops.HeadLayout((1, 3), (8, 4), H), A, 1.7, 0.2)
    dst = torch.tensor([0, 0, 0, 2, 2, 3, 3, 3, 3, 5])          # nodes 1 and 4: no incoming edge
    src = torch.randint(0, 6, (dst.numel(),), generator=g)
    graph = ops.Graph(src, dst, 6)
    E = dst.numel()
    alpha_dot = torch.randn(H, A, generator=g, dtype=dtype).requires_grad_(True)
    t0 = torch.randn(E, lay.width, generator=g, dtype=dtype).requires_grad_(True)
    Vs = [torch.randn(E, 3, 4, generator=g, dtype=dtype).requires_grad_(True)]
    keep = (torch.rand(E, H, generator=g) > 0.3).to(dtype) / 0.7
    return lay, graph, alpha_dot, t0, Vs, keep


@pytest.mark.parametrize("masked", [False, True])
def test_mlp_softmax_aggregate_gradcheck(stand_ins, masked):
    ops = stand_ins
    lay, graph, alpha_dot, t0, Vs, keep = _small_case(ops)
    keep = keep if masked else None
    fn = lambda ad, tt, *vv: ops.MlpSoftmaxAggregate.apply(lay, graph, keep, ad, tt, *vv)
    assert torch.autograd.gradcheck(fn, (alpha_dot, t0, *Vs), eps=1e-6, atol=1e-7)


def _chain(ops, lay, graph, keep, alpha_dot, t0, Vs):
    a = ops.SegSoftmax.apply(ops.mlp_logits_torch(lay, t0, alpha_dot).contiguous(), graph)
    vals = [ops.mlp_value_scalars(lay, t0).contiguous(), *[v.contiguous() for v in Vs]]
    return ops.AttnAggregate.apply(lay.head, graph, a if keep is None else a * keep, *vals)


@pytest.mark.parametrize("masked", [False, True])
def test_create_graph_route_equals_the_chain(stand_ins, masked):
    """First and second derivatives through ``MlpSoftmaxAggregate`` under ``create_graph`` against the chain."""
    ops = stand_ins
    lay, graph, alpha_dot, t0, Vs, keep = _small_case(ops, seed=1)
    keep = keep if masked else None
    g = torch.Generator().manual_seed(5)
    Gs = [torch.randn(6, d, C, generator=g, dtype=torch.float64) for d, C in zip(lay.head.ds, lay.head.Cs)]
    ins = (alpha_dot, t0, *Vs)
    results = []
    for f in (lambda: ops.MlpSoftmaxAggregate.apply(lay, graph, keep, *ins),
              lambda: _chain(ops, lay, graph, keep, alpha_dot, t0, Vs)):
        outs = f()
        first = torch.autograd.grad(outs, ins, Gs, create_graph=True)
        w = [torch.randn(t.shape, generator=torch.Generator().manual_seed(9 + i), dtype=torch.float64)
             for i, t in enumerate(first)]
        second = torch.autograd.grad(sum((a * b).sum() for a, b in zip(first, w)), ins)
        results.append((outs, first, second))
    for a, b in zip(*[sum((list(r) for r in res), []) for res in results]):
        assert rel_err(a.detach(), b.detach()) < 1e-12


def test_predicate_is_false_on_the_stand_ins():
    from equiformer_b200 import ops
    lay = ops.MlpAttnLayout(ops.HeadLayout((1, 3), (256, 128), 8), 32, 1.7, 0.2)
    with emu.emulated_kernels():
        assert not ops.mlp_softmax_aggregate_ok(lay, torch.zeros(4, lay.width), types.SimpleNamespace(n_edges=4))


@pytest.mark.gpu
def test_unsupported_layouts_keep_the_chain(cuda_device):
    """The predicate rejects them and the kernel returns EQF_ERR_UNSUPPORTED for them."""
    from equiformer_b200 import _lib, ops
    odd = ops.MlpAttnLayout(ops.HeadLayout((1, 3, 5), (16, 8, 4), 2), 8, 1.7, 0.2)      # 2 channels per head of 2e
    wide = ops.MlpAttnLayout(ops.HeadLayout((1, 3), (512, 256), 8), 64, 1.7, 0.2)     # 512 alpha channels per edge
    graph = ops.Graph(torch.zeros(4, dtype=torch.long, device=cuda_device),
                      torch.tensor([0, 0, 1, 1], device=cuda_device), 2)
    for bad in (odd, wide):
        t0 = torch.zeros(4, bad.width, device=cuda_device)
        assert not ops.mlp_softmax_aggregate_ok(bad, t0, graph)
        Vs = [torch.zeros(4, d, C, device=cuda_device) for d, C in zip(bad.head.ds[1:], bad.head.Cs[1:])]
        ad = torch.zeros(bad.head.n_heads, bad.n_alpha, device=cuda_device)
        with pytest.raises(_lib.EqfError, match="code -3"):
            ops.mlp_softmax_aggregate_raw(bad, t0, Vs, ad, graph)


# ------------------------------------------------------------------------------------------------ GPU: kernels vs chain
def _graph_case(ops, dev, H, A, ds, Cs, n_nodes, seed):
    """Random destination-sorted graph with zero-in-degree nodes (every 7th node)."""
    g = torch.Generator().manual_seed(seed)
    deg = torch.randint(0, 40, (n_nodes,), generator=g)
    deg[::7] = 0
    dst = torch.repeat_interleave(torch.arange(n_nodes), deg)
    src = torch.randint(0, n_nodes, (dst.numel(),), generator=g)
    graph = ops.Graph(src.to(dev), dst.to(dev), n_nodes)
    lay = ops.MlpAttnLayout(ops.HeadLayout(ds, Cs, H), A, 1.6765, 0.2)
    E = dst.numel()
    alpha_dot = (0.3 * torch.randn(H, A, generator=g)).to(dev)
    t0 = torch.randn(E, lay.width, generator=g).to(dev)
    Vs = [torch.randn(E, d, C, generator=g).to(dev) for d, C in zip(ds[1:], Cs[1:])]
    keep = ((torch.rand(E, H, generator=g) > 0.2).float() / 0.8).to(dev)
    Gs = [torch.randn(n_nodes, d, C, generator=g).to(dev) for d, C in zip(ds, Cs)]
    return lay, graph, alpha_dot, t0, Vs, keep, Gs, deg


def _check_against_chain(ops, lay, graph, alpha_dot, t0, Vs, keep, Gs, deg, tol=TOL):
    ad = alpha_dot.clone().requires_grad_(True)
    tl = t0.clone().requires_grad_(True)
    vl = [v.clone().requires_grad_(True) for v in Vs]
    z = ops.mlp_logits_torch(lay, tl, ad)
    alpha_ref = ops.segment_softmax(z.contiguous(), graph)
    vals = [ops.mlp_value_scalars(lay, tl).contiguous(), *vl]
    outs_ref = ops.attention_aggregate(lay.head, graph, alpha_ref if keep is None else alpha_ref * keep, vals)
    grads_ref = torch.autograd.grad(outs_ref, [ad, tl, *vl], Gs)
    outs, alpha = ops.mlp_softmax_aggregate_raw(lay, t0, Vs, alpha_dot, graph, keep)
    assert rel_err(alpha, alpha_ref) < tol
    for a, b in zip(outs, outs_ref):
        assert rel_err(a, b) < tol
    empty = (deg == 0).nonzero().flatten().to(outs[0].device)
    assert all(bool((o.index_select(0, empty) == 0).all()) for o in outs)
    gt0, gVs, gdot = ops.mlp_softmax_aggregate_bwd_raw(lay, Gs, t0, Vs, alpha_dot, alpha, graph, keep)
    for what, a, b in zip(["alpha_dot", "t0"] + ["V"] * len(gVs), [gdot.view_as(alpha_dot), gt0, *gVs], grads_ref):
        assert rel_err(a, b) < tol, (what, rel_err(a, b))
    return gt0, gVs, gdot


@pytest.mark.gpu
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_kernels_match_the_chain(cuda_device, name, masked):
    """Forward (outputs, alpha) and backward (the whole t0 row, the l >= 1 blocks, alpha_dot) against the chain; every
    7th node has no incoming edge."""
    from equiformer_b200 import ops
    H, A, ds, Cs = LAYOUTS[name]
    lay, graph, alpha_dot, t0, Vs, keep, Gs, deg = _graph_case(ops, cuda_device, H, A, ds, Cs, 300, seed=len(name) + masked)
    assert ops.mlp_softmax_aggregate_ok(lay, t0, graph)
    _check_against_chain(ops, lay, graph, alpha_dot, t0, Vs, keep if masked else None, Gs, deg)


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["two_passes", "partial_third_pass"])
def test_kernels_past_the_grid_cap(cuda_device, size):
    """min(ceil(N / 8), 132 * 16) CTAs of 8 warps, one node per warp step: N = 2 C and 2 C + C / 3 nodes."""
    from equiformer_b200 import ops
    C = 8 * 132 * 16
    n = 2 * C if size == "two_passes" else 2 * C + C // 3
    H, A, ds, Cs = LAYOUTS["qm9_md17_l2"]
    lay, graph, alpha_dot, t0, Vs, keep, Gs, deg = _graph_case(ops, cuda_device, H, A, ds, Cs, n, seed=n)
    _check_against_chain(ops, lay, graph, alpha_dot, t0, Vs, keep, Gs, deg, tol=1e-4)


@pytest.mark.gpu
def test_backward_is_bitwise_repeatable(cuda_device):
    from equiformer_b200 import ops
    H, A, ds, Cs = LAYOUTS["oc20_l1"]
    lay, graph, alpha_dot, t0, Vs, keep, Gs, _deg = _graph_case(ops, cuda_device, H, A, ds, Cs, 400, seed=3)
    _outs, alpha = ops.mlp_softmax_aggregate_raw(lay, t0, Vs, alpha_dot, graph, keep)
    a = ops.mlp_softmax_aggregate_bwd_raw(lay, Gs, t0, Vs, alpha_dot, alpha, graph, keep)
    b = ops.mlp_softmax_aggregate_bwd_raw(lay, Gs, t0, Vs, alpha_dot, alpha, graph, keep)
    for x, y in zip([a[0], *a[1], a[2]], [b[0], *b[1], b[2]]):
        assert torch.equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("masked", [False, True])
def test_double_backward_matches_the_chain(cuda_device, masked):
    from equiformer_b200 import ops
    H, A, ds, Cs = LAYOUTS["qm9_md17_l2"]
    lay, graph, alpha_dot, t0, Vs, keep, Gs, _deg = _graph_case(ops, cuda_device, H, A, ds, Cs, 120, seed=11)
    keep = keep if masked else None
    ins = (alpha_dot.clone().requires_grad_(True), t0.clone().requires_grad_(True),
           *[v.clone().requires_grad_(True) for v in Vs])
    res = []
    for f in (lambda: ops.MlpSoftmaxAggregate.apply(lay, graph, keep, *ins),
              lambda: _chain(ops, lay, graph, keep, ins[0], ins[1], ins[2:])):
        first = torch.autograd.grad(f(), ins, Gs, create_graph=True)
        w = [torch.randn(t.shape, generator=torch.Generator().manual_seed(i)).to(cuda_device) for i, t in enumerate(first)]
        second = torch.autograd.grad(sum((a * b).sum() for a, b in zip(first, w)), ins)
        res.append([*first, *second])
    for a, b in zip(*res):
        assert rel_err(a.detach(), b.detach()) < 1e-4


@pytest.mark.gpu
def test_md17_l2_forces_and_their_training_gradients_match_the_chain(cuda_device, monkeypatch):
    """``graph_attention_transformer_l2_md17`` at full width (two blocks): energy, forces and the parameter gradients of
    the force loss (a double backward through the attention) on the fused route against the chain."""
    from equiformer_b200 import ops
    from equiformer_b200.nets.graph_attention_transformer_md17 import GraphAttentionTransformerMD17
    torch.manual_seed(0)
    # the keyword arguments of the registered graph_attention_transformer_l2_md17, two blocks instead of six
    model = GraphAttentionTransformerMD17(
        irreps_in="64x0e", irreps_node_embedding="128x0e+64x1e+32x2e", num_layers=2, irreps_node_attr="1x0e",
        irreps_sh="1x0e+1x1e+1x2e", max_radius=5.0, number_of_basis=128, fc_neurons=[64, 64], irreps_feature="512x0e",
        irreps_head="32x0e+16x1e+8x2e", num_heads=4, irreps_pre_attn=None, rescale_degree=False, nonlinear_message=False,
        irreps_mlp_mid="384x0e+192x1e+96x2e", norm_layer="layer", alpha_drop=0.2, proj_drop=0.0, out_drop=0.0,
        drop_path_rate=0.0).to(cuda_device).eval()
    g = torch.Generator().manual_seed(2)
    z = torch.tensor([6, 6, 8, 1, 1, 1, 1, 6, 8, 1, 6, 1]).to(cuda_device)
    pos = (1.6 * torch.randn(12, 3, generator=g)).to(cuda_device)
    batch = torch.zeros(12, dtype=torch.long, device=cuda_device)
    calls = []
    orig = ops.mlp_softmax_aggregate_raw

    def counting(*a, **k):
        calls.append(1)
        return orig(*a, **k)

    def run():
        model.zero_grad()
        e, f = model(node_atom=z, pos=pos.clone(), batch=batch)
        (e.sum() + (f ** 2).sum()).backward()
        return [e.detach(), f.detach()] + [p.grad.clone() for p in model.parameters() if p.grad is not None]

    monkeypatch.setattr(ops, "mlp_softmax_aggregate_raw", counting)
    fused = run()
    assert len(calls) >= 2
    monkeypatch.setattr(ops, "mlp_softmax_aggregate_ok", lambda *a: False)
    chain = run()
    for a, b in zip(fused, chain):
        assert rel_err(a, b) < 1e-4


# ------------------------------------------------------------------------------------------------ GPU: model level
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["qm9", "md17", "oc20"])
def test_cuda_linear_message_models_match_reference_model_files(cuda_device, kind):
    from equiformer_b200 import ops
    case = load(FIXTURE, kind)
    model = _mirror(kind, case).to(cuda_device)
    calls = []
    orig = ops.mlp_softmax_aggregate_raw

    def counting(*a, **k):
        calls.append(1)
        return orig(*a, **k)

    ops.mlp_softmax_aggregate_raw = counting
    try:
        energy, forces = run_mirror(kind, model, case, cuda_device, torch.float32)
    finally:
        ops.mlp_softmax_aggregate_raw = orig
    assert len(calls) >= case.cfg["num_layers"]
    assert rel_err(energy, case.t("energy")) < 5e-5
    if forces is not None:
        assert rel_err(forces, case.t("forces")) < 2e-4
    assert worst_grad({k: p.grad for k, p in model.named_parameters()}, case.grads, 51) < 1e-3


@pytest.mark.gpu
def test_full_size_linear_layer_matches_the_chain(cuda_device, monkeypatch):
    """One ``OC20_L1_256`` block's attention at full size (16 frames, ~55 k edges): forward and parameter / input
    gradients of the fused route against the chain on the same seeded inputs."""
    from equiformer_b200 import ops
    from equiformer_b200.nets.graph_attention_transformer_oc20 import OC20_L1_256, GraphAttentionTransformerOC20
    from tests.test_oc20_aux import _frames
    torch.manual_seed(0)
    model = GraphAttentionTransformerOC20(None, None, 1, **dict(OC20_L1_256, num_layers=1)).to(cuda_device).eval()
    attn = model.blocks[0].ga
    pos, batch, _z, _tags, src, dst, _vec = _frames(cuda_device, n_frames=16, seed=0)
    E, n = int(src.numel()), int(pos.shape[0])
    print(f"[full size] {n} atoms, {E} edges")
    assert E > 30000
    g = torch.Generator().manual_seed(1)
    x = torch.randn(n, attn.irreps_node_input.dim, generator=g).to(cuda_device)
    sh = torch.randn(E, 4, generator=g).to(cuda_device)
    rbf = torch.randn(E, 128, generator=g).to(cuda_device)
    G = torch.randn(n, attn.irreps_node_output.dim, generator=g).to(cuda_device)
    graph = ops.Graph(src, dst, n)
    calls = []
    orig = ops.mlp_softmax_aggregate_raw

    def counting(*a, **k):
        calls.append(1)
        return orig(*a, **k)

    def run():
        xi = x.clone().requires_grad_(True)
        attn.zero_grad()
        out = attn(xi, None, src, dst, sh, rbf, batch, graph=graph)
        out.backward(G)
        return [out.detach(), xi.grad] + [p.grad.clone() for p in attn.parameters()]

    monkeypatch.setattr(ops, "mlp_softmax_aggregate_raw", counting)
    fused = run()
    assert calls == [1]
    monkeypatch.setattr(ops, "mlp_softmax_aggregate_ok", lambda *a: False)
    chain = run()
    for a, b in zip(fused, chain):
        assert rel_err(a, b) < 1e-4


@pytest.mark.gpu
def test_graphed_linear_oc20_step_matches_eager(cuda_device):
    """2-block ``OC20_L1_256`` (``alpha_drop=0.2``) through ``graphs.GraphedStep``: each replay's loss and gradients
    equal the eager step's from the same generator state, so the replay draws the same dropout masks."""
    from equiformer_b200 import ops
    from equiformer_b200.graphs import GraphedStep
    from equiformer_b200.nets.graph_attention_transformer_oc20 import OC20_L1_256, GraphAttentionTransformerOC20
    from equiformer_b200.parallel import FlatGradAllReduce
    from tests.test_oc20_aux import _frames
    torch.manual_seed(0)
    model = GraphAttentionTransformerOC20(None, None, 1, **dict(OC20_L1_256, num_layers=2)).to(cuda_device).train()
    assert model.blocks[0].ga.alpha_dropout.p == 0.2
    bucket = FlatGradAllReduce(model.parameters())
    pos, batch, z, tags, src, dst, edge_vec = _frames(cuda_device, seed=3)
    target = torch.randn(4, 1, generator=torch.Generator().manual_seed(7)).to(cuda_device)
    n = int(pos.shape[0])
    row_ptr = torch.zeros(n + 1, dtype=torch.int64, device=cuda_device)
    torch.cumsum(torch.zeros(n, dtype=torch.int64, device=cuda_device).index_add_(0, dst, torch.ones_like(dst)), 0,
                 out=row_ptr[1:])

    def captured(edge_vec, target, batch, z, tags, src, dst, row_ptr):
        csr = ops.Graph.__new__(ops.Graph)
        csr.n_nodes, csr.n_edges, csr.perm = int(batch.shape[0]), int(src.numel()), None
        csr.src, csr.dst, csr.row_ptr = src, dst, row_ptr
        csr._src_perm = csr._src_row_ptr = None
        energy = model.forward_edges(edge_vec, batch, z, tags, src, dst, graph=csr, n_graphs=target.shape[0])
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
