"""The dot-product-attention OC20 model (``nets/dp_attention_transformer_oc20.py``) and the fused dot-product attention
kernels (``eqf_attn_dot_softmax_aggregate`` / ``_bwd``, ``ops.DotSoftmaxAggregate``).

CPU: the mirror's constructor defaults and ``OC20_DP_L1_256`` against the reference file and its yml; the full-size
``state_dict`` / ``no_weight_decay()`` table (tests/golden/reference_state_shapes_oc20_dp.json); the oracle and the mirror
(existing chain, kernels emulated in float64) against the reference-run fixture (tests/golden/reference_model_oc20_dp_small.npz,
tests/golden/make_reference_golden_oc20_dp.py); the host logic of ``DotSoftmaxAggregate`` with float64 stand-ins for the
two raw kernels: gradcheck, and its ``create_graph`` route against the chain it is rebuilt from.

-m gpu: the kernels against the chain (``EdgeDot`` -> ``SegSoftmax`` -> ``* keep`` -> ``AttnAggregate`` on contiguous
key / value halves) on the OC20 DP, QM9 DP and MD17 L3 DP head layouts, with and without the dropout mask, including
zero-in-degree nodes, a segment of 600 edges and node counts past the grid cap; bitwise-repeatable backward; double
backward; the CUDA model against the fixture; a full-size ``OC20_DP_L1_256`` layer against the chain; the graph-captured
training step against the eager step with attention dropout on.
"""
from __future__ import annotations

import json
import os

import pytest
import torch

from tests import _emulation as emu
from tests.helpers import rel_err
from tests.reference_fixtures import GOLDEN, load, mirror, oc20_data, oracle_config, run_mirror, run_oracle, worst_grad

FIXTURE = "reference_model_oc20_dp_small.npz"
SHAPES = os.path.join(GOLDEN, "reference_state_shapes_oc20_dp.json")
TOL = 2e-5                      # kernel vs the float32 chain

# head layouts (irreps of H heads, sorted and simplified): (H, ds, Cs)
LAYOUTS = {"oc20_dp": (8, (1, 3), (256, 128)),                 # 8 x (32x0e+16x1e)
           "qm9_dp": (4, (1, 3, 5), (128, 64, 32)),            # 4 x (32x0e+16x1e+8x2e)
           "md17_l3_dp": (4, (1, 3, 5, 7), (128, 64, 64, 32))}  # 4 x (32x0e+16x1e+16x2e+8x3e)


# ------------------------------------------------------------------------------------------------ constructor, tables
def test_constructor_defaults_and_shipped_configuration_match_the_reference():
    """Defaults of reference nets/dp_attention_transformer_oc20.py:86-103 and the model block of
    oc20/configs/is2re/all/dp_attention_transformer/l1_256_g@2_local.yml, restated."""
    import inspect
    from equiformer_b200.nets import model_entrypoint
    from equiformer_b200.nets.dp_attention_transformer_oc20 import OC20_DP_L1_256, DotProductAttentionTransformerOC20
    ref_defaults = dict(irreps_node_embedding="256x0e+128x1e", num_layers=6, irreps_node_attr="1x0e", use_node_attr=False,
                        irreps_sh="1x0e+1x1e", max_radius=6.0, number_of_basis=128, fc_neurons=[64, 64],
                        use_atom_edge_attr=False, irreps_atom_edge_attr="8x0e", irreps_feature="512x0e",
                        irreps_head="32x0e+16x1e", num_heads=8, irreps_pre_attn=None, rescale_degree=False,
                        nonlinear_message=False, irreps_mlp_mid="768x0e+384x1e", norm_layer="layer", alpha_drop=0.2,
                        proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0, use_auxiliary_task=False, otf_graph=False,
                        use_pbc=True, max_neighbors=50)
    params = inspect.signature(DotProductAttentionTransformerOC20.__init__).parameters
    assert list(params)[1:4] == ["num_atoms", "bond_feat_dim", "num_targets"]
    assert {k: p.default for k, p in params.items() if k in ref_defaults} == ref_defaults
    assert set(params) - {"self", "num_atoms", "bond_feat_dim", "num_targets"} == set(ref_defaults)
    yml = dict(irreps_node_embedding="256x0e+128x1e", num_layers=8, irreps_node_attr="1x0e", use_node_attr=False,
               irreps_sh="1x0e+1x1e", max_radius=5.0, number_of_basis=128, fc_neurons=[64, 64], use_atom_edge_attr=False,
               irreps_atom_edge_attr="1x0e", irreps_feature="512x0e", irreps_head="32x0e+16x1e", num_heads=8,
               irreps_pre_attn="256x0e+128x1e", rescale_degree=False, nonlinear_message=False,
               irreps_mlp_mid="768x0e+384x1e", norm_layer="layer", alpha_drop=0.2, proj_drop=0.0, out_drop=0.0,
               drop_path_rate=0.0, otf_graph=True, use_pbc=True, max_neighbors=500)
    assert OC20_DP_L1_256 == yml
    assert "dp_attention_transformer_oc20" in __import__("equiformer_b200.nets", fromlist=["list_models"]).list_models()
    assert model_entrypoint("dp_attention_transformer_oc20").__module__.endswith("dp_attention_transformer_oc20")


def test_full_size_state_dict_and_no_weight_decay_match_the_reference():
    from equiformer_b200.nets import DPTransBlock, model_entrypoint
    from equiformer_b200.nets.dp_attention_transformer_oc20 import OC20_DP_L1_256
    with open(SHAPES) as f:
        ref = json.load(f)
    model = model_entrypoint("dp_attention_transformer_oc20")(**OC20_DP_L1_256)
    assert len(model.blocks) == 8 and all(isinstance(b, DPTransBlock) for b in model.blocks)
    mine = {k: list(v.shape) for k, v in model.state_dict().items() if not k.endswith("tp.output_mask")}
    assert mine == ref["state"]
    assert sorted(model.no_weight_decay()) == ref["no_weight_decay"]


@pytest.mark.parametrize("option", ["use_auxiliary_task", "use_node_attr", "use_atom_edge_attr"])
def test_unsupported_options_raise(option):
    from equiformer_b200.nets.dp_attention_transformer_oc20 import DotProductAttentionTransformerOC20
    with pytest.raises(NotImplementedError):
        DotProductAttentionTransformerOC20(None, None, 1, irreps_node_embedding="16x0e+8x1e", num_layers=1,
                                           irreps_head="8x0e+4x1e", num_heads=2, irreps_feature="32x0e",
                                           irreps_mlp_mid="48x0e+24x1e", **{option: True})


# ------------------------------------------------------------------------------------------------ reference fixture
def _mirror(case):
    from equiformer_b200.nets.dp_attention_transformer_oc20 import DotProductAttentionTransformerOC20
    return mirror(DotProductAttentionTransformerOC20, case.cfg, case.state, None, None, 1)


def test_oracle_matches_reference_dp_oc20_model_file():
    case = load(FIXTURE)
    energy, _forces, params = run_oracle("oc20", case, oracle_config("oc20", case.cfg, attention="dot_product"))
    assert rel_err(energy.detach(), case.t("energy")) < 1e-11
    assert worst_grad({k: v.grad for k, v in params.items()}, case.grads, 51) < 1e-8


def test_mirror_with_emulated_kernels_matches_reference_dp_oc20_model_file():
    """float64 CPU stand-ins: the predicate of the fused kernel is false, so the existing chain runs."""
    from equiformer_b200.graph import radius_graph_pbc
    from tests._emulation import emulated_kernels
    case = load(FIXTURE)
    model = _mirror(case).double()
    data = oc20_data(case)
    edge, offs, _d2 = radius_graph_pbc(data.pos.float(), data.batch, data.cell.float(), case.cfg["max_radius"],
                                       case.cfg["max_neighbors"])
    assert torch.equal(edge, case.t("edge_index"))
    with emulated_kernels():
        energy, _forces = run_mirror("oc20", model, case)
    assert rel_err(energy.detach(), case.t("energy")) < 1e-10
    assert worst_grad({k: p.grad for k, p in model.named_parameters()}, case.grads, 51) < 1e-7


# ------------------------------------------------------------------------------------------------ host logic (float64)
_halves = emu.kv_halves


@pytest.fixture
def stand_ins(monkeypatch):
    from equiformer_b200 import ops
    monkeypatch.setattr(ops, "dot_softmax_aggregate_raw", emu.dot_softmax_aggregate_raw)
    monkeypatch.setattr(ops, "dot_softmax_aggregate_bwd_raw", emu.dot_softmax_aggregate_bwd_raw)
    with emu.emulated_kernels():
        yield ops


def _small_case(ops, dtype=torch.float64, seed=0):
    g = torch.Generator().manual_seed(seed)
    lay = ops.HeadLayout((1, 3), (8, 4), 2)
    dst = torch.tensor([0, 0, 0, 2, 2, 3, 3, 3, 3, 5])          # nodes 1 and 4: no incoming edge
    src = torch.randint(0, 6, (dst.numel(),), generator=g)
    graph = ops.Graph(src, dst, 6)
    qs = [torch.randn(6, d, C, generator=g, dtype=dtype).requires_grad_(True) for d, C in zip(lay.ds, lay.Cs)]
    kvs = [torch.randn(dst.numel(), d, 2 * C, generator=g, dtype=dtype).requires_grad_(True)
           for d, C in zip(lay.ds, lay.Cs)]
    keep = (torch.rand(dst.numel(), 2, generator=g) > 0.3).to(dtype) / 0.7
    return lay, graph, qs, kvs, keep


@pytest.mark.parametrize("masked", [False, True])
def test_dot_softmax_aggregate_gradcheck(stand_ins, masked):
    ops = stand_ins
    lay, graph, qs, kvs, keep = _small_case(ops)
    keep = keep if masked else None
    fn = lambda *ins: ops.DotSoftmaxAggregate.apply(lay, graph, keep, *ins)
    assert torch.autograd.gradcheck(fn, (*qs, *kvs), eps=1e-6, atol=1e-7)


def _chain(ops, lay, graph, keep, qs, kvs):
    k, v = _halves(lay, kvs)
    a = ops.SegSoftmax.apply(ops.EdgeDot.apply(lay, graph, *[t.contiguous() for t in k], *qs), graph)
    return ops.AttnAggregate.apply(lay, graph, a if keep is None else a * keep, *[t.contiguous() for t in v])


@pytest.mark.parametrize("masked", [False, True])
def test_create_graph_route_equals_the_chain(stand_ins, masked):
    """First and second derivatives through ``DotSoftmaxAggregate`` under ``create_graph`` against the chain."""
    ops = stand_ins
    lay, graph, qs, kvs, keep = _small_case(ops, seed=1)
    keep = keep if masked else None
    g = torch.Generator().manual_seed(5)
    Gs = [torch.randn(6, d, C, generator=g, dtype=torch.float64) for d, C in zip(lay.ds, lay.Cs)]
    ins = (*qs, *kvs)
    results = []
    for f in (lambda: ops.DotSoftmaxAggregate.apply(lay, graph, keep, *ins), lambda: _chain(ops, lay, graph, keep, qs, kvs)):
        outs = f()
        first = torch.autograd.grad(outs, ins, Gs, create_graph=True)
        w = [torch.randn(t.shape, generator=torch.Generator().manual_seed(9 + i), dtype=torch.float64)
             for i, t in enumerate(first)]
        second = torch.autograd.grad(sum((a * b).sum() for a, b in zip(first, w)), ins)
        results.append((outs, first, second))
    for a, b in zip(*[sum((list(r) for r in res), []) for res in results]):
        assert rel_err(a.detach(), b.detach()) < 1e-12


# ------------------------------------------------------------------------------------------------ GPU: kernels vs chain
def _graph_case(ops, dev, H, ds, Cs, n_nodes, seed, long_segment=0):
    """Random destination-sorted graph with zero-in-degree nodes (every 7th node) and optionally one long segment."""
    g = torch.Generator().manual_seed(seed)
    deg = torch.randint(0, 40, (n_nodes,), generator=g)
    deg[::7] = 0
    if long_segment:
        deg[n_nodes // 2] = long_segment
    dst = torch.repeat_interleave(torch.arange(n_nodes), deg)
    src = torch.randint(0, n_nodes, (dst.numel(),), generator=g)
    graph = ops.Graph(src.to(dev), dst.to(dev), n_nodes)
    lay = ops.HeadLayout(ds, Cs, H)
    qs = [torch.randn(n_nodes, d, C, generator=g).to(dev) for d, C in zip(ds, Cs)]
    kvs = [torch.randn(dst.numel(), d, 2 * C, generator=g).to(dev) for d, C in zip(ds, Cs)]
    keep = ((torch.rand(dst.numel(), H, generator=g) > 0.2).float() / 0.8).to(dev)
    Gs = [torch.randn(n_nodes, d, C, generator=g).to(dev) for d, C in zip(ds, Cs)]
    return lay, graph, qs, kvs, keep, Gs, deg


def _check_against_chain(ops, lay, graph, qs, kvs, keep, Gs, deg, tol=TOL):
    # chain forward and backward (autograd through EdgeDot / SegSoftmax / AttnAggregate on contiguous halves)
    ql = [t.clone().requires_grad_(True) for t in qs]
    kl = [t.clone().requires_grad_(True) for t in kvs]
    k, v = _halves(lay, kl)
    z = ops.EdgeDot.apply(lay, graph, *[t.contiguous() for t in k], *ql)
    alpha_ref = ops.segment_softmax(z.contiguous(), graph)
    outs_ref = ops.attention_aggregate(lay, graph, alpha_ref if keep is None else alpha_ref * keep,
                                       [t.contiguous() for t in v])
    grads_ref = torch.autograd.grad(outs_ref, [*ql, *kl], Gs)
    outs, alpha = ops.dot_softmax_aggregate_raw(lay, qs, kvs, graph, keep)
    assert rel_err(alpha, alpha_ref) < tol
    for a, b in zip(outs, outs_ref):
        assert rel_err(a, b) < tol
    empty = (deg == 0).nonzero().flatten().to(outs[0].device)
    assert all(bool((o.index_select(0, empty) == 0).all()) for o in outs)
    gqs, gkvs = ops.dot_softmax_aggregate_bwd_raw(lay, Gs, qs, kvs, alpha, graph, keep)
    for what, a, b in zip(["gq"] * len(gqs) + ["gkv"] * len(gkvs), [*gqs, *gkvs], grads_ref):
        assert rel_err(a, b) < tol, (what, rel_err(a, b))
    return alpha, gqs, gkvs


@pytest.mark.gpu
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_kernels_match_the_chain(cuda_device, name, masked):
    """Forward (outputs, alpha) and backward (gq, the whole key / value gradient) against the chain; node 150 has a
    600-edge segment, every 7th node none."""
    from equiformer_b200 import ops
    H, ds, Cs = LAYOUTS[name]
    lay, graph, qs, kvs, keep, Gs, deg = _graph_case(ops, cuda_device, H, ds, Cs, 300, seed=len(name) + masked,
                                                     long_segment=600)
    assert ops.dot_softmax_aggregate_ok(lay, qs[0], graph)
    _check_against_chain(ops, lay, graph, qs, kvs, keep if masked else None, Gs, deg)


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["two_passes", "partial_third_pass"])
def test_kernels_past_the_grid_cap(cuda_device, size):
    """min(ceil(N / 8), 132 * 16) CTAs of 8 warps, one node per warp step: N = 2 C and 2 C + C / 3 nodes."""
    from equiformer_b200 import ops
    C = 8 * 132 * 16
    n = 2 * C if size == "two_passes" else 2 * C + C // 3
    H, ds, Cs = LAYOUTS["qm9_dp"]
    lay, graph, qs, kvs, keep, Gs, deg = _graph_case(ops, cuda_device, H, ds, Cs, n, seed=n)
    _check_against_chain(ops, lay, graph, qs, kvs, keep, Gs, deg)


@pytest.mark.gpu
def test_backward_is_bitwise_repeatable(cuda_device):
    from equiformer_b200 import ops
    H, ds, Cs = LAYOUTS["oc20_dp"]
    lay, graph, qs, kvs, keep, Gs, _deg = _graph_case(ops, cuda_device, H, ds, Cs, 400, seed=3, long_segment=700)
    _outs, alpha = ops.dot_softmax_aggregate_raw(lay, qs, kvs, graph, keep)
    a = ops.dot_softmax_aggregate_bwd_raw(lay, Gs, qs, kvs, alpha, graph, keep)
    b = ops.dot_softmax_aggregate_bwd_raw(lay, Gs, qs, kvs, alpha, graph, keep)
    for x, y in zip([*a[0], *a[1]], [*b[0], *b[1]]):
        assert torch.equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("masked", [False, True])
def test_double_backward_matches_the_chain(cuda_device, masked):
    from equiformer_b200 import ops
    H, ds, Cs = LAYOUTS["md17_l3_dp"]
    lay, graph, qs, kvs, keep, Gs, _deg = _graph_case(ops, cuda_device, H, ds, Cs, 120, seed=11)
    keep = keep if masked else None
    ql = [t.clone().requires_grad_(True) for t in qs]
    kl = [t.clone().requires_grad_(True) for t in kvs]
    ins = (*ql, *kl)
    res = []
    for f in (lambda: ops.DotSoftmaxAggregate.apply(lay, graph, keep, *ins), lambda: _chain(ops, lay, graph, keep, ql, kl)):
        first = torch.autograd.grad(f(), ins, Gs, create_graph=True)
        w = [torch.randn(t.shape, generator=torch.Generator().manual_seed(i)).to(cuda_device) for i, t in enumerate(first)]
        second = torch.autograd.grad(sum((a * b).sum() for a, b in zip(first, w)), ins)
        res.append([*first, *second])
    for a, b in zip(*res):
        assert rel_err(a.detach(), b.detach()) < 1e-4


# ------------------------------------------------------------------------------------------------ GPU: model level
@pytest.mark.gpu
def test_cuda_dp_oc20_model_matches_reference_model_file(cuda_device):
    from equiformer_b200 import ops
    case = load(FIXTURE)
    model = _mirror(case).to(cuda_device)
    calls = []
    orig = ops.dot_softmax_aggregate_raw

    def counting(*a, **k):
        calls.append(1)
        return orig(*a, **k)

    ops.dot_softmax_aggregate_raw = counting
    try:
        energy = model(oc20_data(case, cuda_device, torch.float32))
    finally:
        ops.dot_softmax_aggregate_raw = orig
    assert len(calls) == case.cfg["num_layers"]
    assert rel_err(energy, case.t("energy")) < 5e-5
    (energy ** 2).sum().backward()
    assert worst_grad({k: p.grad for k, p in model.named_parameters()}, case.grads, 51) < 1e-3


@pytest.mark.gpu
def test_full_size_dp_layer_matches_the_chain(cuda_device, monkeypatch):
    """One ``OC20_DP_L1_256`` block's attention at full size (16 frames, ~55 k edges): forward and parameter / input
    gradients of the fused route against the chain on the same seeded inputs."""
    from equiformer_b200 import ops
    from equiformer_b200.nets.dp_attention_transformer_oc20 import OC20_DP_L1_256, DotProductAttentionTransformerOC20
    from tests.test_oc20_aux import _frames
    torch.manual_seed(0)
    model = DotProductAttentionTransformerOC20(None, None, 1, **dict(OC20_DP_L1_256, num_layers=1)).to(cuda_device).eval()
    attn = model.blocks[0].dpa
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

    def run():
        xi = x.clone().requires_grad_(True)
        attn.zero_grad()
        out = attn(xi, None, src, dst, sh, rbf, batch, graph=graph)
        out.backward(G)
        return [out.detach(), xi.grad] + [p.grad.clone() for p in attn.parameters()]

    fused = run()
    monkeypatch.setattr(ops, "dot_softmax_aggregate_ok", lambda *a: False)
    chain = run()
    for a, b in zip(fused, chain):
        assert rel_err(a, b) < 1e-4


@pytest.mark.gpu
def test_graphed_dp_oc20_step_matches_eager(cuda_device):
    """2-block ``OC20_DP_L1_256`` (``alpha_drop=0.2``) through ``graphs.GraphedStep``: each replay's loss and gradients
    equal the eager step's from the same generator state, so the replay draws the same dropout masks."""
    from equiformer_b200 import ops
    from equiformer_b200.graphs import GraphedStep
    from equiformer_b200.nets.dp_attention_transformer_oc20 import OC20_DP_L1_256, DotProductAttentionTransformerOC20
    from equiformer_b200.parallel import FlatGradAllReduce
    from tests.test_oc20_aux import _frames
    torch.manual_seed(0)
    model = DotProductAttentionTransformerOC20(None, None, 1, **dict(OC20_DP_L1_256, num_layers=2)).to(cuda_device).train()
    assert model.blocks[0].dpa.alpha_dropout.p == 0.2
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
