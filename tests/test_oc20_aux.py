"""The OC20 IS2RS auxiliary task: ``GraphAttentionTransformerOC20(use_auxiliary_task=True)`` and the objective helpers of
``equiformer_b200.oc20_objective``.

Pinned to ``tests/golden/reference_model_oc20_aux_small.npz`` (the reference's OC20 model file itself, float64, two periodic
frames, a ``32x0e+16x1e`` final feature; ``tests/golden/make_reference_golden_oc20_aux.py``) for a nonlinear-message and a
linear-message model: the oracle extension (``tests/oracle_oc20_aux.py``) and the mirror with emulated kernels in float64
on the CPU, the CUDA model on a GPU.  At the full ``l1_256`` sizes the head is checked against the float64 oracle, its
routes (generated ``oc20_l1`` DTP kernels, no edge-sized torch GEMM / scatter) and its CUDA-graph capture.
"""
from __future__ import annotations

import pytest
import torch

from oracle import e3nn_ref as e3
from oracle import equiformer_ref as R
from tests import oracle_oc20_aux as OA
from tests.helpers import rel_err
from tests.reference_fixtures import load, mirror, oc20_data, oracle_config

AUX = "reference_model_oc20_aux_small.npz"
CASES = ["nonlinear", "linear"]


def _load(case):
    """The run of one case and its constructor arguments: both runs share the file's ``cfg/`` and differ only in
    ``nonlinear_message``."""
    run = load(AUX, case)
    return run, dict(run.cfg, nonlinear_message=case == "nonlinear")


def _mirror(cfg, state):
    from equiformer_b200.nets.graph_attention_transformer_oc20 import GraphAttentionTransformerOC20
    return mirror(GraphAttentionTransformerOC20, cfg, state, None, None, 1)


# ------------------------------------------------------------------------------------------- model construction (CPU)

@pytest.mark.parametrize("case", CASES)
def test_mirror_loads_reference_aux_state_dict(case):
    """The reference's ``state_dict`` loads with only ``tp.output_mask`` buffers missing, and the ``auxiliary_head.*``
    parameters have the reference's names and shapes."""
    run, cfg = _load(case)
    state = run.state
    model = _mirror(cfg, state)
    ours = {k: tuple(p.shape) for k, p in model.named_parameters() if k.startswith("auxiliary_head.")}
    ref = {k: tuple(v.shape) for k, v in state.items() if k.startswith("auxiliary_head.") and k in dict(model.named_parameters())}
    assert ours and ours == ref
    assert all(k in ours for k in run.grads if k.startswith("auxiliary_head."))
    assert str(model.auxiliary_head.proj.irreps_out) == "1x1e"        # no 1o block in 32x0e+16x1e


def test_aux_off_model_is_unchanged():
    """Without the option there is no ``auxiliary_head`` and the keys are the reference's aux-off keys."""
    small = load("reference_model_oc20_small.npz")
    cfg = small.cfg
    from equiformer_b200.nets.graph_attention_transformer_oc20 import GraphAttentionTransformerOC20
    off = GraphAttentionTransformerOC20(None, None, 1, **cfg)
    on = GraphAttentionTransformerOC20(None, None, 1, **dict(cfg, use_auxiliary_task=True))
    assert not hasattr(off, "auxiliary_head")
    keys_off = set(off.state_dict())
    assert keys_off == {k for k in on.state_dict() if not k.startswith("auxiliary_head.")}
    ref = set(small.state)
    assert ref <= keys_off and all(k.endswith("tp.output_mask") for k in keys_off - ref)


def test_attention_head_and_node_attributes_still_raise():
    from equiformer_b200.nets.graph_attention_transformer_oc20 import GraphAttentionTransformerOC20
    small = dict(irreps_node_embedding="16x0e+8x1e", num_layers=1, irreps_feature="32x0e+16x1e", irreps_head="8x0e+4x1e",
                 num_heads=2, irreps_mlp_mid="48x0e+24x1e", number_of_basis=16, fc_neurons=[16, 16])
    for flag in ("use_attention_head", "use_node_attr", "use_atom_edge_attr"):
        with pytest.raises(NotImplementedError) as exc:
            GraphAttentionTransformerOC20(None, None, 1, use_auxiliary_task=True, **{flag: True}, **small)
        assert "auxiliary" not in str(exc.value)


def test_aux_configuration_dicts():
    """The ``model:`` blocks of the ``*_aux_*`` configurations: 6 / 18 blocks, a ``1e`` final-feature block, the head's
    ``1x1e`` output and an energy head fed by the ``512x0e`` part only."""
    from equiformer_b200.nets.graph_attention_transformer_oc20 import (OC20_L1_256_BLOCKS18_NONLINEAR_AUX, OC20_L1_256_NONLINEAR,
                                                                       OC20_L1_256_NONLINEAR_AUX, GraphAttentionTransformerOC20)
    assert OC20_L1_256_NONLINEAR_AUX == dict(OC20_L1_256_NONLINEAR, irreps_feature="512x0e+256x1e", drop_path_rate=0.05,
                                             use_auxiliary_task=True)
    assert OC20_L1_256_BLOCKS18_NONLINEAR_AUX == dict(OC20_L1_256_NONLINEAR_AUX, num_layers=18)
    model = GraphAttentionTransformerOC20(None, None, 1, **OC20_L1_256_BLOCKS18_NONLINEAR_AUX)
    assert len(model.blocks) == 18 and model.blocks[-1].ffn_shortcut is not None
    assert str(model.head[0].irreps_out) == "512x0e" and str(model.auxiliary_head.irreps_node_output) == "1x1e"
    assert str(model.auxiliary_head.irreps_pre_attn) == "256x0e+128x1e"
    assert model.auxiliary_head.alpha_dropout is not None and model.auxiliary_head.alpha_dropout.p == 0.2


# ---------------------------------------------------------------------------------------- parity with the reference file

@pytest.mark.parametrize("case", CASES)
def test_oracle_aux_matches_reference_model_file(case):
    run, cfg = _load(case)
    params = {k: v.requires_grad_(v.is_floating_point() and v.numel() > 0)
              for k, v in R.cast_params(run.state, torch.float64).items()}
    t = run.t
    edge = t("edge_index")
    energy, aux = OA.model_forward_oc20_aux(params, oracle_config("oc20", cfg), t("pos").double(), t("cell").double(),
                                            t("batch"), t("z"), t("tags"), 2, edge[0], edge[1], t("cell_offsets"),
                                            cfg["irreps_pre_attn"])
    assert rel_err(energy, t("energy")) < 1e-10
    assert rel_err(aux, t("aux")) < 1e-10
    ((t("c").double() * energy).sum() + (t("W").double() * aux).sum()).backward()
    for k, ref in run.grads.items():
        assert rel_err(params[k].grad, ref) < 1e-6, k


@pytest.mark.parametrize("case", CASES)
def test_mirror_aux_matches_reference_model_file(case):
    """The mirror (own periodic neighbour list, kernels emulated in float64): same edge list as the fixture's, energy and
    aux 1e-10, parameter gradients 1e-6."""
    from equiformer_b200.graph import radius_graph_pbc
    from tests._emulation import emulated_kernels
    run, cfg = _load(case)
    model = _mirror(cfg, run.state).double()
    data = oc20_data(run)
    edge, offs, _d2 = radius_graph_pbc(data.pos.float(), data.batch, data.cell.float(), cfg["max_radius"], cfg["max_neighbors"])
    assert torch.equal(edge, run.t("edge_index"))
    assert torch.equal(offs.long(), run.t("cell_offsets").long())
    t = run.t
    with emulated_kernels():
        energy, aux = model(data)
        ((t("c").double() * energy).sum() + (t("W").double() * aux).sum()).backward()
    assert rel_err(energy, t("energy")) < 1e-10
    assert rel_err(aux, t("aux")) < 1e-10
    for k, ref in run.grads.items():
        assert rel_err(model.get_parameter(k).grad, ref) < 1e-6, k


# --------------------------------------------------------------------------------------------------- objective helpers

def test_masked_l2mae_equals_boolean_index_formula():
    from equiformer_b200.oc20_objective import masked_l2mae
    g = torch.Generator().manual_seed(4)
    pred, target = torch.randn(40, 3, generator=g, dtype=torch.float64), torch.randn(40, 3, generator=g, dtype=torch.float64)
    tags = torch.randint(0, 3, (40,), generator=g)
    keep = tags > 0
    ref = (pred[keep] - target[keep]).norm(p=2, dim=-1).mean()
    assert rel_err(masked_l2mae(pred, target, tags), ref) < 1e-14
    assert masked_l2mae(pred, target, torch.zeros_like(tags)).item() == 0.0


def test_relaxation_target_and_weight_schedule():
    from equiformer_b200.oc20_objective import auxiliary_task_weight, relaxation_target
    pos, relaxed = torch.zeros(2, 3), torch.ones(2, 3)
    assert torch.allclose(relaxation_target(pos, relaxed, 0.5), torch.full((2, 3), 2.0))
    assert auxiliary_task_weight(0, 1000, 15.0) == 15.0
    assert auxiliary_task_weight(500, 1000, 15.0) == 8.0
    assert auxiliary_task_weight(1000, 1000, 15.0) == 1.0
    assert auxiliary_task_weight(2000, 1000, 15.0) == 1.0
    assert auxiliary_task_weight(10, 1000, 1.0) == 1.0


def test_interpolation_is_seeded_moves_only_tagged_atoms_of_drawn_frames():
    from equiformer_b200.oc20_objective import interpolate_init_relaxed_pos
    g = torch.Generator().manual_seed(0)
    n_frames, per = 32, 10
    batch = torch.arange(n_frames).repeat_interleave(per)
    pos = torch.randn(n_frames * per, 3, generator=g, dtype=torch.float64)
    relaxed = pos + torch.randn(pos.shape, generator=g, dtype=torch.float64)
    tags = torch.randint(0, 3, (n_frames * per,), generator=g)
    before = pos.clone()
    a = interpolate_init_relaxed_pos(pos, relaxed, batch, tags, n_frames, torch.Generator().manual_seed(5))
    b = interpolate_init_relaxed_pos(pos, relaxed, batch, tags, n_frames, torch.Generator().manual_seed(5))
    assert torch.equal(a, b) and torch.equal(pos, before)
    moved = (a != pos).any(dim=1)
    assert not moved[tags == 0].any()
    frame_moved = torch.zeros(n_frames, dtype=torch.bool).index_put_((batch[moved],), torch.tensor(True))
    assert 0 < int(frame_moved.sum()) < n_frames           # each frame with probability 1/2: both kinds among 32
    for f in range(n_frames):                                # a frame drawn as "no interpolation" comes back unchanged
        rows = batch == f
        if not frame_moved[f]:
            assert torch.equal(a[rows], pos[rows])
        else:                                                # drawn: every tagged atom moved
            assert moved[rows & (tags > 0)].all()


# ------------------------------------------------------------------------------------------------------------- GPU

@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_cuda_aux_matches_reference_model_file(case, cuda_device):
    from equiformer_b200.graph import radius_graph_pbc
    run, cfg = _load(case)
    model = _mirror(cfg, run.state).to(cuda_device)
    data = oc20_data(run, cuda_device, torch.float32)
    edge, offs, _d2 = radius_graph_pbc(data.pos, data.batch, data.cell, cfg["max_radius"], cfg["max_neighbors"])
    assert torch.equal(edge.cpu(), run.t("edge_index"))
    t = run.t
    energy, aux = model(data)
    ((t("c", cuda_device) * energy).sum() + (t("W", cuda_device) * aux).sum()).backward()
    assert rel_err(energy, t("energy")) < 1e-4
    assert rel_err(aux, t("aux")) < 1e-4
    worst = max(rel_err(model.get_parameter(k).grad, ref) for k, ref in run.grads.items())
    assert worst < 1e-3, worst


def _full_size_model(dev, num_layers=6):
    """``OC20_L1_256_NONLINEAR_AUX`` with dropouts and stochastic depth at 0 and perturbed biases / offsets."""
    from equiformer_b200.nets.graph_attention_transformer_oc20 import GraphAttentionTransformerOC20, OC20_L1_256_NONLINEAR_AUX
    torch.manual_seed(0)
    cfg = dict(OC20_L1_256_NONLINEAR_AUX, alpha_drop=0.0, drop_path_rate=0.0, num_layers=num_layers)
    model = GraphAttentionTransformerOC20(None, None, 1, **cfg)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if p.abs().max() == 0 or "bias" in name or "offset" in name:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
    return model.to(dev).train()


def _frames(dev, n_frames=4, seed=0):
    from equiformer_b200.graph import radius_graph_pbc
    from equiformer_b200.synthetic import oc20_like_frames
    pos, batch, z, tags, side = oc20_like_frames(n_frames, seed=seed)
    cell = torch.diag_embed(side[:, None].expand(-1, 3)).float()
    pos, batch, z, tags, cell = (t.to(dev) for t in (pos, batch, z, tags, cell))
    edge, offs, _ = radius_graph_pbc(pos, batch, cell, 5.0, 500)
    src, dst = edge[0], edge[1]
    edge_vec = (pos.index_select(0, src) - pos.index_select(0, dst)
                + torch.bmm(offs.to(pos.dtype).view(-1, 1, 3), cell.index_select(0, batch.index_select(0, dst))).view(-1, 3))
    return pos, batch, z, tags, src, dst, edge_vec


@pytest.mark.gpu
def test_cuda_aux_head_full_size_matches_oracle_on_library_kernels(cuda_device):
    """``l1_256`` sizes (``512x0e+256x1e`` feature, 4 synthetic periodic frames): the head's output and parameter gradients
    against the float64 oracle fed the same head inputs; its products resolve to the generated ``oc20_l1`` kernels and
    neither its forward nor its backward has an edge-sized torch GEMM or scatter."""
    from equiformer_b200 import ops
    model = _full_size_model(cuda_device)
    head = model.auxiliary_head
    for sep in (head.sep_act, head.sep_value):
        assert sep.dtp.tp.plan.generated
    pos, batch, z, tags, src, dst, edge_vec = _frames(cuda_device)
    E, n = int(src.numel()), int(pos.shape[0])
    seen = {}
    hook = head.register_forward_pre_hook(lambda m, a, kw: seen.update(kw), with_kwargs=True)
    try:
        energy, aux = model.forward_edges(edge_vec, batch, z, tags, src, dst, n_graphs=4)
    finally:
        hook.remove()
    W = torch.randn(aux.shape, generator=torch.Generator().manual_seed(2)).to(cuda_device)
    model.zero_grad(set_to_none=True)
    ((W * aux).sum() + energy.sum()).backward()

    params = {k: v.requires_grad_(v.is_floating_point() and v.numel() > 0)
              for k, v in R.cast_params(model.state_dict(), torch.float64).items() if k.startswith("auxiliary_head.")}
    cpu64 = lambda t: t.detach().cpu().double()
    ref = OA.graph_attention_pre(params, "auxiliary_head", e3.parse_irreps("512x0e+256x1e"), e3.parse_irreps("256x0e+128x1e"),
                                 e3.parse_irreps("1x0e+1x1e"), e3.parse_irreps("32x0e+16x1e"), 8, [(1, 1, 1)], True,
                                 cpu64(seen["node_input"]), seen["edge_src"].cpu(), seen["edge_dst"].cpu(),
                                 cpu64(seen["edge_attr"]), cpu64(seen["edge_scalars"]))
    (ref * W.cpu().double()).sum().backward()
    assert rel_err(aux, ref) < 1e-4
    worst = max((rel_err(model.get_parameter(k).grad, v.grad), k) for k, v in params.items() if v.grad is not None)
    assert worst[0] < 1e-3, worst

    # the head alone, forward + backward, under the torch profiler and the launch accounting of our kernels
    from torch.profiler import ProfilerActivity, profile
    x = seen["node_input"].detach().requires_grad_(True)
    kw = {k: (v.detach() if isinstance(v, torch.Tensor) else v) for k, v in seen.items() if k != "node_input"}
    prof_k = ops.KernelProfile(time_events=True)
    ops.PROFILE = prof_k
    try:
        with profile(activities=[ProfilerActivity.CPU], record_shapes=True) as prof:
            out = head(node_input=x, **kw)
            (out * W).sum().backward()
            torch.cuda.synchronize()
    finally:
        ops.PROFILE = None
    names = {r[0] for r in prof_k.records}
    assert any(k.startswith("dtp_") for k in names) and any(k.startswith("gemm") for k in names), names
    edge_sized = [(e.name, e.input_shapes) for e in prof.events()
                  if e.name in ("aten::mm", "aten::bmm", "aten::addmm", "aten::matmul", "aten::index_add", "aten::index_add_")
                  and any(s and s[0] == E for s in e.input_shapes)]
    assert not edge_sized, edge_sized[:5]
    assert E > 4 * n


@pytest.mark.gpu
def test_graphed_energy_and_aux_step_matches_eager(cuda_device):
    """The energy + auxiliary loss step captured by ``graphs.GraphedStep`` (dropouts at 0) gives the eager loss and
    gradients; weight gradients add with fp32 atomics in no fixed order, hence 1e-5 and not bit equality."""
    from equiformer_b200 import ops
    from equiformer_b200.graphs import GraphedStep
    from equiformer_b200.oc20_objective import masked_l2mae, relaxation_target
    from equiformer_b200.parallel import FlatGradAllReduce
    model = _full_size_model(cuda_device, num_layers=2)
    bucket = FlatGradAllReduce(model.parameters())
    pos, batch, z, tags, src, dst, edge_vec = _frames(cuda_device, seed=3)
    g = torch.Generator().manual_seed(7)
    relaxed = pos + 0.3 * torch.randn(pos.shape, generator=g).to(cuda_device)
    aux_target = relaxation_target(pos, relaxed, 0.9452036023139954)
    target = torch.randn(4, 1, generator=g).to(cuda_device)
    n = int(pos.shape[0])
    row_ptr = torch.zeros(n + 1, dtype=torch.int64, device=cuda_device)
    torch.cumsum(torch.zeros(n, dtype=torch.int64, device=cuda_device).index_add_(0, dst, torch.ones_like(dst)), 0,
                 out=row_ptr[1:])

    def loss_of(energy, aux, tgt, atgt, tg):
        return (energy - tgt).abs().mean() + 15.0 * masked_l2mae(aux, atgt, tg)

    def captured(edge_vec, target, aux_target, batch, z, tags, src, dst, row_ptr):
        csr = ops.Graph.__new__(ops.Graph)
        csr.n_nodes, csr.n_edges, csr.perm = int(batch.shape[0]), int(src.numel()), None
        csr.src, csr.dst, csr.row_ptr = src, dst, row_ptr
        csr._src_perm = csr._src_row_ptr = None
        energy, aux = model.forward_edges(edge_vec, batch, z, tags, src, dst, graph=csr, n_graphs=target.shape[0])
        return loss_of(energy, aux, target, aux_target, tags)

    step = GraphedStep(captured, bucket)
    key = (n, int(src.numel()), 4)
    inputs = [edge_vec, target, aux_target, batch, z, tags, src, dst, row_ptr]
    for _ in range(2):                                  # capture, then a pure replay
        loss_g = step(key, inputs).clone()
    grads_g = bucket.flat.clone()
    assert step.captures == 1
    bucket.zero_grad()
    energy, aux = model.forward_edges(edge_vec, batch, z, tags, src, dst, n_graphs=4)
    loss_e = loss_of(energy, aux, target, aux_target, tags)
    loss_e.backward()
    assert rel_err(loss_g, loss_e) < 1e-5
    assert rel_err(grads_g, bucket.flat) < 1e-5
    head_g = [p.grad for k, p in model.named_parameters() if k.startswith("auxiliary_head.")]
    assert any(float(gr.abs().max()) > 0 for gr in head_g)
