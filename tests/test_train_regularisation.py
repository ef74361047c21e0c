"""Training with the shipped regularisers on the fused, capturable path: attention-weight dropout applied inside K2
(``ops.MaskedSoftmaxAggregate``) and per-graph stochastic depth on the planar blocks, drawn without host reads.

CPU: ``GraphDropPath`` with ``n_graphs`` against the reference fixture, and the planar stochastic-depth route against the
stock e3nn-layout route with emulated kernels in float64 (the masked kernels get the stand-ins below).
GPU: the masked kernel family against float64, the fused route against the unfused one from the same seed (one layer,
the QM9 model, the MD17 energy + force step), and CUDA-graph replays against eager steps from the same generator state.
"""
from __future__ import annotations

import contextlib
import os

import numpy as np
import pytest
import torch

from tests import _emulation as emu
from tests._emulation import emulated_kernels
from tests.helpers import aspirin_like, molecules, rel_err

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_modules.npz")


# ------------------------------------------------------------------------------------------------ emulation with masks

def _softmax_aggregate_raw(lay, z, Vs, graph, keep=None):
    alpha = emu.seg_softmax_raw(z, graph)
    return emu.attn_aggregate_raw(lay, alpha if keep is None else alpha * keep, Vs, graph), alpha


def _seg_softmax_bwd_raw(alpha, ga, graph, keep=None):
    return emu.seg_softmax_bwd_raw(alpha, ga if keep is None else ga * keep, graph)


def _attn_edge_scale_raw(lay, alpha, Gs, graph, keep=None):
    return emu.attn_edge_scale_raw(lay, alpha if keep is None or alpha is None else alpha * keep, Gs, graph)


@contextlib.contextmanager
def emulated_kernels_with_masks():
    """``emulated_kernels`` plus float64 stand-ins for the kernels that take an attention-dropout mask."""
    from equiformer_b200 import ops
    with emulated_kernels():
        saved = {n: getattr(ops, n) for n in ("softmax_aggregate_raw", "seg_softmax_bwd_raw", "attn_edge_scale_raw")}
        try:
            ops.softmax_aggregate_raw = _softmax_aggregate_raw
            ops.seg_softmax_bwd_raw = _seg_softmax_bwd_raw
            ops.attn_edge_scale_raw = _attn_edge_scale_raw
            yield
        finally:
            for n, fn in saved.items():
                setattr(ops, n, fn)


def _model(name, dev=None, dtype=torch.float64, drop_path_rate=0.0, **kw):
    from equiformer_b200.nets import model_entrypoint
    from equiformer_b200.nets.drop import GraphDropPath
    torch.manual_seed(0)
    args = dict(irreps_in="5x0e", radius=5.0, num_basis=128)
    args.update(kw)
    model = model_entrypoint(name)(**args).to(dtype)
    if drop_path_rate > 0.0:                      # what the constructors build for drop_path_rate > 0
        for blk in model.blocks:
            blk.drop_path = GraphDropPath(drop_path_rate)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for p in model.parameters():
            p.add_(torch.randn(p.shape, generator=g, dtype=p.dtype) * 0.05)
    return model.to(dev).train() if dev is not None else model.train()


def _flat_grads(model):
    return torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in model.parameters()])


# ------------------------------------------------------------------------------------------------ CPU

def test_graph_drop_path_with_n_graphs_draws_like_the_reference():
    """Handing over the number of graphs changes nothing but the host read: same draws, same output, bit for bit, and
    the reference's fixture."""
    from equiformer_b200.nets import drop
    gold = np.load(FIXTURE)
    x, batch = torch.from_numpy(gold["drop/x"]).float(), torch.from_numpy(gold["drop/batch"])
    module = drop.GraphDropPath(0.4).train()
    torch.manual_seed(321)
    without = module(x, batch)
    torch.manual_seed(321)
    with_n = module(x, batch, n_graphs=int(batch.max()) + 1)
    assert torch.equal(with_n, without)
    assert torch.equal(with_n, torch.from_numpy(gold["drop/graph_drop_path"]).float())
    # the per-node factor for planar [N, d, C] blocks makes the same draws
    torch.manual_seed(321)
    s = module.node_scale(x.view(x.shape[0], 1, -1), batch, int(batch.max()) + 1)
    assert torch.equal(x * s.view(-1, 1), with_n)


def _run_qm9(model, pos, batch, z, seed, n_graphs):
    model.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    out = model(f_in=None, pos=pos, batch=batch, node_atom=z, n_graphs=n_graphs)
    out.pow(2).sum().backward()
    return out.detach(), _flat_grads(model)


def test_planar_stochastic_depth_matches_the_stock_route():
    """QM9 ``nonlinear_l2`` in training with stochastic depth (rate 0.3: some graphs drop) and attention dropout 0.2: the
    planar blocks draw in the stock order (attention mask, attention branch, FFN branch) and give the same energies and
    parameter gradients as the stock e3nn-layout ``TransBlock.forward``."""
    from equiformer_b200.nets import graph_attention_transformer as G
    model = _model("graph_attention_transformer_nonlinear_l2", drop_path_rate=0.3)
    pos, batch, z = molecules([5, 8, 6, 7, 4, 6], seed=4, dtype=torch.float64)
    assert all(blk.supports_planar for blk in model.blocks[:-1])          # the last block projects to irreps_feature
    calls = {"planar": 0, "stock": 0}
    orig_planar, orig_forward, orig_supports = G.TransBlock.forward_planar, G.TransBlock.forward, G.TransBlock.supports_planar

    def spy_planar(self, *a, **k):
        calls["planar"] += 1
        return orig_planar(self, *a, **k)

    def spy_forward(self, *a, **k):
        calls["stock"] += 1
        return orig_forward(self, *a, **k)

    G.TransBlock.forward_planar, G.TransBlock.forward = spy_planar, spy_forward
    try:
        with emulated_kernels_with_masks():
            out_p, grads_p = _run_qm9(model, pos, batch, z, seed=11, n_graphs=6)
            n_planar = dict(calls)
            G.TransBlock.supports_planar = property(lambda self: False)  # force the stock route
            calls.update(planar=0, stock=0)
            out_s, grads_s = _run_qm9(model, pos, batch, z, seed=11, n_graphs=6)
            # and without n_graphs (host read of batch.max()) the stock route makes the same draws
            out_h, _ = _run_qm9(model, pos, batch, z, seed=11, n_graphs=None)
    finally:
        G.TransBlock.forward_planar, G.TransBlock.forward = orig_planar, orig_forward
        G.TransBlock.supports_planar = orig_supports
    assert n_planar["planar"] == len(model.blocks) - 1 and n_planar["stock"] == 1
    assert calls["planar"] == 0 and calls["stock"] == 2 * len(model.blocks)
    assert rel_err(out_p, out_s) < 1e-10
    assert rel_err(grads_p, grads_s) < 1e-10
    assert torch.equal(out_h, out_s)
    # the regularisers are in effect: another seed gives other energies
    with emulated_kernels_with_masks():
        out_o, _ = _run_qm9(model, pos, batch, z, seed=12, n_graphs=6)
    assert rel_err(out_o, out_p) > 1e-6


def test_md17_force_step_with_attention_dropout_fused_matches_unfused_on_host(monkeypatch):
    """The create_graph path of the masked K2 (``AttnAggregate(SegSoftmax(z) * keep, V)``) against the unfused
    softmax -> nn.Dropout -> aggregate composition, float64 with emulated kernels: energy, forces and the gradient of a
    force loss from the same seed."""
    from equiformer_b200 import ops
    model = _model("graph_attention_transformer_nonlinear_l2_md17", irreps_in="64x0e", num_basis=32)
    assert model.blocks[0].ga.alpha_dropout.p == 0.2
    pos, batch, z = aspirin_like(seed=1, dtype=torch.float64)

    def step():
        model.zero_grad(set_to_none=True)
        torch.manual_seed(5)
        energy, forces = model(node_atom=z, pos=pos.clone(), batch=batch)
        (energy.sum() + (forces ** 2).sum()).backward()
        return energy.detach(), forces.detach(), _flat_grads(model)

    used = []
    orig = ops.MaskedSoftmaxAggregate.apply
    monkeypatch.setattr(ops.MaskedSoftmaxAggregate, "apply", lambda *a: used.append(1) or orig(*a))
    with emulated_kernels_with_masks():
        fused = step()
        assert used
        monkeypatch.setattr(ops, "softmax_aggregate_ok", lambda lay, z: False)
        used.clear()
        unfused = step()
        assert not used
    for a, b in zip(fused, unfused):
        assert rel_err(a, b) < 1e-10


# ------------------------------------------------------------------------------------------------ GPU: kernels

def _graph(n_nodes, E, seed, device):
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(seed)
    dst = torch.randint(0, n_nodes, (E,), generator=g)
    dst[dst == 1] = 0                                                        # node 1 has no incoming edge
    dst = torch.sort(dst).values
    src = torch.randint(0, n_nodes, (E,), generator=g)
    return ops.Graph(src.to(device), dst.to(device), n_nodes), dst


def _ref_masked(lay, z, keep, Vs, dst, n_nodes):
    """float64 torch: PyG softmax, times the mask, weighted scatter over destinations (differentiable)."""
    from oracle import equiformer_ref as R
    a = R.pyg_softmax(z, dst, n_nodes) * keep
    outs = []
    for g, V in enumerate(Vs):
        C = lay.Cs[g]
        head = torch.arange(C) // (C // lay.n_heads)
        outs.append(torch.zeros((n_nodes,) + tuple(V.shape[1:]), dtype=V.dtype).index_add(0, dst, V * a[:, head][:, None, :]))
    return outs


HEAD_LAYOUTS = {"qm9": (4, (1, 3, 5), (128, 64, 32)),     # 4 heads of 32x0e+16x1e+8x2e (also the MD17 l2 layout)
                "oc20": (8, (1, 3), (256, 128))}          # 8 heads of 32x0e+16x1e


@pytest.mark.gpu
@pytest.mark.parametrize("layout", list(HEAD_LAYOUTS))
def test_masked_k2_family_vs_float64(cuda_device, layout):
    """K2 with a p = 0.2 mask: outputs, z- and V-gradients (first-order kernels) and second-order gradients against
    float64; ``keep=None`` and an all-ones mask reproduce the unmasked kernel bit for bit."""
    from equiformer_b200 import ops
    H, dims, chans = HEAD_LAYOUTS[layout]
    n_nodes, E = 97, 2100
    graph, dst = _graph(n_nodes, E, 3, cuda_device)
    lay = ops.HeadLayout(list(dims), list(chans), H)
    g = torch.Generator().manual_seed(8)
    z = torch.randn(E, H, generator=g) * 2
    Vs = [torch.randn(E, d, c, generator=g) for d, c in zip(dims, chans)]
    Gs = [torch.randn(n_nodes, d, c, generator=g) for d, c in zip(dims, chans)]
    keep = (torch.rand(E, H, generator=g) >= 0.2).float() / 0.8
    assert 0 < int((keep == 0).sum()) < E * H
    d = lambda t: t.to(cuda_device)
    assert ops.softmax_aggregate_ok(lay, d(z))

    # forward and first-order gradients
    zz, kk, vv = d(z).requires_grad_(True), d(keep), [d(v).requires_grad_(True) for v in Vs]
    outs = ops.MaskedSoftmaxAggregate.apply(lay, graph, zz, kk, *vv)
    grads = torch.autograd.grad(outs, [zz, *vv], [d(t) for t in Gs])
    z64, v64 = z.double().requires_grad_(True), [v.double().requires_grad_(True) for v in Vs]
    ref = _ref_masked(lay, z64, keep.double(), v64, dst, n_nodes)
    ref_grads = torch.autograd.grad(ref, [z64, *v64], [t.double() for t in Gs])
    for a, b in zip(outs, ref):
        assert rel_err(a, b) < 1e-5
    for a, b in zip(grads, ref_grads):
        assert rel_err(a, b) < 1e-5

    # second order (the MD17 force loss differentiates the first-order gradients again)
    r = torch.Generator().manual_seed(9)
    wz = torch.randn(E, H, generator=r)
    wv = [torch.randn(v.shape, generator=r) for v in Vs]

    def second(apply, z_, vs_, gs_, wz_, wv_):
        gz, *gv = torch.autograd.grad(apply(z_, vs_), [z_, *vs_], gs_, create_graph=True)
        s = (gz * wz_).sum() + sum((a * b).sum() for a, b in zip(gv, wv_))
        return torch.autograd.grad(s, [z_, *vs_])

    zz, vv = d(z).requires_grad_(True), [d(v).requires_grad_(True) for v in Vs]
    g2 = second(lambda z_, vs_: ops.MaskedSoftmaxAggregate.apply(lay, graph, z_, kk, *vs_), zz, vv, [d(t) for t in Gs],
                d(wz), [d(t) for t in wv])
    z64, v64 = z.double().requires_grad_(True), [v.double().requires_grad_(True) for v in Vs]
    g2_ref = second(lambda z_, vs_: _ref_masked(lay, z_, keep.double(), vs_, dst, n_nodes), z64, v64,
                    [t.double() for t in Gs], wz.double(), [t.double() for t in wv])
    for a, b in zip(g2, g2_ref):
        assert rel_err(a, b) < 1e-4

    # no mask: the same launches and bits as the unmasked autograd function
    def first(apply):
        z_, vs_ = d(z).requires_grad_(True), [d(v).requires_grad_(True) for v in Vs]
        o = apply(z_, vs_)
        return list(o) + list(torch.autograd.grad(o, [z_, *vs_], [d(t) for t in Gs]))

    plain = first(lambda z_, vs_: ops.SoftmaxAggregate.apply(lay, graph, z_, *vs_))
    for k in (None, torch.ones_like(kk)):
        other = first(lambda z_, vs_: ops.MaskedSoftmaxAggregate.apply(lay, graph, z_, k, *vs_))
        for a, b in zip(plain, other):
            assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ GPU: same draws

def _fused_and_unfused(monkeypatch, run):
    """``run()`` from the same seed on the fused route (must use the masked K2) and on the unfused one."""
    from equiformer_b200 import ops
    used = []
    orig = ops.MaskedSoftmaxAggregate.apply
    monkeypatch.setattr(ops.MaskedSoftmaxAggregate, "apply", lambda *a: used.append(1) or orig(*a))
    torch.manual_seed(17)
    fused = run()
    assert used, "the fused route did not run"
    monkeypatch.setattr(ops, "softmax_aggregate_ok", lambda lay, z: False)
    used.clear()
    torch.manual_seed(17)
    unfused = run()
    assert not used
    return fused, unfused


@pytest.mark.gpu
def test_graph_attention_dropout_fused_matches_unfused(cuda_device, monkeypatch):
    """One ``GraphAttention`` (QM9 sizes) in training at p = 0.2: output and gradients (input and parameters) of the
    masked K2 route equal those of softmax -> nn.Dropout -> aggregate from the same seed."""
    from equiformer_b200 import o3
    from equiformer_b200.graph import radius_graph
    from equiformer_b200.nets import GraphAttention
    from tests.helpers import qm9_like_batch
    torch.manual_seed(0)
    irreps = "128x0e+64x1e+32x2e"
    ga = GraphAttention(irreps, "1x0e", "1x0e+1x1e+1x2e", irreps, [128, 64, 64], "32x0e+16x1e+8x2e", 4,
                        nonlinear_message=True, alpha_drop=0.2, proj_drop=0.0).to(cuda_device).train()
    pos, batch, _ = qm9_like_batch(16, seed=4)
    src, dst = radius_graph(pos, 5.0, batch, max_num_neighbors=1000)
    sh = o3.spherical_harmonics("1x0e+1x1e+1x2e", pos[src] - pos[dst], True, "component")
    g = torch.Generator().manual_seed(5)
    x = torch.randn(pos.shape[0], 480, generator=g)
    rbf = torch.randn(src.numel(), 128, generator=g)
    cot = torch.randn(pos.shape[0], 480, generator=g)
    d = lambda t: t.to(cuda_device)

    def run():
        ga.zero_grad(set_to_none=True)
        xx = d(x).requires_grad_(True)
        out = ga(xx, None, d(src), d(dst), d(sh), d(rbf), d(batch))
        (out * d(cot)).sum().backward()
        return out.detach(), xx.grad, _flat_grads(ga)

    fused, unfused = _fused_and_unfused(monkeypatch, run)
    for a, b in zip(fused, unfused):
        assert rel_err(a, b) < 1e-5
    with torch.no_grad():
        ga.eval()
        plain = ga(d(x), None, d(src), d(dst), d(sh), d(rbf), d(batch))
    assert rel_err(fused[0], plain) > 1e-4                                # the mask dropped something


@pytest.mark.gpu
def test_qm9_model_attention_dropout_fused_matches_unfused(cuda_device, monkeypatch):
    model = _model("graph_attention_transformer_nonlinear_l2", cuda_device, torch.float32)
    assert model.blocks[0].ga.alpha_dropout.p == 0.2
    pos, batch, z = (t.to(cuda_device) for t in molecules([9, 14, 5, 11, 7], seed=2))

    def run():
        model.zero_grad(set_to_none=True)
        out = model(f_in=None, pos=pos, batch=batch, node_atom=z, n_graphs=5)
        out.pow(2).sum().backward()
        return out.detach(), _flat_grads(model)

    fused, unfused = _fused_and_unfused(monkeypatch, run)
    for a, b in zip(fused, unfused):
        assert rel_err(a, b) < 1e-5


@pytest.mark.gpu
def test_md17_force_step_attention_dropout_fused_matches_unfused(cuda_device, monkeypatch):
    """``nonlinear_l2_md17`` energy + forces and the gradient of a force loss (double backward through the masked K2)."""
    model = _model("graph_attention_transformer_nonlinear_l2_md17", cuda_device, torch.float32, irreps_in="64x0e")
    assert model.blocks[0].ga.alpha_dropout.p == 0.2
    pos, batch, z = (t.to(cuda_device) for t in aspirin_like(seed=1))

    def run():
        model.zero_grad(set_to_none=True)
        energy, forces = model(node_atom=z, pos=pos.clone(), batch=batch)
        (energy.sum() + (forces ** 2).sum()).backward()
        return energy.detach(), forces.detach(), _flat_grads(model)

    fused, unfused = _fused_and_unfused(monkeypatch, run)
    for a, b in zip(fused, unfused):
        assert rel_err(a, b) < 1e-5


# ------------------------------------------------------------------------------------------------ GPU: capture

def _replays_match_eager(replay, eager, bucket):
    """Two replays, each against an eager step started from the generator state the replay started from; the two
    replays draw different masks."""
    losses = []
    for _ in range(2):
        state = torch.cuda.get_rng_state()
        loss_g = replay().clone()
        grads_g = bucket.flat.clone()
        after = torch.cuda.get_rng_state()
        torch.cuda.set_rng_state(state)
        bucket.zero_grad()
        loss_e = eager()
        assert rel_err(loss_g, loss_e) < 1e-5
        assert rel_err(grads_g, bucket.flat) < 1e-5
        assert torch.equal(torch.cuda.get_rng_state(), after)           # the replay advanced the generator as eager did
        losses.append(float(loss_g))
    assert losses[0] != losses[1]                                       # same inputs, fresh draws


@pytest.mark.gpu
def test_graphed_oc20_aux_step_with_regularisers_matches_eager(cuda_device):
    """2-block ``OC20_L1_256_NONLINEAR_AUX`` at ``drop_path_rate=0.5``, ``alpha_drop=0.2`` through ``graphs.GraphedStep``."""
    from equiformer_b200 import ops
    from equiformer_b200.graphs import GraphedStep
    from equiformer_b200.nets.graph_attention_transformer_oc20 import GraphAttentionTransformerOC20, OC20_L1_256_NONLINEAR_AUX
    from equiformer_b200.oc20_objective import masked_l2mae, relaxation_target
    from equiformer_b200.parallel import FlatGradAllReduce
    from tests.test_oc20_aux import _frames
    torch.manual_seed(0)
    cfg = dict(OC20_L1_256_NONLINEAR_AUX, alpha_drop=0.2, drop_path_rate=0.5, num_layers=2)
    model = GraphAttentionTransformerOC20(None, None, 1, **cfg).to(cuda_device).train()
    assert all(blk.supports_planar for blk in model.blocks[:-1])
    bucket = FlatGradAllReduce(model.parameters())
    pos, batch, z, tags, src, dst, edge_vec = _frames(cuda_device, seed=3)
    g = torch.Generator().manual_seed(7)
    aux_target = relaxation_target(pos, pos + 0.3 * torch.randn(pos.shape, generator=g).to(cuda_device), 0.9452036023139954)
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
    step(key, inputs)                                                   # capture (and a first replay)
    assert step.captures == 1

    def eager():
        energy, aux = model.forward_edges(edge_vec, batch, z, tags, src, dst, n_graphs=4)
        loss = loss_of(energy, aux, target, aux_target, tags)
        loss.backward()
        return loss.detach()

    _replays_match_eager(lambda: step(key, inputs), eager, bucket)
    assert step.captures == 1


@pytest.mark.gpu
def test_graphed_qm9_step_with_attention_dropout_matches_eager(cuda_device):
    from equiformer_b200.graphs import GraphedForwardBackward
    from equiformer_b200.parallel import FlatGradAllReduce
    model = _model("graph_attention_transformer_nonlinear_l2", cuda_device, torch.float32)
    assert model.blocks[0].ga.alpha_dropout.p == 0.2
    bucket = FlatGradAllReduce(model.parameters())
    loss_fn = lambda out, tgt: (out - tgt).abs().mean()
    gfb = GraphedForwardBackward(model, loss_fn, bucket, max_radius=5.0)
    pos, batch, z = (t.to(cuda_device) for t in molecules([9, 14, 5, 11, 7], seed=2))
    tgt = torch.linspace(-1, 1, 5).view(5, 1).to(cuda_device)
    gfb(pos, batch, z, tgt)                                             # capture (and a first replay)

    def eager():
        loss = loss_fn(model(f_in=None, pos=pos, batch=batch, node_atom=z, n_graphs=5), tgt)
        loss.backward()
        return loss.detach()

    _replays_match_eager(lambda: gfb(pos, batch, z, tgt), eager, bucket)
    assert gfb.captures == 1
