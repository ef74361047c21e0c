"""DeNS training of the MD17 ``equiformer_dens`` configurations: ``Equiformer_MD17_DeNS.forward_edges``, the objective of
``equiformer_b200.md17_dens_objective`` and the captured, bucketed training step ``graphs.DensTrainStep``.

Pinned to the reference's own code: ``tests/golden/reference_dens_noise.npz`` (the trainer's noise function,
``tests/golden/make_reference_golden_dens_train.py``) and the two DeNS model fixtures, ``reference_model_dens_small.npz``
(L2-like) and ``reference_model_dens_l3_small.npz`` (``1x3e`` harmonics, ``tests/golden/make_reference_golden_dens_l3.py``).
On the CPU in float64 with the kernels emulated; on a GPU the CUDA path, the full-size configurations' kernel routes and
the captured step against the eager one.
"""
from __future__ import annotations

import os
import types

import numpy as np
import pytest
import torch

from tests.helpers import rel_err
from tests.reference_fixtures import GOLDEN, dens_setup

NOISE = os.path.join(GOLDEN, "reference_dens_noise.npz")
FIXTURES = {"l2_small": "reference_model_dens_small.npz", "l3_small": "reference_model_dens_l3_small.npz"}
NOISE_CASES = [(None, 0.0), (None, 0.25), (None, 1.0), (0.25, 0.0), (0.25, 0.25), (0.25, 1.0)]
TASK_MEAN, TASK_STD, STD = -0.37, 1.9, 0.05


def _case_name(corrupt_ratio, prob):
    return f"cr{'none' if corrupt_ratio is None else corrupt_ratio}_p{prob}"


# --------------------------------------------------------------------------------------------------- the objective (CPU)

@pytest.mark.parametrize("corrupt_ratio,prob", NOISE_CASES)
def test_noise_matches_reference_trainer(corrupt_ratio, prob):
    """``add_masked_gaussian_noise`` with a seeded generator makes the reference's draws in its order and dtype: masks,
    noise, noised positions and force encoding are bit for bit the fixture's."""
    from equiformer_b200.md17_dens_objective import add_masked_gaussian_noise
    g = np.load(NOISE)
    t = lambda k: torch.from_numpy(g[k])
    name = _case_name(corrupt_ratio, prob)
    pos, dy, batch = t("pos"), t("dy"), t("batch")
    before = pos.clone()
    gen = torch.Generator().manual_seed(int(g[f"{name}/seed"]))
    pos_n, noise_vec, noise_mask, dpm, force = add_masked_gaussian_noise(pos, dy, batch, 12, float(g["std"]), prob,
                                                                         corrupt_ratio, generator=gen)
    assert torch.equal(pos, before)
    assert torch.equal(noise_mask, t(f"{name}/noise_mask"))
    assert torch.equal(dpm, t(f"{name}/denoising_pos_mask"))
    assert torch.equal(noise_vec, t(f"{name}/noise_vec"))
    assert torch.equal(pos_n, t(f"{name}/pos"))
    assert torch.equal(force, t(f"{name}/force"))


def _boolean_index_loss(pred_y, pred_dy, y, dy, noise_vec, noise_mask, w_e, w_f, w_dn):
    """The reference trainer's statement (main_md17_dens.py:389-403) with ``L2MAELoss``."""
    crit = lambda a, b: torch.norm(a - b, p=2, dim=-1).mean()
    loss_e = crit(pred_y, (y - TASK_MEAN) / TASK_STD)
    loss_f = crit(pred_dy[~noise_mask], dy[~noise_mask] / TASK_STD)
    loss_dn = crit(pred_dy[noise_mask], noise_vec[noise_mask] / STD)
    loss = w_e * loss_e
    if not loss_f.isnan():
        loss = loss + w_f * loss_f
    if not loss_dn.isnan():
        loss = loss + w_dn * loss_dn
    return loss


@pytest.mark.parametrize("case", ["mixed", "none_denoised", "all_noised", "padding"])
def test_dens_loss_equals_boolean_index_statement(case):
    from equiformer_b200.md17_dens_objective import dens_loss
    g = torch.Generator().manual_seed(3)
    G, N = 4, 60
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    pred_y, y, pred_dy, dy, noise_vec = r(G, 1), r(G, 1), r(N, 3), r(N, 3), STD * r(N, 3)
    noise_mask = {"mixed": torch.rand(N, generator=g) < 0.3, "none_denoised": torch.zeros(N, dtype=torch.bool),
                  "all_noised": torch.ones(N, dtype=torch.bool), "padding": torch.rand(N, generator=g) < 0.3}[case]
    w_dn = torch.tensor([2.5], dtype=torch.float64)
    ref = _boolean_index_loss(pred_y, pred_dy, y, dy, noise_vec, noise_mask, 1.0, 80.0, 2.5)
    if case != "padding":
        ours = dens_loss(pred_y, pred_dy, y, dy, noise_vec, noise_mask, TASK_MEAN, TASK_STD, STD, 1.0, 80.0, w_dn)
    else:                                  # 13 padding atoms with arbitrary values, weight 0, half of them "noised"
        P = 13
        pad = lambda t, v: torch.cat([t, v])
        ours = dens_loss(pred_y, pad(pred_dy, r(P, 3)), y, pad(dy, r(P, 3)), pad(noise_vec, r(P, 3)),
                         pad(noise_mask, torch.arange(P) % 2 == 0), TASK_MEAN, TASK_STD, STD, 1.0, 80.0, w_dn,
                         atom_weight=pad(torch.ones(N, dtype=torch.float64), torch.zeros(P, dtype=torch.float64)))
    assert ours.shape == ()
    assert rel_err(ours, ref) < 1e-14
    if case == "none_denoised":            # the denoising term is dropped, as the reference's NaN skip drops it
        assert rel_err(ours, _boolean_index_loss(pred_y, pred_dy, y, dy, noise_vec, noise_mask, 1.0, 80.0, 0.0)) < 1e-14
    if case == "all_noised":               # the force term is dropped
        assert rel_err(ours, _boolean_index_loss(pred_y, pred_dy, y, dy, noise_vec, noise_mask, 1.0, 0.0, 2.5)) < 1e-14


def test_denoising_pos_weight_schedule():
    from equiformer_b200.md17_dens_objective import denoising_pos_weight
    assert denoising_pos_weight(0, 1500, 5.0, True) == 5.0
    assert denoising_pos_weight(750, 1500, 5.0, True) == 2.5
    assert denoising_pos_weight(1500, 1500, 5.0, True) == 0.0
    assert denoising_pos_weight(3000, 1500, 5.0, True) == 0.0
    assert denoising_pos_weight(750, 1500, 5.0, False) == 5.0


def test_dens_configuration_dicts():
    """The ``model:`` blocks of the two ``equiformer_dens`` configurations build, with the head predicting ``1x1e`` from the
    widened final feature and an energy head fed by its ``512x0e`` part."""
    from equiformer_b200.nets.equiformer_md17_dens import MD17_DENS_L2, MD17_DENS_L3, Equiformer_MD17_DeNS
    for cfg, feature in ((MD17_DENS_L2, "512x0e+256x1e+128x2e"), (MD17_DENS_L3, "512x0e+256x1e+256x2e+128x3e")):
        model = Equiformer_MD17_DeNS(**cfg)
        assert str(model.irreps_feature) == feature and len(model.blocks) == 6 and model.use_force_encoding
        assert str(model.energy_head[0].irreps_out) == "512x0e"
        assert str(model.denoising_pos_head.irreps_node_output) == "1x1e"
        assert model.blocks[-1].ffn_shortcut is not None
    assert MD17_DENS_L3["irreps_equivariant_inputs"] == MD17_DENS_L3["irreps_sh"] == "1x0e+1x1e+1x2e+1x3e"


# ----------------------------------------------------------------------------------------------------- the model (CPU)

def _targets(n_atoms, n_graphs, dtype=torch.float64):
    g = torch.Generator().manual_seed(5)
    return (torch.randn(n_graphs, 1, generator=g, dtype=dtype), torch.randn(n_atoms, 3, generator=g, dtype=dtype),
            STD * torch.randn(n_atoms, 3, generator=g, dtype=dtype))


def _grads(model, loss):
    params = [p for p in model.parameters() if p.requires_grad]
    return [gr for gr in torch.autograd.grad(loss, params, allow_unused=True)]


def _worst(ga, gb):
    return max((rel_err(a, b) for a, b in zip(ga, gb) if b is not None and float(b.abs().max()) > 0), default=0.0)


@pytest.mark.parametrize("which", sorted(FIXTURES))
def test_forward_edges_equals_forward(which):
    """``forward_edges`` on the neighbour list ``forward(data)`` builds gives its energies and outputs, and the parameter
    gradients of the DeNS training loss, to 1e-12."""
    from equiformer_b200.graph import radius_graph
    from equiformer_b200.md17_dens_objective import dens_loss
    from tests._emulation import emulated_kernels
    _case, model, data = dens_setup(FIXTURES[which])
    n, G = data.pos.shape[0], int(data.batch.max()) + 1
    y, dy, noise_vec = _targets(n, G)
    loss_of = lambda e, d: dens_loss(e, d, y, dy, noise_vec, data.noise_mask, TASK_MEAN, TASK_STD, STD, 1.0, 80.0, 5.0)
    with emulated_kernels():
        e_ref, d_ref = model(data)
        g_ref = _grads(model, loss_of(e_ref, d_ref))
        pos = data.pos.detach().clone().requires_grad_(True)
        edge = radius_graph(pos, 5.0, data.batch, max_num_neighbors=1000)
        energy, out = model.forward_edges(data.z, pos, data.batch, edge[0], edge[1], force=data.force,
                                          noise_mask=data.noise_mask, n_graphs=G)
        g_new = _grads(model, loss_of(energy, out))
    assert rel_err(energy, e_ref) < 1e-12 and rel_err(out, d_ref) < 1e-12
    assert _worst(g_new, g_ref) < 1e-12


@pytest.mark.parametrize("which", sorted(FIXTURES))
def test_padding_leaves_real_outputs_unchanged(which):
    """A batch padded by ``graphs.pad_to_bucket`` (dummy atoms never noised, zero force encoding, ``atom_weight`` 0, dummy
    energy row dropped) gives the real atoms' outputs and the parameter gradients of the unpadded batch to 1e-12."""
    from equiformer_b200.graph import radius_graph
    from equiformer_b200.graphs import pad_to_bucket
    from equiformer_b200.md17_dens_objective import dens_loss
    from tests._emulation import emulated_kernels
    _case, model, data = dens_setup(FIXTURES[which])
    n, G = data.pos.shape[0], int(data.batch.max()) + 1
    y, dy, noise_vec = _targets(n, G)
    edge = radius_graph(data.pos, 5.0, data.batch, max_num_neighbors=1000)
    (pos_p, batch_p, z_p, src_p, dst_p, _row_ptr), (Nb, Eb) = pad_to_bucket(data.pos, data.batch, data.z, edge[0], edge[1],
                                                                            G, 8, 64)
    P = Nb - n
    assert P >= 2 and Eb > edge.shape[1] and Eb % 64 == 0
    rows = lambda t: torch.cat([t, t.new_zeros((P,) + tuple(t.shape[1:]))])
    with emulated_kernels():
        pos = data.pos.detach().clone().requires_grad_(True)
        e_ref, d_ref = model.forward_edges(data.z, pos, data.batch, edge[0], edge[1], force=data.force,
                                           noise_mask=data.noise_mask, n_graphs=G)
        g_ref = _grads(model, dens_loss(e_ref, d_ref, y, dy, noise_vec, data.noise_mask, TASK_MEAN, TASK_STD, STD, 1.0,
                                        80.0, 5.0))
        pos_p = pos_p.detach().clone().requires_grad_(True)
        noise_p = rows(data.noise_mask)
        energy, out = model.forward_edges(z_p, pos_p, batch_p, src_p, dst_p, force=rows(data.force), noise_mask=noise_p,
                                          n_graphs=G + 1)
        weight = rows(torch.ones(n, dtype=torch.float64))
        g_pad = _grads(model, dens_loss(energy[:G], out, y, rows(dy), rows(noise_vec), noise_p, TASK_MEAN, TASK_STD, STD,
                                        1.0, 80.0, 5.0, atom_weight=weight))
    assert energy.shape[0] == G + 1
    assert rel_err(energy[:G], e_ref) < 1e-12 and rel_err(out[:n], d_ref) < 1e-12
    assert _worst(g_pad, g_ref) < 1e-12


def test_mirror_dens_l3_matches_reference_model_file():
    """The L3 fixture (``1x3e`` harmonics and force encoding, a ``3e`` block in the feature and the head), kernels
    emulated in float64: energies and outputs to 1e-10, parameter gradients of an energy + output loss to 1e-6."""
    from tests._emulation import emulated_kernels
    case, model, data = dens_setup(FIXTURES["l3_small"])
    with emulated_kernels():
        energy, dy = model(data)
        (energy.sum() + (dy ** 2).sum()).backward()
    assert rel_err(energy, case.t("energy")) < 1e-10
    assert rel_err(dy, case.t("dy")) < 1e-10
    for k, ref in case.grads.items():
        assert rel_err(model.get_parameter(k).grad, ref) < 1e-6, k


# ------------------------------------------------------------------------------------------------------------- GPU

@pytest.mark.gpu
def test_cuda_dens_l3_matches_reference_model_file(cuda_device):
    case, model, data = dens_setup(FIXTURES["l3_small"], cuda_device, torch.float32)
    energy, dy = model(data)
    (energy.sum() + (dy ** 2).sum()).backward()
    assert rel_err(energy, case.t("energy")) < 1e-4
    assert rel_err(dy, case.t("dy")) < 3e-4
    worst = max(rel_err(model.get_parameter(k).grad, ref) for k, ref in case.grads.items())
    assert worst < 2e-3, worst


def _full_size_model(name, dev, seed=0):
    """``MD17_DENS_L2`` / ``MD17_DENS_L3`` with perturbed biases / offsets (they start at zero)."""
    from equiformer_b200.nets import equiformer_md17_dens as M
    torch.manual_seed(seed)
    model = M.Equiformer_MD17_DeNS(**getattr(M, name))
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for pname, p in model.named_parameters():
            if p.abs().max() == 0 or "bias" in pname or "offset" in pname:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
    return model.to(dev).train()


def _conformers(n_graphs, seed, dev):
    """``n_graphs`` aspirin-sized conformers with seeded energy / force targets."""
    from equiformer_b200.synthetic import aspirin_like
    confs = [aspirin_like(seed=seed * 64 + s) for s in range(n_graphs)]
    pos = torch.cat([c[0] for c in confs])
    z = torch.cat([c[2] for c in confs])
    batch = torch.arange(n_graphs).repeat_interleave(21)
    g = torch.Generator().manual_seed(seed + 99)
    y, dy = torch.randn(n_graphs, 1, generator=g), torch.randn(21 * n_graphs, 3, generator=g)
    return tuple(t.to(dev) for t in (pos, batch, z, y, dy))


SIZES = {"MD17_DENS_L2": 8, "MD17_DENS_L3": 5}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SIZES))
def test_full_size_routes_take_generated_kernels(name, cuda_device):
    """At full size every block's and the denoising head's tensor products resolve to the generated ``qm9_l2`` /
    ``md17_l3`` kernels, and the head's forward and backward contain no edge-sized torch GEMM or scatter."""
    from torch.profiler import ProfilerActivity, profile

    from equiformer_b200 import ops
    from equiformer_b200.md17_dens_objective import add_masked_gaussian_noise
    model = _full_size_model(name, cuda_device)
    head = model.denoising_pos_head
    for att in [blk.ga for blk in model.blocks] + [head]:
        for sep in (att.sep_act, att.sep_value):
            assert sep.dtp.tp.plan.generated
    B = SIZES[name]
    pos, batch, z, y, dy = _conformers(B, 0, cuda_device)
    pos_n, _nv, noise_mask, _dpm, force = add_masked_gaussian_noise(pos, dy, batch, B, STD, 0.25, 0.25,
                                                                    torch.Generator(device=cuda_device).manual_seed(3))
    data = types.SimpleNamespace(z=z, pos=pos_n, batch=batch, force=force, noise_mask=noise_mask)
    seen = {}
    hook = head.register_forward_pre_hook(lambda m, a, kw: seen.update(kw), with_kwargs=True)
    try:
        energy, out = model(data)
    finally:
        hook.remove()
    assert torch.isfinite(energy).all() and torch.isfinite(out).all()
    E, n = int(seen["edge_src"].numel()), int(pos.shape[0])
    W = torch.randn(n, 3, generator=torch.Generator().manual_seed(2)).to(cuda_device)
    (energy.sum() + (out * W).sum()).backward()       # the whole step once: the graph's source-sorted view is built here
    assert any(float(p.grad.abs().max()) > 0 for p in head.parameters() if p.grad is not None)
    x = seen["node_input"].detach().requires_grad_(True)
    kw = {k: (v.detach() if isinstance(v, torch.Tensor) else v) for k, v in seen.items() if k != "node_input"}
    prof_k = ops.KernelProfile(time_events=True)
    ops.PROFILE = prof_k
    try:
        with profile(activities=[ProfilerActivity.CPU], record_shapes=True) as prof:
            o = head(node_input=x, **kw)
            (o * W).sum().backward()
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


def _trainer(name, dev):
    from equiformer_b200.parallel import FlatAdamW, FlatGradAllReduce
    model = _full_size_model(name, dev)
    bucket = FlatGradAllReduce(model.parameters())
    opt = FlatAdamW(model.named_parameters(), bucket, lr=5e-4, weight_decay=1e-6, no_decay=model.no_weight_decay())
    return model, bucket, opt


@pytest.mark.gpu
@pytest.mark.parametrize("prob,corrupt_ratio", [(0.25, 0.25), (0.0, 0.25), (1.0, None)])
@pytest.mark.parametrize("name", sorted(SIZES))
def test_captured_dens_step_matches_eager(name, prob, corrupt_ratio, cuda_device):
    """Two DeNS training steps through ``graphs.DensTrainStep``: eager noise, neighbour list and padding, then a replay of
    forward + double backward + loss, against the eager unpadded step from the same generator state and the same
    parameters.  Loss, flat gradients and the parameters after AdamW agree; the two batches have different edge counts,
    share one bucket and one capture.
    Weight gradients add with fp32 atomics in no fixed order, hence tolerances and not bit equality."""
    from equiformer_b200.graphs import DensTrainStep
    B, lr = SIZES[name], 5e-4
    model_c, bucket_c, opt_c = _trainer(name, cuda_device)
    model_e, bucket_e, opt_e = _trainer(name, cuda_device)
    kw = dict(task_mean=TASK_MEAN, task_std=TASK_STD, std=STD, prob=prob, corrupt_ratio=corrupt_ratio, w_e=1.0, w_f=80.0)
    step_c = DensTrainStep(model_c, bucket_c, capture=True, **kw)          # default buckets: 32 atoms, 512 edges
    step_e = DensTrainStep(model_e, bucket_e, capture=False, **kw)
    gen_c, gen_e = torch.Generator(device=cuda_device), torch.Generator(device=cuda_device)
    edges = []
    for k, seed in enumerate((0, 1)):
        if k:     # both models start each step from the same parameters and AdamW state (a sign flip of a near-zero
            for a, b in ((opt_c.flat, opt_e.flat), (opt_c.m, opt_e.m), (opt_c.v, opt_e.v)):    # gradient must not carry over)
                a.copy_(b)
        pos, batch, z, y, dy = _conformers(B, seed, cuda_device)
        gen_c.manual_seed(100 + k)
        gen_e.manual_seed(100 + k)
        w_dn = torch.tensor([5.0 * (1 - k / 10)], device=cuda_device)
        loss_c = step_c(pos, batch, z, y, dy, B, w_dn, generator=gen_c).clone()
        loss_e = step_e(pos, batch, z, y, dy, B, w_dn, generator=gen_e)
        assert step_c.last_edges == step_e.last_edges
        edges.append(step_c.last_edges)
        assert torch.isfinite(loss_c) and rel_err(loss_c, loss_e) < 1e-5
        assert rel_err(bucket_c.flat, bucket_e.flat) < 1e-5
        before = opt_e.flat.clone()
        opt_c.step()
        opt_e.step()
        diff = (opt_c.flat - opt_e.flat).abs()
        assert float(diff.max()) <= 2.0 * lr + 1e-6        # at most a sign flip of a near-zero gradient
        g = bucket_e.flat.abs()
        sure = g > 1e-3 * float(g.max())                   # where the gradient is well above its rounding, updates agree
        assert float(diff[sure].max()) < 1e-2 * lr
        assert float((opt_e.flat - before).abs().max()) > 0.5 * lr
    assert edges[0] != edges[1], edges
    assert step_c.captures == 1
