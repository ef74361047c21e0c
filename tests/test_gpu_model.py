"""-m gpu: drop-in modules on the H100 (fp32) against the CPU oracle (fp64, same weights, same inputs).

Tolerances follow north_star: energies / node irreps / forces within 1e-4 relative (to the max magnitude of the
reference quantity); parameter gradients within 1e-3 of the largest gradient entry (they accumulate over all edges).
"""
from __future__ import annotations

import pytest
import torch

from tests.helpers import aspirin_like, molecules, qm9_like_batch, rel_err

pytestmark = pytest.mark.gpu


def _oracle():
    from oracle import equiformer_ref as R
    return R


def _build(name, dev, **kw):
    from equiformer_b200.nets import model_entrypoint
    torch.manual_seed(0)
    args = dict(irreps_in="5x0e", radius=5.0, num_basis=128)
    args.update(kw)
    return model_entrypoint(name)(**args).to(dev).eval()


def _perturb(model, seed=1):
    """Make every parameter non-trivial (biases / affine terms are zero- or one-initialised)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in model.parameters():
            p.add_(torch.randn(p.shape, generator=g).to(p.device) * 0.05)


@pytest.mark.parametrize("name,nonlinear", [("graph_attention_transformer_nonlinear_l2", True),
                                            ("graph_attention_transformer_l2", False)])
def test_qm9_model_energy_and_param_grads(cuda_device, name, nonlinear):
    R = _oracle()
    model = _build(name, cuda_device)
    _perturb(model)
    pos, batch, z = molecules([9, 14, 5, 11, 7], seed=2)
    out = model(f_in=None, pos=pos.to(cuda_device), batch=batch.to(cuda_device), node_atom=z.to(cuda_device))
    out.sum().backward()

    params = {k: v.requires_grad_(v.is_floating_point()) for k, v in R.cast_params(model.state_dict(), torch.float64).items()}
    cfg = R.Config(nonlinear_message=nonlinear)
    ref = R.model_forward(params, cfg, pos.double(), batch, z, 5)
    ref.sum().backward()
    assert rel_err(out, ref) < 1e-4
    worst = 0.0
    for k, p in model.named_parameters():
        if p.grad is None:
            continue
        gref = params[k].grad
        assert gref is not None, k
        worst = max(worst, ((p.grad.double().cpu() - gref).abs().max() / gref.abs().max().clamp_min(1e-12)).item())
    assert worst < 1e-3, worst


def test_graph_attention_layer_node_irreps(cuda_device):
    """One GraphAttention layer: node irreps out (e3nn layout) vs oracle, QM9-shaped batch slice."""
    R = _oracle()
    from oracle import e3nn_ref as e3
    from equiformer_b200 import o3
    from equiformer_b200.graph import radius_graph
    from equiformer_b200.nets import GraphAttention
    torch.manual_seed(0)
    irreps = "128x0e+64x1e+32x2e"
    ga = GraphAttention(irreps, "1x0e", "1x0e+1x1e+1x2e", irreps, [128, 64, 64], "32x0e+16x1e+8x2e", 4,
                        nonlinear_message=True, alpha_drop=0.0, proj_drop=0.0).to(cuda_device).eval()
    _perturb(ga)
    pos, batch, _ = qm9_like_batch(8, seed=4)
    src, dst = radius_graph(pos, 5.0, batch, max_num_neighbors=1000)
    vec = pos[src] - pos[dst]
    sh = o3.spherical_harmonics("1x0e+1x1e+1x2e", vec, True, "component")
    g = torch.Generator().manual_seed(5)
    x = torch.randn(pos.shape[0], 480, generator=g)
    rbf = torch.randn(src.numel(), 128, generator=g)
    d = lambda t: t.to(cuda_device)
    out = ga(d(x), None, d(src), d(dst), d(sh), d(rbf), d(batch))
    params = R.cast_params(ga.state_dict(), torch.float64)
    ir = e3.parse_irreps(irreps)
    params = {"ga." + k: v for k, v in params.items()}
    ref = R.graph_attention(params, "ga", ir, e3.parse_irreps("1x0e+1x1e+1x2e"), e3.parse_irreps("32x0e+16x1e+8x2e"), 4, ir,
                            True, x.double(), src, dst, sh.double(), rbf.double())
    assert rel_err(out, ref) < 1e-4


@pytest.mark.parametrize("name,basis,lmax", [("graph_attention_transformer_nonlinear_exp_l2_md17", 128, 2),
                                             ("graph_attention_transformer_nonlinear_exp_l3_md17", 32, 3)])
def test_md17_energy_forces_and_double_backward(cuda_device, name, basis, lmax):
    """Energy, autograd forces (first backward inside forward) and the gradient of a force loss (backward of backward)."""
    R = _oracle()
    model = _build(name, cuda_device, irreps_in="64x0e", num_basis=basis)
    _perturb(model)
    pos, batch, z = aspirin_like(seed=1)
    energy, forces = model(node_atom=z.to(cuda_device), pos=pos.clone().to(cuda_device), batch=batch.to(cuda_device))
    loss = energy.sum() + (forces ** 2).sum()
    loss.backward()

    params = {k: v.requires_grad_(v.is_floating_point()) for k, v in R.cast_params(model.state_dict(), torch.float64).items()}
    if lmax == 2:
        cfg = R.Config(basis_type="exp", number_of_basis=basis, max_atom_type=64, qm9_atom_remap=False)
    else:
        cfg = R.Config(irreps_node_embedding="128x0e+64x1e+64x2e+32x3e", irreps_sh="1x0e+1x1e+1x2e+1x3e",
                       irreps_head="32x0e+16x1e+16x2e+8x3e", irreps_mlp_mid="384x0e+192x1e+192x2e+96x3e",
                       basis_type="exp", number_of_basis=basis, max_atom_type=64, qm9_atom_remap=False)
    e_ref, f_ref = R.energy_and_forces(params, cfg, pos.double(), batch, z, 1, create_graph=True)
    (e_ref.sum() + (f_ref ** 2).sum()).backward()
    assert rel_err(energy, e_ref) < 1e-4
    assert rel_err(forces, f_ref) < 1e-4
    worst = 0.0
    for k, p in model.named_parameters():
        if p.grad is None or params[k].grad is None:
            continue
        gref = params[k].grad
        worst = max(worst, ((p.grad.double().cpu() - gref).abs().max() / gref.abs().max().clamp_min(1e-12)).item())
    assert worst < 2e-3, worst


def test_qm9_full_batch_invariants(cuda_device):
    """BASELINE config 2 at full size (128 molecules): rotation/translation invariance and permutation of graphs."""
    model = _build("graph_attention_transformer_nonlinear_l2", cuda_device)
    pos, batch, z = qm9_like_batch(128, seed=0)
    d = lambda t: t.to(cuda_device)
    with torch.no_grad():
        e0 = model(f_in=None, pos=d(pos), batch=d(batch), node_atom=d(z))
        g = torch.Generator().manual_seed(9)
        q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
        if torch.det(q) < 0:
            q[:, 0] = -q[:, 0]
        pos_r = (pos.double() @ q.T + torch.tensor([0.3, -1.2, 2.0], dtype=torch.float64)).float()
        e1 = model(f_in=None, pos=d(pos_r), batch=d(batch), node_atom=d(z))
    assert e0.shape == (128, 1)
    assert rel_err(e1, e0) < 1e-4


def test_cuda_graph_replay_matches_eager(cuda_device):
    """GraphedForwardBackward: replayed forward+backward == eager forward+backward (loss and every gradient), also
    after the inputs change (same signature) - the captured graph must read the refreshed static buffers."""
    from equiformer_b200.graphs import GraphedForwardBackward
    from equiformer_b200.parallel import FlatGradAllReduce
    model = _build("graph_attention_transformer_nonlinear_l2", cuda_device)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    bucket = FlatGradAllReduce(model.parameters())
    loss_fn = lambda out, tgt: (out - tgt).abs().mean()
    gfb = GraphedForwardBackward(model, loss_fn, bucket, max_radius=5.0)
    pos, batch, z = molecules([9, 14, 5, 11, 7], seed=2)
    d = lambda t: t.to(cuda_device)
    tgt = torch.linspace(-1, 1, 5).view(5, 1)
    for trial in range(2):
        p = pos if trial == 0 else pos + 0.01 * torch.sin(pos * 3.0)   # small move: same atoms, same edge count expected
        loss_g = gfb(d(p), d(batch), d(z), d(tgt)).clone()
        grads_g = bucket.flat.clone()
        bucket.zero_grad()
        out = model(f_in=None, pos=d(p), batch=d(batch), node_atom=d(z), n_graphs=5)
        loss_e = loss_fn(out, d(tgt))
        loss_e.backward()
        assert rel_err(loss_g, loss_e) < 1e-6
        assert rel_err(grads_g, bucket.flat) < 1e-5
    assert gfb.captures <= 2


def test_oc20_l1_layer_vs_oracle(cuda_device):
    """BASELINE config 4 shapes (l1_256_nonlinear: 256x0e+128x1e, 8 heads of 32x0e+16x1e): one GraphAttention layer."""
    R = _oracle()
    from oracle import e3nn_ref as e3
    from equiformer_b200 import o3
    from equiformer_b200.graph import radius_graph
    from equiformer_b200.nets import GraphAttention
    torch.manual_seed(0)
    irreps, sh, head = "256x0e+128x1e", "1x0e+1x1e", "32x0e+16x1e"
    ga = GraphAttention(irreps, "1x0e", sh, irreps, [128, 64, 64], head, 8, nonlinear_message=True, alpha_drop=0.0,
                        proj_drop=0.0).to(cuda_device).eval()
    _perturb(ga)
    g = torch.Generator().manual_seed(6)
    pos = torch.rand(73, 3, generator=g) * 9.0
    batch = torch.zeros(73, dtype=torch.long)
    src, dst = radius_graph(pos, 5.0, batch, max_num_neighbors=1000)
    sh_e = o3.spherical_harmonics(sh, pos[src] - pos[dst], True, "component")
    x = torch.randn(73, 640, generator=g)
    rbf = torch.randn(src.numel(), 128, generator=g)
    d = lambda t: t.to(cuda_device)
    out = ga(d(x), None, d(src), d(dst), d(sh_e), d(rbf), d(batch))
    params = {"ga." + k: v for k, v in R.cast_params(ga.state_dict(), torch.float64).items()}
    ir = e3.parse_irreps(irreps)
    ref = R.graph_attention(params, "ga", ir, e3.parse_irreps(sh), e3.parse_irreps(head), 8, ir, True, x.double(), src, dst,
                            sh_e.double(), rbf.double())
    assert rel_err(out, ref) < 1e-4


def test_stress_cell_rotation_invariance(cuda_device):
    """BASELINE config 5 size (10 k atoms, ~50 neighbours, E ~ 5e5, Lmax=2): forward energies are rotation invariant."""
    model = _build("graph_attention_transformer_nonlinear_l2", cuda_device)
    g = torch.Generator().manual_seed(0)
    n = 10000
    side = (n / (50.0 / (4.0 / 3.0 * 3.141592653589793 * 125.0))) ** (1.0 / 3.0)
    pos = torch.rand(n, 3, generator=g, dtype=torch.float64) * side
    z = torch.tensor([1, 6, 7, 8, 9])[torch.randint(0, 5, (n,), generator=g)]
    batch = torch.zeros(n, dtype=torch.long)
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    if torch.det(q) < 0:
        q[:, 0] = -q[:, 0]
    d = lambda t: t.to(cuda_device)
    with torch.no_grad():
        e0 = model(f_in=None, pos=d(pos.float()), batch=d(batch), node_atom=d(z))
        e1 = model(f_in=None, pos=d((pos @ q.T).float()), batch=d(batch), node_atom=d(z))
    assert torch.isfinite(e0).all()
    assert rel_err(e1, e0) < 1e-4


def test_bucketed_stream_of_batches_matches_eager(cuda_device):
    """``BucketedForwardBackward``: six different molecule batches replayed through <= 3 captured graphs (atoms / edges
    padded to bucket sizes with a dummy molecule) give the eager loss and gradients of each batch."""
    from equiformer_b200.graphs import BucketedForwardBackward
    from equiformer_b200.parallel import FlatGradAllReduce
    model = _build("graph_attention_transformer_nonlinear_l2", cuda_device)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    bucket = FlatGradAllReduce(model.parameters())
    loss_fn = lambda out, tgt: (out - tgt).abs().mean()
    bfb = BucketedForwardBackward(model, loss_fn, bucket, max_radius=5.0, atom_quantum=32, edge_quantum=512)
    d = lambda t: t.to(cuda_device)
    tgt = torch.linspace(-1, 1, 6).view(6, 1)
    batches = [qm9_like_batch(6, seed=seed) for seed in range(6)]
    replayed = []
    for pos, batch, z in batches:            # the stream first (captures happen here), the eager reference afterwards
        loss_g = bfb(d(pos), d(batch), d(z), d(tgt)).clone()
        replayed.append((loss_g, bucket.flat.clone()))
    assert bfb.captures <= 4, bfb.captures
    for (pos, batch, z), (loss_g, grads_g) in zip(batches, replayed):
        bucket.zero_grad()
        out = model(f_in=None, pos=d(pos), batch=d(batch), node_atom=d(z), n_graphs=6)
        loss_e = loss_fn(out, d(tgt))
        loss_e.backward()
        assert rel_err(loss_g, loss_e) < 1e-5
        assert rel_err(grads_g, bucket.flat) < 2e-5


def test_fused_forward_model_matches_unfused_model(cuda_device, monkeypatch):
    """K1 on (EQF_FUSED=1: every depth-wise product feeds its linears on chip, backward recomputes) against K1 off on the
    same model and batch: energies and every parameter gradient."""
    from equiformer_b200 import ops
    model = _build("graph_attention_transformer_nonlinear_l2", cuda_device)
    _perturb(model)
    pos, batch, z = qm9_like_batch(24, seed=5)
    d = lambda t: t.to(cuda_device)
    res = {}
    for mode in ("0", "1"):
        monkeypatch.setattr(ops, "_FUSED_MODE", mode)
        monkeypatch.setattr(ops, "_FUSED", mode != "0")
        prof = ops.KernelProfile(time_events=False)
        ops.PROFILE = prof
        try:
            model.zero_grad(set_to_none=True)
            out = model(f_in=None, pos=d(pos), batch=d(batch), node_atom=d(z), n_graphs=24)
            (out * torch.linspace(-1, 1, 24, device=cuda_device).view(24, 1)).sum().backward()
        finally:
            ops.PROFILE = None
        res[mode] = (out.detach().clone(), {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None},
                     prof.launches)
    assert rel_err(res["1"][0], res["0"][0]) < 2e-5
    worst = max(rel_err(res["1"][1][k], g) for k, g in res["0"][1].items())
    assert worst < 2e-4, worst
    assert res["1"][2] != res["0"][2]          # the two modes really launched different kernel sets
