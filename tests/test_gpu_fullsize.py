"""-m gpu: parity of the EXACT benchmarked path at BASELINE.json's full sizes against the fp64 CPU oracle.

What these add over ``test_gpu_model.py`` (tiny graphs, where every GEMM is below the tensor-core threshold):
* config 2 (128 molecules, E ~ 32.5 k): forward energies and every parameter gradient of the headline model, eager and
  through ``GraphedForwardBackward`` (the path ``bench.py`` times: wgmma 3xTF32 GEMMs + CUDA-graph replay);
* config 3 (MD17 Lmax=3, batch 5): energy, forces and the parameter gradients of the reference's energy + force loss
  (``main_md17.py:384-390``, weights of ``scripts/train/md17/equiformer/se_l3/target@aspirin.sh:22-23``);
* config 4 (OC20 ``l1_256_nonlinear`` shapes, E ~ 58 k): one GraphAttention layer forward AND backward.

Graphs of a batch are independent, so the oracle runs over chunks of graphs (bounded host memory) and its parameter
gradients are summed over the chunks - exact for losses that are sums over graphs, which is what the tests use.
Tolerances as in test_gpu_model.py: 1e-4 relative for energies / forces / node irreps, 1e-3 of the largest entry for
parameter gradients (they accumulate over all edges).
"""
from __future__ import annotations

import pytest
import torch

from tests.helpers import assert_same_grad_presence, rel_err

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
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in model.parameters():
            p.add_(torch.randn(p.shape, generator=g).to(p.device) * 0.05)


def _worst_grad_err(named_grads, ref_grads):
    worst, where = 0.0, None
    for k, g in named_grads.items():
        gref = ref_grads.get(k)
        if not assert_same_grad_presence(k, g, gref):
            continue
        e = ((g.double().cpu() - gref).abs().max() / gref.abs().max().clamp_min(1e-12)).item()
        if e > worst:
            worst, where = e, k
    return worst, where


@pytest.fixture(scope="module")
def qm9_full(cuda_device):
    """Headline model + the full 128-molecule batch + the fp64 oracle's energies and parameter gradients of
    ``sum_m c_m E_m`` (computed in chunks of 16 molecules)."""
    from equiformer_b200.synthetic import qm9_like_batch
    R = _oracle()
    model = _build("graph_attention_transformer_nonlinear_l2", cuda_device)
    _perturb(model)
    pos, batch, z = qm9_like_batch(128, seed=0)
    coef = torch.linspace(-1.0, 1.0, 128).view(128, 1) + 0.3
    params = {k: v.requires_grad_(v.is_floating_point() and v.numel() > 0)
              for k, v in R.cast_params(model.state_dict(), torch.float64).items()}
    energies = []
    chunk = 16
    for m0 in range(0, 128, chunk):
        keep = (batch >= m0) & (batch < m0 + chunk)
        e = R.model_forward(params, R.Config(), pos[keep].double(), batch[keep] - m0, z[keep], chunk)
        (e * coef[m0:m0 + chunk].double()).sum().backward()
        energies.append(e.detach())
    ref_e = torch.cat(energies)
    ref_g = {k: v.grad.clone() for k, v in params.items() if v.grad is not None}
    return model, (pos, batch, z, coef), ref_e, ref_g


def test_qm9_full_batch_energy_and_param_grads_eager(cuda_device, qm9_full):
    """BASELINE config 2 at full size, eager: every edge-level product has M >= 16 384 rows -> wgmma kernels."""
    from equiformer_b200 import ops
    model, (pos, batch, z, coef), ref_e, ref_g = qm9_full
    d = lambda t: t.to(cuda_device)
    prof = ops.KernelProfile(time_events=False)
    ops.PROFILE = prof
    try:
        model.zero_grad(set_to_none=True)
        out = model(f_in=None, pos=d(pos), batch=d(batch), node_atom=d(z), n_graphs=128)
        (out * d(coef)).sum().backward()
    finally:
        ops.PROFILE = None
    assert prof.launches > 400          # the hand-written kernels ran (count of our launches in one fwd+bwd)
    assert rel_err(out, ref_e) < 1e-4
    worst, where = _worst_grad_err({k: p.grad for k, p in model.named_parameters()}, ref_g)
    assert worst < 1e-3, (worst, where)


def test_qm9_full_batch_graph_replay_matches_oracle(cuda_device, qm9_full):
    """The same through GraphedForwardBackward (capture + replay), the path bench.py times."""
    from equiformer_b200.graphs import GraphedForwardBackward
    from equiformer_b200.parallel import FlatGradAllReduce
    model, (pos, batch, z, coef), ref_e, ref_g = qm9_full
    d = lambda t: t.to(cuda_device)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    model.zero_grad(set_to_none=True)
    bucket = FlatGradAllReduce(model.parameters())
    gfb = GraphedForwardBackward(model, lambda out, c: (out * c).sum(), bucket, max_radius=5.0)
    loss = None
    for _ in range(2):                   # second call = pure replay
        loss = gfb(d(pos), d(batch), d(z), d(coef)).clone()
    ref_loss = (ref_e * coef.double()).sum()
    assert rel_err(loss, ref_loss) < 1e-4
    grads = {k: p.grad for k, p in model.named_parameters()}
    worst, where = _worst_grad_err(grads, ref_g)
    assert worst < 1e-3, (worst, where)
    assert gfb.captures == 1


def _l2mae(pred, target):
    """reference ``L2MAELoss`` (engine of main_md17.py:197): mean over rows of the Euclidean norm of the difference."""
    return (pred - target).norm(p=2, dim=-1).mean()


def test_md17_l3_batch5_energy_force_training_loss(cuda_device):
    """BASELINE config 3: 5 aspirin-sized conformers, energy + force loss with weights 1 / 100, double backward."""
    from equiformer_b200.synthetic import aspirin_like
    R = _oracle()
    model = _build("graph_attention_transformer_nonlinear_exp_l3_md17", cuda_device, irreps_in="64x0e", num_basis=32)
    _perturb(model)
    confs = [aspirin_like(seed=s) for s in range(5)]
    pos = torch.cat([c[0] for c in confs])
    z = torch.cat([c[2] for c in confs])
    batch = torch.cat([torch.full((21,), i, dtype=torch.long) for i in range(5)])
    g = torch.Generator().manual_seed(11)
    te, tf = torch.randn(5, 1, generator=g), torch.randn(105, 3, generator=g)
    d = lambda t: t.to(cuda_device)
    energy, forces = model(node_atom=d(z), pos=d(pos.clone()), batch=d(batch))
    loss = 1.0 * _l2mae(energy, d(te)) + 100.0 * _l2mae(forces, d(tf))
    loss.backward()

    params = {k: v.requires_grad_(v.is_floating_point() and v.numel() > 0)
              for k, v in R.cast_params(model.state_dict(), torch.float64).items()}
    cfg = R.Config(irreps_node_embedding="128x0e+64x1e+64x2e+32x3e", irreps_sh="1x0e+1x1e+1x2e+1x3e",
                   irreps_head="32x0e+16x1e+16x2e+8x3e", irreps_mlp_mid="384x0e+192x1e+192x2e+96x3e",
                   basis_type="exp", number_of_basis=32, max_atom_type=64, qm9_atom_remap=False)
    e_ref, f_ref = R.energy_and_forces(params, cfg, pos.double(), batch, z, 5, create_graph=True)
    ref_loss = 1.0 * _l2mae(e_ref, te.double()) + 100.0 * _l2mae(f_ref, tf.double())
    ref_loss.backward()
    assert rel_err(energy, e_ref) < 1e-4
    assert rel_err(forces, f_ref) < 1e-4
    assert rel_err(loss, ref_loss) < 1e-4
    ref_g = {k: v.grad for k, v in params.items() if v.grad is not None}
    worst, where = _worst_grad_err({k: p.grad for k, p in model.named_parameters()}, ref_g)
    assert worst < 2e-3, (worst, where)


def test_oc20_l1_layer_full_size_forward_and_backward(cuda_device):
    """BASELINE config 4 shapes at the per-GPU size (16 frames, ~73 atoms, ~50 neighbours, E ~ 58 k): one
    ``l1_256_nonlinear`` GraphAttention layer, node irreps out and the gradients w.r.t. node input, edge harmonics,
    radial basis and every parameter."""
    R = _oracle()
    from oracle import e3nn_ref as e3
    from equiformer_b200 import o3
    from equiformer_b200.graph import radius_graph
    from equiformer_b200.nets import GraphAttention
    from equiformer_b200.synthetic import oc20_like_frames
    torch.manual_seed(0)
    irreps, sh, head = "256x0e+128x1e", "1x0e+1x1e", "32x0e+16x1e"
    ga = GraphAttention(irreps, "1x0e", sh, irreps, [128, 64, 64], head, 8, nonlinear_message=True, alpha_drop=0.0,
                        proj_drop=0.0).to(cuda_device).eval()
    _perturb(ga)
    pos, batch, _z, _tags, _cell = oc20_like_frames(16, seed=0, neighbours=110)   # open boundaries: denser, so E ~ 58 k
    src, dst = radius_graph(pos, 5.0, batch, max_num_neighbors=1000)
    E, n = src.numel(), pos.shape[0]
    assert E > 40000, E
    g = torch.Generator().manual_seed(6)
    sh_e = o3.spherical_harmonics(sh, pos[src] - pos[dst], True, "component")
    x = torch.randn(n, 640, generator=g)
    rbf = torch.randn(E, 128, generator=g)
    cot = torch.randn(n, 640, generator=g)
    d = lambda t: t.to(cuda_device)
    xg, shg, rbfg = d(x).requires_grad_(True), d(sh_e).requires_grad_(True), d(rbf).requires_grad_(True)
    out = ga(xg, None, d(src), d(dst), shg, rbfg, d(batch))
    (out * d(cot)).sum().backward()

    params = {"ga." + k: v.requires_grad_(v.is_floating_point() and v.numel() > 0)
              for k, v in R.cast_params(ga.state_dict(), torch.float64).items()}
    ir = e3.parse_irreps(irreps)
    refs, gx, gsh, grbf = [], [], [], []
    for f0 in range(0, 16, 4):                      # frames are independent graphs: chunk the oracle, sum the gradients
        nodes = ((batch >= f0) & (batch < f0 + 4)).nonzero().flatten()
        n0, n1 = int(nodes[0]), int(nodes[-1]) + 1
        em = (dst >= n0) & (dst < n1)
        xc = x[n0:n1].double().requires_grad_(True)
        shc = sh_e[em].double().requires_grad_(True)
        rc = rbf[em].double().requires_grad_(True)
        o = R.graph_attention(params, "ga", ir, e3.parse_irreps(sh), e3.parse_irreps(head), 8, ir, True, xc,
                              src[em] - n0, dst[em] - n0, shc, rc)
        (o * cot[n0:n1].double()).sum().backward()
        refs.append(o.detach()); gx.append(xc.grad); gsh.append(shc.grad); grbf.append(rc.grad)
    ref = torch.cat(refs)
    assert rel_err(out, ref) < 1e-4
    assert rel_err(xg.grad, torch.cat(gx)) < 2e-4
    assert rel_err(shg.grad, torch.cat(gsh)) < 2e-4       # edges are destination-sorted, so chunks concatenate in order
    assert rel_err(rbfg.grad, torch.cat(grbf)) < 2e-4
    ref_g = {k[3:]: v.grad for k, v in params.items() if v.grad is not None}
    worst, where = _worst_grad_err({k: p.grad for k, p in ga.named_parameters()}, ref_g)
    assert worst < 1e-3, (worst, where)
