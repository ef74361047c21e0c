"""CPU: host logic of the drop-in modules (layouts, weight views, autograd families) against the oracle.

The kernels themselves cannot run here; ``tests/_emulation.py`` swaps the raw kernel calls for fp64 torch walks over
the same plan tables so that everything *around* the kernels is exercised end to end in fp64 (tolerance 1e-9).
The kernels are compared with the same oracle on the GPU box (tests/test_gpu_*.py).
"""
from __future__ import annotations

import pytest
import torch

from oracle import equiformer_ref as R
from tests._emulation import emulated_kernels
from tests.helpers import aspirin_like, molecules, rel_err


def _build(name, **kw):
    from equiformer_b200.nets import model_entrypoint
    torch.manual_seed(0)
    args = dict(irreps_in="5x0e", radius=5.0, num_basis=128)
    args.update(kw)
    model = model_entrypoint(name)(**args).double().eval()
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for p in model.parameters():
            p.add_(torch.randn(p.shape, generator=g, dtype=torch.float64) * 0.05)
    return model


def _grads_match(model, params, tol):
    worst = 0.0
    for k, p in model.named_parameters():
        if p.grad is None and params[k].grad is None:
            continue
        assert p.grad is not None and params[k].grad is not None, k
        worst = max(worst, ((p.grad - params[k].grad).abs().max() / params[k].grad.abs().max().clamp_min(1e-12)).item())
    assert worst < tol, worst


@pytest.mark.parametrize("name,nonlinear", [("graph_attention_transformer_nonlinear_l2", True),
                                            ("graph_attention_transformer_l2", False)])
def test_qm9_model_matches_oracle(name, nonlinear):
    model = _build(name)
    pos, batch, z = molecules([6, 9, 4], seed=2, dtype=torch.float64)
    with emulated_kernels():
        out = model(f_in=None, pos=pos, batch=batch, node_atom=z)
        out.sum().backward()
    params = {k: v.requires_grad_(v.is_floating_point()) for k, v in R.cast_params(model.state_dict(), torch.float64).items()}
    ref = R.model_forward(params, R.Config(nonlinear_message=nonlinear), pos, batch, z, 3)
    ref.sum().backward()
    assert rel_err(out, ref) < 1e-10
    _grads_match(model, params, 1e-8)


def test_md17_forces_and_double_backward_match_oracle():
    """BASELINE config 1 geometry (aspirin-like, 21 atoms): energy, forces, and d(force loss)/d(params)."""
    model = _build("graph_attention_transformer_nonlinear_exp_l2_md17", irreps_in="64x0e", num_basis=32)
    pos, batch, z = aspirin_like(seed=1, dtype=torch.float64)
    with emulated_kernels():
        energy, forces = model(node_atom=z, pos=pos.clone(), batch=batch)
        (energy.sum() + (forces ** 2).sum()).backward()
    params = {k: v.requires_grad_(v.is_floating_point()) for k, v in R.cast_params(model.state_dict(), torch.float64).items()}
    cfg = R.Config(basis_type="exp", number_of_basis=32, max_atom_type=64, qm9_atom_remap=False)
    e_ref, f_ref = R.energy_and_forces(params, cfg, pos, batch, z, 1, create_graph=True)
    (e_ref.sum() + (f_ref ** 2).sum()).backward()
    assert rel_err(energy, e_ref) < 1e-10
    assert rel_err(forces, f_ref) < 1e-9
    _grads_match(model, params, 1e-7)


def test_state_dict_keys_follow_reference_names():
    from equiformer_b200.nets import model_entrypoint
    model = model_entrypoint("graph_attention_transformer_nonlinear_l2")(irreps_in="5x0e", radius=5.0)
    keys = set(model.state_dict())
    for k in ["blocks.0.ga.merge_src.tp.weight", "blocks.0.ga.merge_src.bias.0", "blocks.0.ga.sep_act.dtp_rad.net.0.weight",
              "blocks.0.ga.sep_act.dtp_rad.net.6.weight", "blocks.0.ga.sep_act.dtp_rad.offset",
              "blocks.0.ga.sep_act.lin.tp.weight", "blocks.0.ga.sep_act.lin.bias.0", "blocks.0.ga.sep_alpha.tp.weight",
              "blocks.0.ga.sep_value.dtp.tp.weight", "blocks.0.ga.sep_value.lin.tp.weight", "blocks.0.ga.alpha_dot",
              "blocks.0.ga.proj.tp.weight", "blocks.0.norm_1.affine_weight", "blocks.0.norm_2.affine_bias",
              "blocks.0.ffn.fctp_1.tp.weight", "blocks.0.ffn.fctp_2.tp.weight", "blocks.5.ffn_shortcut.tp.weight",
              "edge_deg_embed.exp.tp.weight", "edge_deg_embed.rad.net.6.weight", "edge_deg_embed.proj.tp.weight",
              "atom_embed.atom_type_lin.tp.weight", "rbf.mean", "rbf.std", "norm.affine_weight", "head.0.tp.weight",
              "head.2.tp.weight"]:
        assert k in keys, k
    ga = model.blocks[0].ga
    assert ga.sep_act.dtp.tp.weight_numel == 960 and str(ga.sep_act.dtp.irreps_out.simplify()) == "224x0e+384x1e+352x2e"
    assert ga.sep_act.lin.tp.weight.numel() == 86016 and ga.sep_alpha.tp.weight.numel() == 28672
    assert ga.sep_value.lin.tp.weight.numel() == 64512
    assert sum(p.numel() for p in model.parameters()) == 3531715


def test_product_refuses_cpu_tensors():
    """No CPU fallback: the edge path raises on CPU inputs instead of silently computing somewhere else."""
    from equiformer_b200 import _lib
    from equiformer_b200.nets.graph_attention_transformer import DepthwiseTensorProduct
    dtp = DepthwiseTensorProduct("8x0e+4x1e", "1x0e+1x1e", "8x0e+4x1e", internal_weights=False, bias=False)
    x, y, w = torch.randn(5, 20), torch.randn(5, 4), torch.randn(5, dtp.tp.weight_numel)
    with pytest.raises(_lib.EqfError):
        dtp(x, y, w)


def test_planar_resident_blocks_match_the_e3nn_layout_path():
    """The transformer blocks run on planar node blocks when every sub-layer supports it and fall back to the stock
    e3nn-layout `TransBlock.forward` otherwise (e.g. stochastic depth in training): both routes give the same model."""
    from equiformer_b200.nets import graph_attention_transformer as G
    model = _build("graph_attention_transformer_nonlinear_l2")
    pos, batch, z = molecules([5, 8], seed=4, dtype=torch.float64)
    assert all(blk.supports_planar for blk in model.blocks[:-1])          # the last block projects to irreps_feature
    calls = {"planar": 0, "stock": 0}
    orig_planar, orig_forward = G.TransBlock.forward_planar, G.TransBlock.forward

    def spy_planar(self, *a, **k):
        calls["planar"] += 1
        return orig_planar(self, *a, **k)

    def spy_forward(self, *a, **k):
        calls["stock"] += 1
        return orig_forward(self, *a, **k)

    G.TransBlock.forward_planar, G.TransBlock.forward = spy_planar, spy_forward
    try:
        with emulated_kernels():
            out_planar = model(f_in=None, pos=pos, batch=batch, node_atom=z)
            n_planar = dict(calls)
            class _KeepAll(torch.nn.Module):                              # a drop path that drops nothing
                def forward(self, x, batch):
                    return x

            for blk in model.blocks:                                      # force the fallback route
                blk.drop_path = _KeepAll()
            model.train()
            for m in model.modules():
                if isinstance(m, torch.nn.Dropout):
                    m.p = 0.0
            calls.update(planar=0, stock=0)
            out_stock = model(f_in=None, pos=pos, batch=batch, node_atom=z)
    finally:
        G.TransBlock.forward_planar, G.TransBlock.forward = orig_planar, orig_forward
    assert n_planar["planar"] == len(model.blocks) - 1 and n_planar["stock"] == 1
    assert calls["planar"] == 0 and calls["stock"] == len(model.blocks)
    assert rel_err(out_stock, out_planar) < 1e-10


def test_radius_graph_statement_contract():
    """The torch statement of the neighbour list: centres ascending, neighbours ascending inside a centre, no self
    loops, same graph only, d < r, at most `max_num_neighbors` (the first ones) per centre."""
    from equiformer_b200.graph import radius_graph, radius_graph_csr
    g = torch.Generator().manual_seed(0)
    pos = torch.rand(40, 3, generator=g) * 3.0
    batch = torch.repeat_interleave(torch.arange(4), 10)
    edge = radius_graph(pos, 1.5, batch, max_num_neighbors=1000)
    src, dst = edge
    assert bool((dst[1:] >= dst[:-1]).all()) and bool((src != dst).all()) and bool((batch[src] == batch[dst]).all())
    same = dst[1:] == dst[:-1]
    assert bool((src[1:][same] > src[:-1][same]).all())
    d = (pos[src] - pos[dst]).norm(dim=1)
    assert bool((d < 1.5).all())
    full = ((pos[:, None] - pos[None]).norm(dim=-1) < 1.5) & (batch[:, None] == batch[None]) & ~torch.eye(40, dtype=torch.bool)
    assert int(full.sum()) == edge.shape[1]
    capped, row_ptr = radius_graph_csr(pos, 1.5, batch, max_num_neighbors=2)
    assert int(torch.bincount(capped[1], minlength=40).max()) <= 2 and int(row_ptr[-1]) == capped.shape[1]
    kept = {(int(a), int(b)) for a, b in zip(*capped)}
    assert kept <= {(int(a), int(b)) for a, b in zip(src, dst)}


def test_dot_product_attention_rescale_degree_divides_by_the_average_degree():
    """ref nets/dp_attention_transformer.py:148-152: ``attn * degree / _AVG_DEGREE`` (ADVICE r1: the mirror multiplied by
    the degree only)."""
    from oracle import e3nn_ref as e3
    from oracle import equiformer_ref as R
    from equiformer_b200 import o3
    from equiformer_b200.graph import radius_graph
    from equiformer_b200.nets.dp_attention_transformer import DotProductAttention
    torch.manual_seed(0)
    irreps, sh, head = "16x0e+8x1e", "1x0e+1x1e", "4x0e+2x1e"
    dpa = DotProductAttention(irreps, "1x0e", sh, irreps, [8, 8, 8], head, 4, rescale_degree=True, alpha_drop=0.0,
                              proj_drop=0.0).double().eval()
    pos, batch, _ = molecules([6, 9], seed=3, dtype=torch.float64)
    src, dst = radius_graph(pos, 5.0, batch, max_num_neighbors=1000)
    sh_e = o3.spherical_harmonics(sh, pos[src] - pos[dst], True, "component")
    g = torch.Generator().manual_seed(5)
    x = torch.randn(pos.shape[0], 40, generator=g, dtype=torch.float64)
    rbf = torch.randn(src.numel(), 8, generator=g, dtype=torch.float64)
    with emulated_kernels():
        out = dpa(x, None, src, dst, sh_e, rbf, batch)
    params = {"dpa." + k: v for k, v in R.cast_params(dpa.state_dict(), torch.float64).items()}
    ir = e3.parse_irreps(irreps)
    ref = R.dot_product_attention(params, "dpa", ir, e3.parse_irreps(sh), e3.parse_irreps(head), 4, ir, x, src, dst, sh_e,
                                  rbf, rescale_degree=True)
    assert rel_err(out, ref) < 1e-10


def test_bucketed_step_padding_leaves_loss_and_gradients_unchanged():
    """``graphs.BucketedForwardBackward`` pads atoms / edges to bucket sizes with a dummy molecule whose energy never
    enters the loss: loss and every parameter gradient equal the unpadded step (kernels emulated, no capture)."""
    from equiformer_b200.graphs import BucketedForwardBackward
    from equiformer_b200.parallel import FlatGradAllReduce
    model = _build("graph_attention_transformer_nonlinear_l2")
    pos, batch, z = molecules([5, 7, 4], seed=3, dtype=torch.float64)
    tgt = torch.tensor([[0.3], [-1.0], [2.0]], dtype=torch.float64)
    loss_fn = lambda o, t: (o - t).abs().mean()
    with emulated_kernels():
        out = model(f_in=None, pos=pos, batch=batch, node_atom=z, n_graphs=3)
        l0 = loss_fn(out, tgt)
        g0 = torch.autograd.grad(l0, list(model.parameters()), allow_unused=True)
        bucket = FlatGradAllReduce(model.parameters())
        bfb = BucketedForwardBackward(model, loss_fn, bucket, 5.0, atom_quantum=8, edge_quantum=64, capture=False)
        l1 = bfb(pos, batch, z, tgt)
    assert list(bfb._cache) == [(24, 128, 3)]          # 16 atoms + >= 2 dummies -> 24; 106 edges -> 128
    assert rel_err(l1, l0) < 1e-12
    for p, g in zip(model.parameters(), g0):
        if g is not None:
            assert rel_err(p.grad, g) < 1e-10


def test_radial_first_layers_run_as_one_product(monkeypatch):
    """The first Linear of the 7 radial MLPs of the QM9 model is ONE stacked product (``radial_func.hoist_first_layers``);
    outputs and gradients equal the per-module evaluation (the model with nothing hoisted)."""
    from equiformer_b200 import ops
    from equiformer_b200.nets import graph_attention_transformer
    model = _build("graph_attention_transformer_nonlinear_l2")
    pos, batch, z = molecules([5, 7], seed=3, dtype=torch.float64)
    real = ops.linear_f32
    results = {}
    for hoist in (True, False):
        if not hoist:
            monkeypatch.setattr(graph_attention_transformer, "hoist_first_layers", lambda modules, x: [])
        calls = []
        monkeypatch.setattr(ops, "linear_f32", lambda x, w, b=None: (calls.append(tuple(w.shape)), real(x, w, b))[1])
        model.zero_grad(set_to_none=True)
        with emulated_kernels():
            out = model(f_in=None, pos=pos, batch=batch, node_atom=z)
            out.sum().backward()
        first = [s for s in calls if s[1] == 128]
        results[hoist] = (out.detach().clone(), {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}, first)
    assert results[True][2] == [(7 * 64, 128)] and len(results[False][2]) == 7      # 6 blocks + the degree embedding
    assert rel_err(results[True][0], results[False][0]) < 1e-12
    for k, g in results[False][1].items():
        assert rel_err(results[True][1][k], g) < 1e-10, k
    assert all(getattr(m, "_hoisted", None) is None for m in model.modules())
