"""The per-graph equivariant norms (``norm_layer='graph' | 'instance'``) and the fast layer norm (``'fast_layer'``).

Pinned to ``tests/golden/reference_norms_small.npz`` (``make_reference_golden_norms.py``: the reference's own
``graph_norm.py``, ``instance_norm.py``, ``fast_layer_norm.py`` and model files in float64).

CPU: the torch statements against the fixture to 1e-10; the mirrors load the reference's ``state_dict``s; ``gradcheck``
/ ``gradgradcheck`` of the torch statement and of ``ops.SegmentNorm`` on float64 stand-ins of the kernels (the same
algorithm: fixed-order segment sums, the hand-derived backward); the kernel inventory of ``libeqf_b200_norm.so`` is
claimed by the GPU cases.

GPU: the kernels against float64 under the launch audit's bounds (1-atom, empty, constant-scalar and 5 000-atom
graphs, more graphs than one grid pass); bitwise repeats; the model files against the fixture, eager and captured;
bucket padding; every model family with each norm, captured against eager.
"""
from __future__ import annotations

import contextlib
import os

import numpy as np
import pytest
import torch

from tests.helpers import rel_err
from tests.reference_fixtures import GOLDEN, load, mirror, run_mirror

FIXTURE = "reference_norms_small.npz"
NORMS = ("graph", "instance", "fast_layer")


def _module_names(g):
    return sorted({k.split("/")[1] for k in g.files if k.startswith("mod/")})


MODULE_CASES = _module_names(np.load(os.path.join(GOLDEN, FIXTURE)))


def _module(name, case):
    from equiformer_b200.nets.fast_layer_norm import EquivariantLayerNormFast
    from equiformer_b200.nets.graph_norm import EquivariantGraphNorm
    from equiformer_b200.nets.instance_norm import EquivariantInstanceNorm
    kind, norm, affine, *rest = name.split("_") if not name.startswith("fast_layer") else ["fast_layer", *name.split("_")[2:]]
    irreps = "6x0e+4x1e+3x0o+2x2e+4x0e"
    if kind == "fast_layer":
        m = EquivariantLayerNormFast(irreps, eps=1e-5, affine=affine == "affine", normalization=norm)
    else:
        cls = {"graph": EquivariantGraphNorm, "instance": EquivariantInstanceNorm}[kind]
        m = cls(irreps, eps=1e-5, affine=affine == "affine", reduce=rest[0], normalization=norm)
    m.load_state_dict(case.state, strict=True)
    return m.double()


# ------------------------------------------------------------------------------------------------ CPU: statements
@pytest.mark.parametrize("name", MODULE_CASES)
def test_torch_statement_matches_reference_norm_files(name):
    case = load(FIXTURE, f"mod/{name}")
    m = _module(name, case)
    t = case.t
    x = t("x").clone().requires_grad_(True)
    y = m(x, batch=t("batch"))
    (y * t("gy")).sum().backward()
    assert rel_err(y.detach(), t("y")) < 1e-10
    assert rel_err(x.grad, t("gx")) < 1e-10
    for k, p in m.named_parameters():
        assert rel_err(p.grad, case.grads[k]) < 1e-10, k


def test_get_norm_layer_returns_the_reference_classes():
    from equiformer_b200.nets.fast_layer_norm import EquivariantLayerNormFast
    from equiformer_b200.nets.graph_attention_transformer import SeparableFCTP, get_norm_layer
    from equiformer_b200.nets.graph_norm import EquivariantGraphNorm
    from equiformer_b200.nets.instance_norm import EquivariantInstanceNorm
    from equiformer_b200.nets.layer_norm import EquivariantLayerNormV2
    assert get_norm_layer("graph") is EquivariantGraphNorm
    assert get_norm_layer("instance") is EquivariantInstanceNorm
    assert get_norm_layer("fast_layer") is EquivariantLayerNormFast
    assert get_norm_layer("layer") is EquivariantLayerNormV2 and get_norm_layer(None) is None
    with pytest.raises(ValueError):
        get_norm_layer("batch")
    sep = SeparableFCTP("8x0e+4x1e", "1x0e+1x1e", "8x0e+4x1e", [4, 8])      # default norm_layer='graph'
    assert isinstance(sep.norm, EquivariantGraphNorm)
    assert set(sep.norm.state_dict()) == {"mean_shift", "affine_weight", "affine_bias"}
    with pytest.raises(NotImplementedError):
        sep.planar([torch.zeros(3, 1, 8), torch.zeros(3, 3, 4)], torch.zeros(3, 4), torch.zeros(3, 4))


def test_separable_fctp_forward_with_the_default_graph_norm():
    """``SeparableFCTP``'s stock forward with its default ``norm_layer='graph'``: with a batch vector, and without one,
    which makes all nodes one graph (as ``global_mean_pool`` reads a missing batch)."""
    from equiformer_b200.nets.graph_attention_transformer import SeparableFCTP
    from tests._emulation import emulated_kernels
    torch.manual_seed(2)
    sep = SeparableFCTP("8x0e+4x1e", "1x0e+1x1e", "8x0e+4x1e", [4, 8]).double()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(7, 20, generator=g, dtype=torch.float64)
    sh = torch.randn(7, 4, generator=g, dtype=torch.float64)
    scalars = torch.randn(7, 4, generator=g, dtype=torch.float64)
    batch = torch.tensor([0, 0, 0, 1, 1, 1, 1])
    with emulated_kernels(), emulated_norm_kernels():
        out = sep(x, sh, scalars, batch=batch)
        one = sep(x, sh, scalars)
        ref_one = sep(x, sh, scalars, batch=torch.zeros(7, dtype=torch.long))
        pre = sep.lin(sep.dtp(x, sh, sep.dtp_rad(scalars)))
    # outside the stand-ins the norm runs its torch statement
    assert rel_err(out, sep.norm(pre, batch=batch)) < 1e-12
    assert rel_err(one, ref_one) < 1e-12 and rel_err(one, sep.norm(pre)) < 1e-12
    assert rel_err(one, out) > 1e-3


def test_norm_layout_constant_matches_the_header():
    import ctypes
    import re
    from equiformer_b200 import _lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                               "eqf_b200_norm.h")).read()
    assert int(re.search(r"#define EQF_NORM_MAX_ENTRIES (\d+)", header).group(1)) == _lib.EQF_NORM_MAX_ENTRIES
    assert ctypes.sizeof(_lib.EqfSegNormLayout) == 4 * (1 + 5 * _lib.EQF_NORM_MAX_ENTRIES + 3 + 1)


def test_fast_layer_norm_equals_layer_norm_v2():
    """``F.layer_norm`` on the scalars is the V2 map of a 1-component entry: the two torch statements agree."""
    from equiformer_b200.nets.fast_layer_norm import EquivariantLayerNormFast
    from equiformer_b200.nets.layer_norm import EquivariantLayerNormV2
    g = torch.Generator().manual_seed(3)
    for norm in ("component", "norm"):
        a = EquivariantLayerNormFast("6x0e+4x1e+3x0o+2x2e", normalization=norm).double()
        b = EquivariantLayerNormV2("6x0e+4x1e+3x0o+2x2e", normalization=norm).double()
        with torch.no_grad():
            for p in a.parameters():
                p.copy_(torch.randn(p.shape, generator=g, dtype=torch.float64))
        b.load_state_dict(a.state_dict())
        x = torch.randn(9, a.irreps.dim, generator=g, dtype=torch.float64)
        assert rel_err(a(x), b(x)) < 1e-12


def _mirror(kind, case):
    from equiformer_b200.nets.graph_attention_transformer import GraphAttentionTransformer
    from equiformer_b200.nets.graph_attention_transformer_md17 import GraphAttentionTransformerMD17
    return mirror({"qm9": GraphAttentionTransformer, "md17": GraphAttentionTransformerMD17}[kind], case.cfg, case.state)


MODEL_CASES = [(kind, norm) for kind in ("qm9", "md17") for norm in NORMS]


@pytest.mark.parametrize("kind,norm", MODEL_CASES)
def test_mirror_loads_reference_state_dict(kind, norm):
    case = load(FIXTURE, f"{kind}_{norm}")
    model = _mirror(kind, case)
    norm_keys = {k for k in case.state if ".norm" in k or k.startswith("norm.")}
    assert norm_keys and norm_keys <= set(model.state_dict())
    if norm == "graph":
        assert any(k.endswith("mean_shift") for k in norm_keys)


@pytest.mark.parametrize("kind,norm", MODEL_CASES)
def test_no_weight_decay_matches_reference_model_files(kind, norm):
    """The parameters left out of weight decay are the reference's: the graph and instance norms' ones among them, the
    fast layer norm's not."""
    case = load(FIXTURE, f"{kind}_{norm}")
    model = _mirror(kind, case)
    assert model.no_weight_decay() == set(case.arrays["no_weight_decay"].tolist())


@pytest.mark.parametrize("family", ["oc20", "oc20_dp", "dens"])
def test_no_weight_decay_holds_the_per_graph_norms_of_every_model(family):
    """OC20, dot-product OC20 and DeNS list EquivariantGraphNorm / EquivariantInstanceNorm parameters among those
    without weight decay, as every reference model does (and EquivariantLayerNormFast's not)."""
    for norm in NORMS:
        model = _family_model(family, norm, "cpu")
        model = model[0] if isinstance(model, tuple) else model
        norm_params = {n for n, _ in model.named_parameters() if n.startswith("norm.") or ".norm_" in n}
        assert norm_params
        skip = model.no_weight_decay()
        assert (norm_params <= skip) if norm != "fast_layer" else not (norm_params & skip), (family, norm)


# ------------------------------------------------------------------------------------------------ CPU: kernel stand-ins
def _emu_graph_ptr(batch, n_graphs):
    return torch.searchsorted(batch, torch.arange(n_graphs + 1, dtype=batch.dtype, device=batch.device))


def _emu_fwd(lay, xs, ptr, G, shift, w, b):
    """The forward kernel's algorithm in the inputs' dtype: per (graph, channel) the mean, then the centred square mean."""
    ys = [torch.empty_like(x) for x in xs]
    mean = xs[0].new_zeros((G, lay.n_s))
    rstd = xs[0].new_zeros((G, lay.n_w))
    iw = i_s = 0
    for (m, d, s), x, y in zip(lay.entries, xs, ys):
        for g in range(G):
            n0, n1 = int(ptr[g]), int(ptr[g + 1])
            n = n1 - n0
            blk = x[n0:n1]
            mu = blk[:, 0, :].sum(0) / max(n, 1) if s else x.new_zeros(m)
            msh = (shift[:m] if shift is not None else 1.0) * mu if s else x.new_zeros(m)
            z = blk - msh
            v = (z * z).sum((0, 1)) / max(n, 1) / (d if lay.component else 1)
            r = (v + lay.eps).rsqrt()
            y[n0:n1] = z * (r * w[iw:iw + m]) + (b[i_s:i_s + m] if s else 0.0)
            rstd[g, iw:iw + m] = r
            if s:
                mean[g, i_s:i_s + m] = mu
        iw += m
        i_s += m if s else 0
    return ys, mean, rstd


def _emu_bwd(lay, xs, gys, ptr, G, shift, w, mean, rstd):
    """The backward kernel's formulas (see ``csrc/eqf_norm.cu``), per graph, then the partials summed over the graphs."""
    gxs = [torch.empty_like(x) for x in xs]
    gw = w.new_zeros(lay.n_w)
    gb = w.new_zeros(lay.n_s)
    gs = w.new_zeros(lay.n_s)
    iw = i_s = 0
    for (m, d, s), x, gy, gx in zip(lay.entries, xs, gys, gxs):
        sh = shift[:m] if (s and shift is not None) else x.new_ones(m)
        for g in range(G):
            n0, n1 = int(ptr[g]), int(ptr[g + 1])
            n = n1 - n0
            inv_n = 1.0 / n if n else 0.0
            r = rstd[g, iw:iw + m]
            mu = mean[g, i_s:i_s + m] if s else x.new_zeros(m)
            msh = sh * mu if s else x.new_zeros(m)
            z = x[n0:n1] - msh
            t = gy[n0:n1]
            s0, s1, sz = t.sum((0, 1)), (t * z).sum((0, 1)), z.sum((0, 1))
            sc = r * w[iw:iw + m]
            c1 = r ** 3 * w[iw:iw + m] * s1 * inv_n / (d if lay.component else 1)
            sum_dz = sc * s0 - c1 * sz
            corr = sh * inv_n * sum_dz if s else 0.0
            gx[n0:n1] = t * sc - c1 * z - corr
            gw[iw:iw + m] += r * s1
            if s:
                gb[i_s:i_s + m] += s0
                gs[i_s:i_s + m] += -mu * sum_dz
        iw += m
        i_s += m if s else 0
    gshift = None
    if shift is not None:
        gshift = torch.zeros_like(shift)
        off = 0
        for m, _d, s in lay.entries:
            if s:
                gshift[:m] += gs[off:off + m]
                off += m
    return gxs, gw, gb, gshift


@contextlib.contextmanager
def emulated_norm_kernels():
    from equiformer_b200 import norm_kernels, ops
    saved = (norm_kernels.graph_ptr_raw, norm_kernels.norm_fwd_raw, norm_kernels.norm_bwd_raw, ops.FUSED_ON_ANY_DEVICE)
    try:
        norm_kernels.graph_ptr_raw = _emu_graph_ptr
        norm_kernels.norm_fwd_raw, norm_kernels.norm_bwd_raw = _emu_fwd, _emu_bwd
        ops.FUSED_ON_ANY_DEVICE = True
        yield
    finally:
        norm_kernels.graph_ptr_raw, norm_kernels.norm_fwd_raw, norm_kernels.norm_bwd_raw, ops.FUSED_ON_ANY_DEVICE = saved


def _planar_case(seed, sizes, irreps="5x0e+3x1e+2x0o+2x2e+3x0e", normalization="component", dtype=torch.float64):
    from equiformer_b200.nets.graph_norm import EquivariantGraphNorm
    from equiformer_b200.o3 import Irreps
    g = torch.Generator().manual_seed(seed)
    m = EquivariantGraphNorm(irreps, normalization=normalization)
    lay = m._layout
    N = sum(sizes)
    batch = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
    xs = [torch.randn(N, ir.dim, mul, generator=g, dtype=dtype) for mul, ir in Irreps(irreps)]
    w = 1.0 + 0.3 * torch.randn(lay.n_w, generator=g, dtype=dtype)
    b = 0.3 * torch.randn(lay.n_s, generator=g, dtype=dtype)
    shift = 1.0 + 0.3 * torch.randn(lay.n_s, generator=g, dtype=dtype)
    return lay, xs, batch, len(sizes), w, b, shift


@pytest.mark.parametrize("instance", [False, True])
@pytest.mark.parametrize("normalization", ["component", "norm"])
def test_segment_norm_gradcheck_on_kernel_stand_ins(instance, normalization):
    """First order: the hand-derived backward (float64 stand-in of the kernel) against finite differences; second order
    (``create_graph``): the torch-statement rebuild.  Graphs of 3, 1, 0 (padding) and 4 nodes."""
    from equiformer_b200 import ops
    lay, xs, batch, G, w, b, shift = _planar_case(5, [3, 1, 0, 4], normalization=normalization)
    shift = None if instance else shift
    seg = ops.GraphSegments(batch, G)
    ins = [t.requires_grad_(True) for t in (w, b, *xs)] + ([] if shift is None else [shift.requires_grad_(True)])

    def fn(w_, b_, *rest):
        blocks, sh = (rest, None) if shift is None else (rest[:-1], rest[-1])
        return tuple(ops.SegmentNorm.apply(lay, seg, w_, b_, sh, *blocks))

    with emulated_norm_kernels():
        assert torch.autograd.gradcheck(fn, ins, eps=1e-6, atol=1e-7)
        assert torch.autograd.gradgradcheck(fn, ins, eps=1e-6, atol=1e-6)
        out = fn(*ins)
    ref = ops.segment_norm_planar_torch(lay, xs, batch, G, w, b, shift)
    for o, r in zip(out, ref):
        assert rel_err(o.detach(), r.detach()) < 1e-12


def test_torch_statement_gradcheck():
    from equiformer_b200 import ops
    lay, xs, batch, G, w, b, shift = _planar_case(7, [2, 1, 3])
    ins = [t.requires_grad_(True) for t in (w, b, shift, *xs)]
    fn = lambda w_, b_, s_, *blocks: tuple(ops.segment_norm_planar_torch(lay, list(blocks), batch, G, w_, b_, s_))
    assert torch.autograd.gradcheck(fn, ins)
    assert torch.autograd.gradgradcheck(fn, ins)


@pytest.mark.parametrize("kind,norm", MODEL_CASES)
def test_mirror_with_emulated_kernels_matches_reference_model_files(kind, norm):
    from tests._emulation import emulated_kernels
    case = load(FIXTURE, f"{kind}_{norm}")
    model = _mirror(kind, case).double()
    with emulated_kernels(), emulated_norm_kernels():
        energy, forces = run_mirror(kind, model, case)
    assert rel_err(energy.detach(), case.t("energy")) < 1e-10
    if forces is not None:
        assert rel_err(forces.detach(), case.t("forces")) < 1e-10


# ------------------------------------------------------------------------------------------------ inventory
# every kernel entry of libeqf_b200_norm.so, claimed by test_kernels_under_the_launch_audit
NORM_CLAIMS = {"eqf::norm_graph_ptr_kernel", "eqf::norm_fwd_kernel", "eqf::norm_bwd_kernel", "eqf::norm_param_reduce_kernel"}


def test_norm_library_inventory_is_claimed():
    from equiformer_b200 import _lib
    from tests.test_gpu_kernel_instances import inventory
    inv = inventory(_lib.NORM_LIB_PATH)
    assert inv == NORM_CLAIMS, (sorted(inv - NORM_CLAIMS), sorted(NORM_CLAIMS - inv))


# ------------------------------------------------------------------------------------------------ GPU: kernels
def _audit_refs(name, args, kw):
    """float64 statements of the norm library's launchers (outputs in order, None: not compared)."""
    from equiformer_b200 import ops
    from tests import test_gpu_launch_audit as A
    a = A._map(A._f64, args)
    if name == "graph_ptr_raw":
        batch, n_graphs = a
        return [_emu_graph_ptr(batch, n_graphs)]
    if name == "norm_fwd_raw":
        lay, xs, ptr, G, shift, w, b = a
        batch = torch.repeat_interleave(torch.arange(G, device=ptr.device), ptr[1:] - ptr[:-1])
        ys = ops.segment_norm_planar_torch(lay, list(xs), batch, G, w, b, shift)
        _ys, mean, rstd = _emu_fwd(lay, list(xs), ptr.cpu(), G, shift, w, b)
        return [*ys, mean, rstd]
    if name == "norm_bwd_raw":
        lay, xs, gys, ptr, G, shift, w, _mean, _rstd = a
        batch = torch.repeat_interleave(torch.arange(G, device=ptr.device), ptr[1:] - ptr[:-1])
        b = w.new_zeros(lay.n_s)
        fn = lambda ww, bb, ss, *blocks: tuple(ops.segment_norm_planar_torch(lay, list(blocks), batch, G, ww, bb, ss))
        g = A._vjp(fn, (w, b, shift, *xs), list(gys))
        return [*g[3:], g[0], g[1], g[2]]
    return A._nonlin_ref(name, args, kw)


AUDITED = {"graph_ptr_raw": "fwd", "norm_fwd_raw": "fwd", "norm_bwd_raw": "bwd"}


def _install_audit(audit, monkeypatch):
    from equiformer_b200 import norm_kernels
    from tests import test_gpu_launch_audit as A
    audit.install(monkeypatch)
    for name, kind in AUDITED.items():
        monkeypatch.setitem(A.CRITERIA, name, (kind, A.TOL_FWD if kind == "fwd" else A.TOL_BWD, None))
        monkeypatch.setattr(norm_kernels, name, audit._wrap(name, getattr(norm_kernels, name)))
    monkeypatch.setattr(A, "_nonlin_ref", _audit_refs)


# (name, graph sizes, constant 0e graphs): 1-atom and empty graphs, a constant-scalar graph, one 5 000-atom graph,
# 2 600 graphs (past the 1 024-CTA graph stride of the forward and backward kernels)
KERNEL_CASES = {
    "ragged": ([5, 1, 0, 7, 4, 0, 1, 33], [4]),
    "stress_5000": ([5000], []),
    "past_grid": ([1 + (i * 7) % 5 for i in range(2600)], [3, 2599]),
}


def _kernel_inputs(case, dev, irreps="128x0e+64x1e+32x2e+7x0o+16x0e"):
    from equiformer_b200.nets.graph_norm import EquivariantGraphNorm
    from equiformer_b200.o3 import Irreps
    sizes, constant = KERNEL_CASES[case]
    g = torch.Generator(device=dev).manual_seed(11)
    m = EquivariantGraphNorm(irreps)
    lay = m._layout
    ptr = torch.tensor([0] + list(np.cumsum(sizes)), device=dev)
    batch = torch.repeat_interleave(torch.arange(len(sizes), device=dev), torch.tensor(sizes, device=dev))
    N = int(ptr[-1])
    xs = [torch.randn(N, ir.dim, mul, generator=g, device=dev) + (0.5 if ir.l == 0 else 0.0) for mul, ir in Irreps(irreps)]
    for gi in constant:
        for (mul, d, s), x in zip(lay.entries, xs):
            if s:
                x[int(ptr[gi]):int(ptr[gi + 1])] = 0.625
    rnd = lambda n: torch.randn(n, generator=g, device=dev)
    w, b, shift = 1.0 + 0.3 * rnd(lay.n_w), 0.3 * rnd(lay.n_s), 1.0 + 0.3 * rnd(lay.n_s)
    gys = [torch.randn(x.shape, generator=g, device=dev) for x in xs]
    return lay, xs, gys, batch, len(sizes), w, b, shift


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(KERNEL_CASES))
def test_kernels_under_the_launch_audit(cuda_device, monkeypatch, case):
    """Graph and instance norm, forward and backward, each launch re-evaluated in float64 under the launch audit's
    nonlinear bounds (2e-5 forward, 5e-5 backward of the largest magnitude); the launched kernels are NORM_CLAIMS."""
    from equiformer_b200 import ops
    from tests.test_gpu_kernel_instances import _launched
    from tests.test_gpu_launch_audit import Audit
    lay, xs, gys, batch, G, w, b, shift = _kernel_inputs(case, cuda_device)

    def run(dev):
        for sh in (shift, None):
            seg = ops.GraphSegments(batch, G)
            ins = [t.detach().requires_grad_(True) for t in (w, b, *xs)]
            ys = ops.SegmentNorm.apply(lay, seg, ins[0], ins[1], sh, *ins[2:])
            torch.autograd.backward(ys, gys)
            for y in ys:
                assert bool(torch.isfinite(y).all())

    audit = Audit(f"norm_{case}")
    _install_audit(audit, monkeypatch)
    try:
        launched = _launched(run, cuda_device)
        audit.report()
    finally:
        monkeypatch.undo()
    assert not audit.unaudited, audit.unaudited
    assert not audit.failures, "\n".join(audit.failures[:20])
    assert audit.index == 6
    assert launched == NORM_CLAIMS, (sorted(launched - NORM_CLAIMS), sorted(NORM_CLAIMS - launched))


@pytest.mark.gpu
def test_kernels_are_bitwise_repeatable(cuda_device):
    from equiformer_b200 import ops
    lay, xs, gys, batch, G, w, b, shift = _kernel_inputs("ragged", cuda_device)
    runs = []
    for _ in range(3):
        ins = [t.detach().requires_grad_(True) for t in (w, b, shift, *xs)]
        ys = ops.SegmentNorm.apply(lay, ops.GraphSegments(batch, G), *ins[:3], *ins[3:])
        torch.autograd.backward(ys, gys)
        runs.append([t.detach().clone() for t in ys] + [t.grad.clone() for t in ins])
    for later in runs[1:]:
        assert all(torch.equal(a, c) for a, c in zip(runs[0], later))


# ------------------------------------------------------------------------------------------------ GPU: models
@pytest.mark.gpu
@pytest.mark.parametrize("kind,norm", MODEL_CASES)
def test_cuda_models_match_reference_model_files(cuda_device, kind, norm):
    """The captured step's loss against the fixture's, then the eager energies (and MD17 forces) at 1e-4 (the captured
    step runs first, as in the other capture tests)."""
    from equiformer_b200 import ops
    from equiformer_b200.graphs import GraphedForwardBackward, GraphedStep
    from equiformer_b200.parallel import FlatGradAllReduce
    from oracle import equiformer_ref as R
    case = load(FIXTURE, f"{kind}_{norm}")
    cfg = case.cfg
    model = _mirror(kind, case).to(cuda_device)
    t = lambda k: case.t(k, cuda_device)
    energy_ref = case.t("energy")
    pos, batch, z = t("pos"), t("batch"), t("z")
    n_graphs = int(energy_ref.shape[0])
    bucket = FlatGradAllReduce(model.parameters())
    if kind == "qm9":
        gfb = GraphedForwardBackward(model, lambda out, tgt: ((out - tgt) ** 2).sum(), bucket, max_radius=cfg["max_radius"])
        target = torch.zeros(n_graphs, 1, device=cuda_device)
        for _ in range(2):
            loss = gfb(pos, batch, z, target).clone()
        assert gfb.captures == 1
        ref_loss = (energy_ref ** 2).sum()
    else:
        graph = ops.Graph(*R.radius_graph(pos, cfg["max_radius"], batch), pos.shape[0])

        def captured(pos, batch, z, src, dst, row_ptr):
            from equiformer_b200.graphs import csr_graph
            e, f = model.forward_edges(z, pos.detach().requires_grad_(True), batch, src, dst,
                                       graph=csr_graph(src, dst, row_ptr, pos.shape[0]), n_graphs=n_graphs)
            return e.sum() + (f ** 2).sum()

        step = GraphedStep(captured, bucket)
        for _ in range(2):
            loss = step((int(pos.shape[0]), graph.n_edges), [pos, batch, z, graph.src, graph.dst, graph.row_ptr]).clone()
        assert step.captures == 1
        ref_loss = energy_ref.sum() + (case.t("forces") ** 2).sum()
    assert abs(float(loss) - float(ref_loss)) <= 1e-4 * abs(float(ref_loss))
    energy, forces = run_mirror(kind, model, case, cuda_device, torch.float32)
    assert rel_err(energy.detach(), energy_ref) < 1e-4
    if forces is not None:
        assert rel_err(forces.detach(), case.t("forces")) < 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("norm", ["graph", "instance"])
def test_bucket_padding_is_its_own_graph(cuda_device, norm):
    """The dummy molecule that pads a batch to its bucket is graph ``n_graphs``: the real molecules' energies and
    gradients with padding equal those without, although the norm statistics are per graph."""
    from equiformer_b200.graph import radius_graph_csr
    from equiformer_b200.graphs import csr_graph, pad_to_bucket
    case = load(FIXTURE, f"qm9_{norm}")
    cfg = case.cfg
    model = _mirror("qm9", case).to(cuda_device)
    t = lambda k: case.t(k, cuda_device)
    pos, batch, z = t("pos"), t("batch"), t("z")
    G = int(batch.max()) + 1
    edge, row_ptr = radius_graph_csr(pos, cfg["max_radius"], batch, max_num_neighbors=1000)
    runs = []
    for pad in (False, True):
        model.zero_grad()
        if pad:
            (p, bt, zz, src, dst, rp), _ = pad_to_bucket(pos, batch, z, edge[0], edge[1], G, 32, 512)
            out = model.forward_edges(p, bt, zz, src, dst, graph=csr_graph(src, dst, rp, p.shape[0]), n_graphs=G + 1)[:G]
        else:
            out = model.forward_edges(pos, batch, z, edge[0], edge[1], graph=csr_graph(edge[0], edge[1], row_ptr,
                                                                                        pos.shape[0]), n_graphs=G)
        (out ** 2).sum().backward()
        runs.append((out.detach(), {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}))
    assert rel_err(runs[1][0], runs[0][0]) < 1e-5
    assert rel_err(runs[0][0], case.t("energy")) < 1e-4
    # a gradient that vanishes in exact arithmetic (a bias that the next norm's mean subtraction removes) is rounding
    # noise in both runs: errors are taken against 1e-3 of the largest gradient entry of the model at least
    floor = 1e-3 * max(float(g.abs().max()) for g in runs[0][1].values())
    worst = max((float((g - runs[0][1][k]).abs().max()) / max(float(runs[0][1][k].abs().max()), floor), k)
                for k, g in runs[1][1].items())
    assert worst[0] < 1e-4, worst


def _oc20_step(model, dev):
    from equiformer_b200.graphs import csr_graph
    from tests.test_oc20_aux import _frames
    pos, batch, z, tags, src, dst, edge_vec = _frames(dev, n_frames=2, seed=3)
    n = int(pos.shape[0])
    row_ptr = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    torch.cumsum(torch.zeros(n, dtype=torch.int64, device=dev).index_add_(0, dst, torch.ones_like(dst)), 0, out=row_ptr[1:])

    def loss(edge_vec, batch, z, tags, src, dst, row_ptr):
        out = model.forward_edges(edge_vec, batch, z, tags, src, dst, graph=csr_graph(src, dst, row_ptr, batch.shape[0]),
                                  n_graphs=2)
        out = out[0] if isinstance(out, tuple) else out
        return (out ** 2).sum()
    return loss, (n, int(src.numel())), [edge_vec, batch, z, tags, src, dst, row_ptr]


def _family_model(family, norm, dev):
    torch.manual_seed(0)
    if family in ("oc20", "oc20_dp"):
        from equiformer_b200.nets.dp_attention_transformer_oc20 import DotProductAttentionTransformerOC20
        from equiformer_b200.nets.graph_attention_transformer_oc20 import GraphAttentionTransformerOC20
        cls = DotProductAttentionTransformerOC20 if family == "oc20_dp" else GraphAttentionTransformerOC20
        cfg = dict(irreps_node_embedding="16x0e+8x1e", num_layers=2, irreps_sh="1x0e+1x1e", number_of_basis=16,
                   fc_neurons=[16, 16], irreps_feature="32x0e", irreps_head="8x0e+4x1e", num_heads=2,
                   irreps_pre_attn="16x0e+8x1e", irreps_mlp_mid="48x0e+24x1e", norm_layer=norm, alpha_drop=0.0)
        return cls(None, None, 1, **cfg).to(dev).eval()
    from equiformer_b200.nets.equiformer_md17_dens import Equiformer_MD17_DeNS
    case = load("reference_model_dens_small.npz")
    return Equiformer_MD17_DeNS(**dict(case.cfg, norm_layer=norm)).to(dev).eval(), case


@pytest.mark.gpu
@pytest.mark.parametrize("norm", NORMS)
@pytest.mark.parametrize("family", ["oc20", "oc20_dp", "dens"])
def test_model_families_captured_equal_eager(cuda_device, family, norm):
    """OC20 (graph attention and dot-product attention) and DeNS with each norm: the captured step's loss and gradients
    equal the eager step's; the DeNS step is also padded to its bucket when captured."""
    from equiformer_b200.graphs import DensTrainStep, GraphedStep
    from equiformer_b200.parallel import FlatGradAllReduce
    if family == "dens":
        model, case = _family_model(family, norm, cuda_device)
        t = lambda k: case.t(k, cuda_device)
        pos, batch, z = t("pos").float(), t("batch"), t("z")
        G = int(batch.max()) + 1
        gen = torch.Generator().manual_seed(2)
        y, dy = torch.randn(G, 1, generator=gen).to(cuda_device), torch.randn(pos.shape, generator=gen).to(cuda_device)
        results = []
        for capture in (False, True):
            bucket = FlatGradAllReduce(model.parameters())
            step = DensTrainStep(model, bucket, capture=capture)
            for _ in range(2 if capture else 1):
                loss = step(pos, batch, z, y, dy, G, 0.5, generator=torch.Generator(device=cuda_device).manual_seed(4))
            results.append((float(loss), bucket.flat.clone()))
    else:
        model = _family_model(family, norm, cuda_device)
        loss_fn, key, inputs = _oc20_step(model, cuda_device)
        bucket = FlatGradAllReduce(model.parameters())
        step = GraphedStep(loss_fn, bucket)
        for _ in range(2):
            loss_g = float(step(key, inputs))
        flat_g = bucket.flat.clone()
        bucket.zero_grad()
        loss_e = loss_fn(*inputs)
        loss_e.backward()
        results = [(float(loss_e), bucket.flat.clone()), (loss_g, flat_g)]
    (le, ge), (lc, gc) = results
    assert np.isfinite(le) and abs(lc - le) <= 1e-5 * abs(le)
    assert rel_err(gc, ge) < 1e-4
