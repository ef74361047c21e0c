"""Every compiled kernel instance of ``libeqf_b200.so`` launched by a case of this file and checked against float64.

One entry point of the library covers several compiled kernels: the instance is chosen from the plan and the problem
size (head count, float4 slots per lane, the float4 layout, shared or per-edge weights, gather, output degree, column
tile).  The model tests and the launch audit reach only the instances their configurations select, so an instance with a
wrong lane -> head or slot -> group map can sit in the library untested.  This module closes that gap:

* ``test_inventory_is_read_from_the_binary`` (CPU) lists the kernel entries of the built library with ``cuobjdump`` and
  ``cu++filt`` and normalises them (template arguments as ``16`` / ``true``, no parameter list);
* ``CASES`` runs small problems through the public ``ops`` wrappers and autograd Functions.  Each case names the exact set
  of instances it launches; ``test_case_launches_what_it_claims`` (GPU) runs it under ``torch.profiler`` and asserts that
  the ``eqf::`` device kernels it launched are that set, while every leaf ``*_raw`` call is re-evaluated in float64 by the
  launch audit (``tests/test_gpu_launch_audit.py``: the componentwise ``tau u sqrt(K) |terms|`` bound for multilinear
  calls, 2e-5 / 5e-5 for nonlinear ones, exact zeros at nodes without incoming edges);
* ``test_every_instance_is_claimed`` (CPU): the claims plus ``NOT_LAUNCHED`` are the inventory, in both directions.

The attention graphs have ragged segments, nodes without incoming edges and a hub of 600 edges; the grid-stride dot-product
and linear-message attention kernels run on one more node than two full passes of their grid (``_past_grid_cap``).
"""
from __future__ import annotations

import re
import shutil
import subprocess

import pytest
import torch

from tests.test_gpu_launch_audit import Audit

# ------------------------------------------------------------------------------------------------ names
_CAST = re.compile(r"\((?:int|unsigned int|long long|bool)\)(-?\d+)")


def normalise(name: str) -> str:
    """``void eqf::k<(int)16, (bool)1>(eqf::Args, float *)`` and ``eqf::k<16, true>(...)`` -> ``eqf::k<16,true>``."""
    s = name.strip()
    if s.startswith("void "):
        s = s[5:]
    s = re.sub(r"\(bool\)1\b", "true", s)
    s = re.sub(r"\(bool\)0\b", "false", s)
    s = _CAST.sub(r"\1", s)
    cut = s.find("(")
    if cut >= 0:
        s = s[:cut]
    return re.sub(r"\s+", "", s)


def inventory(lib_path) -> set:
    """Normalised names of the kernel entries (``STO_ENTRY``) of the library's sm_90a code."""
    tools = {t: shutil.which(t) or f"/usr/local/cuda/bin/{t}" for t in ("cuobjdump", "cu++filt")}
    for t, p in tools.items():
        if not shutil.which(p):
            pytest.fail(f"{t} not found (CUDA toolkit bin directory): the kernel inventory is read from the binary")
    dump = subprocess.run([tools["cuobjdump"], "-symbols", str(lib_path)], capture_output=True, text=True, check=True)
    mangled = [line.split()[-1] for line in dump.stdout.splitlines() if "STO_ENTRY" in line]
    demangled = subprocess.run([tools["cu++filt"]], input="\n".join(mangled), capture_output=True, text=True,
                               check=True).stdout.splitlines()
    assert len(demangled) == len(mangled)
    return {normalise(n) for n in demangled}


def _k(name, *targs):
    return f"eqf::{name}" + (f"<{','.join(str(a).lower() for a in targs)}>" if targs else "")


# ------------------------------------------------------------------------------------------------ problem builders
def _past_grid_cap() -> int:
    """Nodes of one warp-per-node grid-stride launch past two full passes: min(ceil(N / 8), 132 * 16) CTAs of 8 warps."""
    return 2 * 8 * 132 * 16 + 1


def _graph(dev, n_nodes, seed, max_deg=40, hub=600):
    """Destination-sorted graph: ragged in-degrees in [0, max_deg), every 7th node none, node n/2 a hub of ``hub`` edges;
    no self-loops (edge lengths are positive)."""
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(seed)
    deg = torch.randint(0, max_deg, (n_nodes,), generator=g)
    deg[::7] = 0
    deg[n_nodes // 2] = hub
    dst = torch.repeat_interleave(torch.arange(n_nodes), deg)
    src = torch.randint(0, n_nodes, (dst.numel(),), generator=g)
    src = torch.where(src == dst, (src + 1) % n_nodes, src)
    return ops.Graph(src.to(dev), dst.to(dev), n_nodes), g


def _randn(g, dev, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(dev)


def _keep(g, dev, E, H):
    return ((torch.rand(E, H, generator=g) > 0.2).float() / 0.8).to(dev)


def _backward(outs, g, dev):
    outs = [o for o in (outs if isinstance(outs, (list, tuple)) else [outs]) if o is not None and o.requires_grad]
    torch.autograd.backward(outs, [_randn(g, dev, *o.shape) for o in outs])


def _leaves(ts):
    return [t.requires_grad_(True) for t in ts]


# ------------------------------------------------------------------------------------------------ attention cases
def _dot_case(H, ds, Cs):
    def run(dev):
        from equiformer_b200 import ops
        graph, g = _graph(dev, _past_grid_cap(), seed=H + sum(Cs), max_deg=3)
        lay = ops.HeadLayout(ds, Cs, H)
        qs = _leaves([_randn(g, dev, graph.n_nodes, d, C) for d, C in zip(ds, Cs)])
        kvs = _leaves([_randn(g, dev, graph.n_edges, d, 2 * C) for d, C in zip(ds, Cs)])
        assert ops.dot_softmax_aggregate_ok(lay, qs[0], graph)
        outs = ops.DotSoftmaxAggregate.apply(lay, graph, _keep(g, dev, graph.n_edges, H), *qs, *kvs)
        _backward(outs, g, dev)
    return run


def _dot_slots(ds, Cs):
    return -(-sum(d * C for d, C in zip(ds, Cs)) // 128)


def _mlp_case(H, A, ds, Cs):
    def run(dev):
        from equiformer_b200 import ops
        graph, g = _graph(dev, _past_grid_cap(), seed=H + A, max_deg=3)
        lay = ops.MlpAttnLayout(ops.HeadLayout(ds, Cs, H), A, 1.6765, 0.2)
        alpha_dot, t0 = _leaves([_randn(g, dev, H, A, scale=0.3), _randn(g, dev, graph.n_edges, lay.width)])
        Vs = _leaves([_randn(g, dev, graph.n_edges, d, C) for d, C in zip(ds[1:], Cs[1:])])
        assert ops.mlp_softmax_aggregate_ok(lay, t0, graph)
        outs = ops.MlpSoftmaxAggregate.apply(lay, graph, _keep(g, dev, graph.n_edges, H), alpha_dot, t0, *Vs)
        _backward(outs, g, dev)
    return run


def _chain_case(H, ds, Cs):
    """EdgeDot -> SegSoftmax -> AttnAggregate and back (the unfused attention family)."""
    def run(dev):
        from equiformer_b200 import ops
        graph, g = _graph(dev, 300, seed=H + sum(Cs))
        lay = ops.HeadLayout(ds, Cs, H)
        ks = _leaves([_randn(g, dev, graph.n_edges, d, C) for d, C in zip(ds, Cs)])
        qs = _leaves([_randn(g, dev, graph.n_nodes, d, C) for d, C in zip(ds, Cs)])
        vs = _leaves([_randn(g, dev, graph.n_edges, d, C) for d, C in zip(ds, Cs)])
        z = ops.EdgeDot.apply(lay, graph, *ks, *qs)
        alpha = ops.SegSoftmax.apply(z, graph)
        _backward(ops.AttnAggregate.apply(lay, graph, alpha, *vs), g, dev)
    return run


def _softmax_aggregate_case(H, ds, Cs):
    def run(dev):
        from equiformer_b200 import ops
        graph, g = _graph(dev, 300, seed=H + 1)
        lay = ops.HeadLayout(ds, Cs, H)
        z = _leaves([_randn(g, dev, graph.n_edges, H)])[0]
        vs = _leaves([_randn(g, dev, graph.n_edges, d, C) for d, C in zip(ds, Cs)])
        assert ops.softmax_aggregate_ok(lay, z)
        _backward(ops.MaskedSoftmaxAggregate.apply(lay, graph, z, _keep(g, dev, graph.n_edges, H), *vs), g, dev)
    return run


# ------------------------------------------------------------------------------------------------ tensor-product cases
PLANS = {
    "qm9_l2": ("128x0e+64x1e+32x2e", "1x0e+1x1e+1x2e"),
    "md17_l3": ("128x0e+64x1e+64x2e+32x3e", "1x0e+1x1e+1x2e+1x3e"),
    "oc20_l1": ("256x0e+128x1e", "1x0e+1x1e"),
    "oc20_l1_e3": ("256x0e+64x0o+64x1e+64x1o", "1x0e+1x1o"),
    "e3_l2": ("128x0e+32x0o+32x1e+32x1o+16x2e+16x2o", "1x0e+1x1o+1x2e"),     # table-driven float4 kernels
    "odd_mul": ("6x0e+3x1e+2x2e", "1x0e+1x1e+1x2e"),                          # table-driven scalar kernels
}
_PLAN_CACHE = {}


def _plan(name):
    if name not in _PLAN_CACHE:
        from equiformer_b200 import codegen
        _PLAN_CACHE[name] = codegen.plan_for(*PLANS[name])
    return _PLAN_CACHE[name]


def _dtp_case(name, shared, grads, gather=False):
    """One depth-wise tensor product forward + backward.  ``grads``: which of x, w, y get a gradient ("xwy", "x", "w")."""
    def run(dev):
        from equiformer_b200 import ops
        plan = _plan(name)
        graph, g = _graph(dev, 97, seed=len(name) + 2 * shared + len(grads) + gather)
        E = graph.n_edges
        y = _randn(g, dev, E, plan.d_y)
        w = _randn(g, dev, *((plan.weight_numel,) if shared else (E, plan.weight_numel)), scale=0.5)
        y.requires_grad_("y" in grads)
        w.requires_grad_("w" in grads)
        if gather:
            As = _leaves([_randn(g, dev, graph.n_nodes, 2 * l + 1, m) for l, m in plan.in1_blocks])
            Bs = _leaves([_randn(g, dev, graph.n_nodes, 2 * l + 1, m) for l, m in plan.in1_blocks])
            outs = ops.DtpOutGathered.apply(plan, graph, len(Bs), y, w, *As, *Bs)
        else:
            xs = [_randn(g, dev, E, 2 * l + 1, m).requires_grad_("x" in grads) for l, m in plan.in1_blocks]
            outs = ops.DtpOut.apply(plan, y, w, *xs)
        _backward(outs, g, dev)
    return run


def _gen(name, kind, *targs):
    return f"eqf::gen_{name}::{kind}_kernel<{','.join('true' if a else 'false' for a in targs)}>"


def _fused_case(name, width):
    """Every output group of a plan times a [K, width] linear (``ops.dtp_linear``, forward): up to 64 columns the fused
    producer + wgmma kernel, wider the group forward + GEMM."""
    def run(dev):
        from equiformer_b200 import ops
        plan = _plan(name)
        graph, g = _graph(dev, 61, seed=width)
        E = graph.n_edges
        As = [_randn(g, dev, graph.n_nodes, 2 * l + 1, m) for l, m in plan.in1_blocks]
        Bs = [_randn(g, dev, graph.n_nodes, 2 * l + 1, m) for l, m in plan.in1_blocks]
        y = _randn(g, dev, E, plan.d_y)
        w = _randn(g, dev, E, plan.weight_numel, scale=0.5)
        off = _randn(g, dev, plan.weight_numel, scale=0.1)
        Ws = [_randn(g, dev, K, width, scale=K ** -0.5) for _l, _p, K in plan.out_groups]
        with torch.no_grad():
            ops.dtp_linear(plan, graph, As, Bs, y, w, off, Ws)
    return run


# ------------------------------------------------------------------------------------------------ GEMM and row cases
def _linear_case(n_out, k_in, rows):
    """``linear_f32`` forward + backward: C = x W^T (mode 1), dx = dC W (mode 0), dW = dC^T x (mode 2)."""
    def run(dev):
        from equiformer_b200 import ops
        g = torch.Generator().manual_seed(n_out + k_in + rows)
        x, W = _leaves([_randn(g, dev, rows, k_in), _randn(g, dev, n_out, k_in, scale=k_in ** -0.5)])
        _backward(ops.linear_f32(x, W), g, dev)
    return run


def _grouped_case(dev):
    """The planar node-level linears' product kernel: matmul_f32 forward + backward below the wgmma row threshold,
    with a bias (its gradient is a column sum) on a row count that is not a multiple of the tile."""
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(5)
    x, W, b = _leaves([_randn(g, dev, 1237, 96), _randn(g, dev, 96, 40, scale=0.1), _randn(g, dev, 40)])
    _backward(ops.add_bias(ops.matmul_f32(x, W), b), g, dev)


def _colsum_scalar_case(dev):
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(6)
    x, b = _leaves([_randn(g, dev, 3001, 37), _randn(g, dev, 37)])
    _backward(ops.add_bias(x, b), g, dev)


def _ln_silu_case(C):
    def run(dev):
        from equiformer_b200 import ops
        g = torch.Generator().manual_seed(C)
        x, gamma, beta, bias = _leaves([_randn(g, dev, 2011, C, scale=2.0), _randn(g, dev, C), _randn(g, dev, C),
                                        _randn(g, dev, C)])
        _backward(ops.ln_silu(x, gamma, beta, 1e-5, bias), g, dev)
    return run


def _gate_case(A0, S, H, ds, Cs):
    def run(dev):
        from equiformer_b200 import ops
        g = torch.Generator().manual_seed(A0 + S)
        lay = ops.GateLayout(A0, S, H, ds, Cs, 1.6791767923989418, 1.8467055342154763, 1.531320475574866, 0.2)
        E = 1999
        t0, bias, ad = _leaves([_randn(g, dev, E, lay.width), _randn(g, dev, lay.width, scale=0.3),
                                _randn(g, dev, H, A0 // H)])
        gated = _leaves([_randn(g, dev, E, d, c) for d, c in zip(ds, Cs)])
        _backward(ops.GateLogits.apply(lay, t0, bias, ad, *gated), g, dev)
    return run


def _eln_case(planar):
    def run(dev):
        from equiformer_b200 import ops
        lay = ops.NormLayout([(128, 1, True), (64, 3, False), (64, 5, False), (32, 7, False)], 1e-5)
        g = torch.Generator().manual_seed(7 + planar)
        x = _randn(g, dev, 1461, lay.dim, scale=1.5)
        w, b = _leaves([_randn(g, dev, lay.n_w), _randn(g, dev, lay.n_b)])
        if planar:          # blocks [N, d, mul]
            xs = _leaves([_randn(g, dev, 1461, d, m, scale=1.5) for m, d, _ in lay.entries])
            _backward(ops.equivariant_layer_norm_planar(lay, xs, w, b), g, dev)
        else:
            _backward(ops.equivariant_layer_norm(lay, x.requires_grad_(True), w, b), g, dev)
    return run


def _radial_case(dev):
    """Edge geometry (vector, length, harmonics to l = 3) feeding the Gaussian, exp-normal and Bessel bases."""
    from equiformer_b200 import ops
    from equiformer_b200.nets.expnorm_rbf import ExpNormalSmearing
    graph, g = _graph(dev, 211, seed=9)
    pos = _leaves([_randn(g, dev, graph.n_nodes, 3, scale=2.0)])[0]
    vec, length, sh = ops.edge_geometry(pos, graph, 3)
    mean, std = _randn(g, dev, 1, 128).abs(), (torch.rand(1, 128, generator=g) * 0.99 + 0.01).to(dev)
    weight, bias = torch.tensor([[1.3]], device=dev), torch.tensor([[-0.05]], device=dev)
    gauss = ops.gaussian_rbf(length, *_leaves([mean, std, weight, bias]), 5.0)
    mod = ExpNormalSmearing(0.0, 5.0, 32, trainable=False)
    expn = ops.expnorm_rbf(length, mod.means.to(dev), mod.betas.to(dev), mod.alpha, 5.0)
    freq = _leaves([(torch.pi * torch.arange(1, 9, dtype=torch.float32)).to(dev)])[0]
    bess = ops.bessel_rbf(length, freq, 5.0)
    _backward([vec, sh, gauss, expn, bess], g, dev)


# ------------------------------------------------------------------------------------------------ the case table
def _cases():
    cases = {}
    # dot-product attention: S = 4 for node rows of <= 512 floats, 5 for 513-640, 8 for 641-1024; channels per head % 4
    for H in (1, 2, 4, 8, 16):
        for ds, Cs in (((1, 3), (64, 64)), ((1, 3, 5), (128, 64, 64)), ((1, 3, 5), (192, 128, 64))):
            slots = _dot_slots(ds, Cs)
            S = 4 if slots <= 4 else 5 if slots == 5 else 8
            cases[f"dot_attention_H{H}_S{S}"] = (_dot_case(H, ds, Cs), {_k("dot_softmax_aggregate_kernel", H, S),
                                                                         _k("dot_softmax_aggregate_bwd_kernel", H, S)})
    # linear-message attention: <H, SA, SV>
    for H, A, ds, Cs, inst in ((2, 32, (1, 3, 5), (64, 64, 32), (2, 1, 4)), (4, 32, (1, 3, 5), (128, 64, 32), (4, 1, 4)),
                               (8, 32, (1, 3), (256, 128), (8, 2, 5))):
        cases[f"mlp_attention_H{H}"] = (_mlp_case(H, A, ds, Cs), {_k("mlp_softmax_aggregate_kernel", *inst),
                                                                 _k("mlp_softmax_aggregate_bwd_kernel", *inst),
                                                                 _k("colsum_kernel", 4)})
    # the unfused attention family: float4 layouts per head count, and a layout off the float4 grid
    for H in (1, 2, 4, 8, 16):
        cases[f"attention_chain_H{H}"] = (_chain_case(H, (1, 3), (64, 64)), {
            _k("edge_dot_vec_kernel", H), _k("seg_softmax_kernel"), _k("seg_softmax_bwd_kernel"),
            _k("aggregate_vec_kernel"), _k("edge_scale_vec_kernel")})
    cases["attention_chain_scalar"] = (_chain_case(2, (1, 3), (6, 2)), {
        _k("edge_dot_kernel"), _k("seg_softmax_kernel"), _k("seg_softmax_bwd_kernel"), _k("aggregate_kernel"),
        _k("edge_scale_kernel")})
    cases["softmax_aggregate_H4"] = (_softmax_aggregate_case(4, (1, 3, 5), (128, 64, 32)), {
        _k("softmax_aggregate_vec_kernel"), _k("edge_dot_vec_kernel", 4), _k("seg_softmax_bwd_kernel"),
        _k("edge_scale_vec_kernel")})
    # plan-specialised tensor products: forward<SHARED, GATHER>, backward<SHARED, GATHER, WITH_W>, grad_y<SHARED>
    for name in ("qm9_l2", "md17_l3", "oc20_l1", "oc20_l1_e3"):
        for shared in (False, True):
            s = "shared" if shared else "edge"
            cases[f"dtp_{name}_{s}_w_xwy"] = (_dtp_case(name, shared, "xwy"), {
                _gen(name, "forward", shared, False), _gen(name, "backward", shared, False, True),
                _gen(name, "grad_y", shared)} | ({_k("colsum_kernel", 4)} if shared else set()))
            cases[f"dtp_{name}_{s}_w_x"] = (_dtp_case(name, shared, "x"), {
                _gen(name, "forward", shared, False), _gen(name, "backward", shared, False, False)})
            cases[f"dtp_{name}_{s}_w_gathered"] = (_dtp_case(name, shared, "xw", gather=True), {
                _gen(name, "forward", shared, True), _gen(name, "backward", shared, True, True),
                _k("aggregate_vec_kernel")} | ({_k("colsum_kernel", 4)} if shared else set()))
    cases["dtp_md17_l3_w_only"] = (_dtp_case("md17_l3", False, "w"), {
        _gen("md17_l3", "forward", False, False), _k("dtp_grad_w_kernel")})
    # table-driven tensor products: float4 (vec_ok) and scalar plans
    for shared in (False, True):
        s = "shared" if shared else "edge"
        cases[f"dtp_e3_l2_{s}_w_xwy"] = (_dtp_case("e3_l2", shared, "xwy"), {
            _k("dtp_forward_vec_kernel", not shared), _k("dtp_grad_x_vec_kernel", True), _k("dtp_grad_y_kernel")}
            | ({_k("colsum_kernel", 4)} if shared else set()))
        cases[f"dtp_odd_mul_{s}_w_xwy"] = (_dtp_case("odd_mul", shared, "xwy"), {
            _k("dtp_forward_kernel"), _k("dtp_grad_x_kernel", True), _k("dtp_grad_y_kernel")}
            | ({_k("colsum_kernel", 4)} if shared else set()))
    cases["dtp_e3_l2_edge_w_x"] = (_dtp_case("e3_l2", False, "x"), {
        _k("dtp_forward_vec_kernel", True), _k("dtp_grad_x_vec_kernel", False)})
    cases["dtp_odd_mul_edge_w_x"] = (_dtp_case("odd_mul", False, "x"), {
        _k("dtp_forward_kernel"), _k("dtp_grad_x_kernel", False)})
    # tensor product fused into the channel-mixing linear (md17_l3: output degrees 0..3)
    for width, bn in ((32, 32), (64, 64)):
        cases[f"dtp_linear_md17_l3_N{width}"] = (_fused_case("md17_l3", width), {
            _k("fused::split_transpose_kernel")} | {_k("fused::dtp_gemm_fwd_kernel", bn, d3) for d3 in (1, 3, 5, 7)})
    cases["dtp_linear_md17_l3_N128"] = (_fused_case("md17_l3", 128), {
        _k("small::grouped_gemm_mma_kernel")} | {_k("fused::dtp_group_forward_kernel", d3) for d3 in (1, 3, 5, 7)})
    # 3xTF32 wgmma GEMMs: column tiles 32 / 64 / 96 / 128 of the forward (mode 1) and data gradient (mode 0), and of the
    # weight gradient (mode 2); 16 411 rows, not a multiple of any tile
    for n_out, k_in in ((32, 96), (64, 128), (96, 32), (128, 64)):
        bn = lambda n: 32 if n <= 32 else 64 if n <= 64 else 96 if n <= 96 else 128
        cases[f"linear_{k_in}_to_{n_out}"] = (_linear_case(n_out, k_in, 16411), {
            _k("tf32x3::split_kernel"), _k("tf32x3::split_transpose_kernel"), _k("tf32x3::gemm_tf32x3_kernel", bn(n_out)),
            _k("tf32x3::gemm_tf32x3_kernel", bn(k_in)), _k("tf32x3::wg::wgrad_tf32x3_kernel", bn(k_in))})
    cases["small_products_with_bias"] = (_grouped_case, {_k("small::grouped_gemm_mma_kernel"), _k("colsum_kernel", 4)})
    cases["bias_37_columns"] = (_colsum_scalar_case, {_k("colsum_kernel", 1)})
    # row kernels
    for C, fwd, bwd in ((64, "ln_silu_fwd64_kernel", "ln_silu_bwd64_kernel"), (48, ("ln_silu_fwd_kernel", 2), None),
                        (96, ("ln_silu_fwd_kernel", 4), None), (256, ("ln_silu_fwd_kernel", 8), None)):
        if C == 64:
            claim = {_k(fwd), _k(bwd)}
        else:
            claim = {_k(*fwd), _k("ln_silu_bwd_kernel", fwd[1])}
        cases[f"ln_silu_C{C}"] = (_ln_silu_case(C), claim | {_k("colsum_kernel", 4 if C % 4 == 0 else 1)})
    cases["gate_logits_vec"] = (_gate_case(128, 128, 4, (3, 5), (64, 32)), {
        _k("gate_logits_fwd_vec_kernel"), _k("gate_logits_bwd_vec_kernel"), _k("colsum_kernel", 4)})
    cases["gate_logits_scalar"] = (_gate_case(64, 20, 4, (3,), (6,)), {
        _k("gate_logits_fwd_kernel"), _k("gate_logits_bwd_kernel"), _k("colsum_kernel", 1), _k("colsum_kernel", 4)})
    cases["equivariant_layer_norm"] = (_eln_case(False), {_k("eln_fwd_kernel"), _k("eln_bwd_kernel"), _k("colsum_kernel", 4)})
    cases["equivariant_layer_norm_planar"] = (_eln_case(True), {_k("eln_fwd_kernel"), _k("eln_bwd_kernel"),
                                                                _k("colsum_kernel", 4)})
    cases["edge_geometry_and_radial_bases"] = (_radial_case, {
        _k("edge_geom_fwd_kernel"), _k("edge_geom_bwd_kernel"), _k("rbf_fwd_kernel"), _k("rbf_bwd_kernel"),
        _k("expnorm_fwd_kernel"), _k("expnorm_bwd_kernel"), _k("bessel_fwd_kernel"), _k("bessel_bwd_kernel"),
        _k("aggregate_kernel"), _k("colsum_kernel", 1), _k("colsum_kernel", 4)})
    return cases


CASES = _cases()

# instances no case launches: integer outputs compared bit for bit against brute force elsewhere
NOT_LAUNCHED = {
    _k("radius_graph_kernel", "false"): "neighbour-list count pass, tested bit for bit against the torch brute force "
                                        "(test_gpu_kernels.py::test_radius_graph_kernels_match_torch_statement)",
    _k("radius_graph_kernel", "true"): "neighbour-list fill pass, as the count pass",
    _k("radius_graph_pbc_kernel", "false"): "periodic neighbour-list count pass, tested against a float64 brute force "
                                            "(test_neighbour_list_pbc.py::test_statement_matches_oracle)",
    _k("radius_graph_pbc_kernel", "true"): "periodic neighbour-list fill pass, as the count pass",
}


# ------------------------------------------------------------------------------------------------ tests
def _lib_path():
    from equiformer_b200 import _lib
    _lib.build()
    return _lib.LIB_PATH


def test_inventory_is_read_from_the_binary():
    inv = inventory(_lib_path())
    print(f"\n[instances] {len(inv)} kernel entries in the library")
    assert inv and all(n.startswith("eqf::") for n in inv), sorted(inv)[:5]
    assert not any("(" in n or " " in n for n in inv)


def test_names_normalise_alike():
    """cu++filt spells template arguments as casts, the profiler as literals: both must map to the same name."""
    a = normalise("void eqf::gen_qm9_l2::backward_kernel<(bool)1, (bool)0, (bool)1>(eqf::EdgeArgs)")
    b = normalise("void eqf::gen_qm9_l2::backward_kernel<true, false, true>(eqf::EdgeArgs)")
    assert a == b == "eqf::gen_qm9_l2::backward_kernel<true,false,true>"
    assert normalise("void eqf::dot_softmax_aggregate_kernel<(int)16, (int)4>(eqf::DotArgs, const float *)") == \
        normalise("void eqf::dot_softmax_aggregate_kernel<16, 4>(eqf::DotArgs, float const*)") == \
        "eqf::dot_softmax_aggregate_kernel<16,4>"
    assert normalise("eqf::seg_softmax_kernel(const float *, long long)") == "eqf::seg_softmax_kernel"


def test_every_instance_is_claimed():
    """The instances the cases claim, plus NOT_LAUNCHED, are exactly the library's kernel entries."""
    inv = inventory(_lib_path())
    claimed = set().union(*(claim for _run, claim in CASES.values()))
    orphans = sorted(inv - claimed - set(NOT_LAUNCHED))
    assert not orphans, f"kernel instances that no case launches: {orphans}"
    stale = sorted((claimed | set(NOT_LAUNCHED)) - inv)
    assert not stale, f"claimed instances that the library does not contain: {stale}"
    assert not claimed & set(NOT_LAUNCHED), sorted(claimed & set(NOT_LAUNCHED))


def _launched(run, dev):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(dev)
        torch.cuda.synchronize()
    return {normalise(e.name) for e in prof.events() if normalise(e.name).startswith("eqf::")}


@pytest.fixture(scope="module")
def profiler_sees_kernels(cuda_device):
    """The profiler reports this library's device kernels at all (otherwise every launch record below is empty)."""
    from equiformer_b200 import ops
    x = torch.randn(333, 20, device=cuda_device)
    seen = _launched(lambda dev: ops.colsum_raw(x), cuda_device)
    assert seen == {_k("colsum_kernel", 4)}, f"the profiler recorded {seen or 'no eqf:: kernel'} for one column sum"
    return True


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_case_launches_what_it_claims(cuda_device, profiler_sees_kernels, case, monkeypatch):
    run, claim = CASES[case]
    torch.manual_seed(0)
    audit = Audit(case)
    audit.install(monkeypatch)
    torch.cuda.reset_peak_memory_stats()
    try:
        launched = _launched(run, cuda_device)
    finally:
        monkeypatch.undo()
    audit.report()
    print(f"[instances] {case}: peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    torch.cuda.empty_cache()
    assert not audit.unaudited, f"{case}: compute launches outside any audited wrapper: {audit.unaudited}"
    assert not audit.failures, "\n".join(audit.failures[:20])
    assert audit.index > 0
    assert launched == claim, (f"{case}: launched but not claimed {sorted(launched - claim)}, "
                               f"claimed but not launched {sorted(claim - launched)}")
