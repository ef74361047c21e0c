"""TEST-ONLY stand-ins for the raw kernel entry points of ``equiformer_b200.ops``.

The product has no CPU path (CPU tensors raise).  To exercise the *host* logic - planar layouts, weight views, head
layouts, the autograd families and their closure under differentiation - without a GPU, the CPU test-suite
monkeypatches the ``*_raw`` functions with these torch restatements that walk the same plan tables the kernels use.
Nothing outside ``tests/`` imports this module.
"""
from __future__ import annotations

import contextlib

import torch

from equiformer_b200 import ops


def _cg(plan, p, like):
    """Coupling block of path ``p`` in the dtype and on the device of ``like`` (the references also run on a GPU in fp64)."""
    d1, d2, d3 = 2 * p.l1 + 1, 2 * p.l2 + 1, 2 * p.l3 + 1
    c = torch.from_numpy(plan.cg64[p.cg_off:p.cg_off + d1 * d2 * d3].copy()).reshape(d1, d2, d3)
    return c.to(device=like.device, dtype=like.dtype)


def _w(plan, p, w):
    wv = w[..., p.w_off:p.w_off + p.mul]
    return wv if wv.dim() == 2 else wv[None, :]


def _gathered(xs, gather):
    if gather is None:
        return xs
    src, dst, x2s = gather
    xs = [x.index_select(0, src) for x in xs]
    if x2s is not None:
        xs = [x + b.index_select(0, dst) for x, b in zip(xs, x2s)]
    return xs


def dtp_forward_raw(plan, xs, y, w, gather=None, w_offset=None):
    xs = _gathered(xs, gather)
    if w_offset is not None:
        w = w + w_offset
    E = y.shape[0]
    outs = [y.new_zeros((E, 2 * l + 1, mul)) for l, _p, mul in plan.out_groups]
    for p in plan.paths:
        M = torch.einsum("ijk,ej->eik", _cg(plan, p, y), y[:, p.in2_off:p.in2_off + 2 * p.l2 + 1])
        val = torch.einsum("eiu,eik->eku", xs[p.in1_block], M) * _w(plan, p, w)[:, None, :]
        outs[p.out_group][:, :, p.out_chan_off:p.out_chan_off + p.mul] = val
    return outs


def dtp_linear_fwd_raw(plan, group, xs, y, w, Wt, gather=None, w_offset=None):
    f = dtp_forward_raw(plan, xs, y, w, gather, w_offset)[group]
    return torch.einsum("eku,un->ekn", f, Wt)


def dtp_group_forward_raw(plan, group, xs, y, w, gather=None, w_offset=None):
    return dtp_forward_raw(plan, xs, y, w, gather, w_offset)[group]


def dtp_grad_x_raw(plan, gs, y, w):
    E = y.shape[0]
    gxs = [y.new_zeros((E, 2 * l + 1, mul)) for l, mul in plan.in1_blocks]
    for p in plan.paths:
        M = torch.einsum("ijk,ej->eik", _cg(plan, p, y), y[:, p.in2_off:p.in2_off + 2 * p.l2 + 1])
        g = gs[p.out_group][:, :, p.out_chan_off:p.out_chan_off + p.mul]
        gxs[p.in1_block] = gxs[p.in1_block] + torch.einsum("eku,eik->eiu", g, M) * _w(plan, p, w)[:, None, :]
    return gxs


def dtp_grad_w_raw(plan, xs, y, gs, shared):
    E = y.shape[0]
    gw = y.new_zeros((E, plan.weight_numel))
    for p in plan.paths:
        M = torch.einsum("ijk,ej->eik", _cg(plan, p, y), y[:, p.in2_off:p.in2_off + 2 * p.l2 + 1])
        g = gs[p.out_group][:, :, p.out_chan_off:p.out_chan_off + p.mul]
        gw[:, p.w_off:p.w_off + p.mul] = torch.einsum("eiu,eik,eku->eu", xs[p.in1_block], M, g)
    return gw.sum(0) if shared else gw


def dtp_grad_y_raw(plan, xs, w, gs, y_like):
    E = y_like.shape[0]
    gy = y_like.new_zeros((E, plan.d_y))
    for p in plan.paths:
        g = gs[p.out_group][:, :, p.out_chan_off:p.out_chan_off + p.mul]
        N = torch.einsum("eiu,eku,eu->eik", xs[p.in1_block], g, _w(plan, p, w).expand(E, -1))
        d2 = 2 * p.l2 + 1
        gy[:, p.in2_off:p.in2_off + d2] = gy[:, p.in2_off:p.in2_off + d2] + torch.einsum(
            "ijk,eik->ej", _cg(plan, p, y_like), N)
    return gy


def dtp_grad_xw_raw(plan, xs, y, w, gs, gather=None, w_offset=None):
    xs = _gathered(xs, gather)
    if w_offset is not None:
        w = w + w_offset
    return dtp_grad_x_raw(plan, gs, y, w), dtp_grad_w_raw(plan, xs, y, gs, w.dim() == 1)


def seg_softmax_bwd_raw(alpha, ga, graph, keep=None):
    t = alpha * (ga if keep is None else ga * keep)
    s = alpha.new_zeros((graph.n_nodes, alpha.shape[1])).index_add(0, graph.dst, t)
    return t - alpha * s.index_select(0, graph.dst)


def _head_of(lay, g, device=None):
    C = lay.Cs[g]
    return torch.arange(C, device=device) // (C // lay.n_heads)


def seg_softmax_raw(z, graph):
    """Segment softmax over destination segments, vectorised (segment maxima by ``index_reduce``)."""
    m = z.new_full((graph.n_nodes, z.shape[1]), float("-inf")).index_reduce(0, graph.dst, z, "amax")
    e = (z - m.index_select(0, graph.dst)).exp()
    s = z.new_zeros((graph.n_nodes, z.shape[1])).index_add(0, graph.dst, e)
    return e / (s.index_select(0, graph.dst) + 1e-16)


def attn_aggregate_raw(lay, alpha, Vs, graph, by_src=False):
    outs = []
    index = graph.src if by_src else graph.dst
    for g, V in enumerate(Vs):
        val = V if alpha is None else V * alpha[:, _head_of(lay, g, V.device)][:, None, :]
        out = V.new_zeros((graph.n_nodes,) + tuple(V.shape[1:]))
        outs.append(out.index_add(0, index, val))
    return outs


def softmax_aggregate_raw(lay, z, Vs, graph, keep=None):
    alpha = seg_softmax_raw(z, graph)
    return attn_aggregate_raw(lay, alpha if keep is None else alpha * keep, Vs, graph), alpha


def attn_edge_dot_raw(lay, Vs, Gs, graph):
    E = graph.n_edges
    out = Vs[0].new_zeros((E, lay.n_heads))
    for g, (V, G) in enumerate(zip(Vs, Gs)):
        prod = (V * G.index_select(0, graph.dst)).sum(dim=1)  # [E, C]
        out = out.index_add(1, _head_of(lay, g, V.device), prod)
    return out


def attn_edge_scale_raw(lay, alpha, Gs, graph, keep=None):
    if keep is not None:
        alpha = alpha * keep
    outs = []
    for g, G in enumerate(Gs):
        val = G.index_select(0, graph.dst)
        if alpha is not None:
            val = val * alpha[:, _head_of(lay, g, G.device)][:, None, :]
        outs.append(val)
    return outs


def kv_halves(lay, kvs):
    """Keys ``[..., :C]`` and values ``[..., C:]`` of the key / value blocks of the dot-product attention."""
    return ([t[..., :C] for t, C in zip(kvs, lay.Cs)], [t[..., C:] for t, C in zip(kvs, lay.Cs)])


def dot_softmax_aggregate_raw(lay, qs, kvs, graph, keep=None):
    k, v = kv_halves(lay, kvs)
    alpha = seg_softmax_raw(attn_edge_dot_raw(lay, k, qs, graph), graph)
    return attn_aggregate_raw(lay, alpha if keep is None else alpha * keep, v, graph), alpha


def dot_softmax_aggregate_bwd_raw(lay, Gs, qs, kvs, alpha, graph, keep=None):
    """The formulas the backward kernel implements, stated on whole tensors."""
    k, v = kv_halves(lay, kvs)
    keep = torch.ones_like(alpha) if keep is None else keep
    ga = attn_edge_dot_raw(lay, v, Gs, graph)
    s = alpha.new_zeros((graph.n_nodes, lay.n_heads)).index_add(0, graph.dst, alpha * keep * ga)
    gz = alpha * (keep * ga - s.index_select(0, graph.dst))
    gk = attn_edge_scale_raw(lay, gz, qs, graph)
    gv = attn_edge_scale_raw(lay, alpha * keep, Gs, graph)
    gq = attn_aggregate_raw(lay, gz, k, graph)
    return gq, [torch.cat([a, b], dim=2) for a, b in zip(gk, gv)]


def mlp_softmax_aggregate_raw(lay, t0, Vs, alpha_dot, graph, keep=None):
    alpha = seg_softmax_raw(ops.mlp_logits_torch(lay, t0, alpha_dot), graph)
    vals = [ops.mlp_value_scalars(lay, t0), *Vs]
    return attn_aggregate_raw(lay.head, alpha if keep is None else alpha * keep, vals, graph), alpha


def mlp_softmax_aggregate_bwd_raw(lay, Gs, t0, Vs, alpha_dot, alpha, graph, keep=None):
    """The formulas the backward kernel implements, stated on whole tensors."""
    hl = lay.head
    E, H, A, R_ = t0.shape[0], hl.n_heads, lay.n_alpha, lay.n_scalars
    keep = torch.ones_like(alpha) if keep is None else keep
    vals = [ops.mlp_value_scalars(lay, t0), *Vs]
    ga = attn_edge_dot_raw(hl, vals, Gs, graph)
    s = alpha.new_zeros((graph.n_nodes, H)).index_add(0, graph.dst, alpha * keep * ga)
    gz = alpha * (keep * ga - s.index_select(0, graph.dst))
    gv = attn_edge_scale_raw(hl, alpha * keep, Gs, graph)
    a = t0.reshape(E, H, A + R_)[:, :, :A]
    sg = torch.sigmoid(a)
    k1, k2 = 0.5 * (1 + lay.slope), 0.5 * (1 - lay.slope)
    act = lay.c_slr * (k1 * a + k2 * a * (2 * sg - 1))
    dact = lay.c_slr * (k1 + k2 * ((2 * sg - 1) + 2 * a * sg * (1 - sg)))
    gt0 = torch.cat([gz[:, :, None] * alpha_dot.reshape(1, H, A) * dact, gv[0].reshape(E, H, R_)], dim=2).reshape(E, -1)
    return gt0, gv[1:], (gz[:, :, None] * act).sum(0).reshape(-1)


def gemm_raw(mode, A, B):
    if mode == 0:
        return A @ B
    return A @ B.t() if mode == 1 else A.t() @ B


def grouped_gemm_raw(problems):
    """``(mode, A, B, C, alpha, accumulate)``: C is written (or added to) in place, like the kernel."""
    for mode, A, B, C, alpha, acc in problems:
        val = alpha * (A @ B if mode == 0 else A @ B.t() if mode == 1 else A.t() @ B)
        if acc:
            C.add_(val)
        else:
            C.copy_(val)


def ln_silu_fwd_raw(x, gamma, beta, eps, bias=None):
    xb = x if bias is None else x + bias
    mean = xb.mean(-1)
    rstd = (xb.var(-1, unbiased=False) + eps).rsqrt()
    return ops.ln_silu_torch(x, gamma, beta, eps, bias), mean, rstd


def rbf_fwd_raw(dist, mean, std, weight, bias, cutoff):
    return ops.gaussian_rbf_torch(dist, mean, std, weight, bias, cutoff)


def rbf_bwd_raw(dist, mean, std, weight, bias, cutoff, g):
    ins = [t.detach().requires_grad_(True) for t in (dist, mean, std, weight, bias)]
    with torch.enable_grad():
        out = ops.gaussian_rbf_torch(*ins, cutoff)
    gd, gm, gs, gw, gb = torch.autograd.grad(out, ins, g)
    return gd, gm.reshape(-1), gs.reshape(-1), gw.reshape(-1), gb.reshape(-1)


def colsum_raw(x):
    return x.sum(0)


def eln_fwd_raw(lay, x, w, b):
    return ops.eln_torch(lay, x, w, b), torch.zeros(x.shape[0], len(lay.entries))


def eln_bwd_raw(lay, x, w, rstd, gy):
    xs = [t.detach().requires_grad_(True) for t in (x, w, b_like(lay, x))]
    with torch.enable_grad():
        y = ops.eln_torch(lay, *xs)
    gx, gw, gb = torch.autograd.grad(y, xs, gy, allow_unused=True)
    return gx, gw, gb if gb is not None else torch.zeros(lay.n_b)


def eln_planar_fwd_raw(lay, xs, w, b):
    return ops.eln_planar_torch(lay, list(xs), w, b), torch.zeros(xs[0].shape[0], len(lay.entries))


def eln_planar_bwd_raw(lay, xs, w, rstd, gys):
    ins = [t.detach().requires_grad_(True) for t in (w, b_like(lay, xs[0]), *xs)]
    with torch.enable_grad():
        ys = ops.eln_planar_torch(lay, ins[2:], ins[0], ins[1])
    g = torch.autograd.grad(ys, ins, list(gys), allow_unused=True)
    return list(g[2:]), g[0], (g[1] if g[1] is not None else torch.zeros(lay.n_b))


def b_like(lay, x):
    return torch.zeros(lay.n_b, dtype=x.dtype)


def ln_silu_bwd_raw(x, gamma, beta, mean, rstd, gy, bias=None):
    with torch.enable_grad():
        xs = [t.detach().requires_grad_(True) for t in (x, gamma, beta)]
        y = ops.ln_silu_torch(xs[0], xs[1], xs[2], 1e-5, bias)
        gx, gg, gb = torch.autograd.grad(y, xs, gy)
    return gx, gg, gb, (gx.sum(0) if bias is not None else None)


def gate_logits_fwd_raw(lay, t0, bias, alpha_dot, gated):
    z, v0, *vout = ops.gate_logits_torch(lay, t0, bias, alpha_dot, *gated)
    return z, v0, list(vout)


def gate_logits_bwd_raw(lay, t0, bias, alpha_dot, gated, gz, gv0, gvout):
    with torch.enable_grad():
        t = t0.detach().requires_grad_(True)
        ad = alpha_dot.detach().requires_grad_(True)
        gs = [g.detach().requires_grad_(True) for g in gated]
        outs = ops.gate_logits_torch(lay, t, bias.detach() if bias is not None else None, ad, *gs)
        pairs = [(o, g) for o, g in zip(outs, [gz, gv0, *gvout]) if o.requires_grad]
        grads = torch.autograd.grad([o for o, _ in pairs], [t, ad, *gs], [g for _, g in pairs], allow_unused=True)
    return grads[0], list(grads[2:]), (grads[1].reshape(-1) if lay.n_alpha > 0 else None)


_PATCHED = ["rbf_fwd_raw", "rbf_bwd_raw", "colsum_raw", "eln_fwd_raw", "eln_bwd_raw", "eln_planar_fwd_raw", "eln_planar_bwd_raw", "ln_silu_fwd_raw", "ln_silu_bwd_raw", "gate_logits_fwd_raw", "gate_logits_bwd_raw", "gemm_raw", "grouped_gemm_raw", "dtp_forward_raw", "dtp_linear_fwd_raw", "dtp_group_forward_raw", "dtp_grad_x_raw", "dtp_grad_w_raw", "dtp_grad_y_raw", "dtp_grad_xw_raw",
            "seg_softmax_raw", "seg_softmax_bwd_raw", "softmax_aggregate_raw", "attn_aggregate_raw", "attn_edge_dot_raw", "attn_edge_scale_raw"]


@contextlib.contextmanager
def emulated_kernels():
    """Swap the raw kernel calls (and the CUDA-only checks) for the torch stand-ins above."""
    saved = {name: getattr(ops, name) for name in _PATCHED}
    saved["_require_cuda"] = ops._require_cuda
    saved["_require_index"] = ops._require_index
    g = globals()
    try:
        for name in _PATCHED:
            setattr(ops, name, g[name])
        ops._require_cuda = lambda t, name: t.contiguous()
        ops._require_index = lambda t, name: t.to(torch.int64).contiguous()
        ops.FUSED_ON_ANY_DEVICE = True
        yield
    finally:
        ops.FUSED_ON_ANY_DEVICE = False
        for name, fn in saved.items():
            setattr(ops, name, fn)
