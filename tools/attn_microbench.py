"""K2 microbenchmark: softmax + aggregation in one kernel (eqf_attn_softmax_aggregate) vs the two round-1 kernels, and K2
with an attention-dropout mask (p = 0.2) against K2 without one, forward and first-order backward (edge_dot ->
seg_softmax_bwd, edge_scale).
usage: python tools/attn_microbench.py [E] [n_nodes] [iters]   (QM9 head layout: 4 heads, groups (1,128) (3,64) (5,32))

       python tools/attn_microbench.py dp [iters]
Dot-product attention: the fused kernels (eqf_attn_dot_softmax_aggregate and its backward) against the chain the DP layer
ran before them, forward and first-order backward timed separately, with and without the dropout mask, at the OC20 DP
layout (55 000 edges over 1 240 nodes, 8 heads of 32x0e+16x1e) and the QM9 DP layout (32 560 edges over 2 324 nodes, 4
heads of 32x0e+16x1e+8x2e).  The chain is timed as its raw launches in sequence (no autograd bookkeeping): forward =
key / value half copies, edge_dot, seg_softmax, the mask multiply, aggregate; backward = edge_dot, edge_scale, the mask
multiply, seg_softmax_bwd, edge_scale, aggregate and the concatenation of the key and value gradients into one block.
Bytes are the fused kernels' algorithmic bytes from shapes (ops._dot_attn_bytes); GB/s = those bytes over each time.

       python tools/attn_microbench.py linear [iters]
Linear-message attention: the fused kernels (eqf_attn_mlp_softmax_aggregate and its backward) against the chain the
linear-message layer runs without them, forward and first-order backward timed separately, with and without the dropout
mask, at the OC20 l1_256 layout (55 000 edges over 1 240 nodes, 8 heads of 32 alpha + 32x0e+16x1e) and the QM9 / MD17
L2 layout (32 560 edges over 2 324 nodes, 4 heads of 32 alpha + 32x0e+16x1e+8x2e).  The chain is timed as its raw
launches in sequence: forward = the activation statement on the alpha channels (elementwise torch ops, * alpha_dot, sum),
the copy of the strided value scalars, K2 (eqf_attn_softmax_aggregate); backward = edge_dot, seg_softmax_bwd and
edge_scale of K2, the activation's backward as torch ops, the alpha_dot sum and the assembly of the t0 gradient.  Bytes
are the fused kernels' algorithmic bytes from shapes (ops._mlp_attn_bytes)."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from equiformer_b200 import ops  # noqa: E402


def main():
    E = int(sys.argv[1]) if len(sys.argv) > 1 else 32560
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 2324
    iters = int(sys.argv[3]) if len(sys.argv) > 3 else 50
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    dst = torch.sort(torch.randint(0, n, (E,), device=dev, generator=g)).values
    src = torch.randint(0, n, (E,), device=dev, generator=g)
    graph = ops.Graph(src, dst, n)
    lay = ops.HeadLayout([1, 3, 5], [128, 64, 32], 4)
    z = torch.randn(E, 4, device=dev, generator=g)
    Vs = [torch.randn(E, d, c, device=dev, generator=g) for d, c in zip(lay.ds, lay.Cs)]
    Gs = [torch.randn(n, d, c, device=dev, generator=g) for d, c in zip(lay.ds, lay.Cs)]
    keep = torch.nn.functional.dropout(torch.ones_like(z), 0.2, True)

    def timeit(fn):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) * 1e3 / iters

    two = timeit(lambda: ops.attn_aggregate_raw(lay, ops.seg_softmax_raw(z, graph), Vs, graph))
    one = timeit(lambda: ops.softmax_aggregate_raw(lay, z, Vs, graph))
    masked = timeit(lambda: ops.softmax_aggregate_raw(lay, z, Vs, graph, keep))
    alpha = ops.softmax_aggregate_raw(lay, z, Vs, graph)[1]

    def backward(*extra):
        ops.seg_softmax_bwd_raw(alpha, ops.attn_edge_dot_raw(lay, Vs, Gs, graph), graph, *extra)
        ops.attn_edge_scale_raw(lay, alpha, Gs, graph, *extra)

    bwd = timeit(backward)
    bwd_masked = timeit(lambda: backward(keep))
    nbytes = 4 * (E * (480 + 4 + 4) + n * 480)
    print(json.dumps({"E": E, "nodes": n, "two_kernels_us": round(two, 1), "fused_us": round(one, 1),
                      "fused_masked_us": round(masked, 1), "bwd_us": round(bwd, 1), "bwd_masked_us": round(bwd_masked, 1),
                      "fused_gb_s": round(nbytes / one / 1e3, 1), "algorithmic_bytes": nbytes,
                      "device": torch.cuda.get_device_name(dev)}))


def _timeit(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / iters


DP_LAYOUTS = {"oc20_dp": (55000, 1240, 8, (1, 3), (256, 128)), "qm9_dp": (32560, 2324, 4, (1, 3, 5), (128, 64, 32))}


def dot_product(iters):
    dev = torch.device("cuda:0")
    for name, (E, n, H, ds, Cs) in DP_LAYOUTS.items():
        g = torch.Generator(device=dev).manual_seed(0)
        dst = torch.sort(torch.randint(0, n, (E,), device=dev, generator=g)).values
        src = torch.randint(0, n, (E,), device=dev, generator=g)
        graph = ops.Graph(src, dst, n)
        lay = ops.HeadLayout(ds, Cs, H)
        qs = [torch.randn(n, d, c, device=dev, generator=g) for d, c in zip(ds, Cs)]
        kvs = [torch.randn(E, d, 2 * c, device=dev, generator=g) for d, c in zip(ds, Cs)]
        Gs = [torch.randn(n, d, c, device=dev, generator=g) for d, c in zip(ds, Cs)]
        keep = torch.nn.functional.dropout(torch.ones(E, H, device=dev), 0.2, True)
        row = {"layout": name, "E": E, "nodes": n, "heads": H}
        for masked in (False, True):
            kp = keep if masked else None
            tag = "masked" if masked else "unmasked"

            def chain_fwd():
                k = [t.narrow(2, 0, c).contiguous() for t, c in zip(kvs, Cs)]
                v = [t.narrow(2, c, c).contiguous() for t, c in zip(kvs, Cs)]
                a = ops.seg_softmax_raw(ops.attn_edge_dot_raw(lay, k, qs, graph), graph)
                return ops.attn_aggregate_raw(lay, a if kp is None else a * kp, v, graph), a, k, v

            _, alpha, k, v = chain_fwd()

            def chain_bwd():
                ga = ops.attn_edge_dot_raw(lay, v, Gs, graph)
                gv = ops.attn_edge_scale_raw(lay, alpha if kp is None else alpha * kp, Gs, graph)
                gz = ops.seg_softmax_bwd_raw(alpha, ga if kp is None else ga * kp, graph)
                gk = ops.attn_edge_scale_raw(lay, gz, qs, graph)
                gq = ops.attn_aggregate_raw(lay, gz, k, graph)
                return gq, [torch.cat([a, b], dim=2) for a, b in zip(gk, gv)]

            fused_fwd = lambda: ops.dot_softmax_aggregate_raw(lay, qs, kvs, graph, kp)
            fused_bwd = lambda: ops.dot_softmax_aggregate_bwd_raw(lay, Gs, qs, kvs, alpha, graph, kp)
            for kind, fused, chain in (("forward", fused_fwd, chain_fwd), ("backward", fused_bwd, chain_bwd)):
                nbytes = ops._dot_attn_bytes(lay, E, n, masked, kind)
                t_f, t_c = _timeit(fused, iters), _timeit(chain, iters)
                row[f"{kind}_{tag}"] = {"fused_us": round(t_f, 1), "chain_us": round(t_c, 1), "bytes": nbytes,
                                        "fused_gb_s": round(nbytes / t_f / 1e3, 1),
                                        "chain_gb_s": round(nbytes / t_c / 1e3, 1)}
        row["device"] = torch.cuda.get_device_name(dev)
        print(json.dumps(row), flush=True)


LINEAR_LAYOUTS = {"oc20_l1": (55000, 1240, 8, 32, (1, 3), (256, 128)),
                  "qm9_md17_l2": (32560, 2324, 4, 32, (1, 3, 5), (128, 64, 32))}


def linear_message(iters):
    dev = torch.device("cuda:0")
    for name, (E, n, H, A, ds, Cs) in LINEAR_LAYOUTS.items():
        g = torch.Generator(device=dev).manual_seed(0)
        dst = torch.sort(torch.randint(0, n, (E,), device=dev, generator=g)).values
        src = torch.randint(0, n, (E,), device=dev, generator=g)
        graph = ops.Graph(src, dst, n)
        hl = ops.HeadLayout(ds, Cs, H)
        lay = ops.MlpAttnLayout(hl, A, 1.6765, 0.2)
        R = lay.n_scalars
        t0 = torch.randn(E, lay.width, device=dev, generator=g)
        Vs = [torch.randn(E, d, c, device=dev, generator=g) for d, c in zip(ds[1:], Cs[1:])]
        ad = 0.3 * torch.randn(H, A, device=dev, generator=g)
        Gs = [torch.randn(n, d, c, device=dev, generator=g) for d, c in zip(ds, Cs)]
        keep = torch.nn.functional.dropout(torch.ones(E, H, device=dev), 0.2, True)
        k1, k2 = 0.5 * (1 + lay.slope), 0.5 * (1 - lay.slope)
        row = {"layout": name, "E": E, "nodes": n, "heads": H}
        for masked in (False, True):
            kp = keep if masked else None
            tag = "masked" if masked else "unmasked"

            def chain_fwd():
                z = ops.mlp_logits_torch(lay, t0, ad)
                vals = [ops.mlp_value_scalars(lay, t0).contiguous(), *Vs]
                return ops.softmax_aggregate_raw(hl, z, vals, graph, *(() if kp is None else (kp,))), vals

            (_, alpha), vals = chain_fwd()

            def chain_bwd():
                ga = ops.attn_edge_dot_raw(hl, vals, Gs, graph)
                gz = ops.seg_softmax_bwd_raw(alpha, ga, graph, *(() if kp is None else (kp,)))
                gv = ops.attn_edge_scale_raw(hl, alpha, Gs, graph, *(() if kp is None else (kp,)))
                a = t0.view(E, H, A + R)[:, :, :A]
                s = torch.sigmoid(a)
                act = lay.c_slr * (k1 * a + k2 * a * (2 * s - 1))
                dact = lay.c_slr * (k1 + k2 * ((2 * s - 1) + 2 * a * s * (1 - s)))
                gdot = (gz[:, :, None] * act).sum(0)
                gt0 = torch.zeros_like(t0).view(E, H, A + R)
                gt0[:, :, :A] = gz[:, :, None] * ad * dact
                gt0[:, :, A:] = gv[0].view(E, H, R)
                return gt0, gv[1:], gdot

            fused_fwd = lambda: ops.mlp_softmax_aggregate_raw(lay, t0, Vs, ad, graph, kp)
            fused_bwd = lambda: ops.mlp_softmax_aggregate_bwd_raw(lay, Gs, t0, Vs, ad, alpha, graph, kp)
            for kind, fused, chain in (("forward", fused_fwd, chain_fwd), ("backward", fused_bwd, chain_bwd)):
                nbytes = ops._mlp_attn_bytes(lay, E, n, masked, kind)
                t_f, t_c = _timeit(fused, iters), _timeit(chain, iters)
                row[f"{kind}_{tag}"] = {"fused_us": round(t_f, 1), "chain_us": round(t_c, 1), "bytes": nbytes,
                                        "fused_gb_s": round(nbytes / t_f / 1e3, 1),
                                        "chain_gb_s": round(nbytes / t_c / 1e3, 1)}
        row["device"] = torch.cuda.get_device_name(dev)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "dp":
        dot_product(int(sys.argv[2]) if len(sys.argv) > 2 else 200)
    elif len(sys.argv) > 1 and sys.argv[1] == "linear":
        linear_message(int(sys.argv[2]) if len(sys.argv) > 2 else 200)
    else:
        main()
