"""K2 microbenchmark: softmax + aggregation in one kernel (eqf_attn_softmax_aggregate) vs the two round-1 kernels, and K2
with an attention-dropout mask (p = 0.2) against K2 without one, forward and first-order backward (edge_dot ->
seg_softmax_bwd, edge_scale).
usage: python tools/attn_microbench.py [E] [n_nodes] [iters]   (QM9 head layout: 4 heads, groups (1,128) (3,64) (5,32))"""
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


if __name__ == "__main__":
    main()
