"""K1 microbenchmark: the fused DTP -> per-degree linear launch (``eqf_dtp_linear_fwd``) against the round-1 pipeline
(DTP kernel writing ``[E, K]`` to HBM + wgmma GEMM reading it back) on the layer shapes of the model.

usage: python tools/fused_microbench.py [config] [E] [iters] > out.jsonl     config in {qm9_l2, md17_l3, oc20_l1}
CUDA-event timing on the launching stream after warm-up; node tables are L2-resident as in the model, the per-edge radial
weights ([E, W], 125 MB at the QM9 size) stream from HBM."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from equiformer_b200 import ops  # noqa: E402
from equiformer_b200.nets.graph_attention_transformer import DepthwiseTensorProduct  # noqa: E402

CONFIGS = {"qm9_l2": ("128x0e+64x1e+32x2e", "1x0e+1x1e+1x2e", {0: (352, 128), 1: (64, 64), 2: (32, 32)}),
           "md17_l3": ("128x0e+64x1e+64x2e+32x3e", "1x0e+1x1e+1x2e+1x3e", {0: (352, 128), 1: (64, 64), 2: (64, 64), 3: (32, 32)}),
           "oc20_l1": ("256x0e+128x1e", "1x0e+1x1e", {0: (768, 256), 1: (128, 128)})}


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "qm9_l2"
    E = int(sys.argv[2]) if len(sys.argv) > 2 else 32560
    iters = int(sys.argv[3]) if len(sys.argv) > 3 else 20
    irreps, sh, widths = CONFIGS[name]
    plan = DepthwiseTensorProduct(irreps, sh, irreps, internal_weights=False, bias=False).tp.plan
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    n_nodes = max(E // 14, 2)
    As = [torch.randn(n_nodes, 2 * l + 1, m, device=dev, generator=g) for l, m in plan.in1_blocks]
    Bs = [torch.randn(n_nodes, 2 * l + 1, m, device=dev, generator=g) for l, m in plan.in1_blocks]
    xe = [torch.randn(E, 2 * l + 1, m, device=dev, generator=g) for l, m in plan.in1_blocks]
    y = torch.randn(E, plan.d_y, device=dev, generator=g)
    w = torch.randn(E, plan.weight_numel, device=dev, generator=g)
    ws = torch.randn(plan.weight_numel, device=dev, generator=g)
    off = torch.randn(plan.weight_numel, device=dev, generator=g)
    dst = torch.sort(torch.randint(0, n_nodes, (E,), device=dev, generator=g)).values
    src = torch.randint(0, n_nodes, (E,), device=dev, generator=g)
    gather = (src, dst, Bs)

    def timeit(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) * 1e3 / iters

    for which, (xs, gat, ww, oo, col) in {"dtp1 (gather, per-edge w)": (As, gather, w, off, 0),
                                          "dtp2 (per-edge x, shared w)": (xe, None, ws, None, 1)}.items():
        Ws = [torch.randn(K, widths[l][col], device=dev, generator=g) / K ** 0.5 for l, _p, K in plan.out_groups]
        us_dtp = timeit(lambda: ops.dtp_forward_raw(plan, xs, y, ww, gather=gat, w_offset=oo))
        f = ops.dtp_forward_raw(plan, xs, y, ww, gather=gat, w_offset=oo)
        row = {"config": name, "E": E, "case": which, "unfused_dtp_us": round(us_dtp, 1), "groups": []}
        tot_f = tot_u = 0.0
        for gi, (l, _p, K) in enumerate(plan.out_groups):
            N = Ws[gi].shape[1]
            d = 2 * l + 1
            a2 = f[gi].reshape(E * d, K)
            us_gemm = timeit(lambda: ops.gemm_tf32x3_raw(a2, Ws[gi], b_is_kn=True))
            us_fused = timeit(lambda: ops.dtp_linear_fwd_raw(plan, gi, xs, y, ww, Ws[gi], gather=gat, w_offset=oo))
            err = ((ops.dtp_linear_fwd_raw(plan, gi, xs, y, ww, Ws[gi], gather=gat, w_offset=oo).reshape(E * d, N)
                    - ops.gemm_tf32x3_raw(a2, Ws[gi], b_is_kn=True)).abs().max() / (a2 @ Ws[gi]).abs().max()).item()
            flops = 2.0 * E * d * K * N
            rec = {"l": l, "rows": E * d, "K": K, "N": N, "gemm_us": round(us_gemm, 1), "fused_us": round(us_fused, 1),
                   "fused_tflops_useful": round(flops / us_fused / 1e6, 1), "rel_diff": err}
            if N > ops._FUSED_MAX_N:       # the route DtpLinear takes for wide linears: one group to HBM + wide GEMM
                us_grp = timeit(lambda: ops.dtp_group_forward_raw(plan, gi, xs, y, ww, gather=gat, w_offset=oo))
                rec["group_forward_us"] = round(us_grp, 1)
                us_fused = us_grp + us_gemm
                rec["route_us"] = round(us_fused, 1)
            row["groups"].append(rec)
            tot_f += us_fused
            tot_u += us_gemm
        row["fused_total_us"] = round(tot_f, 1)
        row["unfused_total_us"] = round(tot_u + us_dtp, 1)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
