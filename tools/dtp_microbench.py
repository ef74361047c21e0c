"""Operator-boundary microbenchmark of the DTP kernels (SURVEY.md section 8d): GB/s vs the measured HBM peak.

usage: python tools/dtp_microbench.py [config] [E] [iters]      config in {qm9_l2, md17_l3, oc20_l1, oc20_l1_e3}
Times each kernel with CUDA events on the launching stream after warm-up; operands (>= 0.5 GB) exceed the 126 MB L2.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from equiformer_b200 import ops  # noqa: E402
from equiformer_b200.nets.graph_attention_transformer import DepthwiseTensorProduct  # noqa: E402

CONFIGS = {"qm9_l2": ("128x0e+64x1e+32x2e", "1x0e+1x1e+1x2e"),
           "md17_l3": ("128x0e+64x1e+64x2e+32x3e", "1x0e+1x1e+1x2e+1x3e"),
           "oc20_l1": ("256x0e+128x1e", "1x0e+1x1e"),
           "oc20_l1_e3": ("256x0e+64x0o+64x1e+64x1o", "1x0e+1x1o")}      # OC20_L1_256_E3_NONLINEAR


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "qm9_l2"
    E = int(sys.argv[2]) if len(sys.argv) > 2 else 32560
    iters = int(sys.argv[3]) if len(sys.argv) > 3 else 20
    irreps, sh = CONFIGS[name]
    plan = DepthwiseTensorProduct(irreps, sh, irreps, internal_weights=False, bias=False).tp.plan
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    xs = [torch.randn(E, 2 * l + 1, m, device=dev, generator=g) for l, m in plan.in1_blocks]
    y = torch.randn(E, plan.d_y, device=dev, generator=g)
    w = torch.randn(E, plan.weight_numel, device=dev, generator=g)
    ws = torch.randn(plan.weight_numel, device=dev, generator=g)
    gs = [torch.randn(E, 2 * l + 1, m, device=dev, generator=g) for l, _p, m in plan.out_groups]
    peak = 6592.2
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        peak = json.load(open(p))["hbm_gbs"]

    def timeit(fn, nbytes):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        us = s.elapsed_time(e) * 1e3 / iters
        gbs = nbytes / (us * 1e-6) / 1e9
        return us, gbs

    rows = {}
    rows["forward(per-edge w)"] = timeit(lambda: ops.dtp_forward_raw(plan, xs, y, w), ops._dtp_bytes(plan, E, False, "forward"))
    rows["forward(shared w)"] = timeit(lambda: ops.dtp_forward_raw(plan, xs, y, ws), ops._dtp_bytes(plan, E, True, "forward"))
    rows["grad_xw(per-edge w)"] = timeit(lambda: ops.dtp_grad_xw_raw(plan, xs, y, w, gs), ops._dtp_bytes(plan, E, False, "grad_xw"))
    rows["grad_xw(shared w)"] = timeit(lambda: ops.dtp_grad_xw_raw(plan, xs, y, ws, gs), ops._dtp_bytes(plan, E, True, "grad_xw"))
    rows["grad_x"] = timeit(lambda: ops.dtp_grad_x_raw(plan, gs, y, w), ops._dtp_bytes(plan, E, False, "grad_x"))
    rows["grad_y"] = timeit(lambda: ops.dtp_grad_y_raw(plan, xs, w, gs, y), ops._dtp_bytes(plan, E, False, "grad_y"))
    out = {"config": name, "E": E, "generated": bool(plan.generated), "peak_gbs": peak}
    for k, (us, gbs) in rows.items():
        out[k] = {"us": round(us, 1), "gb_s": round(gbs, 1), "frac": round(gbs / peak, 3)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
