"""Hand-written wgmma 3xTF32 GEMM vs cuBLAS on the layer shapes (forward / dgrad)."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from equiformer_b200 import ops  # noqa: E402


def timeit(fn, iters=20):
    """GPU time per call: the calls are captured into a CUDA graph and replayed, so host launch overhead (tensor-map
    encodes, Python) is out of the measurement - as it is in the benchmark's graph-replayed step."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    g.replay()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / iters


def main():
    E = int(sys.argv[1]) if len(sys.argv) > 1 else 32560
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    shapes = [("tiny", 100, 32, 16), ("small", 1000, 64, 48), ("val1_l0", E, 224, 224), ("alpha", E, 224, 128),
              ("val1_l1", 3 * E, 384, 64), ("val1_l2", 5 * E, 352, 32), ("dgrad_l2", 5 * E, 32, 352), ("dgrad_l1", 3 * E, 64, 384),
              ("rad_last", E, 64, 960), ("rad_last_dgrad", E, 960, 64), ("rad_first", E, 128, 64), ("node_l0", 2324, 128, 128),
              ("ragged", 3001, 100, 72)]
    g = torch.Generator(device=dev).manual_seed(0)
    for name, M, K, N in shapes:
        A = torch.randn(M, K, device=dev, generator=g)
        Bt = torch.randn(N, K, device=dev, generator=g)
        ref = A.double() @ Bt.double().t()
        out = ops.gemm_tf32x3_raw(A, Bt)
        torch.cuda.synchronize()
        err = ((out.double() - ref).abs().max() / ref.abs().max()).item()
        row = {"shape": name, "M": M, "K": K, "N": N, "rel_err": float(f"{err:.2e}")}
        print(json.dumps(row), flush=True)
        us = timeit(lambda: ops.gemm_tf32x3_raw(A, Bt))
        us_t = timeit(lambda: A @ Bt.t())
        err_t = (((A @ Bt.t()).double() - ref).abs().max() / ref.abs().max()).item()
        nbytes = 4 * (A.numel() + Bt.numel() + out.numel())
        row.update({"us": round(us, 1), "cublas_us": round(us_t, 1), "cublas_err": float(f"{err_t:.2e}"),
                    "gb_s": round(nbytes / us / 1e3, 1), "tflops": round(2 * M * N * K / us / 1e6, 1)})
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
