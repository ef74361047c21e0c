"""Hand-written wgmma 3xTF32 weight-gradient kernel vs cuBLAS on the layer shapes."""
import json, os, sys
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
    shapes = [("tiny", 100, 32, 32), ("small", 1000, 64, 48), ("val1_l0", E, 224, 224), ("alpha", E, 224, 128),
              ("fused_l0", E, 224, 352), ("val1_l1", 3 * E, 384, 64), ("val1_l2", 5 * E, 352, 32), ("val2_l1", 3 * E, 384, 64),
              ("rad_last", E, 64, 960), ("rad_first", E, 128, 64), ("node_l0", 2324, 128, 128), ("node_l2", 11620, 32, 32),
              ("ragged", 3001, 100, 72)]
    g = torch.Generator(device=dev).manual_seed(0)
    for name, R, K1, N in shapes:
        A = torch.randn(R, K1, device=dev, generator=g)
        G = torch.randn(R, N, device=dev, generator=g)
        ref = A.double().t() @ G.double()
        out = ops.gemm_tf32x3_wgrad_raw(A, G)
        torch.cuda.synchronize()
        err = ((out.double() - ref).abs().max() / ref.abs().max()).item()
        row = {"shape": name, "R": R, "K1": K1, "N": N, "rel_err": float(f"{err:.2e}")}
        print(json.dumps(row), flush=True)
        us = timeit(lambda: ops.gemm_tf32x3_wgrad_raw(A, G))
        us_t = timeit(lambda: A.t() @ G)
        row.update({"us": round(us, 1), "cublas_us": round(us_t, 1),
                    "gb_s": round(4 * (A.numel() + G.numel()) / us / 1e3, 1)})
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
