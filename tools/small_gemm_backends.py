"""Which kernel for a mid-size product?  The MD17 edge-level shapes (E = 2 100 edges x (2l+1) rows, DTP group channels ->
head / value channels) and a few node-level ones on three backends: wgmma 3xTF32 (eqf_gemm_tf32x3), the warp-MMA grouped
kernel (one problem), cuBLAS.  CUDA-graph timed."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from equiformer_b200 import ops  # noqa: E402
from tools.tf32x3_microbench import timeit  # noqa: E402


def main():
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator(device=dev).manual_seed(0)
    E = 2100
    shapes = [("md17 l0 fwd", E, 288, 128), ("md17 l1 fwd", 3 * E, 576, 64), ("md17 l2 fwd", 5 * E, 672, 64), ("md17 l3 fwd", 7 * E, 576, 32),
              ("md17 l2 dgrad", 5 * E, 64, 672), ("md17 rad last", E, 64, 2112), ("md17 rad last dgrad", E, 2112, 64),
              ("qm9 node l0", 2324, 128, 128), ("qm9 node l2", 11620, 32, 32), ("4k rows", 4096, 256, 128), ("8k rows", 8192, 256, 128)]
    for name, M, K, N in shapes:
        A = torch.randn(M, K, device=dev, generator=g)
        B = torch.randn(K, N, device=dev, generator=g)
        C = torch.empty(M, N, device=dev)
        row = {"shape": name, "M": M, "K": K, "N": N, "mflop": round(2 * M * K * N / 1e6, 1)}
        row["wgmma_us"] = round(timeit(lambda: ops.gemm_tf32x3_raw(A, B, b_is_kn=True)), 1)
        row["grouped_mma_us"] = round(timeit(lambda: ops.grouped_gemm_raw([(0, A, B, C, 1.0, False)])), 1)
        row["cublas_us"] = round(timeit(lambda: A @ B), 1)
        Bt = B.t().contiguous()
        row["wgmma_nt_us"] = round(timeit(lambda: ops.gemm_tf32x3_raw(A, Bt)), 1)
        G = torch.randn(M, N, device=dev, generator=g)
        W = torch.zeros(K, N, device=dev)
        row["wgrad_wgmma_us"] = round(timeit(lambda: ops.gemm_tf32x3_wgrad_raw(A, G)), 1)
        row["wgrad_grouped_mma_us"] = round(timeit(lambda: ops.grouped_gemm_raw([(2, A, G, W, 1.0, True)])), 1)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
