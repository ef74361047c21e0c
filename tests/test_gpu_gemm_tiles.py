"""The forward / data-gradient wgmma GEMM with many tiles per persistent CTA: shallow reductions (one or two k-tiles per
tile, so the fragment double buffer crosses tile boundaries) with K tails, ragged column blocks, column-block counts that
do not divide the SM count, and a deep reduction."""
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K", [(50000, 96, 36), (40000, 200, 20), (70001, 352, 32), (30000, 960, 64), (30000, 544, 48),
                                   (20000, 64, 200)])
def test_tf32x3_gemm_tile_schedules(cuda_device, M, N, K):
    from equiformer_b200 import ops
    g = torch.Generator().manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g)
    Bt = torch.randn(N, K, generator=g)
    d = lambda t: t.to(cuda_device)
    out = ops.gemm_tf32x3_raw(d(A), d(Bt))
    assert out.shape == (M, N) and rel_err(out, A.double() @ Bt.double().t()) < 6e-6
    Ai = torch.randint(-8, 9, (M, K), generator=g).float()
    Bi = torch.randint(-8, 9, (N, K), generator=g).float()
    assert torch.equal(ops.gemm_tf32x3_raw(d(Ai), d(Bi)).cpu(), Ai @ Bi.t())
