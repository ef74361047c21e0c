"""Shared helpers for the parity tests; the synthetic geometry generators live in ``equiformer_b200.synthetic``."""
from __future__ import annotations

import torch

from equiformer_b200.synthetic import aspirin_like, molecules, qm9_like_batch  # noqa: F401  (re-exported for the tests)


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def assert_same_grad_presence(name: str, got, ref) -> bool:
    """A parameter that one side trains and the other leaves without a gradient fails here instead of being skipped by
    the comparison that follows; an empty gradient counts as none.  Returns whether there is a gradient to compare."""
    has_got = got is not None and got.numel() > 0
    has_ref = ref is not None and ref.numel() > 0
    assert has_got == has_ref, f"{name}: {'the reference' if has_ref else 'the CUDA path'} trains it, the other does not"
    return has_got


def closed_form_tensor(name: str, shape, mean: float, std: float) -> torch.Tensor:
    """A float32 tensor that both the golden generator and the tests can rebuild from (name, shape, mean, std) alone -
    ``mean + std * sqrt(2) * sin(phase(name) + 0.618 i)`` over the flat index - so that full-size models need only two
    numbers per large tensor in a fixture (tests/golden/make_reference_golden.py, "headline" case)."""
    import zlib
    n = 1
    for d in shape:
        n *= int(d)
    phase = (zlib.crc32(name.encode()) % 10007) * 0.001
    i = torch.arange(n, dtype=torch.float64)
    return (mean + std * (2.0 ** 0.5) * torch.sin(phase + 0.6180339887 * i)).float().reshape(tuple(int(d) for d in shape))
