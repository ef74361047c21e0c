"""CPU: what ``bench.py --dump-outputs`` writes - float32 / float64 files only, within the 64 MB budget also for the largest
model (OC20 l1_256: 9 123 331 parameters), and a seeded sample that a reader can recompute."""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def test_dump_of_the_largest_model_stays_within_budget(tmp_path):
    n = 9_123_331
    g = torch.Generator().manual_seed(0)
    grads, params = torch.randn(n, generator=g), torch.randn(n, generator=g)
    bench.dump_outputs(str(tmp_path), 0.25, grads, params)
    files = sorted(os.listdir(tmp_path))
    assert files == ["grads.npy", "loss.npy", "params.npy"]
    assert sum(os.path.getsize(tmp_path / f) for f in files) <= 64 << 20
    loss = np.load(tmp_path / "loss.npy")
    assert loss.dtype == np.float64 and loss.tolist() == [0.25]
    idx = bench.dump_sample(n)
    assert idx.numel() == bench.DUMP_MAX_ELEMENTS and bool((idx[1:] > idx[:-1]).all())
    for name, t in (("grads", grads), ("params", params)):
        a = np.load(tmp_path / f"{name}.npy")
        assert a.dtype == np.float32 and a.shape == (bench.DUMP_MAX_ELEMENTS,)
        assert np.array_equal(a, t[idx].numpy())


def test_small_arrays_are_dumped_whole(tmp_path):
    grads, params = torch.arange(10, dtype=torch.float32), -torch.arange(10, dtype=torch.float32)
    bench.dump_outputs(str(tmp_path), 1.0, grads, params)
    assert np.array_equal(np.load(tmp_path / "grads.npy"), grads.numpy())
    assert np.array_equal(np.load(tmp_path / "params.npy"), params.numpy())


def test_reference_arms_reject_dump_outputs(tmp_path):
    proc = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--dump-outputs",
                           str(tmp_path / "d")], capture_output=True, text=True, timeout=300)
    assert proc.returncode == 2 and "--dump-outputs" in proc.stderr
    assert not (tmp_path / "d").exists()
