"""CPU: host logic around the small-product kernel - dispatch thresholds, the column-split Function, the problem table that
``grouped_gemm_raw`` would hand to ``eqf_gemm_grouped`` (layout flags and leading dimensions), without launching anything."""
import ctypes

import torch

from equiformer_b200 import _lib, ops


def test_tcgen05_dispatch_thresholds(monkeypatch):
    monkeypatch.setattr(ops, "_GEMM_MIN_M", 16384)
    monkeypatch.setattr(ops, "_GEMM_MIN_FLOP", float("inf"))
    assert ops._use_tensor_cores(32560, 64, 128) and not ops._use_tensor_cores(11620, 32, 32)
    assert not ops._use_tensor_cores(14700, 32, 576)              # the MD17 edge-level products stay on the grouped kernel
    monkeypatch.setattr(ops, "_GEMM_MIN_FLOP", 4e8)
    assert ops._use_tensor_cores(14700, 32, 576) and not ops._use_tensor_cores(2324, 128, 128)
    assert not ops._use_tensor_cores(512, 4096, 4096)             # a flop-heavy product with too few rows for 128-row tiles
    monkeypatch.setattr(ops, "_GEMM_MIN_M", 1)               # smoke() / the tensor-core-forced parity tests
    assert ops._use_tensor_cores(7, 4, 4)


def test_split_columns_backward_is_one_concatenation():
    x = torch.randn(5, 12, dtype=torch.float64, requires_grad=True)

    def f(x):
        a, b, c = ops.split_columns(x, [4, 4, 4])
        return a * 2.0, c.sin()          # the middle block gets no gradient: the backward must fill it with zeros

    assert torch.autograd.gradcheck(f, (x,))
    assert torch.autograd.gradgradcheck(f, (x,))
    parts = ops.split_columns(x, [4, 8])
    assert all(p.is_contiguous() for p in parts) and torch.equal(torch.cat(parts, 1), x)


def test_problem_table_matches_the_c_struct():
    """``_lib.EqfGemmProblem`` mirrors ``EqfGemmProblem`` of include/eqf_b200.h: 3 pointers, 6 int64, 2 int32, float, pad."""
    assert ctypes.sizeof(_lib.EqfGemmProblem) == 3 * 8 + 6 * 8 + 4 * 4
    names = [f[0] for f in _lib.EqfGemmProblem._fields_]
    assert names == ["A", "B", "C", "M", "N", "K", "lda", "ldb", "ldc", "mode", "accumulate", "alpha", "pad"]
    header = (_lib.INCLUDE_DIR / "eqf_b200.h").read_text()
    body = header[header.index("typedef struct {\n  const float* A;"):header.index("} EqfGemmProblem;")]
    order = [tok.strip(" ;*") for line in body.splitlines()[1:] for tok in line.replace("const float*", "").replace("float*", "")
             .replace("int64_t", "").replace("int32_t", "").replace("float", "").split(",") if tok.strip(" ;*")]
    assert order == names
    assert f"#define EQF_GROUP_MAX {_lib.EQF_GROUP_MAX}" in header


def test_linear_spec_alignment_rules():
    ok = ops.LinearSpec([(0, 0, 0, 128, 128, 1.0), (1, 1, 16384, 64, 64, 0.5)], 16384 + 4096)
    assert ok.aligned()
    assert not ops.LinearSpec([(0, 0, 0, 128, 1, 1.0)], 128).aligned()                       # a 1-column head output
    assert not ops.LinearSpec([(0, 0, 0, 8, 8, 1.0), (1, 0, 64, 8, 8, 1.0)], 128).aligned()  # two paths into one output
    assert not ops.LinearSpec([(i, i, 64 * i, 8, 8, 1.0) for i in range(9)], 576).aligned()  # more paths than a launch takes
