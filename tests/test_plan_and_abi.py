"""CPU: the path tables the kernels consume (walked in numpy) equal the oracle's per-instruction einsum; the C-ABI
library loads and exports every symbol include/eqf_b200.h declares (no compute calls without a GPU)."""
import ctypes
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from equiformer_b200 import _lib
from oracle import e3nn_ref as e3
from oracle import equiformer_ref as R

CASES = [("128x0e+64x1e+32x2e", "1x0e+1x1e+1x2e"), ("128x0e+64x1e+64x2e+32x3e", "1x0e+1x1e+1x2e+1x3e"),
         ("256x0e+128x1e", "1x0e+1x1e"), ("12x0e+4x0o+4x1e+4x1o+4x2e+4x2o", "1x0e+1x1o+1x2e")]


@pytest.mark.parametrize("irreps,sh", CASES)
def test_plan_tables_reproduce_oracle_tensor_product(irreps, sh):
    from equiformer_b200 import ops
    from equiformer_b200.nets.graph_attention_transformer import DepthwiseTensorProduct
    dtp = DepthwiseTensorProduct(irreps, sh, irreps, internal_weights=False, bias=False)
    plan = dtp.tp.plan
    E = 6
    g = torch.Generator().manual_seed(0)
    x = torch.randn(E, dtp.irreps_in1.dim, generator=g, dtype=torch.float64)
    y = torch.randn(E, dtp.irreps_in2.dim, generator=g, dtype=torch.float64)
    w = torch.randn(E, plan.weight_numel, generator=g, dtype=torch.float64)
    xs = [t.numpy() for t in ops.to_planar(x, dtp.irreps_in1)]
    groups = plan.emulate_forward(xs, y.numpy(), w.numpy())
    out = ops.from_planar([torch.from_numpy(t) for t in groups])
    irr_out, ins = R.dtp_instructions(e3.parse_irreps(irreps), e3.parse_irreps(sh), e3.parse_irreps(irreps))
    ref = e3.tensor_product(x, y, w, e3.parse_irreps(irreps), e3.parse_irreps(sh), irr_out, ins, False)
    assert (out - ref).abs().max() < 1e-6 * ref.abs().max()   # cg table is stored in fp32 for the device
    assert plan.weight_numel == dtp.tp.weight_numel


def _generated_signatures():
    """tag -> the signature literal a committed ``csrc/gen/dtp_gen_<tag>.cu`` registers its kernels under."""
    from equiformer_b200 import codegen
    out = {}
    for tag, _irreps, _sh in codegen.KNOWN_CONFIGS:
        text = (codegen.GEN_DIR / f"dtp_gen_{tag}.cu").read_text()
        found = re.findall(r'GeneratedKernels kernels = \{0x([0-9a-f]{16})ULL, "([a-z0-9_]+)"', text)
        assert [t for _s, t in found] == [tag], (tag, found)
        out[tag] = int(found[0][0], 16)
    return out


def test_generated_kernel_signatures_match_the_shipped_plans():
    """The plan-specialised kernels run only when a plan's hash equals the literal in its generated file: every committed
    file matches its configuration, and the depth-wise products of the QM9 and MD17-L3 models (radial degree embedding,
    attention value) land on one of them - a drift would move the shipped models onto the generic kernels silently."""
    from equiformer_b200 import codegen
    from equiformer_b200.nets import model_entrypoint
    sigs = _generated_signatures()
    for tag, irreps, sh in codegen.KNOWN_CONFIGS:
        assert sigs[tag] == codegen.plan_signature(codegen.plan_for(irreps, sh)), tag
    for name, irreps_in, tag in (("graph_attention_transformer_nonlinear_l2", "5x0e", "qm9_l2"),
                                 ("graph_attention_transformer_nonlinear_exp_l3_md17", "64x0e", "md17_l3")):
        model = model_entrypoint(name)(irreps_in=irreps_in, radius=5.0, num_basis=128)
        plans = [model.edge_deg_embed.dw.tp.plan] + [blk.ga.sep_value.dtp.tp.plan for blk in model.blocks]
        for plan in plans:
            assert codegen.plan_signature(plan) == sigs[tag], (name, tag)


def _known_tags():
    from equiformer_b200 import codegen
    return [tag for tag, _irreps, _sh in codegen.KNOWN_CONFIGS]


@pytest.mark.parametrize("tag", _known_tags())
def test_committed_generated_file_is_what_the_generator_emits(tag):
    """``build()`` regenerates ``csrc/gen`` before it compiles: a committed file that the generator no longer emits
    byte for byte would be reviewed as one kernel and compiled as another."""
    from equiformer_b200 import codegen
    irreps, sh = next((i, s) for t, i, s in codegen.KNOWN_CONFIGS if t == tag)
    committed = (codegen.GEN_DIR / f"dtp_gen_{tag}.cu").read_text()
    assert codegen.generate(codegen.plan_for(irreps, sh), tag) == committed, tag


def test_plan_info_and_bytes(built_lib):
    from equiformer_b200.nets.graph_attention_transformer import DepthwiseTensorProduct
    irreps = "128x0e+64x1e+32x2e"
    plan = DepthwiseTensorProduct(irreps, "1x0e+1x1e+1x2e", irreps, internal_weights=False, bias=False).tp.plan
    info = plan.info()
    assert info["n_paths"] == 15 and info["m_size"] == 179 and info["n_wtasks"] == 30 and info["n_xtasks"] == 7
    assert info["weight_numel"] == 960 and info["smem_bytes"] < 48 * 1024
    assert plan.algorithmic_bytes()["forward"] == 18340          # SURVEY.md section 8d
    assert built_lib.eqf_plan_partial_rows(plan.handle, 36000) >= 1


def test_library_exports_every_declared_symbol(built_lib):
    header = (Path(_lib.INCLUDE_DIR) / "eqf_b200.h").read_text()
    declared = set(re.findall(r"\b(eqf_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    bound = set(_lib.SIGNATURES)
    assert declared == bound, declared ^ bound
    for name in _lib.SIGNATURES:
        assert hasattr(built_lib, name), name
    assert built_lib.eqf_version() == 100
    assert built_lib.eqf_last_error() is not None


def test_plan_create_rejects_bad_input(built_lib):
    h = ctypes.c_void_p()
    desc = (_lib.EqfPathDesc * 1)(_lib.EqfPathDesc(1, 1, 3, 8, 0, 0, 0, 0, 0, 0))   # (1,1,3) violates the triangle rule
    one = (ctypes.c_int32 * 1)
    cg = (ctypes.c_float * 64)()
    rc = built_lib.eqf_plan_create(desc, 1, one(1), one(8), 1, one(3), one(8), 1, 4, 8, cg, 64, ctypes.byref(h))
    assert rc < 0 and b"triangle" in built_lib.eqf_last_error()
    desc[0] = _lib.EqfPathDesc(4, 0, 4, 8, 0, 0, 0, 0, 0, 0)                       # l = 4 is not compiled in
    rc = built_lib.eqf_plan_create(desc, 1, one(4), one(8), 1, one(4), one(8), 1, 1, 8, cg, 64, ctypes.byref(h))
    assert rc == -3
