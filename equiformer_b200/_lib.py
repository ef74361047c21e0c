"""ctypes binding of ``libeqf_b200.so`` (C ABI declared in ``include/eqf_b200.h``).

The shared library is built in-tree by :func:`build` (``nvcc -gencode arch=compute_90a,code=sm_90a``)
and loaded lazily.  There is deliberately **no fallback**: if the library is missing or a kernel entry
point fails, the call raises - the product path never routes through a CPU or eager-torch restatement
(the only CPU restatement lives in ``oracle/`` and is test infrastructure).
"""
from __future__ import annotations

import ctypes
import os
import shutil
import subprocess
import threading
from ctypes import POINTER, c_char_p, c_float, c_int32, c_int64, c_void_p
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC_DIR = PKG_DIR / "csrc"
INCLUDE_DIR = PKG_DIR.parent / "include"
LIB_PATH = PKG_DIR / "libeqf_b200.so"
SOURCES = ("eqf_abi.cu", "eqf_dtp.cu", "eqf_dtp_vec.cu", "eqf_dtp_v3.cu", "eqf_attn.cu", "eqf_pointwise.cu", "eqf_gemm_tf32x3.cu", "eqf_graph.cu",
           "eqf_fused.cu", "eqf_edge.cu", "eqf_gemm_small.cu")

EQF_COLSUM_COUNTERS = 16384
EQF_MAX_BLOCKS = 8
EQF_MAX_HEADS = 16

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17", "--shared", "-Xcompiler", "-fPIC",
]


class EqfPathDesc(ctypes.Structure):
    _fields_ = [
        ("l1", c_int32), ("l2", c_int32), ("l3", c_int32), ("mul", c_int32),
        ("in1_block", c_int32), ("in2_off", c_int32), ("out_group", c_int32),
        ("out_chan_off", c_int32), ("w_off", c_int32), ("cg_off", c_int32),
    ]


class EqfEdgeOperands(ctypes.Structure):
    _fields_ = [
        ("x", c_void_p * EQF_MAX_BLOCKS),
        ("x2", c_void_p * EQF_MAX_BLOCKS),
        ("src", c_void_p),
        ("dst", c_void_p),
        ("y", c_void_p),
        ("w", c_void_p),
        ("w_shared", c_int32),
        ("g", c_void_p * EQF_MAX_BLOCKS),
        ("w_offset", c_void_p),
    ]


class EqfGateLayout(ctypes.Structure):
    _fields_ = [
        ("n_gated", c_int32),
        ("d", c_int32 * EQF_MAX_BLOCKS),
        ("C", c_int32 * EQF_MAX_BLOCKS),
        ("n_alpha", c_int32), ("n_scalars", c_int32), ("n_heads", c_int32),
        ("c_silu", c_float), ("c_sigmoid", c_float), ("c_slr", c_float), ("slr_slope", c_float),
    ]


class EqfNormLayout(ctypes.Structure):
    _fields_ = [
        ("n_entries", c_int32),
        ("mul", c_int32 * EQF_MAX_BLOCKS),
        ("d", c_int32 * EQF_MAX_BLOCKS),
        ("is_scalar", c_int32 * EQF_MAX_BLOCKS),
        ("eps", c_float),
    ]


class EqfHeadLayout(ctypes.Structure):
    _fields_ = [
        ("n_groups", c_int32),
        ("d", c_int32 * EQF_MAX_BLOCKS),
        ("C", c_int32 * EQF_MAX_BLOCKS),
        ("n_heads", c_int32),
    ]


EQF_GROUP_MAX = 8


class EqfGemmProblem(ctypes.Structure):
    _fields_ = [
        ("A", c_void_p), ("B", c_void_p), ("C", c_void_p),
        ("M", c_int64), ("N", c_int64), ("K", c_int64), ("lda", c_int64), ("ldb", c_int64), ("ldc", c_int64),
        ("mode", c_int32), ("accumulate", c_int32), ("alpha", c_float), ("pad", c_int32),
    ]


PtrArray = c_void_p * EQF_MAX_BLOCKS

# name -> (restype, argtypes); every symbol include/eqf_b200.h declares
SIGNATURES = {
    "eqf_version": (c_int32, []),
    "eqf_last_error": (c_char_p, []),
    "eqf_device_sm_count": (c_int32, []),
    "eqf_plan_create": (c_int32, [POINTER(EqfPathDesc), c_int32, POINTER(c_int32), POINTER(c_int32), c_int32,
                                  POINTER(c_int32), POINTER(c_int32), c_int32, c_int32, c_int32,
                                  POINTER(c_float), c_int32, POINTER(c_void_p)]),
    "eqf_plan_destroy": (None, [c_void_p]),
    "eqf_plan_info": (c_int32, [c_void_p, POINTER(c_int32), c_int32]),
    "eqf_plan_partial_rows": (c_int32, [c_void_p, c_int64]),
    "eqf_dtp_forward": (c_int32, [c_void_p, POINTER(EqfEdgeOperands), c_int64, POINTER(c_void_p), c_void_p]),
    "eqf_dtp_grad_x": (c_int32, [c_void_p, POINTER(EqfEdgeOperands), c_int64, POINTER(c_void_p), c_void_p]),
    "eqf_dtp_grad_w": (c_int32, [c_void_p, POINTER(EqfEdgeOperands), c_int64, c_void_p, c_void_p]),
    "eqf_dtp_grad_y": (c_int32, [c_void_p, POINTER(EqfEdgeOperands), c_int64, c_void_p, c_void_p]),
    "eqf_dtp_grad_xw": (c_int32, [c_void_p, POINTER(EqfEdgeOperands), c_int64, POINTER(c_void_p), c_void_p, c_void_p]),
    "eqf_seg_softmax": (c_int32, [c_void_p, c_void_p, c_int64, c_int32, c_void_p, c_void_p]),
    "eqf_seg_softmax_bwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_void_p, c_void_p]),
    "eqf_attn_aggregate": (c_int32, [POINTER(EqfHeadLayout), c_void_p, POINTER(c_void_p), c_void_p, c_void_p, c_int64,
                                     POINTER(c_void_p), c_void_p]),
    "eqf_attn_softmax_aggregate": (c_int32, [POINTER(EqfHeadLayout), c_void_p, POINTER(c_void_p), c_void_p, c_int64,
                                             POINTER(c_void_p), c_void_p, c_void_p]),
    "eqf_attn_edge_dot": (c_int32, [POINTER(EqfHeadLayout), POINTER(c_void_p), POINTER(c_void_p), c_void_p, c_int64,
                                    c_void_p, c_void_p]),
    "eqf_attn_edge_scale": (c_int32, [POINTER(EqfHeadLayout), c_void_p, POINTER(c_void_p), c_void_p, c_int64,
                                      POINTER(c_void_p), c_void_p]),
    "eqf_pointwise_rows": (c_int32, [c_int64]),
    "eqf_ln_silu_fwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int64, c_int32, c_void_p, c_void_p,
                                  c_void_p, c_void_p]),
    "eqf_ln_silu_bwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32,
                                  c_void_p, c_void_p, c_void_p]),
    "eqf_gemm_tf32x3": (c_int32, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_int32,
                                  c_void_p, c_void_p]),
    "eqf_gemm_tf32x3_wgrad_slices": (c_int64, [c_int64, c_int64, c_int64]),
    "eqf_gemm_tf32x3_wgrad": (c_int32, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p]),
    "eqf_gemm_tf32x3_wgrad_accumulate": (c_int32, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64,
                                                   c_void_p]),
    "eqf_dtp_linear_supported": (c_int32, [c_void_p, c_int32]),
    "eqf_fused_set_timeline": (None, [c_void_p]),
    "eqf_dtp_group_forward": (c_int32, [c_void_p, POINTER(EqfEdgeOperands), c_int64, c_int32, c_void_p, c_void_p]),
    "eqf_dtp_linear_fwd": (c_int32, [c_void_p, POINTER(EqfEdgeOperands), c_int64, c_int32, c_void_p, c_int64, c_int64, c_void_p,
                                     c_int64, c_void_p, c_void_p]),
    "eqf_radius_graph_count": (c_int32, [c_void_p, c_void_p, c_int64, c_float, c_int32, c_int64, c_void_p, c_void_p]),
    "eqf_radius_graph_fill": (c_int32, [c_void_p, c_void_p, c_int64, c_float, c_int32, c_int64, c_void_p, c_void_p, c_void_p,
                                        c_void_p]),
    "eqf_radius_graph_pbc_count": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_float, c_int32, c_int32, c_int32,
                                             c_void_p, c_void_p]),
    "eqf_radius_graph_pbc_fill": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_float, c_int32, c_int32, c_int32,
                                            c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "eqf_edge_geom_fwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_void_p,
                                    c_void_p, c_void_p, c_void_p]),
    "eqf_edge_geom_bwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "eqf_expnorm_fwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_float, c_float, c_int64, c_int32, c_void_p, c_void_p]),
    "eqf_expnorm_bwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_float, c_float, c_int64, c_int32, c_void_p, c_void_p, c_void_p]),
    "eqf_rbf_fwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int64, c_void_p, c_void_p]),
    "eqf_rbf_bwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_int64, c_void_p, c_void_p,
                              c_void_p]),
    "eqf_colsum_scratch_floats": (c_int64, [c_int64, c_int64]),
    "eqf_colsum": (c_int32, [c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "eqf_gemm_grouped": (c_int32, [ctypes.POINTER(EqfGemmProblem), c_int32, c_void_p]),
    "eqf_eln_rows": (c_int32, [POINTER(EqfNormLayout), c_int64]),
    "eqf_eln_fwd": (c_int32, [POINTER(EqfNormLayout), c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "eqf_eln_bwd": (c_int32, [POINTER(EqfNormLayout), c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p,
                              c_void_p]),
    "eqf_eln_fwd_planar": (c_int32, [POINTER(EqfNormLayout), c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "eqf_eln_bwd_planar": (c_int32, [POINTER(EqfNormLayout), c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p,
                                     c_void_p]),
    "eqf_gate_logits_fwd": (c_int32, [POINTER(EqfGateLayout), c_void_p, c_void_p, POINTER(c_void_p), c_void_p, c_int64,
                                      c_void_p, c_void_p, POINTER(c_void_p), c_void_p]),
    "eqf_gate_logits_bwd": (c_int32, [POINTER(EqfGateLayout), c_void_p, c_void_p, POINTER(c_void_p), c_void_p, c_void_p,
                                      c_void_p, POINTER(c_void_p), c_int64, c_void_p, POINTER(c_void_p), c_void_p,
                                      c_void_p]),
}


class EqfError(RuntimeError):
    pass


_lock = threading.Lock()
_lib = None


def sources():
    gen = sorted((CSRC_DIR / "gen").glob("dtp_gen_*.cu")) if (CSRC_DIR / "gen").exists() else []
    return [CSRC_DIR / s for s in SOURCES if (CSRC_DIR / s).exists()] + gen


def generate_sources():
    """Emit the plan-specialised kernels for the registered model configurations (csrc/gen/*.cu)."""
    from . import codegen
    return codegen.write_all()


def needs_build() -> bool:
    if not LIB_PATH.exists():
        return True
    mtime = LIB_PATH.stat().st_mtime
    deps = sources() + list(CSRC_DIR.glob("*.cuh")) + [INCLUDE_DIR / "eqf_b200.h"]
    return any(p.stat().st_mtime > mtime for p in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile ``csrc/*.cu`` for sm_90a into ``equiformer_b200/libeqf_b200.so`` (in-tree)."""
    generate_sources()
    if not force and not needs_build():
        return LIB_PATH
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise EqfError("nvcc not found: cannot build libeqf_b200.so")
    # one nvcc per source file, in parallel (the plan-specialised files take a minute each), then one
    # link step; objects live in a scratch directory next to the library
    from concurrent.futures import ThreadPoolExecutor
    obj_dir = PKG_DIR / "build" / ("obj%d" % os.getpid())
    obj_dir.mkdir(parents=True, exist_ok=True)
    compile_flags = [f for f in NVCC_FLAGS if f != "--shared"]

    def compile_one(src: Path):
        obj = obj_dir / (src.stem + ".o")
        cmd = [nvcc, *compile_flags, "-I", str(INCLUDE_DIR), "-c", "-o", str(obj), str(src)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        return obj, subprocess.run(cmd, capture_output=True, text=True)

    try:
        with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as pool:
            results = list(pool.map(compile_one, sources()))
        for _obj, proc in results:
            if proc.returncode != 0:
                raise EqfError("nvcc failed:\n" + proc.stdout + proc.stderr)
            if verbose:
                print(proc.stderr)
        tmp = LIB_PATH.with_suffix(".so.tmp%d" % os.getpid())
        link = subprocess.run([nvcc, "--shared", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a",
                               "-o", str(tmp), *[str(o) for o, _ in results]], capture_output=True, text=True)
        if link.returncode != 0:
            raise EqfError("nvcc link failed:\n" + link.stdout + link.stderr)
        os.replace(tmp, LIB_PATH)
    finally:
        shutil.rmtree(obj_dir, ignore_errors=True)
    return LIB_PATH


def load():
    """Return the loaded library (raises :class:`EqfError` when it is absent - no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not LIB_PATH.exists():
            raise EqfError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(the sm_90a kernels are the only implementation of the edge path)")
        lib = ctypes.CDLL(str(LIB_PATH))
        for name, (restype, argtypes) in SIGNATURES.items():
            try:
                fn = getattr(lib, name)
            except AttributeError as exc:  # stale build
                raise EqfError(f"libeqf_b200.so does not export {name}; rebuild it") from exc
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().eqf_last_error()
        raise EqfError(f"{what} failed (code {rc}): {msg.decode() if msg else '?'}")
