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
from ctypes import POINTER, c_char_p, c_double, c_float, c_int32, c_int64, c_void_p
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC_DIR = PKG_DIR / "csrc"
INCLUDE_DIR = PKG_DIR.parent / "include"
LIB_PATH = PKG_DIR / "libeqf_b200.so"
# depth-wise plans with an in1 / output degree of 4: the plan and table-walk DTP sources built once more with
# -DEQF_MAX_DEGREE=4, so that the degree-4 branches stay out of the kernels of the main library
L4_LIB_PATH = PKG_DIR / "libeqf_b200_l4.so"
L4_SOURCES = ("eqf_abi.cu", "eqf_dtp.cu", "eqf_dtp_vec.cu")
# the per-graph equivariant norms (EquivariantGraphNorm / EquivariantInstanceNorm): their own library and header
# (include/eqf_b200_norm.h), bound by load_norm()
NORM_LIB_PATH = PKG_DIR / "libeqf_b200_norm.so"
NORM_SOURCES = ("eqf_norm.cu",)
EQF_NORM_MAX_ENTRIES = 8      # include/eqf_b200_norm.h: irreps entries per norm layout
# gradient clipping, AdamW and the model EMA on the flat parameter buffers: their own library and header
# (include/eqf_b200_optim.h), bound by load_optim()
OPTIM_LIB_PATH = PKG_DIR / "libeqf_b200_optim.so"
OPTIM_SOURCES = ("eqf_optim.cu",)
EQF_OPTIM_THREADS = 256       # include/eqf_b200_optim.h: threads per CTA, 4 elements each per pass
EQF_OPTIM_MAX_CTAS = 1024     # include/eqf_b200_optim.h: grid cap (and length of the partial-sum scratch)
EQF_LR_MAX_MILESTONES = 8     # include/eqf_b200_optim.h: milestones of a multistep schedule
EQF_LR_KINDS = {"oc20_cosine": 1, "oc20_multistep": 2, "timm_cosine": 3}   # EQF_LR_* of include/eqf_b200_optim.h
# the metric terms of the evaluation passes (evaluation.EvalPass): their own library and header (include/eqf_b200_eval.h),
# bound by load_eval()
EVAL_LIB_PATH = PKG_DIR / "libeqf_b200_eval.so"
EVAL_SOURCES = ("eqf_eval.cu",)
EQF_EVAL_THREADS = 256        # include/eqf_b200_eval.h: threads per CTA, one row each per pass
EQF_EVAL_MAX_CTAS = 128       # include/eqf_b200_eval.h: grid cap
EQF_EVAL_SCRATCH = 512        # include/eqf_b200_eval.h: doubles of the partials scratch
EQF_EVAL_GRAPH_SLOTS = 5      # include/eqf_b200_eval.h: accumulator slots of eqf_eval_graph / _atom / _batch
EQF_EVAL_ATOM_SLOTS = 3
EQF_EVAL_BATCH_SLOTS = 2
# the de-normalised OC20 predictions of a predict pass (evaluation.EvalPass.predict): their own library and header
# (include/eqf_b200_predict.h), bound by load_predict()
PREDICT_LIB_PATH = PKG_DIR / "libeqf_b200_predict.so"
PREDICT_SOURCES = ("eqf_predict.cu",)
EQF_PREDICT_THREADS = 256     # include/eqf_b200_predict.h: threads per CTA, one row each per pass
EQF_PREDICT_MAX_CTAS = 128    # include/eqf_b200_predict.h: grid cap
SOURCES = ("eqf_abi.cu", "eqf_dtp.cu", "eqf_dtp_vec.cu", "eqf_attn.cu", "eqf_pointwise.cu", "eqf_gemm_tf32x3.cu", "eqf_graph.cu",
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


class EqfSegNormLayout(ctypes.Structure):
    _fields_ = [
        ("n_entries", c_int32),
        ("mul", c_int32 * EQF_NORM_MAX_ENTRIES),
        ("d", c_int32 * EQF_NORM_MAX_ENTRIES),
        ("is_scalar", c_int32 * EQF_NORM_MAX_ENTRIES),
        ("w_off", c_int32 * EQF_NORM_MAX_ENTRIES),
        ("s_off", c_int32 * EQF_NORM_MAX_ENTRIES),
        ("n_w", c_int32), ("n_s", c_int32), ("component", c_int32),
        ("eps", c_float),
    ]


class EqfHeadLayout(ctypes.Structure):
    _fields_ = [
        ("n_groups", c_int32),
        ("d", c_int32 * EQF_MAX_BLOCKS),
        ("C", c_int32 * EQF_MAX_BLOCKS),
        ("n_heads", c_int32),
    ]


class EqfLrSchedule(ctypes.Structure):
    _fields_ = [
        ("kind", c_int32), ("n_milestones", c_int32), ("steps_per_unit", c_int64),
        ("base_lr", c_double), ("warmup", c_double), ("warmup_start", c_double), ("total", c_double),
        ("min_value", c_double), ("gamma", c_double), ("milestones", c_double * EQF_LR_MAX_MILESTONES),
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
    "eqf_seg_softmax_bwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_void_p, c_void_p]),
    "eqf_attn_aggregate": (c_int32, [POINTER(EqfHeadLayout), c_void_p, POINTER(c_void_p), c_void_p, c_void_p, c_int64,
                                     POINTER(c_void_p), c_void_p]),
    "eqf_attn_softmax_aggregate": (c_int32, [POINTER(EqfHeadLayout), c_void_p, c_void_p, POINTER(c_void_p), c_void_p,
                                             c_int64, POINTER(c_void_p), c_void_p, c_void_p]),
    "eqf_attn_dot_softmax_aggregate": (c_int32, [POINTER(EqfHeadLayout), POINTER(c_void_p), POINTER(c_void_p), c_void_p,
                                                 c_void_p, c_int64, POINTER(c_void_p), c_void_p, c_void_p]),
    "eqf_attn_dot_softmax_aggregate_bwd": (c_int32, [POINTER(EqfHeadLayout), POINTER(c_void_p), POINTER(c_void_p),
                                                     POINTER(c_void_p), c_void_p, c_void_p, c_void_p, c_int64,
                                                     POINTER(c_void_p), POINTER(c_void_p), c_void_p, c_void_p]),
    "eqf_attn_mlp_rows": (c_int32, [c_int64]),
    "eqf_attn_mlp_softmax_aggregate": (c_int32, [POINTER(EqfHeadLayout), c_int32, c_float, c_float, c_void_p,
                                                 POINTER(c_void_p), c_void_p, c_void_p, c_void_p, c_int64,
                                                 POINTER(c_void_p), c_void_p, c_void_p]),
    "eqf_attn_mlp_softmax_aggregate_bwd": (c_int32, [POINTER(EqfHeadLayout), c_int32, c_float, c_float, POINTER(c_void_p),
                                                     c_void_p, POINTER(c_void_p), c_void_p, c_void_p, c_void_p, c_void_p,
                                                     c_int64, c_void_p, POINTER(c_void_p), c_void_p, c_void_p, c_void_p]),
    "eqf_attn_edge_dot": (c_int32, [POINTER(EqfHeadLayout), POINTER(c_void_p), POINTER(c_void_p), c_void_p, c_int64,
                                    c_void_p, c_void_p]),
    "eqf_attn_edge_scale": (c_int32, [POINTER(EqfHeadLayout), c_void_p, c_void_p, POINTER(c_void_p), c_void_p, c_int64,
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
    "eqf_edge_geom_fwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32,
                                    c_void_p, c_void_p, c_void_p, c_void_p]),
    "eqf_edge_geom_bwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_void_p,
                                    c_void_p]),
    "eqf_expnorm_fwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_float, c_float, c_int64, c_int32, c_void_p, c_void_p]),
    "eqf_expnorm_bwd": (c_int32, [c_void_p, c_void_p, c_void_p, c_float, c_float, c_int64, c_int32, c_void_p, c_void_p, c_void_p]),
    "eqf_bessel_fwd": (c_int32, [c_void_p, c_void_p, c_float, c_int64, c_int32, c_void_p, c_void_p]),
    "eqf_bessel_bwd": (c_int32, [c_void_p, c_void_p, c_float, c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_void_p]),
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

# every symbol include/eqf_b200_norm.h declares
NORM_SIGNATURES = {
    "eqf_last_error": (c_char_p, []),
    "eqf_norm_graph_ptr": (c_int32, [c_void_p, c_int64, c_int64, c_void_p, c_void_p]),
    "eqf_norm_fwd": (c_int32, [POINTER(EqfSegNormLayout), POINTER(c_void_p), c_void_p, c_int64, c_void_p, c_void_p,
                               c_void_p, POINTER(c_void_p), c_void_p, c_void_p, c_void_p]),
    "eqf_norm_bwd": (c_int32, [POINTER(EqfSegNormLayout), POINTER(c_void_p), POINTER(c_void_p), c_void_p, c_int64,
                               c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_void_p), c_void_p, c_void_p]),
    "eqf_norm_param_reduce": (c_int32, [c_void_p, c_int64, c_int32, c_void_p, c_void_p]),
}

# every symbol include/eqf_b200_optim.h declares
OPTIM_SIGNATURES = {
    "eqf_last_error": (c_char_p, []),
    "eqf_flat_sqnorm": (c_int32, [c_void_p, c_int64, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "eqf_flat_adamw": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p,
                                 c_void_p, c_double, c_double, c_float, c_double, c_void_p, c_void_p]),
    "eqf_flat_sqnorm_check": (c_int32, [c_void_p, c_int64, c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "eqf_flat_adamw_check": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p,
                                       c_void_p, c_void_p, c_double, c_double, c_void_p]),
    "eqf_lr_schedule_check": (c_int32, [POINTER(EqfLrSchedule)]),
    "eqf_lr_at": (c_int32, [POINTER(EqfLrSchedule), c_int64, POINTER(c_double)]),
    "eqf_flat_adamw_scheduled": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p,
                                           c_void_p, c_void_p, c_double, c_double, c_float, c_double, c_void_p,
                                           POINTER(EqfLrSchedule), c_void_p]),
}

# every symbol include/eqf_b200_eval.h declares
EVAL_SIGNATURES = {
    "eqf_last_error": (c_char_p, []),
    "eqf_eval_graph": (c_int32, [c_void_p, c_void_p, c_int64, c_float, c_float, c_float, c_void_p, c_void_p, c_void_p,
                                 c_void_p]),
    "eqf_eval_atom": (c_int32, [c_void_p, c_void_p, c_int64, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "eqf_eval_batch": (c_int32, [c_void_p, c_void_p, c_void_p]),
    "eqf_eval_graph_check": (c_int32, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "eqf_eval_atom_check": (c_int32, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "eqf_eval_batch_check": (c_int32, [c_void_p, c_void_p]),
}

# every symbol include/eqf_b200_predict.h declares
PREDICT_SIGNATURES = {
    "eqf_last_error": (c_char_p, []),
    "eqf_predict_is2re": (c_int32, [c_void_p, c_int64, c_float, c_float, c_void_p, c_void_p, c_void_p, c_int64, c_float,
                                    c_void_p, c_void_p, c_void_p]),
    "eqf_predict_is2re_check": (c_int32, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p]),
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
    libs = (LIB_PATH, L4_LIB_PATH, NORM_LIB_PATH, OPTIM_LIB_PATH, EVAL_LIB_PATH, PREDICT_LIB_PATH)
    if not all(p.exists() for p in libs):
        return True
    mtime = min(p.stat().st_mtime for p in libs)
    deps = (sources() + [CSRC_DIR / s for s in NORM_SOURCES + OPTIM_SOURCES + EVAL_SOURCES + PREDICT_SOURCES]
            + list(CSRC_DIR.glob("*.cuh"))
            + [INCLUDE_DIR / "eqf_b200.h", INCLUDE_DIR / "eqf_b200_norm.h", INCLUDE_DIR / "eqf_b200_optim.h",
               INCLUDE_DIR / "eqf_b200_eval.h", INCLUDE_DIR / "eqf_b200_predict.h"])
    return any(p.stat().st_mtime > mtime for p in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile ``csrc/*.cu`` for sm_90a into ``equiformer_b200/libeqf_b200.so``, ``L4_SOURCES`` with
    ``-DEQF_MAX_DEGREE=4`` into ``equiformer_b200/libeqf_b200_l4.so``, ``NORM_SOURCES`` into
    ``equiformer_b200/libeqf_b200_norm.so``, ``OPTIM_SOURCES`` into ``equiformer_b200/libeqf_b200_optim.so``,
    ``EVAL_SOURCES`` into ``equiformer_b200/libeqf_b200_eval.so`` and ``PREDICT_SOURCES`` into
    ``equiformer_b200/libeqf_b200_predict.so`` (in-tree)."""
    generate_sources()
    if not force and not needs_build():
        return LIB_PATH
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise EqfError("nvcc not found: cannot build libeqf_b200.so")
    # one nvcc per source file, in parallel (the plan-specialised files take a minute each), then one
    # link step per library; objects live in a scratch directory next to the libraries
    from concurrent.futures import ThreadPoolExecutor
    obj_dir = PKG_DIR / "build" / ("obj%d" % os.getpid())
    obj_dir.mkdir(parents=True, exist_ok=True)
    compile_flags = [f for f in NVCC_FLAGS if f != "--shared"]
    jobs = ([(src, "", []) for src in sources()] + [(CSRC_DIR / s, "_l4", ["-DEQF_MAX_DEGREE=4"]) for s in L4_SOURCES]
            + [(CSRC_DIR / s, "_norm", []) for s in NORM_SOURCES] + [(CSRC_DIR / s, "_optim", []) for s in OPTIM_SOURCES]
            + [(CSRC_DIR / s, "_eval", []) for s in EVAL_SOURCES] + [(CSRC_DIR / s, "_predict", []) for s in PREDICT_SOURCES])

    def compile_one(job):
        src, suffix, defines = job
        obj = obj_dir / (src.stem + suffix + ".o")
        cmd = [nvcc, *compile_flags, *defines, "-I", str(INCLUDE_DIR), "-c", "-o", str(obj), str(src)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        return obj, suffix, subprocess.run(cmd, capture_output=True, text=True)

    def link(path: Path, objs):
        tmp = path.with_suffix(".so.tmp%d" % os.getpid())
        proc = subprocess.run([nvcc, "--shared", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a",
                               "-o", str(tmp), *[str(o) for o in objs]], capture_output=True, text=True)
        if proc.returncode != 0:
            raise EqfError("nvcc link failed:\n" + proc.stdout + proc.stderr)
        os.replace(tmp, path)

    try:
        with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as pool:
            results = list(pool.map(compile_one, jobs))
        for _obj, _suffix, proc in results:
            if proc.returncode != 0:
                raise EqfError("nvcc failed:\n" + proc.stdout + proc.stderr)
            if verbose:
                print(proc.stderr)
        link(LIB_PATH, [o for o, suffix, _ in results if suffix == ""])
        link(L4_LIB_PATH, [o for o, suffix, _ in results if suffix == "_l4"])
        link(NORM_LIB_PATH, [o for o, suffix, _ in results if suffix == "_norm"])
        link(OPTIM_LIB_PATH, [o for o, suffix, _ in results if suffix == "_optim"])
        link(EVAL_LIB_PATH, [o for o, suffix, _ in results if suffix == "_eval"])
        link(PREDICT_LIB_PATH, [o for o, suffix, _ in results if suffix == "_predict"])
    finally:
        shutil.rmtree(obj_dir, ignore_errors=True)
    return LIB_PATH


def _open(path: Path, required: bool):
    if not path.exists():
        raise EqfError(
            f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(the sm_90a kernels are the only implementation of the edge path)")
    lib = ctypes.CDLL(str(path))
    for name, (restype, argtypes) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as exc:  # stale build (the degree-4 library exports the plan and DTP entry points only)
            if required:
                raise EqfError(f"{path.name} does not export {name}; rebuild it") from exc
            continue
        fn.restype = restype
        fn.argtypes = argtypes
    return lib


_lib_l4 = None


def load_l4():
    """Return the loaded degree-4 library (plan creation and the table-walk DTP kernels with in1 / output degree <= 4)."""
    global _lib_l4
    with _lock:
        if _lib_l4 is None:
            lib = _open(L4_LIB_PATH, required=False)
            if not hasattr(lib, "eqf_dtp_forward"):
                raise EqfError(f"{L4_LIB_PATH.name} does not export eqf_dtp_forward; rebuild it")
            _lib_l4 = lib
    return _lib_l4


_side_libs = {}


def _load_side(path: Path, signatures: dict):
    """Load a library of its own (every symbol of ``signatures`` required), once."""
    with _lock:
        if path not in _side_libs:
            if not path.exists():
                raise EqfError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
            lib = ctypes.CDLL(str(path))
            for name, (restype, argtypes) in signatures.items():
                try:
                    fn = getattr(lib, name)
                except AttributeError as exc:
                    raise EqfError(f"{path.name} does not export {name}; rebuild it") from exc
                fn.restype, fn.argtypes = restype, argtypes
            _side_libs[path] = lib
    return _side_libs[path]


def load_norm():
    """Return the loaded norm library (``include/eqf_b200_norm.h``)."""
    return _load_side(NORM_LIB_PATH, NORM_SIGNATURES)


def load_optim():
    """Return the loaded optimiser library (``include/eqf_b200_optim.h``)."""
    return _load_side(OPTIM_LIB_PATH, OPTIM_SIGNATURES)


def load_eval():
    """Return the loaded evaluation-metric library (``include/eqf_b200_eval.h``)."""
    return _load_side(EVAL_LIB_PATH, EVAL_SIGNATURES)


def load_predict():
    """Return the loaded prediction library (``include/eqf_b200_predict.h``)."""
    return _load_side(PREDICT_LIB_PATH, PREDICT_SIGNATURES)


def load():
    """Return the loaded library (raises :class:`EqfError` when it is absent - no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        _lib = _open(LIB_PATH, required=True)
    return _lib


def check(rc: int, what: str, lib=None) -> None:
    """Raise with the library's last error message when ``rc`` is not ``EQF_OK`` (``lib``: the library that returned it,
    default the main one)."""
    if rc != 0:
        msg = (lib if lib is not None else load()).eqf_last_error()
        raise EqfError(f"{what} failed (code {rc}): {msg.decode() if msg else '?'}")
