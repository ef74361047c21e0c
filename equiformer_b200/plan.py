"""Host-side construction of the DTP path tables consumed by ``eqf_plan_create``.

Everything the edge kernels need is fixed when the reference builds its modules
(``DepthwiseTensorProduct``, ``nets/graph_attention_transformer.py:157-183``; instruction
normalisation in ``TensorProductRescale.__init__``, ``nets/tensor_product_rescale.py:33-37``):
the Clebsch-Gordan paths, where each path reads its weights (instruction order) and where it
writes its output (sorted order).  This module turns ``(irreps_in1, irreps_in2, irreps_out,
instructions)`` into that table once, on the host.

Planar layout: an irreps row ``[mul x (2l+1)]*`` is stored per *block* as ``[rows, 2l+1, mul]``.
Inputs are split per ``irreps_in1`` entry; outputs per *group* = maximal run of equal irreps in
``irreps_out`` (i.e. the entries of ``irreps_out.simplify()``), because that is exactly the input
of the per-degree linear that follows (``SeparableFCTP.lin``, ``:215``).
"""
from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass
from typing import List, Sequence, Tuple

import numpy as np

from . import _lib
from .o3.irreps import Irreps
from .o3.wigner import wigner_3j_np


@dataclass(frozen=True)
class Path:
    l1: int
    l2: int
    l3: int
    mul: int
    in1_block: int
    in2_off: int
    out_group: int
    out_chan_off: int
    w_off: int
    cg_off: int
    i_out: int          # index of the irreps_out entry (for e3nn-layout conversion)


class DtpPlan:
    """Path table of one depth-wise ('uvu') tensor product + lazily created native handle."""

    def __init__(self, irreps_in1, irreps_in2, irreps_out, instructions: Sequence[tuple]):
        self.irreps_in1 = Irreps(irreps_in1)
        self.irreps_in2 = Irreps(irreps_in2)
        self.irreps_out = Irreps(irreps_out)
        if any(mul != 1 for mul, _ in self.irreps_in2):
            raise NotImplementedError("depth-wise kernels need multiplicity-1 edge irreps (spherical harmonics)")
        if len(self.irreps_in1) > _lib.EQF_MAX_BLOCKS:
            raise NotImplementedError("too many in1 irrep blocks for the edge kernels")

        in2_offs = [s.start for s in self.irreps_in2.slices()]
        # output groups = runs of equal irreps
        self.group_of_entry: List[int] = []
        self.chan_off_of_entry: List[int] = []
        groups: List[List] = []  # [ir, mul_total]
        for mul, ir in self.irreps_out:
            if groups and groups[-1][0] == ir:
                self.group_of_entry.append(len(groups) - 1)
                self.chan_off_of_entry.append(groups[-1][1])
                groups[-1][1] += mul
            else:
                self.group_of_entry.append(len(groups))
                self.chan_off_of_entry.append(0)
                groups.append([ir, mul])
        if len(groups) > _lib.EQF_MAX_BLOCKS:
            raise NotImplementedError("too many output groups for the edge kernels")
        self.out_groups: List[Tuple[int, int, int]] = [(ir.l, ir.p, mul) for ir, mul in groups]
        self.irreps_out_grouped = Irreps([(mul, (l, p)) for l, p, mul in self.out_groups])
        self.in1_blocks: List[Tuple[int, int]] = [(ir.l, mul) for mul, ir in self.irreps_in1]

        paths: List[Path] = []
        cg_chunks: List[np.ndarray] = []
        cg_off = 0
        w_off = 0
        written = set()
        for ins in instructions:
            i1, i2, io, mode, has_weight = ins[0], ins[1], ins[2], ins[3], ins[4]
            extra_pw = float(ins[5]) if len(ins) > 5 else 1.0
            if mode != "uvu" or not has_weight:
                raise NotImplementedError("edge kernels implement weighted 'uvu' instructions only")
            mul1, ir1 = self.irreps_in1[i1]
            _, ir2 = self.irreps_in2[i2]
            mul3, ir3 = self.irreps_out[io]
            if mul3 != mul1:
                raise ValueError("'uvu' instruction with mismatching multiplicities")
            if ir3 not in ir1 * ir2:
                raise ValueError(f"instruction {ins} violates the selection rule")
            if io in written:
                raise NotImplementedError("several instructions writing one output block are not supported")
            written.add(io)
            # e3nn: irrep_normalization='component' -> alpha = ir_out.dim; path_normalization='none'
            path_weight = math.sqrt(ir3.dim * extra_pw)
            c = wigner_3j_np(ir1.l, ir2.l, ir3.l) * path_weight
            cg_chunks.append(c.reshape(-1))
            paths.append(Path(ir1.l, ir2.l, ir3.l, mul1, i1, in2_offs[i2], self.group_of_entry[io],
                              self.chan_off_of_entry[io], w_off, cg_off, io))
            cg_off += c.size
            w_off += mul1
        if len(written) != len(self.irreps_out):
            raise NotImplementedError("every output block must be produced by exactly one instruction")
        self.paths = paths
        self.weight_numel = w_off
        self.cg = np.concatenate(cg_chunks).astype(np.float32)
        self.cg64 = np.concatenate(cg_chunks)
        self.d_y = self.irreps_in2.dim
        # in1 / output degree 4 runs on libeqf_b200_l4.so (the table-walk kernels built with the degree-4 branches)
        self.max_degree = max([l for l, _ in self.in1_blocks] + [l for l, _, _ in self.out_groups])
        self._handle = None

    # ------------------------------------------------------------------ native handle
    @property
    def lib(self):
        """The library whose kernels run this plan (its handle belongs to that library)."""
        return _lib.load_l4() if self.max_degree > 3 else _lib.load()

    @property
    def handle(self):
        if self._handle is None:
            lib = self.lib
            n = len(self.paths)
            arr = (_lib.EqfPathDesc * n)()
            for i, p in enumerate(self.paths):
                arr[i] = _lib.EqfPathDesc(p.l1, p.l2, p.l3, p.mul, p.in1_block, p.in2_off, p.out_group,
                                          p.out_chan_off, p.w_off, p.cg_off)
            in1_l = (ctypes.c_int32 * len(self.in1_blocks))(*[l for l, _ in self.in1_blocks])
            in1_mul = (ctypes.c_int32 * len(self.in1_blocks))(*[m for _, m in self.in1_blocks])
            out_l = (ctypes.c_int32 * len(self.out_groups))(*[l for l, _, _ in self.out_groups])
            out_mul = (ctypes.c_int32 * len(self.out_groups))(*[m for _, _, m in self.out_groups])
            cg = np.ascontiguousarray(self.cg)
            h = ctypes.c_void_p()
            rc = lib.eqf_plan_create(arr, n, in1_l, in1_mul, len(self.in1_blocks), out_l, out_mul,
                                     len(self.out_groups), self.d_y, self.weight_numel,
                                     cg.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), cg.size, ctypes.byref(h))
            _lib.check(rc, "eqf_plan_create", lib)
            self._handle = h
        return self._handle

    def info(self) -> dict:
        out = (ctypes.c_int32 * 13)()
        _lib.check(self.lib.eqf_plan_info(self.handle, out, 13), "eqf_plan_info", self.lib)
        keys = ("n_paths", "m_size", "n_wtasks", "n_xtasks", "tile_edges", "smem_bytes", "blob_words", "weight_numel",
                "vec_ok", "n_vwtasks", "n_vxtasks", "smem_bytes_vec_fwd", "generated")
        return dict(zip(keys, list(out)))

    @property
    def generated(self) -> bool:
        """True when the plan-specialised kernels (codegen.py) will run for this plan."""
        g = getattr(self, "_generated", None)
        if g is None:
            g = bool(self.info()["generated"])
            self._generated = g
        return g

    def __del__(self):
        h, self._handle = getattr(self, "_handle", None), None
        if h is not None:
            try:
                self.lib.eqf_plan_destroy(h)
            except Exception:
                pass

    # ------------------------------------------------------------------ bytes / flops accounting
    def algorithmic_bytes(self, shared_weights: bool = False) -> dict:
        """fp32 bytes per edge at the operator boundary (SURVEY.md section 8d)."""
        d_in, d_out, w = self.irreps_in1.dim, self.irreps_out.dim, self.weight_numel
        wt = 0 if shared_weights else w
        fwd = 4 * (d_in + self.d_y + wt + d_out)
        bwd_xw = 4 * (d_out + d_in + self.d_y + wt) + 4 * (d_in + wt)
        return {"forward": fwd, "grad_xw": bwd_xw, "grad_y": 4 * (d_out + d_in + self.d_y + wt) + 4 * self.d_y}

    def fma_per_edge(self) -> int:
        return sum(p.mul * (2 * p.l1 + 1) * (2 * p.l3 + 1) for p in self.paths)

    # ------------------------------------------------------------------ table interpreter (host check)
    def emulate_forward(self, xs: Sequence[np.ndarray], y: np.ndarray, w: np.ndarray) -> List[np.ndarray]:
        """Numpy walk over the *same tables the kernel uses* (planar in, planar out); float64.

        Used by the CPU tests to validate the tables against the oracle; never on the product path.
        """
        E = y.shape[0]
        outs = [np.zeros((E, 2 * l + 1, mul)) for l, _, mul in self.out_groups]
        for p in self.paths:
            d1, d2, d3 = 2 * p.l1 + 1, 2 * p.l2 + 1, 2 * p.l3 + 1
            c = self.cg64[p.cg_off:p.cg_off + d1 * d2 * d3].reshape(d1, d2, d3)
            M = np.einsum("ijk,ej->eik", c, y[:, p.in2_off:p.in2_off + d2])
            wv = w[..., p.w_off:p.w_off + p.mul]
            if wv.ndim == 1:
                wv = wv[None, :]
            val = np.einsum("eiu,eik->eku", xs[p.in1_block], M) * wv[:, None, :]
            outs[p.out_group][:, :, p.out_chan_off:p.out_chan_off + p.mul] = val
        return outs
