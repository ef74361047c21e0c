"""The periodic neighbour list ``graph.radius_graph_pbc``: the count / fill kernels of eqf_graph.cu, the torch statement
``radius_graph_pbc_torch`` and the nearest-``max_neighbors`` cut ``_cap_neighbours``.

The independent reference is ``oracle.equiformer_ref.radius_graph_pbc``: float64, one image shell more than the
repetition count needs, its own exact cut.  The inputs are a small cell zoo - cubic OC20-like frames, the two triclinic
cells of the OC20 fixture, a strongly sheared cell whose heights are far below its edge lengths, a cell smaller than the
cutoff (atoms see their own images), a slab with vacuum, a one-atom frame, and a batch whose frames need different
repetition counts around a frame with no atoms - and two constructed frames: pairs exactly at, and a few ulp either side
of, r and the 1e-4 floor; and pairs whose hit decision depends on how the float32 image offset ``n . cell`` is rounded.

Against the statement the kernels must agree bit for bit.  Against the float64 oracle, a pair whose float64 d^2 lies
within its float32 rounding error (a first-order bound from the pair's coordinates and image offset) of r^2 or of 1e-4
may go either way; every other pair must match, with its cell offset, in the same order.
"""
from __future__ import annotations

import functools
import os

import numpy as np
import pytest
import torch

from equiformer_b200.graph import _cap_neighbours, _pbc_repetitions, radius_graph_pbc, radius_graph_pbc_torch
from equiformer_b200.synthetic import oc20_like_frames, stress_cell
from oracle import equiformer_ref as R

R_CUT = 5.0
U32 = 2.0 ** -24                                   # unit roundoff of float32
OC20_SMALL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_model_oc20_small.npz")
SHEARED = [[6.0, 0.0, 0.0], [5.5, 2.0, 0.0], [0.5, 0.5, 7.0]]             # heights 2.05, 2.00, 7.0 A
SMALL_TRICLINIC = [[1.5, 0.0, 0.0], [0.35, 1.6, 0.0], [0.15, -0.2, 1.7]]  # non-dyadic entries: n . cell rounds


# ------------------------------------------------------------------------------------------------ inputs
def _frames(frames, seed):
    """``frames``: list of (cell rows [3, 3], n_atoms, z_max) with atoms uniform in fractional coordinates, the third
    one below ``z_max``.  Returns float32 (pos [N, 3], batch [N], cell [F, 3, 3])."""
    g = torch.Generator().manual_seed(seed)
    pos, batch, cells = [], [], []
    for f, (cell, n, z_max) in enumerate(frames):
        cell = torch.tensor(cell, dtype=torch.float64)
        frac = torch.rand(n, 3, generator=g, dtype=torch.float64) * torch.tensor([1.0, 1.0, z_max], dtype=torch.float64)
        pos.append(frac @ cell)
        batch.append(torch.full((n,), f, dtype=torch.long))
        cells.append(cell)
    return torch.cat(pos).float(), torch.cat(batch), torch.stack(cells).float()


def _cubic(side):
    return [[side, 0.0, 0.0], [0.0, side, 0.0], [0.0, 0.0, side]]


def _exact_boundary_frame():
    """A 10 A cubic cell with exactly representable coordinates: pairs at exactly r inside the cell and across a face
    (kept: d^2 <= r^2), pairs 2 and 4 ulp of 25 inside and outside r^2 (d_y = 4 + k 2^-21 exactly, d^2 = 25 + k 2^-18
    in every rounding), and two atoms 0.01 A apart (d^2 just below 1e-4, excluded as the atom itself) next to two 0.02 A
    apart (kept).  Returns the case and the expected decision of each named pair ``(j, i, offset)``."""
    eps = 2.0 ** -21                                                  # ulp of 5 and of 4
    pts, expect = [], {}

    def pair(pi, pj, offset, kept, name):
        pts.extend([pi, pj])
        expect[name] = (len(pts) - 1, len(pts) - 2, offset, kept)

    pair([1.0, 1.0, 1.0], [4.0, 5.0, 1.0], (0, 0, 0), True, "at r")
    pair([8.0, 1.0, 3.0], [1.0, 5.0, 3.0], (1, 0, 0), True, "at r across a face")
    for z, k in zip((5.0, 6.5, 8.0, 9.5), (-2, -1, 1, 2)):
        pair([1.0, 1.0, z], [4.0, 5.0 + k * eps, z], (0, 0, 0), k < 0, f"{2 * k:+d} ulp of r^2")
    pair([2.0, 8.0, 6.0], [2.01, 8.0, 6.0], (0, 0, 0), False, "0.01 A apart")
    pair([2.0, 8.0, 8.5], [2.02, 8.0, 8.5], (0, 0, 0), True, "0.02 A apart")
    pos = torch.tensor(pts, dtype=torch.float32)
    return (pos, torch.zeros(len(pts), dtype=torch.long), torch.tensor([_cubic(10.0)], dtype=torch.float32)), expect


def _fma32(x, y, z):
    """float32 fused multiply-add ``x * y + z`` rounded once: the product of two float32 is exact in float64, the sum
    is made exact by a two-sum, whose error breaks the float64 result's ties at float32 midpoints."""
    f32, f64 = np.float32, np.float64
    p, z = f64(x) * f64(y), f64(z)
    s = p + z
    t = s - p
    err = (p - (s - t)) + (z - t)
    r = f32(s)
    if err != 0 and f64(r) != s:
        lo, hi = (r, np.nextafter(r, f32(np.inf))) if f64(r) < s else (np.nextafter(r, f32(-np.inf)), r)
        if s - f64(lo) == f64(hi) - s:                        # s is a float32 midpoint: the exact value is off it
            r = hi if err > 0 else lo
    return r


def _offset_roundings(n, cell):
    """The float32 image offset ``n . cell`` in three roundings: separately rounded products summed a, b, c (the
    kernels and the statement); ``fma(n_c, c, fma(n_a, a, n_b b))`` (nvcc's contraction of ``n_a * a + n_b * b + n_c *
    c``: the b product is the rounded one); ``fma(n_c, c, fma(n_b, b, n_a a))`` (the a product rounded, as a float32
    ``imgs @ cell`` gives on x86 CPU torch)."""
    f32 = np.float32
    separate = (n[0] * cell[0] + n[1] * cell[1]) + n[2] * cell[2]
    b_first = np.array([_fma32(n[2], cell[2, k], _fma32(n[0], cell[0, k], n[1] * cell[1, k])) for k in range(3)], f32)
    a_first = np.array([_fma32(n[2], cell[2, k], _fma32(n[1], cell[1, k], n[0] * cell[0, k])) for k in range(3)], f32)
    return separate, b_first, a_first


def _offset_rounding_frame(per_chain=6, seed=11):
    """Pairs within a few ulp of r whose keep / drop decision under separately rounded image offsets differs from the
    decision under each FMA chain of ``_offset_roundings``: ``per_chain`` pairs for each, so a kernel or a statement
    that forms the offset either way disagrees with the other on some of them.  Found by seeded search inside
    ``SMALL_TRICLINIC``, whose heights of 1.46, 1.59 and 1.70 A put images with |n| = 3 along every lattice vector well
    inside the range (products by 3 round; by 1, 2 and 4 they are exact)."""
    f32, f64 = np.float32, np.float64
    cell = np.array(SMALL_TRICLINIC, dtype=f32)
    cell64 = cell.astype(f64)
    rep = np.array(_pbc_repetitions(torch.tensor([SMALL_TRICLINIC], dtype=torch.float64), R_CUT))
    r2 = f32(R_CUT * R_CUT)
    rng = np.random.default_rng(seed)

    def d2(pi, pj, off):
        d = (pj + off) - pi
        return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]

    pts, found = [], [0, 0]
    while min(found) < per_chain:
        n = rng.integers(-rep, rep + 1).astype(f32)
        separate, *chains = _offset_roundings(n, cell)
        wanted = [found[c] < per_chain and not np.array_equal(separate, chain) for c, chain in enumerate(chains)]
        if not any(wanted):
            continue
        # j on the sphere of radius r around pos_i - n . cell, aimed at a random point of the cell; kept when inside
        pi = (rng.random(3) @ cell64).astype(f32)
        centre = pi.astype(f64) - n.astype(f64) @ cell64
        u = rng.random(3) @ cell64 - centre
        pj = (centre + R_CUT * u / np.linalg.norm(u)).astype(f32)
        frac = np.linalg.solve(cell64.T, pj.astype(f64))
        if not ((frac >= 0) & (frac < 1)).all():
            continue
        for k in range(-8, 9):
            q = pi.copy()
            q[0] = q[0] + f32(k) * np.spacing(q[0])
            keep = d2(q, pj, separate) <= r2
            flips = [w and (d2(q, pj, chain) <= r2) != keep for w, chain in zip(wanted, chains)]
            if any(flips):
                pts.extend([q, pj])
                found = [f + fl for f, fl in zip(found, flips)]
                break
    pos = torch.from_numpy(np.stack(pts))
    return pos, torch.zeros(len(pts), dtype=torch.long), torch.tensor([SMALL_TRICLINIC], dtype=torch.float32)


@functools.lru_cache(maxsize=None)
def _case(name):
    if name == "cubic":
        pos, batch, _z, _tags, side = oc20_like_frames(3, seed=3)
        return pos, batch, torch.diag_embed(side[:, None].expand(-1, 3)).float()
    if name == "triclinic":
        fx = np.load(OC20_SMALL)
        return torch.from_numpy(fx["pos"]), torch.from_numpy(fx["batch"]), torch.from_numpy(fx["cell"])
    if name == "sheared":
        return _frames([(SHEARED, 40, 1.0)], seed=1)
    if name == "smaller_than_cutoff":
        return _frames([(_cubic(2.5), 3, 1.0)], seed=2)
    if name == "slab":
        return _frames([([[8.0, 0, 0], [0, 8.0, 0], [0, 0, 30.0]], 40, 1.0 / 3.0)], seed=3)
    if name == "one_atom":
        return _frames([(_cubic(4.0), 1, 1.0)], seed=4)
    if name == "mixed_batch":      # repetitions (3, 3, 1), none, (1, 1, 1), (2, 2, 2): the batch enumerates (3, 3, 2)
        return _frames([(SHEARED, 20, 1.0), (_cubic(9.0), 0, 1.0), (_cubic(9.0), 30, 1.0), (_cubic(2.5), 2, 1.0)], seed=5)
    if name == "exact_boundary":
        return _exact_boundary_frame()[0]
    if name == "offset_rounding":
        return _offset_rounding_frame()
    raise ValueError(name)


ZOO = ["cubic", "triclinic", "sheared", "smaller_than_cutoff", "slab", "one_atom", "mixed_batch"]
BOUNDARY = ["exact_boundary", "offset_rounding"]
CAPS = [None, 12]                  # uncapped, and a cap that cuts most centres of the denser cases


# ------------------------------------------------------------------------------------------------ comparisons
def _keys(edge, offsets, n):
    """One int64 per pair, ascending in (centre i, atom j, image a, b, c): the list order of the contract."""
    o = offsets.long().cpu() + 8
    return (((edge[1].cpu() * n + edge[0].cpu()) * 17 + o[:, 0]) * 17 + o[:, 1]) * 17 + o[:, 2]


def _d2_and_error_bound(pos, cell, batch, edge, offsets):
    """Float64 d^2 of each pair ``(j, i, n)`` and a bound on how far the float32 d^2 of the kernels and the statement
    can lie from it.  Per component d_k = (pos_jk + o_k) - pos_ik with o_k = (n_a a_k + n_b b_k) + n_c c_k: the three
    products and two sums of o_k err by at most 3 u S_k (S_k = sum_m |n_m c_mk|), the two sums after it by u |pos_jk +
    o_k| and u |d_k|, so e_k = u (3 S_k + |pos_jk + o_k| + |d_k|) to first order; the squares and sums of d^2 add
    2 |d_k| e_k per component and 3 u d^2.  Doubled for the terms of second order."""
    p, c = pos.double().cpu(), cell.double().cpu()
    src, dst = edge[0].cpu(), edge[1].cpu()
    terms = offsets.double().cpu()[:, :, None] * c[batch.cpu()[dst]]                  # [E, m, k]: n_m c_mk
    q = p[src] + terms.sum(1)
    d = q - p[dst]
    e = U32 * (3.0 * terms.abs().sum(1) + q.abs() + d.abs())
    d2 = d.pow(2).sum(-1)
    return d2, 2.0 * ((2.0 * d.abs() * e).sum(-1) + 3.0 * U32 * d2)


def _describe(pos, cell, batch, edge, offsets, sel, limit=6):
    d2, bound = _d2_and_error_bound(pos, cell, batch, edge[:, sel], offsets[sel])
    rows = [f"(j={int(j)}, i={int(i)}, n={tuple(int(v) for v in o)}, d2_64={float(x)!r} +- {float(b):.1e})"
            for j, i, o, x, b in zip(edge[0][sel].tolist(), edge[1][sel].tolist(), offsets[sel].tolist(), d2.tolist(),
                                     bound.tolist())]
    return ", ".join(rows[:limit]) + (" ..." if len(rows) > limit else "")


def _assert_same(out, ref, case):
    """Bit for bit: edge index, cell offsets, d^2 and row counts; a mismatch names the pairs only one side has."""
    pos, batch, cell = case
    (edge, offs, d2), (redge, roffs, rd2) = [tuple(t.cpu() for t in x) for x in (out, ref)]
    k, rk = _keys(edge, offs, pos.shape[0]), _keys(redge, roffs, pos.shape[0])
    only, ronly = ~torch.isin(k, rk), ~torch.isin(rk, k)
    assert not only.any() and not ronly.any(), (
        f"{int(only.sum())} pairs only in the kernel output: {_describe(pos, cell, batch, edge, offs, only)}; "
        f"{int(ronly.sum())} only in the statement: {_describe(pos, cell, batch, redge, roffs, ronly)}")
    assert torch.equal(edge, redge) and torch.equal(offs.int(), roffs.int())
    assert d2.dtype == rd2.dtype == torch.float32 and torch.equal(d2, rd2), (d2 - rd2).abs().max()
    n = pos.shape[0]
    assert torch.equal(torch.bincount(edge[1], minlength=n), torch.bincount(redge[1], minlength=n))


def _assert_matches_oracle(out, ref, case, r=R_CUT):
    """Float32 neighbour list ``out`` vs the float64 oracle ``ref`` (both uncapped): same pairs in the same order, except
    pairs whose float64 d^2 lies within their float32 error bound (``_d2_and_error_bound``) of r^2 or 1e-4; float32 d^2
    within that bound of the float64 one.  Returns the number of pairs that went the other way."""
    pos, batch, cell = case
    (edge, offs, d2), (redge, roffs, rd2) = [tuple(t.cpu() for t in x) for x in (out, ref)]
    n = pos.shape[0]
    k, rk = _keys(edge, offs, n), _keys(redge, roffs, n)
    assert bool((k[1:] > k[:-1]).all()), "not ordered by (centre, j, image)"
    assert bool((rk[1:] > rk[:-1]).all()), "oracle not ordered by (centre, j, image)"

    def either_way(x, bound):
        return ((x - r * r).abs() <= bound) | ((x - 1e-4).abs() <= bound)

    in_ref, in_out = torch.isin(k, rk), torch.isin(rk, k)
    extra, bound = _d2_and_error_bound(pos, cell, batch, edge[:, ~in_ref], offs[~in_ref])
    ok = either_way(extra, bound)
    assert bool(ok.all()), (
        f"pairs the oracle does not have: {_describe(pos, cell, batch, edge, offs, (~in_ref).nonzero().flatten()[~ok])}")
    _, bound = _d2_and_error_bound(pos, cell, batch, redge[:, ~in_out], roffs[~in_out])
    ok = either_way(rd2[~in_out], bound)
    assert bool(ok.all()), (
        f"oracle pairs missing: {_describe(pos, cell, batch, redge, roffs, (~in_out).nonzero().flatten()[~ok])}")
    assert torch.equal(k[in_ref], rk[in_out])
    _, bound = _d2_and_error_bound(pos, cell, batch, edge[:, in_ref], offs[in_ref])
    err = (d2[in_ref].double() - rd2[in_out]).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    return int((~in_ref).sum() + (~in_out).sum())


def _assert_exact_cut(capped, uncapped, k):
    """``capped`` == the uncapped list cut to each centre's ``k`` nearest by (d^2, list position), order kept."""
    edge, offs, d2 = (t.cpu() for t in uncapped)
    keep = R.nearest_neighbours_mask(edge[1], d2, k)
    ce, co, cd = (t.cpu() for t in capped)
    assert torch.equal(ce, edge[:, keep]) and torch.equal(co, offs[keep]) and torch.equal(cd, d2[keep])


# ------------------------------------------------------------------------------------------------ CPU
def test_cap_is_exact_on_near_ties_at_a_high_centre_index():
    """A centre at index 1 199 (a 16-frame OC20 batch has about 1 100 atoms) with 60 hits at d^2 in [20.000, 20.010] and a
    cap of 30: the kept hits are exactly its 30 nearest, equal d^2 keeping list order; other centres are untouched."""
    g = torch.Generator().manual_seed(0)
    n, centre = 1200, 1199
    other = torch.repeat_interleave(torch.arange(0, centre, 37), 20)                 # earlier centres below the cap
    dst = torch.cat([other, torch.full((60,), centre)])
    src = torch.randint(0, n, (dst.numel(),), generator=g)
    d2 = torch.cat([torch.rand(other.numel(), generator=g) * 25.0, 20.0 + torch.rand(60, generator=g) * 0.01]).float()
    d2[-10:-5] = d2[-5:]                                                              # exact ties, too
    offsets = torch.randint(-2, 3, (dst.numel(), 3), generator=g, dtype=torch.int32)
    edge = torch.stack([src, dst])
    ce, co, cd = _cap_neighbours(edge, offsets, d2, n, 30)
    keep = R.nearest_neighbours_mask(dst, d2, 30)
    assert torch.equal(ce, edge[:, keep]) and torch.equal(co, offsets[keep]) and torch.equal(cd, d2[keep])
    mine = d2[-60:]
    assert torch.equal(torch.sort(cd[ce[1] == centre]).values, torch.sort(mine).values[:30])
    assert int((ce[1] != centre).sum()) == other.numel()


@pytest.mark.parametrize("name", ZOO + BOUNDARY)
def test_statement_matches_oracle(name):
    """The torch statement against the float64 oracle (uncapped); capped, it is the exact cut of its uncapped list."""
    case = _case(name)
    out = radius_graph_pbc_torch(*case, R_CUT, None)
    either = _assert_matches_oracle(out, R.radius_graph_pbc(*case, R_CUT), case)
    print(f"[{name}] {out[0].shape[1]} pairs, {either} differ from the oracle, all within their rounding error of r^2 / 1e-4")
    _assert_exact_cut(radius_graph_pbc_torch(*case, R_CUT, CAPS[1]), out, CAPS[1])


@pytest.mark.parametrize("name", ZOO + BOUNDARY)
def test_oracle_extra_image_shell_is_empty(name):
    """The oracle enumerates ceil(r / height) + 1 images per lattice vector; no hit lies in the outermost shell, and
    each frame's hits stay within the repetitions ``_pbc_repetitions`` gives its own cell (so also the batch's)."""
    pos, batch, cell = _case(name)
    edge, offs, _d2 = R.radius_graph_pbc(pos, batch, cell, R_CUT)
    frame = batch[edge[1]]
    for f in range(cell.shape[0]):
        rep = torch.tensor(_pbc_repetitions(cell[f:f + 1].double(), R_CUT))
        assert bool((offs[frame == f].abs() <= rep).all()), (f, rep, offs[frame == f].abs().amax(0))
    assert bool((offs.abs() <= torch.tensor(_pbc_repetitions(cell.double(), R_CUT))).all())


def test_exact_boundary_pairs_cpu():
    """Exactly at r: kept; 2 and 4 ulp either side of r^2: decided by the side; 0.01 A apart: excluded; 0.02 A: kept -
    by the statement and by the oracle."""
    case, expect = _exact_boundary_frame()
    n = case[0].shape[0]
    for out in (radius_graph_pbc_torch(*case, R_CUT, None), R.radius_graph_pbc(*case, R_CUT)):
        k = _keys(out[0], out[1], n)
        for name, (j, i, offset, kept) in expect.items():
            key = _keys(torch.tensor([[j], [i]]), torch.tensor([offset]), n)
            assert bool(torch.isin(key, k)) == kept, name


# ------------------------------------------------------------------------------------------------ GPU
def _to(case, dev):
    return tuple(t.to(dev) for t in case)


@pytest.mark.gpu
@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("name", ZOO + BOUNDARY)
def test_kernels_match_statement(cuda_device, name, cap):
    """Count / fill kernels == the torch statement bit for bit: pairs, order, cell offsets, d^2, row counts."""
    case = _case(name)
    out = radius_graph_pbc(*_to(case, cuda_device), R_CUT, cap)
    _assert_same(out, radius_graph_pbc_torch(*case, R_CUT, cap), case)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ZOO + BOUNDARY)
def test_kernels_match_oracle(cuda_device, name):
    """Count / fill kernels (uncapped) against the float64 oracle."""
    case = _case(name)
    out = radius_graph_pbc(*_to(case, cuda_device), R_CUT, None)
    either = _assert_matches_oracle(out, R.radius_graph_pbc(*case, R_CUT), case)
    print(f"[{name}] {out[0].shape[1]} pairs, {either} differ from the oracle, all within their rounding error of r^2 / 1e-4")


@pytest.mark.gpu
def test_exact_boundary_pairs_cuda(cuda_device):
    """The decisions of ``test_exact_boundary_pairs_cpu``, by the kernels."""
    case, expect = _exact_boundary_frame()
    edge, offs, _d2 = radius_graph_pbc(*_to(case, cuda_device), R_CUT, None)
    n = case[0].shape[0]
    k = _keys(edge, offs, n)
    for name, (j, i, offset, kept) in expect.items():
        assert bool(torch.isin(_keys(torch.tensor([[j], [i]]), torch.tensor([offset]), n), k)) == kept, name


@pytest.mark.gpu
def test_kernel_cut_is_exact_on_an_oc20_batch(cuda_device):
    """16 OC20-like frames (about 50 neighbours per centre) with ``max_neighbors=50``: many centres are cut, and the
    capped list is the exact (centre, d^2, list position) cut of the uncapped kernel output - and the statement's."""
    pos, batch, _z, _tags, side = oc20_like_frames(16, seed=0)
    case = (pos, batch, torch.diag_embed(side[:, None].expand(-1, 3)).float())
    dev = _to(case, cuda_device)
    uncapped = radius_graph_pbc(*dev, R_CUT, None)
    capped = radius_graph_pbc(*dev, R_CUT, 50)
    deg = torch.bincount(uncapped[0][1].cpu(), minlength=pos.shape[0])
    assert int((deg > 50).sum()) > pos.shape[0] // 4, int((deg > 50).sum())
    _assert_exact_cut(capped, uncapped, 50)
    _assert_same(capped, radius_graph_pbc_torch(*case, R_CUT, 50), case)


@pytest.mark.gpu
def test_kernels_match_oracle_on_a_stress_frame(cuda_device):
    """One 5 000-atom periodic frame (``bench.py --workload stress``; many ballot rounds per warp) against the oracle,
    which evaluates its centres in chunks on the GPU: the statement's [i, j, image, 3] tensor would take several GB."""
    pos, batch, _z, side = stress_cell(5000, seed=0)
    case = (pos, batch, (torch.eye(3) * side).view(1, 3, 3).float())
    dev = _to(case, cuda_device)
    try:
        torch.cuda.reset_peak_memory_stats()
        out = radius_graph_pbc(*dev, R_CUT, None)
        ref = R.radius_graph_pbc(*dev, R_CUT)
        either = _assert_matches_oracle(out, ref, case)
        print(f"[stress] {out[0].shape[1]} pairs, {either} differ from the oracle, all within their rounding error of r^2 / 1e-4; "
              f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    finally:
        torch.cuda.empty_cache()
