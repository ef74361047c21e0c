"""Neighbour-list construction (stand-in for ``torch_cluster.radius_graph``, SURVEY.md 8f-3).

The ordering contract the hot path relies on - ``edge_index[1]`` (the centre atom, ``edge_dst``) ascending, neighbours
in index order, no self loops, ``d < r``, at most ``max_num_neighbors`` per centre - as used at
``nets/graph_attention_transformer.py:866-867``.  On CUDA fp32 inputs two small kernels (count, fill) around one
prefix sum do it (``eqf_radius_graph_count / _fill``); the torch brute force below is the statement they are tested
against and the path for CPU tensors (host-side tests, oracle inputs).
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch


def radius_graph(pos: torch.Tensor, r: float, batch: Optional[torch.Tensor] = None,
                 max_num_neighbors: int = 32, loop: bool = False, chunk: int = 4096) -> torch.Tensor:
    """Return ``edge_index [2, E]`` with row 0 = neighbour (source) and row 1 = centre (destination, ascending)."""
    n = pos.shape[0]
    if pos.is_cuda and pos.dtype == torch.float32 and n > 0 and (batch is None or batch.dtype == torch.long):
        return _radius_graph_cuda(pos, r, batch, max_num_neighbors, loop)
    return radius_graph_torch(pos, r, batch, max_num_neighbors, loop, chunk)


def radius_graph_csr(pos: torch.Tensor, r: float, batch: Optional[torch.Tensor] = None, max_num_neighbors: int = 32,
                     loop: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(edge_index [2, E], row_ptr [N + 1])``: the neighbour list and the CSR offsets of its (sorted) centres."""
    n = pos.shape[0]
    if pos.is_cuda and pos.dtype == torch.float32 and n > 0 and (batch is None or batch.dtype == torch.long):
        return _radius_graph_cuda(pos, r, batch, max_num_neighbors, loop, with_row_ptr=True)
    edge = radius_graph_torch(pos, r, batch, max_num_neighbors, loop)
    row_ptr = torch.zeros(n + 1, dtype=torch.int64, device=pos.device)
    torch.cumsum(torch.bincount(edge[1], minlength=n), 0, out=row_ptr[1:])
    return edge, row_ptr


def _radius_graph_cuda(pos, r, batch, max_num_neighbors, loop, with_row_ptr: bool = False):
    import ctypes

    from . import _lib
    lib = _lib.load()
    n = pos.shape[0]
    p = pos.detach().contiguous()
    b = batch.contiguous() if batch is not None else None
    cap = int(max_num_neighbors) if max_num_neighbors is not None else n
    stream = ctypes.c_void_p(torch.cuda.current_stream(pos.device).cuda_stream)
    row_ptr = torch.zeros(n + 1, dtype=torch.int64, device=pos.device)
    deg = torch.empty(n, dtype=torch.int64, device=pos.device)
    with torch.cuda.device(pos.device):
        rc = lib.eqf_radius_graph_count(p.data_ptr(), b.data_ptr() if b is not None else None, n, float(r) * float(r),
                                        1 if loop else 0, cap, deg.data_ptr(), stream)
        _lib.check(rc, "eqf_radius_graph_count")
        torch.cumsum(deg, 0, out=row_ptr[1:])
        n_edges = int(row_ptr[-1].item())          # the one host synchronisation of the neighbour search
        edge = torch.empty((2, n_edges), dtype=torch.int64, device=pos.device)
        if n_edges > 0:
            rc = lib.eqf_radius_graph_fill(p.data_ptr(), b.data_ptr() if b is not None else None, n, float(r) * float(r),
                                           1 if loop else 0, cap, row_ptr.data_ptr(), edge[0].data_ptr(), edge[1].data_ptr(),
                                           stream)
            _lib.check(rc, "eqf_radius_graph_fill")
    return (edge, row_ptr) if with_row_ptr else edge


def radius_graph_torch(pos: torch.Tensor, r: float, batch: Optional[torch.Tensor] = None,
                       max_num_neighbors: int = 32, loop: bool = False, chunk: int = 4096) -> torch.Tensor:
    """The plain torch brute force over same-graph pairs (reference statement of the contract above)."""
    n = pos.shape[0]
    if batch is None:
        batch = torch.zeros(n, dtype=torch.long, device=pos.device)
    pos_d = pos.detach()
    srcs, dsts = [], []
    for start in range(0, n, chunk):
        stop = min(start + chunk, n)
        d2 = (pos_d[start:stop, None, :] - pos_d[None, :, :]).pow(2).sum(-1)
        mask = (d2 < r * r) & (batch[start:stop, None] == batch[None, :])
        if not loop:
            idx = torch.arange(start, stop, device=pos.device)
            mask[idx - start, idx] = False
        if max_num_neighbors is not None and max_num_neighbors < n:
            rank = mask.cumsum(dim=1)
            mask &= rank <= max_num_neighbors
        dst, src = mask.nonzero(as_tuple=True)
        srcs.append(src)
        dsts.append(dst + start)
    return torch.stack([torch.cat(srcs), torch.cat(dsts)], dim=0)


def scatter_sum(x: torch.Tensor, index: torch.Tensor, dim: int = 0, dim_size: Optional[int] = None) -> torch.Tensor:
    """``torch_scatter.scatter(x, index, dim=0, dim_size=..)`` with the default ``sum`` reduce (node/graph level)."""
    if dim != 0:
        raise NotImplementedError("scatter_sum: only dim=0 is used by the reference")
    if dim_size is None:
        dim_size = int(index.max()) + 1 if index.numel() > 0 else 0
    out = torch.zeros((dim_size,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    return out.index_add(0, index, x)


# ----------------------------------------------------------------------------------------------- periodic cells
def _pbc_repetitions(cell: torch.Tensor, r: float):
    """Images per lattice vector that can hold a neighbour within ``r``: ceil(r / height) of each frame, max over the
    batch (ocpmodels ``radius_graph_pbc``: ``rep_a = ceil(radius * |b x c| / volume)``)."""
    a, b, c = cell[:, 0], cell[:, 1], cell[:, 2]
    bc, ca, ab = torch.cross(b, c, dim=-1), torch.cross(c, a, dim=-1), torch.cross(a, b, dim=-1)
    vol = (a * bc).sum(-1).abs()
    reps = [torch.ceil(r * x.norm(dim=-1) / vol).max() for x in (bc, ca, ab)]
    return [int(v.item()) for v in reps]


def radius_graph_pbc_torch(pos, batch, cell, r: float, max_neighbors: int = 500):
    """Plain torch statement of the periodic neighbour list (ocpmodels ``radius_graph_pbc`` as the OC20 model consumes it,
    nets/graph_attention_transformer_oc20.py:267-302): returns ``(edge_index [2, E], cell_offsets [E, 3] int, dist2 [E])``
    with ``edge_index[0]`` = neighbour j, ``edge_index[1]`` = centre i (ascending), then j, then image index; a pair is
    kept when ``1e-4 < d^2 <= r^2``; centres with more than ``max_neighbors`` hits keep the nearest ones."""
    rep = _pbc_repetitions(cell.double(), r)
    grids = [torch.arange(-k, k + 1, device=pos.device) for k in rep]
    imgs = torch.stack(torch.meshgrid(*grids, indexing="ij"), dim=-1).reshape(-1, 3)         # a slowest, c fastest
    srcs, dsts, offs, d2s = [], [], [], []
    for f in range(int(batch.max()) + 1 if batch.numel() else 0):
        idx = (batch == f).nonzero().flatten()
        p = pos[idx].float()
        # n_a a + n_b b + n_c c as separately rounded products summed in that order, as the kernels form it (a matmul
        # leaves the rounding order to the library)
        n, c = imgs.to(pos.dtype), cell[f].to(pos.dtype)
        shift = ((n[:, 0:1] * c[0] + n[:, 1:2] * c[1]) + n[:, 2:3] * c[2]).float()           # [n_img, 3]
        d = p[None, :, None, :] + shift[None, None, :, :] - p[:, None, None, :]             # [i, j, img, 3]
        d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        hit = (d2 <= r * r) & (d2 > 1e-4)
        i, j, m = hit.nonzero(as_tuple=True)
        srcs.append(idx[j]); dsts.append(idx[i]); offs.append(imgs[m]); d2s.append(d2[i, j, m])
    edge = torch.stack([torch.cat(srcs), torch.cat(dsts)])
    return _cap_neighbours(edge, torch.cat(offs).to(torch.int32), torch.cat(d2s), pos.shape[0], max_neighbors)


def _cap_neighbours(edge, offsets, d2, n, max_neighbors):
    """Keep the ``max_neighbors`` nearest hits of every centre (ocpmodels ``get_max_neighbors_mask``), exact on the
    given ``d2``; of equal ``d2`` the earlier hit in the list is kept.  Order preserved."""
    deg = torch.bincount(edge[1], minlength=n)
    if max_neighbors is None or edge.shape[1] == 0 or int(deg.max()) <= max_neighbors:
        return edge, offsets, d2
    row_ptr = torch.zeros(n + 1, dtype=torch.long, device=edge.device)
    torch.cumsum(deg, 0, out=row_ptr[1:])
    # by centre, then distance, then list position: two stable sorts, so that no combined float key rounds near-equal
    # distances of high-index centres into ties
    order = torch.argsort(d2, stable=True)
    order = order[torch.argsort(edge[1][order], stable=True)]
    rank = torch.empty_like(order)
    rank[order] = torch.arange(order.numel(), device=order.device) - row_ptr[edge[1][order]]
    keep = rank < max_neighbors
    return edge[:, keep], offsets[keep], d2[keep]


def radius_graph_pbc(pos, batch, cell, r: float, max_neighbors: int = 500):
    """Periodic neighbour list: CUDA kernels (``eqf_radius_graph_pbc_count / _fill``) on fp32 device tensors, the torch
    statement otherwise.  ``cell``: ``[n_frames, 3, 3]`` rows = lattice vectors; ``batch`` ascending."""
    if not (pos.is_cuda and pos.dtype == torch.float32 and pos.shape[0] > 0):
        return radius_graph_pbc_torch(pos, batch, cell, r, max_neighbors)
    import ctypes

    from . import _lib
    lib = _lib.load()
    n = pos.shape[0]
    cell32 = cell.to(device=pos.device, dtype=torch.float32).contiguous()
    rep = _pbc_repetitions(cell.to(pos.device).double(), r)
    n_frames = cell32.shape[0]
    frame_ptr = torch.zeros(n_frames + 1, dtype=torch.int64, device=pos.device)
    torch.cumsum(torch.bincount(batch, minlength=n_frames), 0, out=frame_ptr[1:])
    p, b = pos.detach().contiguous(), batch.contiguous()
    stream = ctypes.c_void_p(torch.cuda.current_stream(pos.device).cuda_stream)
    deg = torch.empty(n, dtype=torch.int64, device=pos.device)
    row_ptr = torch.zeros(n + 1, dtype=torch.int64, device=pos.device)
    with torch.cuda.device(pos.device):
        rc = lib.eqf_radius_graph_pbc_count(p.data_ptr(), b.data_ptr(), frame_ptr.data_ptr(), cell32.data_ptr(), n,
                                            float(r) * float(r), rep[0], rep[1], rep[2], deg.data_ptr(), stream)
        _lib.check(rc, "eqf_radius_graph_pbc_count")
        torch.cumsum(deg, 0, out=row_ptr[1:])
        n_edges = int(row_ptr[-1].item())
        edge = torch.empty((2, n_edges), dtype=torch.int64, device=pos.device)
        offsets = torch.empty((n_edges, 3), dtype=torch.int32, device=pos.device)
        d2 = torch.empty(n_edges, dtype=torch.float32, device=pos.device)
        if n_edges > 0:
            rc = lib.eqf_radius_graph_pbc_fill(p.data_ptr(), b.data_ptr(), frame_ptr.data_ptr(), cell32.data_ptr(), n,
                                               float(r) * float(r), rep[0], rep[1], rep[2], row_ptr.data_ptr(),
                                               edge[0].data_ptr(), edge[1].data_ptr(), offsets.data_ptr(), d2.data_ptr(), stream)
            _lib.check(rc, "eqf_radius_graph_pbc_fill")
    return _cap_neighbours(edge, offsets, d2, n, max_neighbors)
