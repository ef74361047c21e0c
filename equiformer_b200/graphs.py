"""CUDA-graph replay of the forward+backward of a model step (launch-bound inner loop -> one graph launch).

A training step of the unfused pipeline issues a few thousand small kernels; at ~7 us of host time each the host,
not the GPU, bounds the step.  Everything after neighbour search is free of host synchronisation
(``GraphAttentionTransformer.forward_edges``), so it is captured once per input signature ``(atoms, edges, graphs)``
and replayed: inputs are copied into static buffers, ``graph.replay()`` runs forward, loss and backward, gradients
land in the flat bucket of :class:`equiformer_b200.parallel.FlatGradAllReduce`.  A new signature triggers a new
capture (cached), so variable-size batches still work - they just pay the capture when a size is first seen.
Neighbour search, the gradient all-reduce and the optimiser stay outside the graph.
"""
from __future__ import annotations

import gc
from typing import Callable, Dict, Tuple

import torch

from . import ops
from .graph import radius_graph_csr


def pad_to_bucket(pos, batch, z, src, dst, n_graphs: int, atom_quantum: int, edge_quantum: int):
    """Pad a batch of ``n_graphs`` molecules to bucket sizes with a DUMMY molecule (graph index ``n_graphs``) appended
    after the real ones.  Returns the padded ``(pos, batch, z, src, dst, row_ptr)`` and the bucket ``(atoms_b, edges_b)``:
    multiples of ``atom_quantum`` / ``edge_quantum``, with at least two dummy atoms.

    The dummy atoms sit on a line far away and the dummy edges connect dummy atoms only, destination-sorted after every
    real edge (so a destination-sorted ``dst`` stays sorted).  Real atoms share no edge with the dummy molecule and every
    per-node / per-graph op of the models is local, so the real molecules' outputs and parameter gradients do not change
    as long as the dummy's outputs (energy row ``n_graphs``, its atoms' rows) stay out of the loss."""
    N, E = int(pos.shape[0]), int(src.numel())
    Nb = -(-(N + 2) // atom_quantum) * atom_quantum       # at least two dummy atoms (a dummy edge needs src != dst)
    Eb = -(-max(E, 1) // edge_quantum) * edge_quantum
    n_pa, n_pe = Nb - N, Eb - E
    dev = pos.device
    i = torch.arange(n_pa, device=dev)
    pos_p = torch.cat([pos, torch.stack([1000.0 + 1.7 * i.to(pos.dtype), torch.zeros_like(i, dtype=pos.dtype),
                                         torch.zeros_like(i, dtype=pos.dtype)], dim=1)])
    batch_p = torch.cat([batch, torch.full((n_pa,), n_graphs, dtype=batch.dtype, device=dev)])
    z_p = torch.cat([z, torch.ones(n_pa, dtype=z.dtype, device=dev)])
    k = torch.arange(n_pe, device=dev)
    dst_pad = N + (k * n_pa) // max(n_pe, 1)                # ascending over the dummy atoms
    src_pad = N + ((dst_pad - N + 1) % n_pa)
    src_p, dst_p = torch.cat([src, src_pad]), torch.cat([dst, dst_pad])
    counts = torch.zeros(Nb, dtype=torch.int64, device=dev).index_add_(0, dst_p, torch.ones_like(dst_p))
    row_ptr = torch.zeros(Nb + 1, dtype=torch.int64, device=dev)
    torch.cumsum(counts, 0, out=row_ptr[1:])
    return (pos_p, batch_p, z_p, src_p, dst_p, row_ptr), (Nb, Eb)


def csr_graph(src, dst, row_ptr, n_nodes: int) -> ops.Graph:
    """An ``ops.Graph`` over a destination-sorted edge list and its CSR offsets, built without host synchronisation."""
    csr = ops.Graph.__new__(ops.Graph)
    csr.n_nodes, csr.n_edges, csr.perm = int(n_nodes), int(src.numel()), None
    csr.src, csr.dst, csr.row_ptr = src, dst, row_ptr
    csr._src_perm = csr._src_row_ptr = None
    return csr


class _Captured:
    __slots__ = ("graph", "pos", "batch", "z", "target", "src", "dst", "row_ptr", "csr", "loss")


class GraphedForwardBackward:
    def __init__(self, model: torch.nn.Module, loss_fn: Callable[[torch.Tensor, torch.Tensor], torch.Tensor],
                 bucket, max_radius: float, warmup: int = 3, max_cached: int = 8):
        self.model, self.loss_fn, self.bucket = model, loss_fn, bucket
        self.max_radius, self.warmup, self.max_cached = max_radius, warmup, max_cached
        self._cache: Dict[Tuple[int, int, int], _Captured] = {}
        self.captures = 0

    def _fwd_bwd(self, c: _Captured) -> torch.Tensor:
        # the source-sorted (CSC) view of the edge list is rebuilt inside the captured region from the static `src`
        # buffer (sort + scatter-add + scan, no host synchronisation): nothing of it is left on the host's critical path
        c.csr._src_perm = c.csr._src_row_ptr = None
        out = self.model.forward_edges(c.pos, c.batch, c.z, c.src, c.dst, graph=c.csr, n_graphs=c.target.shape[0])
        loss = self.loss_fn(out, c.target)
        # gradients as a list + one multi-tensor copy into the flat bucket (autograd's per-parameter accumulation into
        # the bucket views would be ~290 tiny `grad += g` launches per step)
        self.bucket.store(torch.autograd.grad(loss, self.bucket.params, allow_unused=True))
        return loss.detach()

    def _capture(self, pos, batch, z, target, src, dst, row_ptr) -> _Captured:
        c = _Captured()
        c.pos, c.batch, c.z, c.target = pos.clone(), batch.clone(), z.clone(), target.clone()
        c.src, c.dst, c.row_ptr = src.clone(), dst.clone(), row_ptr.clone()
        csr = ops.Graph.__new__(ops.Graph)
        csr.n_nodes, csr.n_edges, csr.perm = int(pos.shape[0]), int(src.numel()), None
        csr.src, csr.dst, csr.row_ptr = c.src, c.dst, c.row_ptr
        csr._src_perm = csr._src_row_ptr = None
        c.csr = csr
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(self.warmup):
                self._fwd_bwd(c)
        torch.cuda.current_stream().wait_stream(side)
        c.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(c.graph):
            c.loss = self._fwd_bwd(c)
        self.captures += 1
        return c

    def __call__(self, pos, batch, z, target) -> torch.Tensor:
        """Neighbour search (eager) + replay of the captured forward/backward; returns the (static) loss tensor."""
        edge, row_ptr = radius_graph_csr(pos, self.max_radius, batch, max_num_neighbors=1000)
        src, dst = edge[0], edge[1]
        key = (int(pos.shape[0]), int(src.numel()), int(target.shape[0]))
        c = self._cache.get(key)
        if c is None:
            if len(self._cache) >= self.max_cached:
                self._cache.pop(next(iter(self._cache)))
            c = self._capture(pos, batch, z, target, src, dst, row_ptr)
            self._cache[key] = c
        # inputs -> static buffers: one multi-tensor copy per dtype instead of seven small launches
        torch._foreach_copy_([c.pos, c.target], [pos, target])
        torch._foreach_copy_([c.batch, c.z, c.src, c.dst, c.row_ptr], [batch, z, src, dst, row_ptr])
        c.graph.replay()
        return c.loss


class GraphedStep:
    """Generic capture / replay: ``fn(*static_tensors) -> loss`` (forward + loss of any model) is captured once per ``key``
    together with its backward (gradients stored into the flat bucket) and replayed on refreshed static buffers.  Used by
    ``bench.py`` for the OC20 and periodic-cell workloads, whose neighbour search stays eager."""

    def __init__(self, fn: Callable[..., torch.Tensor], bucket, warmup: int = 3, max_cached: int = 8):
        self.fn, self.bucket, self.warmup, self.max_cached = fn, bucket, warmup, max_cached
        self._cache: Dict[tuple, tuple] = {}
        self.captures = 0

    def _fwd_bwd(self, static) -> torch.Tensor:
        loss = self.fn(*static)
        self.bucket.store(torch.autograd.grad(loss, self.bucket.params, allow_unused=True))
        return loss.detach()

    def __call__(self, key, tensors) -> torch.Tensor:
        hit = self._cache.get(key)
        if hit is None:
            if len(self._cache) >= self.max_cached:
                self._cache.pop(next(iter(self._cache)))
            static = [t.clone() for t in tensors]
            # release dead models now: a DtpPlan finalised by the garbage collector in the middle of the capture would
            # free device memory there and invalidate it (torch no longer collects when a capture begins)
            gc.collect()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(self.warmup):
                    self._fwd_bwd(static)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                loss = self._fwd_bwd(static)
            self.captures += 1
            hit = (graph, static, loss)
            self._cache[key] = hit
        graph, static, loss = hit
        fl = [(s, t) for s, t in zip(static, tensors) if s.is_floating_point()]
        ix = [(s, t) for s, t in zip(static, tensors) if not s.is_floating_point()]
        if fl:
            torch._foreach_copy_([s for s, _ in fl], [t for _, t in fl])
        if ix:
            torch._foreach_copy_([s for s, _ in ix], [t for _, t in ix])
        graph.replay()
        return loss


class BucketedForwardBackward:
    """A STREAM of different batches through a handful of captured graphs (reference loop: a new batch every iteration,
    ``engine.py:58-59``).

    ``GraphedForwardBackward`` keys its captures on the exact ``(atoms, edges, graphs)`` signature, so real training would
    re-capture almost every step.  Here atoms and edges are padded up to bucket sizes (multiples of ``atom_quantum`` /
    ``edge_quantum``) with a DUMMY molecule appended after the real ones: its atoms sit on a line far away, its edges
    connect dummy atoms only (destination-sorted, after every real edge), and its energy - output row ``n_graphs`` - never
    enters the loss.  Real atoms share no edge with it and every per-node / per-graph op of the model is local, so outputs
    and parameter gradients of the real molecules are unchanged (the dummy's cotangent is exactly zero); the price is
    <= one quantum of extra atoms and edges per step.  One capture per ``(atoms_b, edges_b, graphs)`` bucket.
    """

    def __init__(self, model: torch.nn.Module, loss_fn: Callable[[torch.Tensor, torch.Tensor], torch.Tensor], bucket,
                 max_radius: float, atom_quantum: int = 128, edge_quantum: int = 2048, warmup: int = 2, max_cached: int = 16,
                 capture: bool = True):
        self.model, self.loss_fn, self.bucket = model, loss_fn, bucket
        self.max_radius, self.warmup, self.max_cached = max_radius, warmup, max_cached
        self.aq, self.eq, self.capture = int(atom_quantum), int(edge_quantum), capture
        self._cache: Dict[Tuple[int, int, int], _Captured] = {}
        self.captures = 0

    # ------------------------------------------------------------------ padding (pure torch, any device)
    def pad(self, pos, batch, z, src, dst):
        """Returns the padded ``(pos, batch, z, src, dst, row_ptr)`` and the bucket ``(atoms_b, edges_b)``."""
        G = int(batch.max()) + 1 if self._n_graphs is None else self._n_graphs
        return pad_to_bucket(pos, batch, z, src, dst, G, self.aq, self.eq)

    _n_graphs = None

    def _fwd_bwd(self, c: _Captured) -> torch.Tensor:
        c.csr._src_perm = c.csr._src_row_ptr = None
        G = c.target.shape[0]
        out = self.model.forward_edges(c.pos, c.batch, c.z, c.src, c.dst, graph=c.csr, n_graphs=G + 1)
        loss = self.loss_fn(out[:G], c.target)
        self.bucket.store(torch.autograd.grad(loss, self.bucket.params, allow_unused=True))
        return loss.detach()

    def _new(self, padded, target) -> _Captured:
        pos, batch, z, src, dst, row_ptr = padded
        c = _Captured()
        c.pos, c.batch, c.z, c.target = pos.clone(), batch.clone(), z.clone(), target.clone()
        c.src, c.dst, c.row_ptr = src.clone(), dst.clone(), row_ptr.clone()
        csr = ops.Graph.__new__(ops.Graph)
        csr.n_nodes, csr.n_edges, csr.perm = int(pos.shape[0]), int(src.numel()), None
        csr.src, csr.dst, csr.row_ptr = c.src, c.dst, c.row_ptr
        csr._src_perm = csr._src_row_ptr = None
        c.csr = csr
        c.graph = None
        if self.capture:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(self.warmup):
                    self._fwd_bwd(c)
            torch.cuda.current_stream().wait_stream(side)
            c.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(c.graph):
                c.loss = self._fwd_bwd(c)
            self.captures += 1
        return c

    def __call__(self, pos, batch, z, target) -> torch.Tensor:
        edge, _row_ptr = radius_graph_csr(pos, self.max_radius, batch, max_num_neighbors=1000)
        self._n_graphs = int(target.shape[0])
        padded, (Nb, Eb) = self.pad(pos, batch, z, edge[0], edge[1])
        key = (Nb, Eb, self._n_graphs)
        c = self._cache.get(key)
        if c is None:
            if len(self._cache) >= self.max_cached:
                self._cache.pop(next(iter(self._cache)))
            c = self._new(padded, target)
            self._cache[key] = c
        torch._foreach_copy_([c.pos, c.target], [padded[0], target])
        torch._foreach_copy_([c.batch, c.z, c.src, c.dst, c.row_ptr], [padded[1], padded[2], padded[3], padded[4], padded[5]])
        if c.graph is not None:
            c.graph.replay()
            return c.loss
        return self._fwd_bwd(c)


class DensTrainStep:
    """One DeNS training step of ``Equiformer_MD17_DeNS`` (reference ``main_md17_dens.py:379-406``, up to the optimiser):
    the noise of ``md17_dens_objective.add_masked_gaussian_noise``, the neighbour list, then forward (energy, forces by a
    ``create_graph`` backward, the denoising head), ``dens_loss`` and the backward to the parameters.

    Real training draws new conformers and new noise every step, so the edge count changes from step to step.  With
    ``capture=True`` the batch is padded by :func:`pad_to_bucket` (dummy atoms: ``atom_weight`` 0, never noised, zero force
    encoding; the dummy molecule's energy row stays out of the loss) and the forward + loss + backward is captured once per
    ``(atoms_b, edges_b, graphs)`` bucket through :class:`GraphedStep`, then replayed.  With ``capture=False`` the same step
    runs eagerly on the unpadded batch.  Noise, neighbour list and padding are eager in both cases.  Gradients land in
    ``bucket`` (a ``FlatGradAllReduce`` over the model's parameters); the call returns the loss."""

    def __init__(self, model: torch.nn.Module, bucket, task_mean=0.0, task_std=1.0, std: float = 0.05, prob: float = 0.25,
                 corrupt_ratio=0.25, w_e: float = 1.0, w_f: float = 80.0, atom_quantum: int = 32, edge_quantum: int = 512,
                 capture: bool = True, warmup: int = 2, max_cached: int = 16):
        self.model, self.bucket = model, bucket
        self.task_mean, self.task_std, self.std, self.prob, self.corrupt_ratio = task_mean, task_std, std, prob, corrupt_ratio
        self.w_e, self.w_f, self.aq, self.eq = w_e, w_f, int(atom_quantum), int(edge_quantum)
        self.graphed = GraphedStep(self._captured, bucket, warmup, max_cached) if capture else None
        self.last_edges = None

    @property
    def captures(self) -> int:
        return 0 if self.graphed is None else self.graphed.captures

    def _loss(self, pos, force, y, dy, noise_vec, atom_weight, w_dn, noise_mask, batch, z, graph, n_graphs):
        from .md17_dens_objective import dens_loss
        p = pos.detach().requires_grad_(True)
        energy, pred_dy = self.model.forward_edges(z, p, batch, graph.src, graph.dst, force=force, noise_mask=noise_mask,
                                                   graph=graph, n_graphs=n_graphs)
        return dens_loss(energy[:y.shape[0]], pred_dy, y, dy, noise_vec, noise_mask, self.task_mean, self.task_std, self.std,
                         self.w_e, self.w_f, w_dn, atom_weight)

    def _captured(self, pos, force, y, dy, noise_vec, atom_weight, w_dn, noise_mask, batch, z, src, dst, row_ptr):
        graph = csr_graph(src, dst, row_ptr, pos.shape[0])
        return self._loss(pos, force, y, dy, noise_vec, atom_weight, w_dn, noise_mask, batch, z, graph, y.shape[0] + 1)

    def __call__(self, pos, batch, z, y, dy, n_graphs: int, w_dn, generator=None) -> torch.Tensor:
        """``pos`` / ``dy`` ``[N, 3]``, ``batch`` / ``z`` ``[N]``, ``y`` ``[n_graphs, 1]``: the clean batch; ``w_dn`` the
        denoising weight of this step; ``generator`` the source of the noise draws."""
        from .md17_dens_objective import add_masked_gaussian_noise
        pos_n, noise_vec, noise_mask, _dpm, force = add_masked_gaussian_noise(
            pos, dy, batch, n_graphs, self.std, self.prob, self.corrupt_ratio, generator)
        edge, row_ptr = radius_graph_csr(pos_n, self.model.max_radius, batch, max_num_neighbors=1000)
        src, dst = edge[0], edge[1]
        self.last_edges = int(src.numel())
        w = w_dn.reshape(1) if isinstance(w_dn, torch.Tensor) else torch.full((1,), float(w_dn), dtype=pos.dtype,
                                                                                device=pos.device)
        if self.graphed is None:
            self.bucket.zero_grad()
            loss = self._loss(pos_n, force, y, dy, noise_vec, None, w, noise_mask, batch, z,
                              csr_graph(src, dst, row_ptr, pos.shape[0]), n_graphs)
            loss.backward()
            return loss.detach()
        (pos_p, batch_p, z_p, src_p, dst_p, row_ptr_p), (Nb, Eb) = pad_to_bucket(pos_n, batch, z, src, dst, n_graphs,
                                                                                  self.aq, self.eq)
        n_pad = Nb - int(pos.shape[0])
        rows = lambda t: torch.cat([t, t.new_zeros((n_pad,) + tuple(t.shape[1:]))])
        atom_weight = rows(torch.ones_like(pos[:, 0]))
        tensors = [pos_p, rows(force), y, rows(dy), rows(noise_vec), atom_weight, w, rows(noise_mask), batch_p, z_p, src_p,
                   dst_p, row_ptr_p]
        return self.graphed((Nb, Eb, n_graphs), tensors)
