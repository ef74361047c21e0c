"""Captured evaluation passes with the reference drivers' validation metrics.

:class:`EvalPass` runs a model over a loader in eval mode and returns the metrics of the reference's evaluation loop for
its task family, in ocpmodels' evaluator layout ``{name: {"total", "numel", "metric"}}`` (``metric = total / numel``), so
the dict can go into ``checkpoint.save_training_state(..., val_metrics=...)``:

==============  ========================================================================================================
``qm9``         ``mae`` = sum |E std + mean - y| / graphs, ``loss`` = sum |E - (y - mean) / std| / graphs
                (``engine.evaluate``; its criterion is ``L1Loss`` whatever the training loss was)
``md17``        ``energy_mae`` = sum |E std + mean - y| / graphs, ``force_mae`` = sum |F std - dy| / (3 atoms),
                ``energy_loss`` = sum |E - (y - mean) / std| / graphs (the L2MAE of a one-wide output),
                ``force_loss`` = sum ||F - dy / std||_2 / atoms (``main_md17.evaluate``, ``main_md17_dens.evaluate``)
``oc20_is2re``  ``energy_mae``, ``energy_mse`` and ``energy_within_threshold`` (``|err| < 0.02``) per frame on the
                de-normalised energy; ``loss`` = the sum of the per-batch losses over the number of batches
                (``base_trainer_v2.validate`` with ocpmodels' ``Evaluator`` for ``is2re``)
==============  ========================================================================================================

Each entry equals the reference's ``AverageMeter.avg`` (a batch mean weighted by the batch's rows) in exact arithmetic.

Per batch, the neighbour list runs eagerly (``radius_graph_csr``, or ``radius_graph_pbc`` for OC20) and the batch is padded
to a bucket by ``graphs.pad_to_bucket``, with a dummy molecule after the real ones.  The forward and the metric kernels
of ``libeqf_b200_eval.so`` are captured once per ``(atoms_b, edges_b, graphs)`` bucket through ``graphs.GraphedStep`` and
replayed on static buffers; the kernels add each batch's terms to a float64 accumulator on the device, and the pass reads
it once at the end.  The MD17 and DeNS forces come from ``forward_edges`` as it is (a ``create_graph`` backward to the
positions), as in the reference's ``evaluate``; QM9 and OC20 run under ``no_grad``.

The captures hold the addresses of the parameters and buffers.  ``CapturableFlatAdamW.ema_weights()`` and
``checkpoint.load_training_state`` write the weights in place, so ``with opt.ema_weights(): ev.run(loader)`` evaluates
the EMA through the same captures, and a pass after a load evaluates the loaded weights.  Loading a state dict by
reassigning parameters would leave the captures reading the old storage.

:meth:`EvalPass.predict` is the OC20 trainer's ``predict`` (``energy_trainer_v2.py:134-225``) on the same padding and
captures: per bucket, the forward and ``eqf_predict_is2re`` of ``libeqf_b200_predict.so``, which de-normalises the energy
and, with ``write_pos``, adds the auxiliary head's de-normalised displacement to the moving atoms.  The batches need no
labels.  :func:`save_predictions` and :func:`save_pos_predictions` write the reference's results files.
"""
from __future__ import annotations

import os
from collections import defaultdict
from typing import Dict, Iterable, Optional

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from .checkpoint import atomic_write
from .eval_kernels import eval_atom_raw, eval_batch_raw, eval_graph_raw, new_scratch, predict_is2re_raw
from .graph import radius_graph_csr, radius_graph_pbc
from .graphs import GraphedStep, csr_graph, pad_to_bucket

TASKS = ("qm9", "md17", "oc20_is2re")
_G, _A = 0, _lib.EQF_EVAL_GRAPH_SLOTS                 # graph slots, then the atom (md17) or batch (oc20) slots
SLOTS = {"qm9": _A, "md17": _A + _lib.EQF_EVAL_ATOM_SLOTS, "oc20_is2re": _A + _lib.EQF_EVAL_BATCH_SLOTS}


def metrics_from_accumulator(task: str, acc) -> Dict[str, dict]:
    """The metrics of ``task`` from a filled accumulator (any float64 tensor of ``SLOTS[task]`` elements, read here)."""
    a = [float(x) for x in torch.as_tensor(acc).detach().double().cpu().reshape(-1)]
    graphs = int(a[_G + 4])
    if task == "qm9":
        pairs = {"mae": (a[_G], graphs), "loss": (a[_G + 3], graphs)}
    elif task == "md17":
        atoms = int(a[_A + 2])
        pairs = {"energy_mae": (a[_G], graphs), "force_mae": (a[_A], 3 * atoms),
                 "energy_loss": (a[_G + 3], graphs), "force_loss": (a[_A + 1], atoms)}
    elif task == "oc20_is2re":
        pairs = {"energy_mae": (a[_G], graphs), "energy_mse": (a[_G + 1], graphs),
                 "energy_within_threshold": (a[_G + 2], graphs), "loss": (a[_A], int(a[_A + 1]))}
    else:
        raise ValueError(f"task must be one of {TASKS}, got {task!r}")
    return {k: {"total": t, "numel": n, "metric": t / n if n else float("nan")} for k, (t, n) in pairs.items()}


def reduce_accumulator(acc: torch.Tensor, process_group=None) -> torch.Tensor:
    """Sum ``acc`` over the processes of ``process_group`` in place (one ``all_reduce``), as the OC20 trainer's
    ``distutils.all_reduce(total)`` / ``all_reduce(numel)`` does.  A no-op without ``torch.distributed``."""
    if dist.is_initialized() and dist.get_world_size(process_group) > 1:
        dist.all_reduce(acc, op=dist.ReduceOp.SUM, group=process_group)
    return acc


def pad_oc20(pos, batch, atomic_numbers, tags, src, dst, edge_vec, n_graphs: int, atom_quantum: int, edge_quantum: int):
    """:func:`graphs.pad_to_bucket` for a periodic OC20 batch.  Returns ``(edge_vec, batch, atomic_numbers, tags, src,
    dst, row_ptr)`` padded, and the bucket ``(atoms_b, edges_b)``.  The real edges keep their ``edge_vec`` (image offsets
    included); the dummy edges get ``pos[src] - pos[dst]`` of the padded positions, and the dummy atoms tag 0, outside
    the auxiliary task's mask."""
    (pos_p, batch_p, z_p, src_p, dst_p, row_ptr), (Nb, Eb) = pad_to_bucket(pos, batch, atomic_numbers, src, dst, n_graphs,
                                                                            atom_quantum, edge_quantum)
    E, N = int(src.numel()), int(pos.shape[0])
    dummy = pos_p.index_select(0, src_p[E:]) - pos_p.index_select(0, dst_p[E:])
    edge_vec_p = torch.cat([edge_vec, dummy.to(edge_vec.dtype)])
    tags_p = torch.cat([tags, tags.new_zeros(Nb - N)])
    return (edge_vec_p, batch_p, z_p, tags_p, src_p, dst_p, row_ptr), (Nb, Eb)


class EvalPass:
    """One evaluation pass of ``model`` over a loader: ``run(loader)`` returns the metrics (module docstring), and for
    ``oc20_is2re`` ``predict(loader)`` the de-normalised predictions of an unlabelled split.

    * ``task``: ``"qm9"`` (``GraphAttentionTransformer``), ``"md17"`` (the MD17 models and ``Equiformer_MD17_DeNS``,
      evaluated on clean data) or ``"oc20_is2re"`` (``GraphAttentionTransformerOC20``, with or without the auxiliary head).
    * ``task_mean`` / ``task_std``: the target normalisation; ``threshold``: the OC20 energy threshold.
    * ``target``: the QM9 column of ``y`` (None: ``y`` is the target itself).
    * ``positions_std``: the OC20 positions normaliser of the auxiliary target; ``aux_weight``: the initial weight of the
      auxiliary loss, a device scalar that :meth:`set_aux_weight` changes without a new capture.
    * ``max_neighbors``: the OC20 periodic neighbour cap (default: the model's).
    * ``capture=False`` runs the same kernels eagerly on the padded batches; ``max_cached`` bounds the captures, which
      live next to the training steps' own.

    Batches are read by attribute: ``pos``, ``batch``, ``z``, ``y`` (QM9: ``y[:, target]``; MD17 also ``dy``); OC20:
    ``pos``, ``batch``, ``atomic_numbers``, ``tags``, ``cell``, ``y_relaxed`` and, with the auxiliary head,
    ``pos_relaxed``.  The graph count is the target's length.

    A pass sets ``model.eval()`` and restores the previous mode afterwards, and leaves the parameters, the buffers, the
    gradient bucket and the CPU and CUDA generator states as it found them.  With ``all_reduce=True`` the accumulator is
    summed over ``process_group`` before it is read (a sharded loader); the QM9 and MD17 mains evaluate the whole loader
    on every rank and do not ask for it.
    """

    def __init__(self, model: torch.nn.Module, task: str, max_radius: float, task_mean: float = 0.0, task_std: float = 1.0,
                 *, target: Optional[int] = None, threshold: float = 0.02, positions_std: float = 1.0,
                 aux_weight: float = 1.0, max_neighbors: Optional[int] = None, atom_quantum: int = 128,
                 edge_quantum: int = 2048, capture: bool = True, warmup: int = 2, max_cached: int = 16,
                 process_group=None):
        if task not in TASKS:
            raise ValueError(f"task must be one of {TASKS}, got {task!r}")
        self.model, self.task, self.max_radius = model, task, float(max_radius)
        self.mean, self.std, self.threshold = float(task_mean), float(task_std), float(threshold)
        self.target, self.positions_std, self.group = target, float(positions_std), process_group
        self.max_neighbors = max_neighbors if max_neighbors is not None else getattr(model, "max_neighbors", 500)
        self.aux = task == "oc20_is2re" and bool(getattr(model, "use_auxiliary_task", False))
        self.aq, self.eq, self.capture = int(atom_quantum), int(edge_quantum), bool(capture)
        self.device = next(model.parameters()).device
        self.acc = torch.zeros(SLOTS[task], dtype=torch.float64, device=self.device)
        self._warm = torch.zeros_like(self.acc)          # the warm-up passes before a capture add here
        self._scratch = new_scratch(self.device)
        self.aux_weight = torch.full((1,), float(aux_weight), dtype=torch.float32, device=self.device)
        fn = {"qm9": self._qm9, "md17": self._md17, "oc20_is2re": self._oc20}[task]
        self._fn = fn
        self._graphed = GraphedStep(fn, None, warmup=warmup, max_cached=max_cached) if self.capture else None
        self._predicting = (GraphedStep(self._oc20_predict, None, warmup=warmup, max_cached=max_cached)
                            if self.capture and task == "oc20_is2re" else None)

    @property
    def captures(self) -> int:
        return 0 if self._graphed is None else self._graphed.captures

    @property
    def predict_captures(self) -> int:
        return 0 if self._predicting is None else self._predicting.captures

    def set_aux_weight(self, value: float) -> None:
        """The weight of the OC20 auxiliary loss in the following passes (a device write: no capture is invalidated)."""
        self.aux_weight.fill_(float(value))

    def run(self, loader: Iterable, all_reduce: bool = False) -> Dict[str, dict]:
        """One pass over ``loader``; returns ``{name: {"total", "numel", "metric"}}``."""
        was_training = self.model.training
        self.acc.zero_()
        self.model.eval()
        try:
            with torch.random.fork_rng(devices=[self.device] if self.device.type == "cuda" else []):
                for batch in loader:
                    self._update(batch)
        finally:
            self.model.train(was_training)
        if all_reduce:
            reduce_accumulator(self.acc, self.group)
        return metrics_from_accumulator(self.task, self.acc)

    def predict(self, loader: Iterable, write_pos: bool = False) -> dict:
        """The OC20 trainer's ``predict(loader, per_image=True)``: ``{"id": [str(sid), ...], "energy": [float, ...]}`` in
        loader order, the energies de-normalised with ``task_mean`` / ``task_std``.  With ``write_pos`` (the auxiliary
        head only) also ``"pos": {sid: float32 [natoms, 3] CPU tensor}``: the input positions plus the head's
        displacement times ``positions_std`` on the atoms with ``tags > 0``.

        Batches are read by attribute: ``pos``, ``batch``, ``atomic_numbers``, ``tags``, ``cell``, ``natoms`` and ``sid``;
        the frame count is ``natoms.numel()``.  The results stay on the device until the end of the pass, which reads
        them once.  Mode, weights and generator states are left as :meth:`run` leaves them."""
        if self.task != "oc20_is2re":
            raise ValueError(f"predict is the OC20 IS2RE trainer's pass; this EvalPass is for {self.task!r}")
        if write_pos and not self.aux:
            raise ValueError("write_pos needs the auxiliary head (use_auxiliary_task=True): it predicts the positions")
        was_training = self.model.training
        sids, natoms, energies, positions = [], [], [], []
        self.model.eval()
        try:
            with torch.random.fork_rng(devices=[self.device] if self.device.type == "cuda" else []):
                for batch in loader:
                    n_atoms = self._get(batch, "natoms").reshape(-1)
                    G = int(n_atoms.numel())
                    pos, padded, (Nb, Eb) = self._oc20_inputs(batch, G)
                    tensors = [*padded, n_atoms]
                    if write_pos:
                        tensors.append(torch.cat([pos.float(), pos.new_zeros(Nb - pos.shape[0], 3, dtype=torch.float32)]))
                    if self._predicting is not None:
                        energy, pos_out = self._predicting((Nb, Eb, G, write_pos), tensors)
                    else:
                        energy, pos_out = self._oc20_predict(*tensors)
                    energies.append(energy.clone())
                    if write_pos:
                        positions.append(pos_out[:pos.shape[0]].clone())
                        natoms.append(n_atoms)
                    sids.append(batch.sid)
        finally:
            self.model.train(was_training)
        out = {"id": [str(i) for s in sids for i in torch.as_tensor(s).reshape(-1).tolist()],
               "energy": torch.cat(energies).tolist() if energies else []}
        if write_pos:
            split = torch.split(torch.cat(positions).cpu(), torch.cat(natoms).tolist()) if positions else ()
            out["pos"] = {sid: p.clone() for sid, p in zip(out["id"], split)}
        return out

    # ------------------------------------------------------------------------------------------ per batch (eager)
    def _get(self, batch, name):
        return getattr(batch, name).to(self.device)

    def _oc20_inputs(self, batch, n_graphs: int):
        """The eager part of an OC20 batch: the periodic neighbour list, ``edge_vec`` with the image offsets, and
        :func:`pad_oc20`.  Returns ``(pos, padded, (atoms_b, edges_b))``."""
        pos, b, cell = self._get(batch, "pos"), self._get(batch, "batch"), self._get(batch, "cell")
        z, tags = self._get(batch, "atomic_numbers").long(), self._get(batch, "tags").long()
        edge, offs, _ = radius_graph_pbc(pos, b, cell, self.max_radius, self.max_neighbors)
        src, dst = edge[0], edge[1]
        cells = cell.to(pos.dtype).index_select(0, b.index_select(0, dst))
        edge_vec = (pos.index_select(0, src) - pos.index_select(0, dst)
                    + torch.bmm(offs.to(pos.dtype).view(-1, 1, 3), cells).view(-1, 3))
        padded, bucket = pad_oc20(pos, b, z, tags, src, dst, edge_vec, n_graphs, self.aq, self.eq)
        return pos, padded, bucket

    def _update(self, batch) -> None:
        dev = self.device
        if self.task == "oc20_is2re":
            y = self._get(batch, "y_relaxed").reshape(-1).float().contiguous()
            G = int(y.shape[0])
            pos, padded, (Nb, Eb) = self._oc20_inputs(batch, G)
            tensors = [padded[0], y, *padded[1:]]
            if self.aux:
                from .oc20_objective import relaxation_target
                aux_t = relaxation_target(pos, self._get(batch, "pos_relaxed"), self.positions_std)
                tensors.append(torch.cat([aux_t, aux_t.new_zeros(Nb - pos.shape[0], 3)]))
        else:
            pos, b, z = self._get(batch, "pos"), self._get(batch, "batch"), self._get(batch, "z")
            y = self._get(batch, "y")
            y = (y if self.target is None else y[:, self.target]).reshape(-1).float().contiguous()
            G = int(y.shape[0])
            edge, _ = radius_graph_csr(pos, self.max_radius, b, max_num_neighbors=1000)
            (pos_p, batch_p, z_p, src_p, dst_p, row_ptr), (Nb, Eb) = pad_to_bucket(pos, b, z, edge[0], edge[1], G,
                                                                                    self.aq, self.eq)
            if self.task == "qm9":
                tensors = [pos_p, y, batch_p, z_p, src_p, dst_p, row_ptr]
            else:
                dy = self._get(batch, "dy").float()
                n = int(pos.shape[0])
                dy_p = torch.cat([dy, dy.new_zeros(Nb - n, 3)])
                tensors = [pos_p, y, dy_p, torch.full((1,), n, dtype=torch.int64, device=dev), batch_p, z_p, src_p,
                           dst_p, row_ptr]
        if self._graphed is not None:
            self._graphed((Nb, Eb, G), tensors)
        else:
            self._fn(*tensors)

    # ------------------------------------------------------------------------------------------ captured region
    def _slots(self) -> torch.Tensor:
        # GraphedStep runs `warmup` eager passes before it captures: those must not count
        capturing = torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()
        return self.acc if (self._graphed is None or capturing) else self._warm

    def _graph_terms(self, energy, y, acc) -> None:
        eval_graph_raw(energy.detach().reshape(-1), y, y.shape[0], self.mean, self.std, self.threshold, acc[_G:_A],
                       self._scratch)

    def _qm9(self, pos, y, batch, z, src, dst, row_ptr):
        with torch.no_grad():
            energy = self.model.forward_edges(pos, batch, z, src, dst, graph=csr_graph(src, dst, row_ptr, pos.shape[0]),
                                              n_graphs=y.shape[0] + 1)
        self._graph_terms(energy, y, self._slots())

    def _md17(self, pos, y, dy, n_atoms, batch, z, src, dst, row_ptr):
        with torch.enable_grad():
            p = pos.detach().requires_grad_(True)
            energy, forces = self.model.forward_edges(z, p, batch, src, dst, graph=csr_graph(src, dst, row_ptr, p.shape[0]),
                                                      n_graphs=y.shape[0] + 1)
        acc = self._slots()
        self._graph_terms(energy, y, acc)
        eval_atom_raw(forces.detach().contiguous(), dy, n_atoms, self.std, acc[_A:], self._scratch)

    def _oc20(self, edge_vec, y, batch, z, tags, src, dst, row_ptr, *aux_target):
        from .oc20_objective import masked_l2mae
        G = y.shape[0]
        with torch.no_grad():
            out = self.model.forward_edges(edge_vec, batch, z, tags, src, dst,
                                           graph=csr_graph(src, dst, row_ptr, batch.shape[0]), n_graphs=G + 1)
            energy, aux = out if isinstance(out, tuple) else (out, None)
            # _compute_loss: L1 of the normalised energy, plus w * L2MAE of the auxiliary head on the moving atoms
            loss = (energy[:G].reshape(-1) - (y - self.mean) / self.std).abs().mean()
            if aux is not None:
                loss = loss + self.aux_weight[0] * masked_l2mae(aux, aux_target[0], tags)
        acc = self._slots()
        self._graph_terms(energy, y, acc)
        eval_batch_raw(loss.float().reshape(1), acc[_A:])

    def _oc20_predict(self, edge_vec, batch, z, tags, src, dst, row_ptr, n_atoms, *pos):
        """Captured per bucket: the forward, then the de-normalised energies ``[G]`` and, given the padded positions,
        the predicted positions ``[atoms_b, 3]`` (the dummy atoms, tag 0, keep their input rows)."""
        G = n_atoms.shape[0]
        with torch.no_grad():
            out = self.model.forward_edges(edge_vec, batch, z, tags, src, dst,
                                           graph=csr_graph(src, dst, row_ptr, batch.shape[0]), n_graphs=G + 1)
        energy, aux = out if isinstance(out, tuple) else (out, None)
        energy_out = torch.empty(G, dtype=torch.float32, device=edge_vec.device)
        if not pos:
            predict_is2re_raw(energy.reshape(-1), G, self.mean, self.std, energy_out)
            return energy_out, None
        pos_out = torch.empty_like(pos[0])
        predict_is2re_raw(energy.reshape(-1), G, self.mean, self.std, energy_out, pos[0], aux.contiguous(), tags,
                          self.positions_std, pos_out)
        return energy_out, pos_out


# ------------------------------------------------------------------------------------------------ results files
def _rank_world():
    distributed = dist.is_initialized() and dist.get_world_size() > 1
    return (dist.get_rank(), dist.get_world_size(), True) if distributed else (0, 1, False)


def save_predictions(predictions: dict, results_dir, results_file: str = "predictions", name: str = "is2re") -> str:
    """The OC20 trainer's ``save_results(predictions, results_file, keys=["energy"])`` (``base_trainer_oc20.py:707-757``).

    Every process writes its ``{name}_{results_file}_{rank}.npz`` (``ids`` as a numpy string array, ``energy`` as the
    float64 array numpy makes of the floats), then waits for the others.  Rank 0 reads the files in rank order, removes
    them, keeps each id once with ``np.unique(ids, return_index=True)`` (so the ids come out sorted as strings; a
    ``DistributedSampler`` repeats samples to even out the ranks) and writes ``{name}_{results_file}.npz``.  Every
    process returns its path once it is written.  Files are written under a temporary name and renamed."""
    rank, world, distributed = _rank_world()
    path_of = lambda suffix: os.path.join(os.fspath(results_dir), f"{name}_{results_file}{suffix}.npz")
    atomic_write(path_of(f"_{rank}"), lambda f: np.savez_compressed(f, ids=predictions["id"],
                                                                    energy=predictions["energy"]))
    if distributed:
        dist.barrier()
    if rank == 0:
        gathered = defaultdict(list)
        for i in range(world):
            with np.load(path_of(f"_{i}"), allow_pickle=True) as r:
                gathered["ids"].extend(r["ids"])
                gathered["energy"].extend(r["energy"])
            os.remove(path_of(f"_{i}"))
        _, idx = np.unique(gathered["ids"], return_index=True)
        result = {k: np.array(v)[idx] for k, v in gathered.items()}
        atomic_write(path_of(""), lambda f: np.savez_compressed(f, **result))
    if distributed:
        dist.barrier()
    return path_of("")


def save_pos_predictions(pos: dict, run_dir) -> str:
    """The ``write_pos`` files of the OC20 trainer's ``predict`` (``energy_trainer_v2.py:208-222``): every process writes
    ``pos_pred_{rank}.pt`` (``{sid: [natoms, 3] tensor}``, kept afterwards), then rank 0 gathers them in rank order into
    ``pos_pred.pt``, the first occurrence of an id winning.  Every process returns its path once it is written."""
    rank, world, distributed = _rank_world()
    run_dir = os.fspath(run_dir)
    atomic_write(os.path.join(run_dir, f"pos_pred_{rank}.pt"), lambda f: torch.save(pos, f))
    if distributed:
        dist.barrier()
    full = os.path.join(run_dir, "pos_pred.pt")
    if rank == 0:
        gathered = {}
        for i in range(world):
            for k, v in torch.load(os.path.join(run_dir, f"pos_pred_{i}.pt")).items():
                if k not in gathered:
                    gathered[k] = v
        atomic_write(full, lambda f: torch.save(gathered, f))
    if distributed:
        dist.barrier()
    return full
