"""Save and resume a training run in the reference trainers' checkpoint layout.

The file is a ``torch.save`` dict with the top-level keys of the OC20 trainer's training-state checkpoint
(``oc20/trainer/base_trainer_oc20.py:502-554``): ``epoch``, ``step``, ``state_dict``, ``optimizer`` (in
``torch.optim.AdamW``'s format), ``scheduler``, ``normalizers``, ``config``, ``val_metrics``, ``ema`` and ``amp``.  Two keys
are added: ``state_dict_ema`` (timm's key) when the optimiser keeps an EMA, and ``rng``.  ``ema`` and ``amp`` are ``None``:
the ocpmodels EMA format is not the one kept here, and the runs are fp32.

Loading writes into the existing tensors.  ``flatten_parameters`` made every parameter a view of one flat buffer, and the
captured steps of ``graphs`` hold the addresses of the parameters, the optimiser state and the EMA, so a load into live
objects is picked up by the next replay without a new capture.
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist


def _ddp_prefix(key: str) -> str:
    n = 0
    while key.startswith("module.", 7 * n):
        n += 1
    return "module." * n


def match_state_dict(state: dict, target: dict) -> dict:
    """``state`` keyed and ordered like ``target`` (a model's ``state_dict``).

    The ``module.`` prefixes of ``DistributedDataParallel`` / ``OCPDataParallel`` are stripped or added as the first keys
    of the two dicts call for, as the OC20 trainer does (``base_trainer_oc20.py:397-412``).  e3nn's ``…tp._w3j_*``
    buffers, which do not exist here, are dropped.  Any other missing or unexpected key, or a changed shape, raises a
    ``ValueError`` that names it."""
    theirs = _ddp_prefix(next(iter(state), ""))
    ours = _ddp_prefix(next(iter(target), ""))
    renamed, unexpected = {}, []
    for k, v in state.items():
        if k.rsplit(".", 1)[-1].startswith("_w3j_"):
            continue
        if k.startswith(theirs) and ours + k[len(theirs):] in target:
            renamed[ours + k[len(theirs):]] = v
        else:
            unexpected.append(k)
    missing = [k for k in target if k not in renamed]
    if missing or unexpected:
        raise ValueError(f"state_dict does not fit the model: missing keys {missing[:5]}"
                         f"{' ...' if len(missing) > 5 else ''}, unexpected keys {unexpected[:5]}"
                         f"{' ...' if len(unexpected) > 5 else ''}")
    for k, t in target.items():
        if tuple(renamed[k].shape) != tuple(t.shape):
            raise ValueError(f"state_dict: {k} has shape {tuple(renamed[k].shape)}, the model's has {tuple(t.shape)}")
    return {k: renamed[k] for k in target}


def _rng_state(generators) -> dict:
    return {"cpu": torch.get_rng_state(),
            "cuda": torch.cuda.get_rng_state() if torch.cuda.is_available() else None,
            "generators": [g.get_state() for g in generators]}


def save_training_state(path, model: torch.nn.Module, optimizer, *, epoch: int, step: int, scheduler=None,
                        normalizers=None, config=None, val_metrics=None, generators=()) -> None:
    """Write the training state of ``model`` and ``optimizer`` (``parallel.FlatAdamW`` or ``CapturableFlatAdamW``) to
    ``path``.

    ``scheduler`` and ``normalizers`` are stored as given, so pass them already serialisable (their ``state_dict()``).
    ``rng`` holds, per process, the CPU and current-CUDA generator states and those of ``generators`` (for example the
    noise generator of ``graphs.DensTrainStep``).  The file is written to a temporary name in the same directory and then
    renamed over ``path``, so an interrupted save leaves the previous checkpoint intact.  Under ``torch.distributed`` every
    process must call this: the RNG states are gathered, rank 0 writes, and all processes wait until the file is there."""
    rng = _rng_state(generators)
    distributed = dist.is_initialized() and dist.get_world_size() > 1
    if distributed:
        states = [None] * dist.get_world_size()
        dist.all_gather_object(states, rng)
    else:
        states = [rng]
    if not distributed or dist.get_rank() == 0:
        ckpt = {"epoch": epoch, "step": step, "state_dict": model.state_dict(), "optimizer": optimizer.state_dict(),
                "scheduler": scheduler, "normalizers": normalizers, "config": config, "val_metrics": val_metrics,
                "ema": None, "amp": None}
        if getattr(optimizer, "ema", None) is not None:
            ckpt["state_dict_ema"] = optimizer.ema_state_dict()
        ckpt["rng"] = states
        path = os.fspath(path)
        tmp = f"{path}.tmp{os.getpid()}"
        try:
            with open(tmp, "wb") as f:
                torch.save(ckpt, f)
                f.flush()
                os.fsync(f.fileno())
            os.replace(tmp, path)
        finally:
            if os.path.exists(tmp):
                os.remove(tmp)
    if distributed:
        dist.barrier()


def load_training_state(path, model: torch.nn.Module, optimizer=None, *, map_location=None, generators=()) -> dict:
    """Resume from a checkpoint of :func:`save_training_state`, of the reference's OC20 trainer, or an MD17 file
    (``{'state_dict': ...}`` alone, ``main_md17.py:248-265``, which loads the model only).

    The model is loaded in place through :func:`match_state_dict`, so its parameters stay views of the optimiser's flat
    buffer.  Then, with an ``optimizer``: its state when the file has one, and its EMA from ``state_dict_ema``; an
    optimiser that keeps an EMA restarts it from the loaded weights when the file has none, as timm's EMA does when it is
    built after the checkpoint is loaded.  Last, the RNG states, when the file was written by as many processes as are
    running now; each process takes its own.  ``generators`` must be the ones that were saved, in the same order.

    The file is unpickled, as the reference's trainers unpickle theirs: load only files you trust.  Returns ``epoch``,
    ``step``, ``scheduler``, ``normalizers`` and ``config``."""
    ckpt = torch.load(path, map_location=map_location, weights_only=False)
    states = ckpt.get("rng")
    distributed = dist.is_initialized() and dist.get_world_size() > 1
    world, rank = (dist.get_world_size(), dist.get_rank()) if distributed else (1, 0)
    rng = states[rank] if states is not None and len(states) == world else None
    if rng is not None and len(rng["generators"]) != len(generators):
        raise ValueError(f"rng: the file holds {len(rng['generators'])} generator states, {len(generators)} generators "
                         "were passed")
    model.load_state_dict(match_state_dict(ckpt["state_dict"], model.state_dict()))
    if optimizer is not None:
        if ckpt.get("optimizer") is not None:
            optimizer.load_state_dict(ckpt["optimizer"])
        if getattr(optimizer, "ema", None) is not None:
            ema = ckpt.get("state_dict_ema")
            optimizer.load_ema_state_dict(ema if ema is not None else model.state_dict())
    if rng is not None:
        torch.set_rng_state(rng["cpu"].cpu())
        if rng["cuda"] is not None and torch.cuda.is_available():
            torch.cuda.set_rng_state(rng["cuda"].cpu())
        for g, s in zip(generators, rng["generators"]):
            g.set_state(s.cpu())
    return {k: ckpt.get(k, 0 if k in ("epoch", "step") else None)
            for k in ("epoch", "step", "scheduler", "normalizers", "config")}
