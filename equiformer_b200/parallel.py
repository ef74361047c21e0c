"""Data-parallel plumbing: one process per GPU, one flat gradient bucket, one all-reduce per step.

Mirrors what the reference gets from ``DistributedDataParallel`` (``main_qm9.py:178-179``): molecules are
independent, so the forward/backward of the edge path needs no communication; only parameter gradients are
averaged.  The model has ~3.5 M fp32 parameters (14 MB) - latency-bound on NVLink 4 / NVSwitch - so all gradients
live as views of ONE contiguous buffer and a single NCCL all-reduce (in-switch NVLS reduction when available) is
issued per step; nothing is bucketed or copied.  Works with any ``torch.distributed`` backend (gloo in the CPU tests).
"""
from __future__ import annotations

import math
import os
from typing import Iterable, Optional

import torch
import torch.distributed as dist


def init_distributed(backend: Optional[str] = None) -> tuple:
    """env:// rendezvous like the reference's ``utils.init_distributed_mode`` (``utils.py:46-69``)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend == "nccl":
            torch.cuda.set_device(local)
            dist.init_process_group(backend, init_method="env://", world_size=world, rank=rank,
                                    device_id=torch.device("cuda", local))
        else:
            dist.init_process_group(backend, init_method="env://", world_size=world, rank=rank)
    return rank, local, world


class FlatGradAllReduce:
    """Gradients of ``params`` are views into one flat buffer; ``reduce()`` averages it across ranks in one call."""

    def __init__(self, params: Iterable[torch.nn.Parameter], process_group=None):
        self.params = [p for p in params if p.requires_grad]
        if not self.params:
            raise ValueError("no trainable parameters")
        first = self.params[0]
        # every tensor starts on a 256-byte boundary of the flat buffer (TMA / vector loads need 16-byte aligned rows)
        self.offsets, total = [], 0
        for p in self.params:
            self.offsets.append(total)
            total += (p.numel() + 63) // 64 * 64
        self.flat = torch.zeros(total, dtype=first.dtype, device=first.device)
        self.group = process_group
        for p, off in zip(self.params, self.offsets):
            p.grad = self.flat[off:off + p.numel()].view_as(p)
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1

    def zero_grad(self) -> None:
        self.flat.zero_()
        base = self.flat.untyped_storage().data_ptr()
        for p in self.params:  # keep the views attached even if an optimizer called zero_grad(set_to_none=True)
            if p.grad is None or p.grad.untyped_storage().data_ptr() != base:
                self._reattach()
                break

    def _reattach(self) -> None:
        for p, off in zip(self.params, self.offsets):
            p.grad = self.flat[off:off + p.numel()].view_as(p)

    def store(self, grads) -> None:
        """Write a list of gradients (``torch.autograd.grad(loss, self.params, allow_unused=True)``) into the flat
        buffer with one multi-tensor copy - instead of ~290 ``grad += g`` launches from autograd's accumulation."""
        views = [p.grad for p in self.params]
        if any(g is None for g in grads):
            self.flat.zero_()
        pairs = [(v, g) for v, g in zip(views, grads) if g is not None]
        torch._foreach_copy_([v for v, _ in pairs], [g.view_as(v) if g.shape != v.shape else g for v, g in pairs])

    def reduce(self, async_op: bool = False):
        """Average gradients over ranks (no-op for a single process)."""
        if self.world == 1:
            return None
        self.flat.div_(self.world)
        return dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=self.group, async_op=async_op)

    @property
    def nbytes(self) -> int:
        return self.flat.numel() * self.flat.element_size()


def broadcast_parameters(module: torch.nn.Module, src: int = 0) -> None:
    """Make every rank start from rank ``src``'s weights (what DDP does at construction)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return
    for t in list(module.parameters()) + list(module.buffers()):
        if t.numel() > 0:
            dist.broadcast(t.data, src)


def is_no_decay(name: str, skip_list=()) -> bool:
    """The reference's weight-decay exemption rule (``optim_factory.py:33-36``): by parameter name only."""
    return (name.endswith(".bias") or name.endswith(".affine_weight") or name.endswith(".affine_bias")
            or name.endswith(".mean_shift") or "bias." in name or name in skip_list)


class FlatAdamW:
    """AdamW over ONE flat parameter buffer (decoupled weight decay, bias correction as torch.optim.AdamW).

    The model has ~290 small parameter tensors; a multi-tensor optimiser step costs more GPU time in launch slots
    than the 14 MB of state deserve.  Parameters are re-pointed to views of one flat buffer (gradients already are,
    see :class:`FlatGradAllReduce`), so a step is six element-wise kernels on 3.5 M floats.  Weight decay follows the
    reference's ``add_weight_decay`` (``optim_factory.py:27-42``) by NAME, not by shape - e3nn keeps every
    ``tp.weight`` as a flat 1-D tensor and those are decayed: exempt are ``*.bias``, ``*.affine_weight``,
    ``*.affine_bias``, ``*.mean_shift``, names containing ``bias.`` (the ``ParameterList`` biases) and ``no_decay``
    (the model's ``no_weight_decay()`` skip list).
    """

    def __init__(self, named_params, bucket: FlatGradAllReduce, lr=5e-4, betas=(0.9, 0.999), eps=1e-8,
                 weight_decay=5e-3, no_decay=()):
        named = [(n, p) for n, p in named_params if p.requires_grad]
        if [p for _, p in named] != bucket.params and any(a is not b for (_, a), b in zip(named, bucket.params)):
            raise ValueError("FlatAdamW: parameter order must match the gradient bucket")
        self.bucket, self.lr, self.betas, self.eps = bucket, lr, betas, eps
        flat = torch.zeros_like(bucket.flat)
        decay = torch.zeros_like(bucket.flat)
        with torch.no_grad():
            for (name, p), off in zip(named, bucket.offsets):
                n = p.numel()
                flat[off:off + n].copy_(p.reshape(-1))
                p.data = flat[off:off + n].view_as(p)
                decay[off:off + n] = 0.0 if is_no_decay(name, no_decay) else weight_decay
        self.flat, self.decay = flat, decay
        self.m = torch.zeros_like(flat)
        self.v = torch.zeros_like(flat)
        self.t = 0

    @torch.no_grad()
    def step(self) -> None:
        self.t += 1
        b1, b2 = self.betas
        g = self.bucket.flat
        self.m.mul_(b1).add_(g, alpha=1 - b1)
        self.v.mul_(b2).addcmul_(g, g, value=1 - b2)
        self.flat.addcmul_(self.flat, self.decay, value=-self.lr)                 # p -= lr * wd * p
        denom = self.v.sqrt().div_(math.sqrt(1 - b2 ** self.t)).add_(self.eps)
        self.flat.addcdiv_(self.m, denom, value=-self.lr / (1 - b1 ** self.t))
