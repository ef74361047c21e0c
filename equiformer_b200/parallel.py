"""Data-parallel plumbing: one process per GPU, one flat gradient bucket, one all-reduce per step.

Mirrors what the reference gets from ``DistributedDataParallel`` (``main_qm9.py:178-179``): molecules are
independent, so the forward/backward of the edge path needs no communication; only parameter gradients are
averaged.  The model has ~3.5 M fp32 parameters (14 MB) - latency-bound on NVLink 4 / NVSwitch - so all gradients
live as views of ONE contiguous buffer and a single NCCL all-reduce (in-switch NVLS reduction when available) is
issued per step; nothing is bucketed or copied.  Works with any ``torch.distributed`` backend (gloo in the CPU tests).
"""
from __future__ import annotations

import contextlib
import math
import os
from typing import Iterable, Optional

import torch
import torch.distributed as dist

from . import _lib


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


def flatten_parameters(named_params, bucket: FlatGradAllReduce, weight_decay: float, no_decay=()):
    """Re-point the trainable parameters to views of one flat buffer laid out as ``bucket.flat`` (same offsets, zero
    padding) and build the per-element weight decay by ``is_no_decay``.  Returns ``(names, flat, decay)``."""
    named = [(n, p) for n, p in named_params if p.requires_grad]
    if [p for _, p in named] != bucket.params and any(a is not b for (_, a), b in zip(named, bucket.params)):
        raise ValueError("the parameter order must match the gradient bucket")
    flat = torch.zeros_like(bucket.flat)
    decay = torch.zeros_like(bucket.flat)
    with torch.no_grad():
        for (name, p), off in zip(named, bucket.offsets):
            n = p.numel()
            flat[off:off + n].copy_(p.reshape(-1))
            p.data = flat[off:off + n].view_as(p)
            decay[off:off + n] = 0.0 if is_no_decay(name, no_decay) else weight_decay
    return [n for n, _ in named], flat, decay


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
        self.bucket, self.lr, self.betas, self.eps = bucket, lr, betas, eps
        _, self.flat, self.decay = flatten_parameters(named_params, bucket, weight_decay, no_decay)
        self.m = torch.zeros_like(self.flat)
        self.v = torch.zeros_like(self.flat)
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


class CapturableFlatAdamW:
    """:class:`FlatAdamW` with gradient-norm clipping and a model EMA, on the fused kernels of ``libeqf_b200_optim.so``.

    The learning rate ``lr`` and the step count ``t`` are device tensors, and :meth:`step` reads nothing from the host,
    so the step can run inside a captured CUDA graph (the ``after_backward`` hook of the steps in ``graphs``) and a
    schedule computed on the host changes the rate between replays through :meth:`set_lr`.

    * ``max_grad_norm``: ``torch.nn.utils.clip_grad_norm_`` over the flat gradient before the update (the OC20 trainer's
      ``clip_grad_norm``, timm's ``dispatch_clip_grad(mode='norm')``).  The clipped gradient is left in the bucket, as
      ``clip_grad_norm_`` leaves it in ``.grad``; ``grad_norm`` holds the norm before clipping (a device tensor).
    * ``ema_decay``: timm's ``ModelEmaV2`` of ``model``, updated after every step: ``ema = d ema + (1 - d) p`` for the
      parameters (in the AdamW kernel) and the floating-point buffers, a copy for the other buffers.
      :meth:`ema_state_dict` and :meth:`ema_weights` read it.

    Across processes, call ``bucket.reduce()`` and then :meth:`step` eagerly, so the averaged gradient is clipped, as
    DDP with ``clip_grad_norm_`` does.
    """

    def __init__(self, named_params, bucket: FlatGradAllReduce, lr=5e-4, betas=(0.9, 0.999), eps=1e-8,
                 weight_decay=5e-3, no_decay=(), max_grad_norm: Optional[float] = None,
                 ema_decay: Optional[float] = None, model: Optional[torch.nn.Module] = None):
        from . import optim_kernels
        if max_grad_norm is not None and not max_grad_norm > 0:
            raise ValueError("max_grad_norm must be positive")
        if ema_decay is not None and not (0.0 <= ema_decay <= 1.0 and model is not None):
            raise ValueError("ema_decay must be in [0, 1] and needs the model whose buffers the EMA follows")
        self.bucket, self.betas, self.eps = bucket, betas, eps
        self.max_grad_norm, self.ema_decay = max_grad_norm, ema_decay
        self._names, self.flat, self.decay = flatten_parameters(named_params, bucket, weight_decay, no_decay)
        dev = self.flat.device
        self.m = torch.zeros_like(self.flat)
        self.v = torch.zeros_like(self.flat)
        self.lr = torch.full((1,), float(lr), dtype=torch.float32, device=dev)
        self.t = torch.zeros(1, dtype=torch.int64, device=dev)
        self.coef = torch.ones(1, dtype=torch.float32, device=dev)
        self.grad_norm = torch.zeros(1, dtype=torch.float32, device=dev) if max_grad_norm is not None else None
        self._partials = torch.zeros(_lib.EQF_OPTIM_MAX_CTAS, dtype=torch.float64, device=dev)
        self._tickets = torch.zeros(2, dtype=torch.int32, device=dev)
        self.model, self.ema = model, None
        if ema_decay is not None:
            self.ema = self.flat.clone()
            params = set(self._names)
            # the model's persistent state other than the flat parameters, by state_dict key
            self._others = [(k, t.detach()) for k, t in model.state_dict(keep_vars=True).items() if k not in params]
            self._ema_others = [t.clone() for _, t in self._others]
            pairs = [(e, t) for e, (_, t) in zip(self._ema_others, self._others) if e.numel()]
            self._lerp = ([e for e, _ in pairs if e.is_floating_point()], [t for e, t in pairs if e.is_floating_point()])
            self._copy = ([e for e, _ in pairs if not e.is_floating_point()], [t for e, t in pairs if not e.is_floating_point()])
        # load both kernels now, on a 4-float scratch, so that a first step inside a capture only launches them
        s = torch.zeros(8, 4, dtype=torch.float32, device=dev)
        optim_kernels.flat_sqnorm_raw(s[0], 1.0, self._partials, self._tickets[0:1], s[1, :1], s[1, 1:2])
        optim_kernels.flat_adamw_raw(s[2], s[3], s[4], s[5], s[6], s[7], s[1, 2:3], s[1, 2:3], self.t.clone(),
                                     betas, eps, 0.0, self._tickets[1:2])

    def set_lr(self, value: float) -> None:
        """Write the learning rate of the following steps (a device write: no capture is invalidated)."""
        self.lr.fill_(float(value))

    @torch.no_grad()
    def step(self) -> None:
        from . import optim_kernels
        if self.bucket.world > 1 and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("CapturableFlatAdamW.step() inside a capture across processes would step on this rank's "
                               "gradient before the all-reduce: call bucket.reduce() and then step() eagerly")
        g = self.bucket.flat
        if self.max_grad_norm is not None:
            optim_kernels.flat_sqnorm_raw(g, self.max_grad_norm, self._partials, self._tickets[0:1], self.grad_norm,
                                          self.coef)
        optim_kernels.flat_adamw_raw(g, self.flat, self.m, self.v, self.decay, self.ema, self.coef, self.lr, self.t,
                                     self.betas, self.eps, self.ema_decay, self._tickets[1:2])
        if self.ema is not None:
            if self._lerp[0]:
                torch._foreach_lerp_(*self._lerp, 1.0 - self.ema_decay)
            if self._copy[0]:
                torch._foreach_copy_(*self._copy)

    def ema_state_dict(self) -> dict:
        """The EMA weights under the model's own ``state_dict`` keys (views of the optimiser's EMA state)."""
        if self.ema is None:
            raise RuntimeError("no EMA: construct the optimiser with ema_decay")
        out = {}
        for name, off, p in zip(self._names, self.bucket.offsets, self.bucket.params):
            out[name] = self.ema[off:off + p.numel()].view_as(p)
        out.update({k: e for (k, _), e in zip(self._others, self._ema_others)})
        keys = list(self.model.state_dict(keep_vars=True).keys())
        return {k: out[k] for k in keys}

    @contextlib.contextmanager
    def ema_weights(self):
        """Run the body with the EMA weights in the model (evaluation of ``model_ema.module``); the live weights come
        back bit for bit afterwards."""
        if self.ema is None:
            raise RuntimeError("no EMA: construct the optimiser with ema_decay")
        others = [t for _, t in self._others]
        with torch.no_grad():
            live, live_others = self.flat.clone(), [t.clone() for t in others]
            self.flat.copy_(self.ema)
            for t, e in zip(others, self._ema_others):
                t.copy_(e)
        try:
            yield self.model
        finally:
            with torch.no_grad():
                self.flat.copy_(live)
                for t, b in zip(others, live_others):
                    t.copy_(b)
