"""Learning-rate schedules of the reference trainers, evaluated on the device inside the fused AdamW step.

A schedule is a function of the optimiser step count ``t`` (the count before the step: the k-th step, k = 0, 1, ...,
runs at ``lr_at(k)``).  :class:`LrSchedule` packs the ``EqfLrSchedule`` descriptor of ``include/eqf_b200_optim.h``; the
AdamW kernel evaluates it from the step count it already keeps, so a captured step replays a whole run with no host
write, and a resumed run lands on the right rate because the position is ``t``.  :meth:`LrSchedule.lr_at` evaluates the
same C function on the host (``eqf_lr_at``); there is no second formula in Python.

Kinds:
  * ``oc20_cosine`` / ``oc20_multistep``: ``oc20/trainer/lr_scheduler.py``'s ``CosineLRLambda`` / ``MultistepLRLambda``
    under torch's ``LambdaLR``, stepped every iteration (``energy_trainer_v2.py``), lengths in iterations.
  * ``timm_cosine``: timm 0.4.12's ``CosineLRScheduler`` as ``create_scheduler`` builds it for ``--sched cosine`` (the
    QM9, MD17 and DeNS mains), stepped at the start of every epoch, lengths in epochs.  Its expression is restated from
    timm 0.4.12's source, not executed against timm.

Scheduler state goes through the optimiser (``CapturableFlatAdamW.lr_schedule_state_dict`` / ``load_lr_schedule_state_dict``):
the OC20 kinds in ``LambdaLR.state_dict()``'s format, so a reference trainer's ``scheduler.scheduler.load_state_dict``
takes it and a reference checkpoint's ``scheduler`` entry loads here.
"""
from __future__ import annotations

import copy
import ctypes
from typing import Optional, Sequence

from . import _lib

N_GROUPS = 2          # the optimiser's groups (no weight decay, weight decay): both run at the one rate


def _lambda_lr_format() -> dict:
    """The keys of this torch's ``LambdaLR.state_dict()`` with the values a fresh scheduler holds, read from a
    ``LambdaLR`` over a one-parameter optimiser (as ``parallel._adamw_format`` reads ``AdamW``'s)."""
    import torch

    class _Probe:
        def __call__(self, step):
            return 1.0

    opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=1.0)
    return torch.optim.lr_scheduler.LambdaLR(opt, _Probe()).state_dict()


def _same(a, b) -> bool:
    if isinstance(a, (list, tuple)) or isinstance(b, (list, tuple)):
        return (isinstance(a, (list, tuple)) and isinstance(b, (list, tuple)) and len(a) == len(b)
                and all(_same(x, y) for x, y in zip(a, b)))
    try:
        return float(a) == float(b)
    except (TypeError, ValueError):
        return a == b


class LrSchedule:
    """One learning-rate schedule: the descriptor the AdamW kernel evaluates, and the reference's own parameters
    (``params``: the ``LambdaLR`` lambda's ``__dict__``, or timm's attribute names) for the state dicts.

    Build it with :meth:`from_oc20_optim`, :meth:`oc20_lambda_lr` or :meth:`timm_cosine`.  The descriptor is checked by
    ``eqf_lr_schedule_check``; a refused one raises ``ValueError`` with the library's reason."""

    def __init__(self, kind: str, base_lr: float, warmup: float, warmup_start: float, *, total: float = 0.0,
                 min_value: float = 0.0, milestones: Sequence[float] = (), gamma: float = 1.0, steps_per_unit: int = 1,
                 params: Optional[dict] = None):
        if kind not in _lib.EQF_LR_KINDS:
            raise ValueError(f"unknown schedule kind {kind!r}: one of {sorted(_lib.EQF_LR_KINDS)}")
        milestones = [float(x) for x in milestones]
        if len(milestones) > _lib.EQF_LR_MAX_MILESTONES:
            raise ValueError(f"{len(milestones)} milestones: at most {_lib.EQF_LR_MAX_MILESTONES} (EQF_LR_MAX_MILESTONES)")
        d = _lib.EqfLrSchedule()
        d.kind, d.n_milestones, d.steps_per_unit = _lib.EQF_LR_KINDS[kind], len(milestones), int(steps_per_unit)
        d.base_lr, d.warmup, d.warmup_start = float(base_lr), float(warmup), float(warmup_start)
        d.total, d.min_value, d.gamma = float(total), float(min_value), float(gamma)
        for i, x in enumerate(milestones):
            d.milestones[i] = x
        lib = _lib.load_optim()
        if lib.eqf_lr_schedule_check(ctypes.byref(d)) != 0:
            raise ValueError(lib.eqf_last_error().decode())
        self.kind, self.descriptor, self.params = kind, d, dict(params or {})

    # ------------------------------------------------------------------------------------------------ constructors
    @classmethod
    def oc20_lambda_lr(cls, lr: float, lambda_type: str, warmup_steps: float, warmup_factor: float, *,
                       max_steps: Optional[float] = None, lr_min_factor: Optional[float] = None,
                       decay_steps: Sequence[float] = (), decay_rate: Optional[float] = None) -> "LrSchedule":
        """The OC20 trainer's ``LambdaLR`` from step counts: ``lambda_type`` ``'cosine'`` (``max_steps``,
        ``lr_min_factor``) or ``'multistep'`` (``decay_steps``, ``decay_rate``); lengths in iterations."""
        if lambda_type == "cosine":
            if max_steps is None or lr_min_factor is None:
                raise ValueError("a cosine LambdaLR needs max_steps and lr_min_factor")
            params = {"warmup_epochs": warmup_steps, "lr_warmup_factor": warmup_factor, "max_epochs": max_steps,
                      "lr_min_factor": lr_min_factor}
            return cls("oc20_cosine", lr, warmup_steps, warmup_factor, total=max_steps, min_value=lr_min_factor,
                       params=params)
        if lambda_type == "multistep":
            if decay_rate is None:
                raise ValueError("a multistep LambdaLR needs decay_rate")
            params = {"warmup_epochs": warmup_steps, "lr_warmup_factor": warmup_factor,
                      "lr_decay_epochs": list(decay_steps), "lr_gamma": decay_rate}
            return cls("oc20_multistep", lr, warmup_steps, warmup_factor, milestones=decay_steps, gamma=decay_rate,
                       params=params)
        raise ValueError(f"lambda_type {lambda_type!r}: the OC20 LRScheduler accepts 'cosine' and 'multistep'")

    @classmethod
    def from_oc20_optim(cls, optim_cfg: dict, n_iter_per_epoch: int) -> "LrSchedule":
        """The schedule an OC20 config's ``optim`` block gives, mapped as ``base_trainer_v2.py``'s ``load_extras`` maps
        it: ``epochs = max_epochs``, ``lr = lr_initial``, and every ``scheduler_params`` key containing ``epochs``
        (lists included) multiplied by ``n_iter_per_epoch``.  ``optim_cfg`` is not modified."""
        if int(optim_cfg.get("grad_accumulation_steps", 1)) != 1:
            raise ValueError("grad_accumulation_steps != 1: gradient accumulation is not supported")
        if optim_cfg.get("scheduler") != "LambdaLR":
            raise ValueError(f"scheduler {optim_cfg.get('scheduler')!r}: only LambdaLR (cosine or multistep) runs on "
                             "the device")
        sp = copy.deepcopy(optim_cfg["scheduler_params"])
        sp["epochs"] = optim_cfg["max_epochs"]
        sp["lr"] = optim_cfg["lr_initial"]
        for k in sp:
            if "epochs" in k:
                if isinstance(sp[k], list):
                    sp[k] = [x * n_iter_per_epoch for x in sp[k]]
                elif isinstance(sp[k], (int, float)):
                    sp[k] = sp[k] * n_iter_per_epoch
        kind = sp.get("lambda_type")
        if kind not in ("cosine", "multistep"):
            raise ValueError(f"lambda_type {kind!r}: the OC20 LRScheduler accepts 'cosine' and 'multistep'")
        if kind == "cosine":
            return cls.oc20_lambda_lr(sp["lr"], kind, sp["warmup_epochs"], sp["warmup_factor"], max_steps=sp["epochs"],
                                      lr_min_factor=sp["lr_min_factor"])
        return cls.oc20_lambda_lr(sp["lr"], kind, sp["warmup_epochs"], sp["warmup_factor"],
                                  decay_steps=sp["decay_epochs"], decay_rate=sp["decay_rate"])

    @classmethod
    def timm_cosine(cls, steps_per_epoch: int, lr: float = 5e-4, epochs: int = 300, warmup_epochs: int = 5,
                    warmup_lr: float = 1e-6, min_lr: float = 1e-5) -> "LrSchedule":
        """timm's cosine schedule of the QM9 / MD17 / DeNS mains, one rate per epoch of ``steps_per_epoch`` iterations
        (their loaders drop the last batch, so every epoch has as many).  The defaults are ``main_qm9.py``'s; the MD17
        and DeNS mains use ``epochs=1000, warmup_epochs=10, min_lr=1e-6``."""
        params = {"base_values": [float(lr)] * N_GROUPS, "t_initial": epochs, "lr_min": min_lr,
                  "warmup_t": warmup_epochs, "warmup_lr_init": warmup_lr, "t_mul": 1.0, "cycle_limit": 1,
                  "warmup_prefix": False, "steps_per_epoch": int(steps_per_epoch)}
        return cls("timm_cosine", lr, warmup_epochs, warmup_lr, total=epochs, min_value=min_lr,
                   steps_per_unit=steps_per_epoch, params=params)

    # ------------------------------------------------------------------------------------------------ evaluation
    @property
    def base_lr(self) -> float:
        return float(self.descriptor.base_lr)

    @property
    def is_oc20(self) -> bool:
        return self.kind.startswith("oc20_")

    def lr_at(self, t: int) -> float:
        """The rate of the step whose count before the step is ``t``, by the C function the kernel runs."""
        out = ctypes.c_double()
        lib = _lib.load_optim()
        if lib.eqf_lr_at(ctypes.byref(self.descriptor), int(t), ctypes.byref(out)) != 0:
            raise ValueError(lib.eqf_last_error().decode())
        return out.value

    # ------------------------------------------------------------------------------------------------ state
    def state_dict(self, t: int) -> dict:
        """The scheduler state at step count ``t``.  OC20 kinds: this torch's ``LambdaLR.state_dict()`` layout with
        ``last_epoch = t`` (the trainer steps the scheduler once per optimiser step), ``_step_count = t + 1`` and the
        lambda's attributes under ``lr_lambdas``.  timm kind: its parameters under timm's attribute names and
        ``last_epoch = t``, the optimiser step count (no reference main saves a timm scheduler, so this layout is ours)."""
        t = int(t)
        if not self.is_oc20:
            return dict(copy.deepcopy(self.params), last_epoch=t)
        out = {}
        for k, v in _lambda_lr_format().items():
            if k == "base_lrs":
                out[k] = [self.base_lr] * N_GROUPS
            elif k == "last_epoch":
                out[k] = t
            elif k == "_step_count":
                out[k] = t + 1
            elif k == "_last_lr":
                out[k] = [self.lr_at(t)] * N_GROUPS
            elif k == "lr_lambdas":
                out[k] = [copy.deepcopy(self.params) for _ in range(N_GROUPS)]
            else:
                out[k] = v
        return out

    def check_state_dict(self, state: dict, t: int) -> None:
        """Raise ``ValueError`` naming the key when ``state`` (ours or a reference checkpoint's ``scheduler``) is not
        this schedule at step count ``t``: other base rates or group count, other lambda / timm parameters, or
        ``last_epoch != t``.  Other keys (``_step_count``, ``_last_lr`` and the bookkeeping of other torch versions:
        ``verbose``, ``_is_initial``, ``_get_lr_called_within_step``) follow from these and are ignored."""
        if not isinstance(state, dict):
            raise ValueError(f"scheduler state: expected a dict, got {type(state).__name__}")
        if self.is_oc20:
            for key in ("base_lrs", "last_epoch", "lr_lambdas"):
                if key not in state:
                    raise ValueError(f"scheduler state: no {key} (not a LambdaLR state_dict)")
            base = list(state["base_lrs"])
            if len(base) != N_GROUPS:
                raise ValueError(f"base_lrs: {len(base)} groups, the optimiser has {N_GROUPS}")
            if not all(float(b) == self.base_lr for b in base):
                raise ValueError(f"base_lrs: {base} differ from the schedule's base rate {self.base_lr}")
            lambdas = list(state["lr_lambdas"])
            if len(lambdas) != N_GROUPS:
                raise ValueError(f"lr_lambdas: {len(lambdas)} lambdas, the optimiser has {N_GROUPS} groups")
            for i, lam in enumerate(lambdas):
                if not isinstance(lam, dict) or set(lam) != set(self.params):
                    got = sorted(lam) if isinstance(lam, dict) else lam
                    raise ValueError(f"lr_lambdas[{i}]: attributes {got}, the schedule's lambda has "
                                     f"{sorted(self.params)}")
                for k, v in self.params.items():
                    if not _same(lam[k], v):
                        raise ValueError(f"lr_lambdas[{i}]: {k} = {lam[k]}, the schedule has {v}")
        else:
            for k, v in self.params.items():
                if k not in state:
                    raise ValueError(f"scheduler state: no {k} (not a timm_cosine state)")
                if not _same(state[k], v):
                    raise ValueError(f"{k} = {state[k]}, the schedule has {v}")
            if "last_epoch" not in state:
                raise ValueError("scheduler state: no last_epoch")
        last = state["last_epoch"]
        if float(last) != int(t):
            raise ValueError(f"last_epoch = {last}, but the optimiser's step count is {int(t)}: load the optimiser "
                             "state first (without gradient accumulation the two are equal)")
