"""Learning-rate schedules from the reference's OWN ``oc20/trainer/lr_scheduler.py`` -> ``reference_lr_schedules.json``.

For each case an OC20 ``optim`` block is mapped as the trainer's ``load_extras`` (``base_trainer_v2.py``) maps it
(``epochs = max_epochs``, ``lr = lr_initial``, every ``scheduler_params`` key containing ``epochs`` multiplied by
``n_iter_per_epoch``) and handed to the reference's ``LRScheduler`` over a two-group ``torch.optim.AdamW`` (the groups of
``add_weight_decay``).  The run then does what ``energy_trainer_v2.py`` does every iteration: an optimiser step at the
group rate, then ``scheduler.step()``.  Stored per case:

  * ``optim``, ``n_iter_per_epoch``: the inputs;
  * ``rates``: the group rate of iterations 0 .. ``n_steps - 1``, past the end of the schedule;
  * ``states``: ``{step: {"scheduler": LambdaLR.state_dict(), "param_groups": the AdamW groups without params}}`` at a
    step inside the warm-up and one inside the cosine / between milestones, taken after ``step`` iterations.

Cases: the ``l1_256_nonlinear`` optim block (cosine) and a multistep block with three milestones.

Run where the reference checkout is: ``python tests/golden/make_reference_golden_lr.py <reference checkout>``.
"""
from __future__ import annotations

import copy
import importlib.util
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))

CASES = {
    # oc20/configs/is2re/all/graph_attention_transformer/l1_256_nonlinear_g@2_local.yml, optim block
    "oc20_cosine": {"optim": {"lr_initial": 0.0002, "max_epochs": 20, "scheduler": "LambdaLR",
                              "scheduler_params": {"lambda_type": "cosine", "warmup_factor": 0.2, "warmup_epochs": 2,
                                                   "lr_min_factor": 1.e-2}},
                    "n_iter_per_epoch": 7, "n_steps": 160, "state_steps": [9, 77]},
    "oc20_multistep": {"optim": {"lr_initial": 0.0005, "max_epochs": 20, "scheduler": "LambdaLR",
                                 "scheduler_params": {"lambda_type": "multistep", "warmup_factor": 0.1,
                                                      "warmup_epochs": 1, "decay_epochs": [4, 9, 15],
                                                      "decay_rate": 0.3}},
                       "n_iter_per_epoch": 7, "n_steps": 150, "state_steps": [3, 70]},
}


def _map(optim, n_iter_per_epoch):
    """base_trainer_v2.py load_extras: the epochs -> iterations mapping of the scheduler parameters."""
    optim = copy.deepcopy(optim)
    sp = optim["scheduler_params"]
    sp["epochs"] = optim["max_epochs"]
    sp["lr"] = optim["lr_initial"]
    for k in sp:
        if "epochs" in k:
            if isinstance(sp[k], list):
                sp[k] = [x * n_iter_per_epoch for x in sp[k]]
            elif isinstance(sp[k], (int, float)):
                sp[k] = sp[k] * n_iter_per_epoch
    return optim


def _jsonable(x):
    if isinstance(x, dict):
        return {str(k): _jsonable(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_jsonable(v) for v in x]
    if isinstance(x, torch.Tensor):
        return x.item()
    return x


def run_case(lr_scheduler, case):
    optim = _map(case["optim"], case["n_iter_per_epoch"])
    p0, p1 = torch.nn.Parameter(torch.zeros(3)), torch.nn.Parameter(torch.zeros(2, 2))
    opt = torch.optim.AdamW([{"params": [p0], "weight_decay": 0.0}, {"params": [p1], "weight_decay": 1e-3}],
                            lr=optim["lr_initial"])
    sched = lr_scheduler.LRScheduler(opt, optim)
    rates, states = [], {}
    for k in range(case["n_steps"]):
        if k in case["state_steps"]:
            groups = [{key: v for key, v in g.items() if key != "params"} for g in opt.state_dict()["param_groups"]]
            states[str(k)] = {"scheduler": sched.scheduler.state_dict(), "param_groups": groups}
        assert opt.param_groups[0]["lr"] == opt.param_groups[1]["lr"]
        rates.append(opt.param_groups[0]["lr"])
        for p in (p0, p1):
            p.grad = torch.zeros_like(p)
        opt.step()
        sched.step()
    return {"optim": case["optim"], "n_iter_per_epoch": case["n_iter_per_epoch"], "rates": rates, "states": states}


def main():
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    path = os.path.join(sys.argv[1], "oc20", "trainer", "lr_scheduler.py")
    spec = importlib.util.spec_from_file_location("ref_lr_scheduler", path)
    lr_scheduler = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(lr_scheduler)
    out = {"torch": torch.__version__, "cases": {name: run_case(lr_scheduler, case) for name, case in CASES.items()}}
    dest = os.path.join(HERE, "reference_lr_schedules.json")
    with open(dest, "w") as f:
        json.dump(_jsonable(out), f, indent=1)
    print("wrote", dest)


if __name__ == "__main__":
    main()
