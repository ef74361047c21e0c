"""Learning-rate schedules evaluated inside the fused AdamW step (``lr_schedule.LrSchedule``, ``eqf_flat_adamw_scheduled``).

CPU: ``eqf_lr_at`` (the C function the kernel runs) against the rates of the reference's own ``LRScheduler``
(``tests/golden/reference_lr_schedules.json``) and against a restatement of timm 0.4.12's cosine schedule; the OC20 config
mapping; every refusal of ``eqf_lr_schedule_check`` and of the state loads; the ``LambdaLR`` state dicts both ways.

GPU: the scheduled kernel over 150 seeded steps against the float64 recipe of ``test_optim.py`` at the reference's rates;
a captured QM9 step following the schedule replay by replay, against host ``set_lr``; bitwise resume through
``save_training_state`` / ``load_training_state``; resume from the reference's state dicts; the floor at t ~ 1e9.
"""
from __future__ import annotations

import ctypes
import json
import math
import os
import re

import numpy as np
import pytest
import torch

from tests.helpers import rel_err

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "reference_lr_schedules.json")
TIMM = dict(lr=1e-2, epochs=25, warmup_epochs=3, warmup_lr=1e-6, min_lr=1e-5)     # 5 iterations per epoch below


def _fixture():
    with open(FIXTURE) as f:
        return json.load(f)["cases"]


def _schedule(name):
    from equiformer_b200.lr_schedule import LrSchedule
    if name == "timm_cosine":
        return LrSchedule.timm_cosine(5, **TIMM)
    case = _fixture()[name]
    return LrSchedule.from_oc20_optim(case["optim"], case["n_iter_per_epoch"])


def timm_0412_cosine(epoch, lr, epochs, warmup_epochs, warmup_lr, min_lr):
    """timm 0.4.12 CosineLRScheduler._get_lr with create_scheduler's arguments (t_mul 1, decay_rate 0.1, cycle_limit 1,
    warmup_prefix False), restated from its source."""
    t, t_initial, t_mul, decay_rate, cycle_limit = epoch, epochs, 1.0, 0.1, 1
    if t < warmup_epochs:
        return warmup_lr + t * ((lr - warmup_lr) / warmup_epochs)
    i = t // t_initial
    t_i = t_initial
    t_curr = t - (t_initial * i)
    gamma = decay_rate ** i
    lr_min = min_lr * gamma
    lr_max = lr * gamma
    if cycle_limit == 0 or (cycle_limit > 0 and i < cycle_limit):
        return lr_min + 0.5 * (lr_max - lr_min) * (1 + math.cos(math.pi * t_curr / t_i))
    return min_lr


def _rates(name, n):
    """The reference's rate of iterations 0 .. n - 1."""
    if name == "timm_cosine":
        return [timm_0412_cosine(k // 5, **TIMM) for k in range(n)]
    return _fixture()[name]["rates"][:n]


def _f32_ulps(a, b):
    """Distance of two float32 values in units in the last place."""
    ia, ib = np.array([a], np.float32).view(np.int32)[0], np.array([b], np.float32).view(np.int32)[0]
    return abs(int(ia) - int(ib))


# ------------------------------------------------------------------------------------------------ CPU: the function
def test_header_layout_matches_ctypes():
    from equiformer_b200 import _lib
    header = open(os.path.join(os.path.dirname(HERE), "include", "eqf_b200_optim.h")).read()
    assert int(re.search(r"#define EQF_LR_MAX_MILESTONES (\d+)", header).group(1)) == _lib.EQF_LR_MAX_MILESTONES
    for name, value in _lib.EQF_LR_KINDS.items():
        assert re.search(rf"EQF_LR_{name.upper()} = (\d+)", header).group(1) == str(value)
    body = re.search(r"typedef struct EqfLrSchedule \{(.*?)\} EqfLrSchedule;", header, re.S).group(1)
    fields = re.findall(r"^\s*\w+ (\w+)(?:\[\w+\])?;", body, re.M)
    assert fields == [f for f, _ in _lib.EqfLrSchedule._fields_]


@pytest.mark.parametrize("name", ["oc20_cosine", "oc20_multistep"])
def test_lr_at_matches_the_reference_scheduler(built_lib, name):
    """Every iteration of the reference's LRScheduler, past the end of the schedule, within 2 ulp in double."""
    sched, rates = _schedule(name), _fixture()[name]["rates"]
    for k, r in enumerate(rates):
        got = sched.lr_at(k)
        assert abs(got - r) <= 2 * math.ulp(r), (k, got, r)
    assert sched.lr_at(10 ** 9) == rates[-1]


def test_timm_cosine_matches_the_restatement(built_lib):
    """Every epoch, from the warm-up start through the switch at W, T - 1 and past T; every iteration of an epoch runs
    at the epoch's rate."""
    from equiformer_b200.lr_schedule import LrSchedule
    for spe in (1, 5):
        sched = LrSchedule.timm_cosine(spe, **TIMM)
        for e in list(range(TIMM["epochs"] + 3)) + [10 ** 6]:
            ref = timm_0412_cosine(e, **TIMM)
            for j in {0, spe - 1}:
                got = sched.lr_at(e * spe + j)
                assert abs(got - ref) <= 2 * math.ulp(ref), (spe, e, j, got, ref)
    s = LrSchedule.timm_cosine(4)                                       # main_qm9.py's defaults
    assert s.lr_at(0) == 1e-6 and s.lr_at(4 * 300) == 1e-5
    assert LrSchedule.timm_cosine(3, warmup_epochs=0).lr_at(0) == 5e-4          # timm: no warm-up when warmup_t = 0


def test_oc20_config_mapping(built_lib):
    """base_trainer_v2.py load_extras: epochs -> iterations for every key containing `epochs`, lists included; the
    lambda parameters are the reference lambdas' attributes; the config is left as it was."""
    from equiformer_b200.lr_schedule import LrSchedule
    for name, case in _fixture().items():
        before = json.dumps(case["optim"], sort_keys=True)
        sched = LrSchedule.from_oc20_optim(case["optim"], case["n_iter_per_epoch"])
        assert json.dumps(case["optim"], sort_keys=True) == before
        ref = next(iter(case["states"].values()))["scheduler"]["lr_lambdas"][0]
        assert sched.params == ref and sched.kind == name
    sp = {"lambda_type": "cosine", "warmup_factor": 0.2, "warmup_epochs": 0.5, "lr_min_factor": 0.01}
    s = LrSchedule.from_oc20_optim({"lr_initial": 1e-3, "max_epochs": 3, "scheduler": "LambdaLR",
                                    "scheduler_params": sp}, 10)
    assert s.params == {"warmup_epochs": 5.0, "lr_warmup_factor": 0.2, "max_epochs": 30, "lr_min_factor": 0.01}
    explicit = LrSchedule.oc20_lambda_lr(1e-3, "cosine", 5.0, 0.2, max_steps=30, lr_min_factor=0.01)
    assert [explicit.lr_at(k) for k in range(40)] == [s.lr_at(k) for k in range(40)]
    base = {"lr_initial": 1e-3, "max_epochs": 3, "scheduler": "LambdaLR", "scheduler_params": sp}
    for bad, match in (({"grad_accumulation_steps": 2}, "accumulation"), ({"scheduler": "ReduceLROnPlateau"}, "LambdaLR"),
                       ({"scheduler_params": dict(sp, lambda_type="step")}, "lambda_type")):
        with pytest.raises(ValueError, match=match):
            LrSchedule.from_oc20_optim(dict(base, **bad), 10)


def _desc(**kw):
    from equiformer_b200 import _lib
    d = _lib.EqfLrSchedule()
    vals = dict(kind=1, n_milestones=0, steps_per_unit=1, base_lr=1e-3, warmup=10.0, warmup_start=0.2, total=100.0,
                min_value=0.01, gamma=0.5)
    vals.update(kw)
    ms = vals.pop("milestones", ())
    for k, v in vals.items():
        setattr(d, k, v)
    for i, x in enumerate(ms):
        d.milestones[i] = x
    return d


def test_schedule_check_refusals(built_lib):
    from equiformer_b200 import _lib
    lib = _lib.load_optim()
    check = lambda d: lib.eqf_lr_schedule_check(ctypes.byref(d))
    msg = lambda: lib.eqf_last_error().decode()
    assert check(_desc()) == 0 and check(_desc(kind=2, total=0.0, n_milestones=3, milestones=(5, 5, 9))) == 0
    assert check(_desc(kind=3, warmup=0.0)) == 0
    cases = [(_desc(kind=0), "kind"), (_desc(kind=7), "kind"), (_desc(warmup=0.0), "warm-up"),
             (_desc(warmup=-1.0), "warm-up"), (_desc(kind=3, warmup=-1.0), "warm-up"),
             (_desc(warmup=float("nan")), "warm-up"), (_desc(total=0.0), "total"), (_desc(kind=3, total=-5.0), "total"),
             (_desc(steps_per_unit=0), "steps_per_unit"), (_desc(kind=2, n_milestones=9), "milestones"),
             (_desc(kind=2, n_milestones=-1), "milestones"),
             (_desc(kind=2, n_milestones=3, milestones=(5, 9, 7)), "sorted"),
             (_desc(kind=2, n_milestones=1, milestones=(float("inf"),)), "finite"),
             (_desc(base_lr=-1e-3), "negative"), (_desc(base_lr=float("inf")), "negative"),
             (_desc(min_value=float("nan")), "negative"), (_desc(kind=3, warmup_start=-1e-6), "negative"),
             (_desc(kind=2, gamma=-0.5), "negative"),
             (_desc(kind=2, gamma=1e200, n_milestones=2, milestones=(1, 2)), "non-finite")]
    for d, match in cases:
        assert check(d) != 0 and match in msg(), (match, msg())
    out = ctypes.c_double()
    assert lib.eqf_lr_at(ctypes.byref(_desc()), -1, ctypes.byref(out)) != 0 and ">= 0" in msg()
    assert lib.eqf_lr_at(ctypes.byref(_desc(total=0.0)), 3, ctypes.byref(out)) != 0
    from equiformer_b200.lr_schedule import LrSchedule
    with pytest.raises(ValueError, match="warm-up"):
        LrSchedule.oc20_lambda_lr(1e-3, "cosine", 0, 0.2, max_steps=10, lr_min_factor=0.01)
    with pytest.raises(ValueError, match="at most"):
        LrSchedule.oc20_lambda_lr(1e-3, "multistep", 2, 0.2, decay_steps=list(range(3, 12)), decay_rate=0.1)


# ------------------------------------------------------------------------------------------------ CPU: state dicts
class _CosineLambda:
    """A lambda with the attribute names of the reference's CosineLRLambda (its formula is not needed here)."""

    def __init__(self):
        self.warmup_epochs, self.lr_warmup_factor, self.max_epochs, self.lr_min_factor = 1, 0.5, 2, 0.5

    def __call__(self, step):
        return 1.0


def test_our_state_loads_into_torch_lambda_lr(built_lib):
    """The dict of an OC20 cosine schedule at t = 50 loads into a torch LambdaLR over two groups; the scheduler then
    holds our step count, base rates, rate and lambda attributes."""
    sched = _schedule("oc20_cosine")
    sd = sched.state_dict(50)
    params = [torch.nn.Parameter(torch.zeros(2)) for _ in range(2)]
    opt = torch.optim.AdamW([{"params": [params[0]]}, {"params": [params[1]]}], lr=0.123)
    lam = _CosineLambda()
    torch_sched = torch.optim.lr_scheduler.LambdaLR(opt, lam)
    assert set(sd) == set(torch_sched.state_dict())
    torch_sched.load_state_dict(sd)
    assert torch_sched.last_epoch == 50 and torch_sched._step_count == 51
    assert torch_sched.base_lrs == [sched.base_lr] * 2 and torch_sched.get_last_lr() == [sched.lr_at(50)] * 2
    assert lam.__dict__ == sched.params
    sched.check_state_dict(sd, 50)


@pytest.mark.parametrize("name", ["oc20_cosine", "oc20_multistep"])
def test_reference_state_loads_and_refusals(built_lib, name):
    """The reference's LambdaLR dicts (and a torch 1.10 variant with `verbose`) fit the schedule at their step; every
    mismatch raises ValueError naming the key."""
    sched = _schedule(name)
    for step, st in _fixture()[name]["states"].items():
        ref, t = st["scheduler"], int(step)
        sched.check_state_dict(ref, t)
        sched.check_state_dict(dict(ref, verbose=False), t)
        assert ref["_last_lr"][0] == sched.lr_at(t)
        ours = sched.state_dict(t)
        assert {k: ours[k] for k in ref} == ref
        lam_key = next(iter(ref["lr_lambdas"][0]))
        bad = [(dict(ref, base_lrs=[1.0, 1.0]), "base_lrs"), (dict(ref, base_lrs=ref["base_lrs"] * 2), "base_lrs"),
               (dict(ref, last_epoch=t + 1), "last_epoch"), (dict(ref, lr_lambdas=ref["lr_lambdas"][:1]), "lr_lambdas"),
               (dict(ref, lr_lambdas=[dict(ref["lr_lambdas"][0], **{lam_key: 999})] * 2), lam_key),
               (dict(ref, lr_lambdas=[{"other": 1}] * 2), "lr_lambdas"),
               ({k: v for k, v in ref.items() if k != "last_epoch"}, "last_epoch"), ("state", "dict")]
        for state, match in bad:
            with pytest.raises(ValueError, match=match):
                sched.check_state_dict(state, t)
    other = "oc20_multistep" if name == "oc20_cosine" else "oc20_cosine"
    theirs = next(iter(_fixture()[other]["states"].values()))["scheduler"]
    with pytest.raises(ValueError, match="lr_lambdas"):
        sched.check_state_dict(dict(theirs, base_lrs=[sched.base_lr] * 2), theirs["last_epoch"])


def test_timm_state_round_trip_and_refusals(built_lib):
    sched = _schedule("timm_cosine")
    sd = sched.state_dict(17)
    assert sd["last_epoch"] == 17 and sd["t_initial"] == TIMM["epochs"] and sd["warmup_lr_init"] == TIMM["warmup_lr"]
    sched.check_state_dict(sd, 17)
    for key, value in (("lr_min", 1.0), ("t_initial", 26), ("steps_per_epoch", 4), ("base_values", [1e-2] * 3),
                       ("last_epoch", 18)):
        with pytest.raises(ValueError, match=key):
            sched.check_state_dict(dict(sd, **{key: value}), 17)
    with pytest.raises(ValueError, match="warmup_t"):
        sched.check_state_dict({k: v for k, v in sd.items() if k != "warmup_t"}, 17)
    with pytest.raises(ValueError, match="base_values"):
        sched.check_state_dict(_schedule("oc20_cosine").state_dict(17), 17)


# ------------------------------------------------------------------------------------------------ GPU
def _opt(model, schedule, max_norm=None, ema_decay=None, eps=1e-8, wd=5e-3):
    from equiformer_b200.parallel import CapturableFlatAdamW, FlatGradAllReduce
    bucket = FlatGradAllReduce(model.parameters())
    opt = CapturableFlatAdamW(model.named_parameters(), bucket, betas=(0.9, 0.999), eps=eps, weight_decay=wd,
                              no_decay=model.no_weight_decay(), max_grad_norm=max_norm, ema_decay=ema_decay,
                              model=model, lr_schedule=schedule)
    return bucket, opt


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["oc20_cosine", "oc20_multistep", "timm_cosine"])
def test_scheduled_kernel_matches_the_float64_recipe(cuda_device, name):
    """About 150 steps of seeded gradients (clip and EMA on), through the warm-up, the decay and past the end:
      * after every step ``opt.lr`` holds float32(rate(t)) of the reference's rates to 1 ulp;
      * the run is bitwise the run of the unscheduled kernel with the host writing eqf_lr_at's rate through set_lr;
      * against clip_grad_norm_ + torch.optim.AdamW + the timm EMA in float64 at the reference's rates.  Over 150 steps
        the float32 moments drift from float64 further than in test_optim's five steps, and at the floor rate (2e-6
        for OC20 cosine) one step moves a parameter by a few float32 ulps, so the parameter bounds are wider here."""
    from tests.test_optim import WD, Float64Recipe, _load_grads, _qm9_model, _seeded_grads, _view
    n = 150 if name == "timm_cosine" else len(_fixture()[name]["rates"]) - 1
    rates = _rates(name, n + 1)
    sched = _schedule(name)
    model, twin_model = _qm9_model(cuda_device), _qm9_model(cuda_device)
    ref = Float64Recipe(model, 100.0, 0.9)
    p0 = [p.detach().double().clone() for p in model.parameters()]
    bucket, opt = _opt(model, sched, 100.0, 0.9, wd=WD)
    twin_bucket, twin = _opt(twin_model, None, 100.0, 0.9, wd=WD)
    assert _f32_ulps(float(opt.lr), rates[0]) <= 1
    for step in range(n):
        grads = [g.to(cuda_device) for g in _seeded_grads(model, step)]
        _load_grads(bucket, grads)
        _load_grads(twin_bucket, grads)
        opt.step()
        twin.set_lr(sched.lr_at(step))
        twin.step()
        for g in ref.opt.param_groups:
            g["lr"] = rates[step]
        ref.step(grads)
        assert _f32_ulps(float(opt.lr), rates[step + 1]) <= 1, (step, float(opt.lr), rates[step + 1])
    assert int(opt.t) == n and len(set(rates)) > 10
    for a, b in ((opt.flat, twin.flat), (opt.m, twin.m), (opt.v, twin.v), (opt.ema, twin.ema)):
        assert torch.equal(a, b)
    worst = {}
    for i, ((_, r), p) in enumerate(zip(ref.named, model.parameters())):
        st = ref.opt.state[r]
        checks = {"p": (p, r), "dp": (p.double() - p0[i], r.detach() - p0[i]), "grad": (p.grad, r.grad),
                  "m": (_view(opt.m, bucket, i, p), st["exp_avg"]), "v": (_view(opt.v, bucket, i, p), st["exp_avg_sq"]),
                  "ema": (_view(opt.ema, bucket, i, p), ref.ema[i])}
        for k, (a, b) in checks.items():
            worst[k] = max(worst.get(k, 0.0), rel_err(a, b))
    bounds = {"p": 1e-4, "dp": 3e-3, "grad": 1e-6, "m": 1e-5, "v": 1e-5, "ema": 1e-4}
    assert all(worst[k] <= bounds[k] for k in worst), worst


@pytest.mark.gpu
def test_captured_step_follows_the_schedule(cuda_device):
    """A captured QM9 step (clip + scheduled AdamW + EMA inside the graph) replayed 10 times through the warm-up and into
    the cosine with no host write, against the same captured step with the host writing eqf_lr_at's rate through
    set_lr before each replay.  eps = 1e-3 as in test_optim's captured case."""
    from equiformer_b200.graphs import GraphedForwardBackward
    from equiformer_b200.lr_schedule import LrSchedule
    from equiformer_b200.synthetic import qm9_like_batch
    from tests.test_optim import _qm9_model
    sched = LrSchedule.oc20_lambda_lr(2e-3, "cosine", 4, 0.2, max_steps=12, lr_min_factor=0.01)
    pos, batch, z = qm9_like_batch(32, seed=0)
    target = torch.randn(32, 1, generator=torch.Generator().manual_seed(1))
    inp = [t.to(cuda_device) for t in (pos, batch, z, target)]
    l1 = lambda out, tgt: (out - tgt).abs().mean()
    runs = []
    for scheduled in (True, False):
        model = _qm9_model(cuda_device)
        bucket, opt = _opt(model, sched if scheduled else None, 0.5, 0.9, eps=1e-3)
        gfb = GraphedForwardBackward(model, l1, bucket, max_radius=5.0, after_backward=opt.step)
        losses, lrs = [], []
        for k in range(10):
            if not scheduled:
                opt.set_lr(sched.lr_at(k))
            losses.append(float(gfb(*inp)))
            lrs.append(float(opt.lr))
        assert gfb.captures == 1 and int(opt.t) == 10
        if scheduled:
            assert all(_f32_ulps(lr, sched.lr_at(k + 1)) <= 1 for k, lr in enumerate(lrs)), lrs
            assert len(set(lrs)) == 10
            with pytest.raises(RuntimeError, match="lr_schedule"):
                opt.set_lr(1e-3)
        runs.append((losses, opt.flat.clone(), opt.m.clone(), opt.v.clone(), opt.ema.clone()))
    (ls, *ts), (lh, *th) = runs
    assert all(abs(a - b) <= 1e-5 * abs(b) for a, b in zip(ls, lh)), (ls, lh)
    errs = [rel_err(a, b) for a, b in zip(ts, th)]
    assert max(errs) <= 1e-5, errs


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["oc20_cosine", "timm_cosine"])
def test_resume_is_bitwise(cuda_device, tmp_path, name):
    """60 steps uninterrupted against 25 steps, save_training_state, load_training_state into fresh objects and 35
    more steps: parameters, moments, EMA, rate and step count are bitwise equal."""
    from equiformer_b200.checkpoint import load_training_state, save_training_state
    from tests.test_optim import _load_grads, _qm9_model, _seeded_grads

    def run(steps, model, bucket, opt, start=0):
        for k in range(start, start + steps):
            _load_grads(bucket, [g.to(cuda_device) for g in _seeded_grads(model, k)])
            opt.step()

    model = _qm9_model(cuda_device)
    bucket, opt = _opt(model, _schedule(name), 100.0, 0.9)
    run(60, model, bucket, opt)
    whole = [opt.flat.clone(), opt.m.clone(), opt.v.clone(), opt.ema.clone(), opt.lr.clone(), opt.t.clone()]

    model = _qm9_model(cuda_device)
    bucket, opt = _opt(model, _schedule(name), 100.0, 0.9)
    run(25, model, bucket, opt)
    path = tmp_path / "ckpt.pt"
    save_training_state(path, model, opt, epoch=0, step=25, scheduler=opt.lr_schedule_state_dict())
    model = _qm9_model(cuda_device)
    bucket, opt = _opt(model, _schedule(name), 100.0, 0.9)
    info = load_training_state(path, model, opt)
    opt.load_lr_schedule_state_dict(info["scheduler"])
    assert int(opt.t) == 25 and _f32_ulps(float(opt.lr), opt.lr_schedule.lr_at(25)) <= 1
    run(35, model, bucket, opt, start=25)
    resumed = [opt.flat, opt.m, opt.v, opt.ema, opt.lr, opt.t]
    assert all(torch.equal(a, b) for a, b in zip(whole, resumed))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["oc20_cosine", "oc20_multistep"])
def test_resume_from_the_reference_state(cuda_device, name):
    """A reference checkpoint's optimizer groups (lr = the rate of step t, initial_lr) and LambdaLR state at its step t:
    after both loads the rate is the reference's at t, and one step later at t + 1.  A scheduler state of another step
    is refused before anything is written."""
    from tests.test_optim import _qm9_model
    case = _fixture()[name]
    model = _qm9_model(cuda_device)
    bucket, opt = _opt(model, _schedule(name), wd=1e-3)
    for step, st in case["states"].items():
        t = int(step)
        sd = opt.state_dict()
        if not sd["state"]:
            sd["state"] = {i: {"step": torch.tensor(float(t)), "exp_avg": torch.zeros(p.shape),
                               "exp_avg_sq": torch.zeros(p.shape)} for i, p in enumerate(
                               [bucket.params[j] for j in opt._groups()[0] + opt._groups()[1]])}
        for s in sd["state"].values():
            s["step"] = torch.tensor(float(t))
        sd["param_groups"] = [dict(g, params=ours["params"]) for g, ours in zip(st["param_groups"], sd["param_groups"])]
        opt.load_state_dict(sd)
        with pytest.raises(ValueError, match="last_epoch"):
            opt.load_lr_schedule_state_dict(dict(st["scheduler"], last_epoch=t + 1))
        opt.load_lr_schedule_state_dict(st["scheduler"])
        assert int(opt.t) == t and _f32_ulps(float(opt.lr), case["rates"][t]) <= 1
        assert opt.state_dict()["param_groups"][0]["lr"] == case["rates"][t]
        assert opt.state_dict()["param_groups"][0]["initial_lr"] == st["param_groups"][0]["initial_lr"]
        assert opt.lr_schedule_state_dict()["_last_lr"] == st["scheduler"]["_last_lr"]
        bucket.zero_grad()
        opt.step()
        assert _f32_ulps(float(opt.lr), case["rates"][t + 1]) <= 1


@pytest.mark.gpu
def test_floor_at_a_billion_steps_and_unscheduled_rate_is_left_alone(cuda_device):
    from tests.test_optim import _qm9_model
    model = _qm9_model(cuda_device)
    bucket, opt = _opt(model, _schedule("oc20_cosine"))
    floor = _fixture()["oc20_cosine"]["rates"][-1]
    sd = opt.state_dict()
    t = 10 ** 9                          # AdamW's state keeps the step in float32: 1e9 is exact
    sd["state"] = {i: {"step": torch.tensor(float(t)), "exp_avg": torch.zeros(bucket.params[j].shape),
                       "exp_avg_sq": torch.zeros(bucket.params[j].shape)}
                   for i, j in enumerate(opt._groups()[0] + opt._groups()[1])}
    opt.load_state_dict(sd)
    assert int(opt.t) == t and _f32_ulps(float(opt.lr), floor) == 0
    bucket.zero_grad()
    opt.step()
    assert int(opt.t) == t + 1 and _f32_ulps(float(opt.lr), floor) == 0
    model = _qm9_model(cuda_device)
    bucket, opt = _opt(model, None)
    opt.set_lr(3e-3)
    for _ in range(3):
        bucket.zero_grad()
        opt.step()
    assert float(opt.lr) == float(np.float32(3e-3)) and int(opt.t) == 3
