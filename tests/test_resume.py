"""Saving and resuming a training run: the flat optimisers' state in ``torch.optim.AdamW``'s format
(``parallel.FlatAdamW`` / ``CapturableFlatAdamW`` ``state_dict`` / ``load_state_dict``, ``load_ema_state_dict``) and the
checkpoint files of ``equiformer_b200.checkpoint`` in the reference trainers' layout.

CPU: ``FlatAdamW`` against ``torch.optim.AdamW`` with the reference's ``[no_decay, decay]`` groups on the QM9 model in
float64, both ways of cross-loading, loads that keep every buffer in place, the refusals, reference-layout and MD17 files,
the saved file's keys and RNG states, and two gloo processes of which only rank 0 writes.

GPU: ``CapturableFlatAdamW`` against ``torch.optim.AdamW`` and its own round trip, the EMA load, and a captured QM9 step
(clip, AdamW and EMA inside the graph) that continues bit for bit after a save and a load, into new objects and into the
live captures.
"""
from __future__ import annotations

import json
import os
import socket
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.helpers import rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
QM9 = "graph_attention_transformer_nonlinear_l2"
LR, WD, BETAS, EPS = 1e-2, 5e-3, (0.9, 0.999), 1e-8
REFERENCE_KEYS = ["epoch", "step", "state_dict", "optimizer", "scheduler", "normalizers", "config", "val_metrics", "ema",
                  "amp"]


def _qm9(dtype=torch.float64, seed=0, dev="cpu"):
    from equiformer_b200.nets import model_entrypoint
    torch.manual_seed(seed)
    return model_entrypoint(QM9)(irreps_in="5x0e", radius=5.0, num_basis=128).to(device=dev, dtype=dtype)


class _Net(torch.nn.Module):
    """Small model with both decay groups: ``lin.tp.weight`` and ``fc.weight`` decayed, ``lin.bias.0`` and ``fc.bias``
    exempt, and a buffer."""

    def __init__(self):
        super().__init__()
        from equiformer_b200.nets.tensor_product_rescale import LinearRS
        self.lin = LinearRS("6x0e", "5x0e", bias=True)
        self.fc = torch.nn.Linear(5, 3)
        self.register_buffer("scale", torch.full((3,), 2.0))


def _flat_adamw(model):
    from equiformer_b200.parallel import FlatAdamW, FlatGradAllReduce
    bucket = FlatGradAllReduce(model.parameters())
    skip = model.no_weight_decay() if hasattr(model, "no_weight_decay") else ()
    return bucket, FlatAdamW(model.named_parameters(), bucket, lr=LR, betas=BETAS, eps=EPS, weight_decay=WD,
                             no_decay=skip)


def _torch_adamw(model):
    """``torch.optim.AdamW(add_weight_decay(model, WD, model.no_weight_decay()))`` as the reference builds it."""
    from equiformer_b200.parallel import is_no_decay
    skip = model.no_weight_decay() if hasattr(model, "no_weight_decay") else ()
    named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
    return torch.optim.AdamW([{"params": [p for n, p in named if is_no_decay(n, skip)], "weight_decay": 0.0},
                              {"params": [p for n, p in named if not is_no_decay(n, skip)], "weight_decay": WD}],
                             lr=LR, betas=BETAS, eps=EPS)


def _group_names(model):
    """Parameter names in the order of the optimiser state's indices: exempt ones, then decayed ones."""
    from equiformer_b200.parallel import is_no_decay
    skip = model.no_weight_decay() if hasattr(model, "no_weight_decay") else ()
    names = [n for n, p in model.named_parameters() if p.requires_grad]
    return [n for n in names if is_no_decay(n, skip)] + [n for n in names if not is_no_decay(n, skip)]


def _grads(model, step, dev=None):
    g = torch.Generator().manual_seed(100 + step)
    return [(torch.randn(p.shape, generator=g, dtype=torch.float64) * (1.0 + i % 7)).to(dev or p.device, p.dtype)
            for i, p in enumerate(model.parameters())]


def _step_ours(bucket, opt, grads):
    bucket.zero_grad()
    for p, g in zip(bucket.params, grads):
        p.grad.copy_(g)
    opt.step()


def _step_torch(model, opt, grads):
    for p, g in zip(model.parameters(), grads):
        p.grad = g.clone()
    opt.step()


def _padding(bucket):
    mask = torch.ones(bucket.flat.numel(), dtype=torch.bool, device=bucket.flat.device)
    for off, p in zip(bucket.offsets, bucket.params):
        mask[off:off + p.numel()] = False
    return mask


def _ptrs(opt, *extra):
    return [t.data_ptr() for t in (opt.flat, opt.m, opt.v, opt.decay, *extra, *opt.bucket.params)]


def _assert_same_layout(ours, theirs, tol):
    """Same top-level keys, groups (keys in order, hyperparameters, indices), state indices and state keys; the
    tensors agree within ``tol`` (``step`` exactly, in torch's dtype)."""
    assert list(ours) == list(theirs) == ["state", "param_groups"]
    assert len(ours["param_groups"]) == len(theirs["param_groups"]) == 2
    for a, b in zip(ours["param_groups"], theirs["param_groups"]):
        assert list(a) == list(b)
        for k in a:
            if k == "lr":
                assert abs(a[k] - b[k]) <= 1e-7 * b[k], (a[k], b[k])
            else:
                assert a[k] == b[k], k
    assert list(ours["state"]) == list(theirs["state"])
    for k, s in theirs["state"].items():
        assert list(ours["state"][k]) == list(s)
        assert ours["state"][k]["step"].dtype == s["step"].dtype and float(ours["state"][k]["step"]) == float(s["step"])
        for key in ("exp_avg", "exp_avg_sq"):
            assert ours["state"][k][key].shape == s[key].shape, (k, key)
            assert rel_err(ours["state"][k][key], s[key]) <= tol, (k, key)


# ------------------------------------------------------------------------------------------------ CPU: optimiser state
def test_flat_adamw_state_dict_is_torch_adamw_state_dict_and_cross_loads():
    """Three steps on the QM9 model in float64 beside ``torch.optim.AdamW``: the two ``state_dict()``s agree (keys, index
    to parameter, hyperparameters, tensors within 1e-12).  Each optimiser's state is then loaded into a new optimiser of
    the other kind, on a copy of the weights; three more steps keep them within 1e-12 of the run they continue."""
    a, b = _qm9(), _qm9()
    assert all(torch.equal(x, y) for x, y in zip(a.parameters(), b.parameters()))
    bucket_a, opt_a = _flat_adamw(a)
    opt_b = _torch_adamw(b)
    for step in range(3):
        grads = _grads(a, step)
        _step_ours(bucket_a, opt_a, grads)
        _step_torch(b, opt_b, grads)
    sa, sb = opt_a.state_dict(), opt_b.state_dict()
    _assert_same_layout(sa, sb, 1e-12)
    params = dict(b.named_parameters())
    for k, name in enumerate(_group_names(b)):                       # torch's index k is the parameter we put there
        assert opt_b.state[params[name]]["exp_avg"] is sb["state"][k]["exp_avg"], name

    c = _qm9(seed=1)                                                 # ours, resumed from torch's state
    c.load_state_dict(b.state_dict())
    bucket_c, opt_c = _flat_adamw(c)
    opt_c.load_state_dict(sb)
    d = _qm9(seed=1)                                                 # torch's, resumed from ours
    d.load_state_dict(a.state_dict())
    opt_d = _torch_adamw(d)
    opt_d.load_state_dict(sa)
    assert opt_c.t == 3 and rel_err(opt_c.m, opt_a.m) <= 1e-12
    for step in range(3, 6):
        grads = _grads(a, step)
        _step_ours(bucket_a, opt_a, grads)
        _step_torch(b, opt_b, grads)
        _step_ours(bucket_c, opt_c, grads)
        _step_torch(d, opt_d, grads)
    for (n, pa), pb, pc, pd in zip(a.named_parameters(), b.parameters(), c.parameters(), d.parameters()):
        assert torch.allclose(pc, pb, rtol=0, atol=1e-12), (n, (pc - pb).abs().max())
        assert torch.allclose(pd, pa, rtol=0, atol=1e-12), (n, (pd - pa).abs().max())


def test_load_writes_in_place_and_adopts_the_groups():
    """``load_state_dict`` keeps the storage of ``flat``, ``m``, ``v``, ``decay`` and every parameter, restores the step
    count and the moments exactly, leaves the padding zero, and adopts ``lr`` and a changed ``weight_decay``."""
    model = _Net()
    bucket, opt = _flat_adamw(model)
    for step in range(2):
        _step_ours(bucket, opt, _grads(model, step))
    sd = opt.state_dict()
    m, v = opt.m.clone(), opt.v.clone()
    ptrs = _ptrs(opt)
    _step_ours(bucket, opt, _grads(model, 2))
    for g in sd["param_groups"]:
        g["lr"] = 3e-3
    sd["param_groups"][1]["weight_decay"] = 0.25
    opt.load_state_dict(sd)
    assert _ptrs(opt) == ptrs
    assert opt.t == 2 and opt.lr == 3e-3 and torch.equal(opt.m, m) and torch.equal(opt.v, v)
    pad = _padding(bucket)
    assert pad.any() and not opt.m[pad].any() and not opt.v[pad].any() and not opt.decay[pad].any()
    decayed = set(_group_names(model)[len(sd["param_groups"][0]["params"]):])
    for (name, p), off in zip(model.named_parameters(), bucket.offsets):
        assert bool((opt.decay[off:off + p.numel()] == (0.25 if name in decayed else 0.0)).all()), name
    assert [g["weight_decay"] for g in opt.state_dict()["param_groups"]] == [0.0, 0.25]

    opt.load_state_dict(_torch_adamw(_Net()).state_dict())            # a torch optimiser that never stepped
    assert opt.t == 0 and not opt.m.any() and not opt.v.any() and _ptrs(opt) == ptrs
    assert opt.state_dict()["state"] == {}


def _refuse_count(sd, names):
    k = sd["param_groups"][1]["params"].pop()
    sd["state"].pop(k)
    return "param_groups"


def _refuse_shape(sd, names):
    sd["state"][2]["exp_avg"] = torch.zeros(7, dtype=torch.float64)
    return names[2]


def _refuse_group(sd, names):
    g0, g1 = sd["param_groups"][0]["params"], sd["param_groups"][1]["params"]
    g1.insert(0, g0.pop())                                           # the last exempt parameter, now decayed
    return names[len(g0)]


def _refuse_step(sd, names):
    sd["state"][3]["step"] = torch.tensor(7.0)
    return names[3]


def _refuse_amsgrad(sd, names):
    sd["param_groups"][1]["amsgrad"] = True
    return "amsgrad"


def _refuse_lr(sd, names):
    sd["param_groups"][0]["lr"] = 1e-3
    return "lr"


@pytest.mark.parametrize("case", [_refuse_count, _refuse_shape, _refuse_group, _refuse_step, _refuse_amsgrad, _refuse_lr],
                         ids=lambda f: f.__name__[len("_refuse_"):])
def test_load_refuses_a_state_that_does_not_fit(case):
    """Each misfit raises a ``ValueError`` naming the parameter or key, and the optimiser is left as it was."""
    model, twin = _Net().double(), _Net().double()
    bucket, opt = _flat_adamw(model)
    ref = _torch_adamw(twin)
    for step in range(2):
        _step_ours(bucket, opt, _grads(model, step))
        _step_torch(twin, ref, _grads(model, step))
    sd = ref.state_dict()
    before = [opt.flat.clone(), opt.m.clone(), opt.v.clone(), opt.decay.clone(), opt.t, opt.lr]
    expect = case(sd, _group_names(model))
    with pytest.raises(ValueError, match=expect.replace(".", r"\.")):
        opt.load_state_dict(sd)
    after = [opt.flat, opt.m, opt.v, opt.decay, opt.t, opt.lr]
    assert all(torch.equal(x, y) if isinstance(x, torch.Tensor) else x == y for x, y in zip(before, after))


# ------------------------------------------------------------------------------------------------ CPU: checkpoint files
def test_reference_trainer_checkpoint_loads(tmp_path):
    """A file as the OC20 trainer writes it (``module.``-prefixed model keys, e3nn's ``_w3j_`` buffers, a real
    ``torch.optim.AdamW`` state) loads into a new model and ``FlatAdamW``: weights, moments and step count as saved, the
    parameters still views of the flat buffer, and the trainer's other entries returned."""
    from equiformer_b200.checkpoint import load_training_state
    b = _qm9(torch.float32)
    opt_b = _torch_adamw(b)
    for step in range(2):
        _step_torch(b, opt_b, _grads(b, step))
    state = {f"module.{k}": v for k, v in b.state_dict().items()}
    state["module.blocks.0.ga.sep_act.dtp.tp._w3j_1e_1e_2e"] = torch.ones(3, 3, 5)
    path = tmp_path / "checkpoint.pt"
    torch.save({"epoch": 3, "step": 1234, "state_dict": state, "optimizer": opt_b.state_dict(),
                "scheduler": {"last_epoch": 3}, "normalizers": {"target": {"mean": 1.5, "std": 2.0}},
                "config": {"optim": {"lr_initial": LR}}, "val_metrics": None, "ema": None, "amp": None}, path)

    a = _qm9(torch.float32, seed=1)
    bucket, opt = _flat_adamw(a)
    ptrs = _ptrs(opt)
    out = load_training_state(path, a, opt)
    assert out == {"epoch": 3, "step": 1234, "scheduler": {"last_epoch": 3},
                   "normalizers": {"target": {"mean": 1.5, "std": 2.0}}, "config": {"optim": {"lr_initial": LR}}}
    assert _ptrs(opt) == ptrs
    for (k, x), y in zip(a.state_dict().items(), b.state_dict().values()):
        assert torch.equal(x, y), k
    params = dict(b.named_parameters())
    assert opt.t == 2
    for i, name in enumerate(n for n, _ in a.named_parameters()):
        st = opt_b.state[params[name]]
        assert torch.equal(opt._view(opt.m, i), st["exp_avg"]) and torch.equal(opt._view(opt.v, i), st["exp_avg_sq"])


def test_md17_checkpoint_loads_the_model_only(tmp_path):
    from equiformer_b200.checkpoint import load_training_state
    src, dst = _Net(), _Net()
    bucket, opt = _flat_adamw(dst)
    _step_ours(bucket, opt, _grads(dst, 0))
    m = opt.m.clone()
    torch.save({"state_dict": src.state_dict()}, tmp_path / "best.pth.tar")
    out = load_training_state(tmp_path / "best.pth.tar", dst, opt)
    assert out == {"epoch": 0, "step": 0, "scheduler": None, "normalizers": None, "config": None}
    assert all(torch.equal(x, y) for x, y in zip(dst.state_dict().values(), src.state_dict().values()))
    assert opt.t == 1 and torch.equal(opt.m, m)


def test_saved_file_has_the_reference_keys_and_round_trips(tmp_path):
    """``save_training_state`` writes the trainer's keys plus ``rng``; loading it restores model, optimiser, the CPU RNG
    and a caller's generator, and a wrong number of generators is refused before anything is loaded."""
    from equiformer_b200.checkpoint import load_training_state, save_training_state
    model = _Net()
    bucket, opt = _flat_adamw(model)
    for step in range(3):
        _step_ours(bucket, opt, _grads(model, step))
    noise = torch.Generator().manual_seed(9)
    torch.manual_seed(5)
    path = tmp_path / "checkpoint.pt"
    save_training_state(path, model, opt, epoch=1, step=30, scheduler={"last_epoch": 1}, normalizers={},
                        config={"name": "run"}, val_metrics={"energy_mae": 0.1}, generators=(noise,))
    assert os.listdir(tmp_path) == ["checkpoint.pt"]
    raw = torch.load(path, weights_only=False)
    assert list(raw) == REFERENCE_KEYS + ["rng"]
    assert raw["ema"] is None and raw["amp"] is None and raw["val_metrics"] == {"energy_mae": 0.1}
    draws = (torch.rand(4), torch.rand(4, generator=noise))
    saved = [opt.flat.clone(), opt.m.clone(), opt.v.clone()]

    fresh = _Net()
    bucket_f, opt_f = _flat_adamw(fresh)
    with pytest.raises(ValueError, match="generator"):
        load_training_state(path, fresh, opt_f)
    assert opt_f.t == 0
    out = load_training_state(path, fresh, opt_f, generators=(noise,))
    assert out["epoch"] == 1 and out["step"] == 30 and out["config"] == {"name": "run"}
    assert opt_f.t == 3 and all(torch.equal(x, y) for x, y in zip([opt_f.flat, opt_f.m, opt_f.v], saved))
    assert torch.equal(torch.rand(4), draws[0]) and torch.equal(torch.rand(4, generator=noise), draws[1])


def test_state_dict_keys_are_matched_as_the_reference_trainer_matches_them():
    from equiformer_b200.checkpoint import match_state_dict
    target = {"a.weight": torch.zeros(2, 3), "a.bias": torch.zeros(2)}
    state = {"a.weight": torch.ones(2, 3), "a.bias": torch.ones(2)}
    for prefix in ("", "module.", "module.module."):                 # plain, DDP or OCPDataParallel, both
        got = match_state_dict({prefix + k: v for k, v in state.items()}, target)
        assert list(got) == list(target) and got["a.bias"] is state["a.bias"]
        ddp = match_state_dict({prefix + k: v for k, v in state.items()}, {"module." + k: v for k, v in target.items()})
        assert list(ddp) == ["module.a.weight", "module.a.bias"]
    assert list(match_state_dict(dict(state, **{"a.tp._w3j_1e_1e_0e": torch.ones(1)}), target)) == list(target)
    with pytest.raises(ValueError, match="a.bias"):
        match_state_dict({"a.weight": state["a.weight"]}, target)
    with pytest.raises(ValueError, match="a.extra"):
        match_state_dict(dict(state, **{"a.extra": torch.ones(1)}), target)
    with pytest.raises(ValueError, match="a.bias"):
        match_state_dict(dict(state, **{"a.bias": torch.ones(3)}), target)


# ------------------------------------------------------------------------------------------------ CPU: two processes
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank_worker(rank, world, port, path, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    from equiformer_b200.checkpoint import load_training_state, save_training_state
    from equiformer_b200.parallel import broadcast_parameters, init_distributed
    init_distributed("gloo")
    torch.manual_seed(100 + rank)
    model = _Net().double()
    broadcast_parameters(model)
    bucket, opt = _flat_adamw(model)
    for step in range(2):
        bucket.zero_grad()
        for p, g in zip(bucket.params, _grads(model, 10 * rank + step)):
            p.grad.copy_(g)
        bucket.reduce()
        opt.step()
    writes = []
    replace = os.replace
    os.replace = lambda src, dst: (writes.append(dst), replace(src, dst))[1]
    torch.manual_seed(rank)                                           # each rank its own stream
    save_training_state(path, model, opt, epoch=0, step=2)
    os.replace = replace
    saved = torch.cat([opt.flat, opt.m, opt.v])
    draw = torch.rand(3)
    _step_ours(bucket, opt, _grads(model, 50 + rank))                 # the ranks drift apart
    load_training_state(path, model, opt)
    state = torch.cat([opt.flat, opt.m, opt.v, torch.tensor([float(opt.t)], dtype=torch.float64)])
    states = [torch.zeros_like(state) for _ in range(world)]
    dist.all_gather(states, state)
    draws = [torch.zeros(3) for _ in range(world)]
    dist.all_gather(draws, torch.rand(3))
    ret[rank] = {"writes": len(writes), "equal": all(torch.equal(s, states[0]) for s in states),
                 "as_saved": torch.equal(state[:-1], saved) and float(state[-1]) == 2.0,
                 "rng": torch.equal(draws[rank], draw) and not torch.equal(draws[0], draws[1])}
    dist.destroy_process_group()


def test_two_processes_rank_zero_writes_and_both_resume(tmp_path):
    """Two gloo processes: only rank 0 writes the file, both load it and end with equal states, and each rank gets its
    own RNG stream back."""
    world = 2
    with mp.Manager() as mgr:
        ret = mgr.dict()
        mp.spawn(_rank_worker, args=(world, _free_port(), str(tmp_path / "checkpoint.pt"), ret), nprocs=world, join=True)
        ret = dict(ret)
    assert [ret[r]["writes"] for r in range(world)] == [1, 0]
    assert all(ret[r]["equal"] and ret[r]["as_saved"] and ret[r]["rng"] for r in range(world)), ret
    assert os.listdir(tmp_path) == ["checkpoint.pt"]


# ------------------------------------------------------------------------------------------------ GPU: capturable
def _capturable(model, max_norm=None, ema_decay=None, lr=LR):
    from equiformer_b200.parallel import CapturableFlatAdamW, FlatGradAllReduce
    bucket = FlatGradAllReduce(model.parameters())
    return bucket, CapturableFlatAdamW(model.named_parameters(), bucket, lr=lr, betas=BETAS, eps=EPS, weight_decay=WD,
                                       no_decay=model.no_weight_decay(), max_grad_norm=max_norm, ema_decay=ema_decay,
                                       model=model)


@pytest.mark.gpu
def test_capturable_state_dict_matches_torch_adamw_and_round_trips(cuda_device):
    """Five steps (clip and EMA off) beside ``torch.optim.AdamW`` in fp32 on the device: the ``state_dict()``s agree to
    the kernel's tolerance against ``FlatAdamW.step()``.  The optimiser's own dict loads back bit for bit after two more
    steps, torch's loads too, every buffer keeps its storage, and other betas are refused."""
    a, b = _qm9(torch.float32, dev=cuda_device), _qm9(torch.float32, dev=cuda_device)
    bucket, opt = _capturable(a)
    ref = _torch_adamw(b)
    for step in range(5):
        grads = _grads(a, step)
        _step_ours(bucket, opt, grads)
        _step_torch(b, ref, grads)
    sa, sb = opt.state_dict(), ref.state_dict()
    _assert_same_layout(sa, sb, 1e-6)
    ptrs = _ptrs(opt, opt.lr, opt.t)
    m, v = opt.m.clone(), opt.v.clone()
    for step in range(5, 7):
        _step_ours(bucket, opt, _grads(a, step))
    opt.set_lr(1e-3)
    opt.load_state_dict(sa)
    assert _ptrs(opt, opt.lr, opt.t) == ptrs
    assert int(opt.t) == 5 and float(opt.lr) == float(torch.tensor(LR, dtype=torch.float32))
    assert torch.equal(opt.m, m) and torch.equal(opt.v, v)
    opt.load_state_dict(sb)
    assert _ptrs(opt, opt.lr, opt.t) == ptrs and int(opt.t) == 5
    assert rel_err(opt.m, m) <= 1e-6 and rel_err(opt.v, v) <= 1e-6
    pad = _padding(bucket)
    assert not opt.m[pad].any() and not opt.v[pad].any() and not opt.decay[pad].any()
    for g in sb["param_groups"]:
        g["betas"] = (0.95, 0.999)
    with pytest.raises(ValueError, match="betas"):
        opt.load_state_dict(sb)


@pytest.mark.gpu
def test_ema_loads_in_place(cuda_device):
    """``load_ema_state_dict`` is the inverse of ``ema_state_dict``: a saved EMA (here ``module.``-prefixed, as a DDP
    run saves it) comes back bit for bit into the same buffers, and a missing key is refused."""
    model = _qm9(torch.float32, dev=cuda_device)
    bucket, opt = _capturable(model, ema_decay=0.5)
    for step in range(3):
        _step_ours(bucket, opt, _grads(model, step))
    saved = {k: t.clone() for k, t in opt.ema_state_dict().items()}
    ptrs = [opt.ema.data_ptr()] + [e.data_ptr() for e in opt._ema_others]
    for step in range(3, 5):
        _step_ours(bucket, opt, _grads(model, step))
    assert not torch.equal(opt.ema_state_dict()[next(iter(saved))], next(iter(saved.values())))
    opt.load_ema_state_dict({f"module.{k}": t for k, t in saved.items()})
    assert [opt.ema.data_ptr()] + [e.data_ptr() for e in opt._ema_others] == ptrs
    for (k, x), y in zip(opt.ema_state_dict().items(), saved.values()):
        assert torch.equal(x, y), k
    first = next(iter(saved))
    with pytest.raises(ValueError, match=first.replace(".", r"\.")):
        opt.load_ema_state_dict({k: t for k, t in saved.items() if k != first})


# ------------------------------------------------------------------------------------------------ GPU: continuation
N_STEPS = 4


def continuation_runs(out_path: str) -> None:
    """The continuation runs, in a process of their own started with ``EQF_DETERMINISTIC=1`` (read when ``ops`` is
    imported: the GEMM weight gradients are summed in a fixed order).  The ``bench.py`` QM9 batch trains through
    ``GraphedForwardBackward`` with clip (max norm 5), AdamW and the EMA (decay 0.9999) inside the captured graph.

    (a) Attention dropout off: 2N uninterrupted steps, against N steps, a save, a new model, optimiser and graphed step
    (from another seed), a load and N more steps.  A twin of the uninterrupted run measures how far two runs of the same
    step drift apart.  (b) Attention dropout 0.2: N steps, a save, N more steps; then the step-N file loaded into the same
    live objects and the N steps replayed without a new capture.  As a control, the same replay after reseeding the CUDA
    generator instead of restoring it.  Writes a JSON summary to ``out_path``."""
    import bench
    from equiformer_b200.checkpoint import load_training_state, save_training_state
    from equiformer_b200.graphs import GraphedForwardBackward
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    inp = bench.make_inputs("qm9", seed=0)
    inp = [inp[k].to(dev) for k in ("pos", "batch", "z", "target")]
    l1 = lambda out, tgt: (out - tgt).abs().mean()
    keep = []      # every model lives to the end: one freed during a later capture would free device memory inside it

    def setup(seed, alpha_drop):
        model = _qm9(torch.float32, seed=seed, dev=dev).train()
        for m in model.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = alpha_drop
        bucket, opt = _capturable(model, max_norm=5.0, ema_decay=0.9999, lr=5e-4)
        step = GraphedForwardBackward(model, l1, bucket, max_radius=5.0, after_backward=opt.step)
        keep.append((model, bucket, opt, step))
        return model, opt, step

    def run(step, n):
        return [float(step(*inp)) for _ in range(n)]

    def state(opt):
        return {"flat": opt.flat.clone(), "m": opt.m.clone(), "v": opt.v.clone(), "t": opt.t.clone(),
                "ema": torch.cat([t.detach().double().reshape(-1) for t in opt.ema_state_dict().values()])}

    def compare(x, y):
        return {k: {"equal": torch.equal(x[k], y[k]), "rel": rel_err(x[k].double(), y[k].double())} for k in x}

    def losses(x, y):
        return {"equal": x == y, "rel": max(abs(a - b) / abs(b) for a, b in zip(x, y)), "values": [x, y]}

    out = {}
    # (a) fresh objects; a twin of the uninterrupted run measures how far two runs of the same step drift apart
    _m, opt_u, step_u = setup(0, 0.0)
    losses_u = run(step_u, 2 * N_STEPS)
    _m, opt_w, step_w = setup(0, 0.0)
    losses_w = run(step_w, 2 * N_STEPS)
    model_1, opt_1, step_1 = setup(0, 0.0)
    run(step_1, N_STEPS)
    path_a = os.path.join(os.path.dirname(out_path), "fresh.pt")
    save_training_state(path_a, model_1, opt_1, epoch=0, step=N_STEPS)
    saved = state(opt_1)
    model_2, opt_2, step_2 = setup(1, 0.0)
    load_training_state(path_a, model_2, opt_2)
    out["fresh_loaded"] = compare(state(opt_2), saved)
    losses_2 = run(step_2, N_STEPS)
    out["fresh"] = dict(compare(state(opt_2), state(opt_u)), loss=losses(losses_2[-1:], losses_u[-1:]))
    out["twin"] = dict(compare(state(opt_w), state(opt_u)), loss=losses(losses_w, losses_u))
    # (b) rewinding live captures, attention dropout on
    model_b, opt_b, step_b = setup(0, 0.2)
    run(step_b, N_STEPS)
    path_b = os.path.join(os.path.dirname(out_path), "live.pt")
    save_training_state(path_b, model_b, opt_b, epoch=0, step=N_STEPS)
    saved = state(opt_b)
    first, s1 = run(step_b, N_STEPS), state(opt_b)
    load_training_state(path_b, model_b, opt_b)
    out["live_loaded"] = compare(state(opt_b), saved)
    again, s2 = run(step_b, N_STEPS), state(opt_b)
    load_training_state(path_b, model_b, opt_b)
    torch.cuda.manual_seed(8)
    control = run(step_b, N_STEPS)
    out["live"] = dict(compare(s2, s1), loss=losses(again, first))
    out["live_captures"] = step_b.captures
    out["control"] = losses(control, first)
    for f in (path_a, path_b):
        os.remove(f)
    torch.cuda.synchronize()
    with open(out_path, "w") as f:
        json.dump(out, f, indent=1)


@pytest.mark.gpu
def test_captured_step_continues_after_save_and_load(cuda_device, tmp_path):
    """A load restores parameters, ``m``, ``v``, ``t`` and the EMA bit for bit, into new objects and into the live
    captures, and the replay with the restored CUDA generator draws the dropout masks of the first continuation.

    The continued runs themselves are compared at last-bit tolerance: even with ``EQF_DETERMINISTIC=1`` the QM9 step is
    not run-to-run reproducible.  Two passes on the same inputs and weights give forward outputs that differ in the last
    bits, and gradients that differ in the parameters whose reductions go through per-CTA partials accumulated with
    shared-memory float ``atomicAdd`` (``ln_silu_bwd_kernel`` for the radial networks' layer norms, ``gate_logits_bwd``
    for ``alpha_dot``, ``eln_bwd_kernel`` for the norms' affine parameters, ``rbf_bwd_kernel`` for ``rbf.weight``), while
    every GEMM weight gradient is bitwise equal.  Two uninterrupted runs of 8 steps drift apart by about 3e-7 relative
    (the ``twin`` entry), and the resumed runs stay as close as that."""
    out = tmp_path / "continuation.json"
    env = dict(os.environ, EQF_DETERMINISTIC="1")
    code = "import sys; from tests.test_resume import continuation_runs; continuation_runs(sys.argv[1])"
    flags = ["-s"] if sys.flags.no_user_site else []
    proc = subprocess.run([sys.executable, *flags, "-c", code, str(out)], cwd=ROOT, env=env, capture_output=True,
                          text=True, timeout=1200)
    assert proc.returncode == 0, proc.stderr[-4000:]
    res = json.loads(out.read_text())
    assert all(r["equal"] for r in res["fresh_loaded"].values()), res["fresh_loaded"]
    assert all(r["equal"] for r in res["live_loaded"].values()), res["live_loaded"]
    assert res["live_captures"] == 1 and res["control"]["rel"] > 1e-4, res["control"]
    for run in ("fresh", "live"):
        assert res[run]["t"]["equal"], res[run]
        assert all(r["rel"] <= 3e-6 for r in res[run].values()), (run, res[run], res["twin"])
