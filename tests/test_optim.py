"""Gradient-norm clipping, AdamW and the model EMA on ``libeqf_b200_optim.so`` (``parallel.CapturableFlatAdamW``).

CPU: the library builds for sm_90a, its kernel entries are the ones the GPU cases launch, ``libeqf_b200.so`` holds none
of them, and the launchers and entry points refuse CPU tensors, other dtypes, misaligned buffers and empty ones.

GPU: five steps on the QM9 model with seeded gradients against a float64 restatement of the reference's recipe
(``torch.nn.utils.clip_grad_norm_`` over the parameters, ``torch.optim.AdamW`` with the name-based decay groups, timm's
``ModelEmaV2``); the kernel without clip and EMA against ``FlatAdamW.step()``; bitwise repeatability; odd lengths and
lengths past the grid cap; NaN / Inf gradients; the step captured inside ``GraphedForwardBackward``; the EMA's
``state_dict`` and weight swap.
"""
from __future__ import annotations

import copy
import os
import re

import pytest
import torch

from tests.helpers import rel_err

# every kernel entry of libeqf_b200_optim.so, claimed by test_raw_kernels_at_odd_lengths_and_past_the_grid_cap: its
# first step runs eqf_flat_sqnorm and eqf_flat_adamw with an EMA buffer, its second without one, and both steps'
# results are checked against float64
OPTIM_CLAIMS = {"eqf::flat_sqnorm_kernel", "eqf::flat_adamw_kernel<true>", "eqf::flat_adamw_kernel<false>"}
QM9 = "graph_attention_transformer_nonlinear_l2"
LR, WD, BETAS, EPS = 1e-2, 5e-3, (0.9, 0.999), 1e-8


# ------------------------------------------------------------------------------------------------ CPU
def test_header_constants_match():
    from equiformer_b200 import _lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                               "eqf_b200_optim.h")).read()
    assert int(re.search(r"#define EQF_OPTIM_THREADS (\d+)", header).group(1)) == _lib.EQF_OPTIM_THREADS
    assert int(re.search(r"#define EQF_OPTIM_MAX_CTAS (\d+)", header).group(1)) == _lib.EQF_OPTIM_MAX_CTAS


def test_optim_library_inventory_is_claimed(built_lib):
    from equiformer_b200 import _lib
    from tests.test_gpu_kernel_instances import inventory
    inv = inventory(_lib.OPTIM_LIB_PATH)
    assert inv == OPTIM_CLAIMS, (sorted(inv - OPTIM_CLAIMS), sorted(OPTIM_CLAIMS - inv))


def test_main_library_holds_no_optimiser_kernel(built_lib):
    from equiformer_b200 import _lib
    from tests.test_gpu_kernel_instances import inventory
    assert not {n for n in inventory(_lib.LIB_PATH) if n.startswith("eqf::flat_")}
    assert "eqf_flat_adamw" not in _lib.SIGNATURES and "eqf_optim.cu" not in _lib.SOURCES


def test_launchers_refuse_cpu_and_non_fp32_buffers():
    from equiformer_b200 import _lib, optim_kernels
    one = lambda dtype=torch.float32: torch.zeros(1, dtype=dtype)
    scratch = torch.zeros(_lib.EQF_OPTIM_MAX_CTAS, dtype=torch.float64)
    ticket = one(torch.int32)
    with pytest.raises(_lib.EqfError, match="CUDA-only"):
        optim_kernels.flat_sqnorm_raw(torch.zeros(8), 1.0, scratch, ticket, one(), one())
    with pytest.raises(_lib.EqfError, match="float32"):
        optim_kernels.flat_sqnorm_raw(torch.zeros(8, dtype=torch.float64), 1.0, scratch, ticket, one(), one())
    bufs = [torch.zeros(8) for _ in range(5)]
    with pytest.raises(_lib.EqfError, match="CUDA-only"):
        optim_kernels.flat_adamw_raw(*bufs, None, one(), one(), one(torch.int64), BETAS, EPS, None, ticket)
    bufs[0] = bufs[0].double()
    with pytest.raises(_lib.EqfError, match="float32"):
        optim_kernels.flat_adamw_raw(*bufs, None, one(), one(), one(torch.int64), BETAS, EPS, None, ticket)


def test_argument_checks_refuse_misaligned_and_empty_buffers(built_lib):
    """The entry points' argument checks, called on their own: host code that launches and dereferences nothing, so
    addresses that name no memory exercise them."""
    from equiformer_b200 import _lib
    lib = _lib.load_optim()
    ok, off = 1 << 20, (1 << 20) + 4
    msg = lambda: lib.eqf_last_error().decode()
    assert lib.eqf_flat_sqnorm_check(ok, 63, 1.0, ok, ok, ok, ok) == 0
    assert lib.eqf_flat_sqnorm_check(off, 64, 1.0, ok, ok, ok, ok) != 0 and "aligned" in msg()
    assert lib.eqf_flat_sqnorm_check(ok, 0, 1.0, ok, ok, ok, ok) != 0 and "positive" in msg()
    assert lib.eqf_flat_adamw_check(ok, ok, ok, ok, ok, None, 63, ok, ok, ok, 0.9, 0.999, ok) == 0
    for bad in range(6):
        ptrs = [off if i == bad else ok for i in range(6)]
        rc = lib.eqf_flat_adamw_check(*ptrs, 64, ok, ok, ok, 0.9, 0.999, ok)
        assert rc != 0 and "aligned" in msg(), bad
    assert lib.eqf_flat_adamw_check(ok, ok, ok, ok, ok, None, 0, ok, ok, ok, 0.9, 0.999, ok) != 0
    assert "positive" in msg()


def test_constructor_refuses_bad_settings():
    from equiformer_b200.parallel import CapturableFlatAdamW, FlatGradAllReduce
    net = torch.nn.Linear(3, 2)
    bucket = FlatGradAllReduce(net.parameters())
    with pytest.raises(ValueError, match="max_grad_norm"):
        CapturableFlatAdamW(net.named_parameters(), bucket, max_grad_norm=0.0)
    with pytest.raises(ValueError, match="ema_decay"):
        CapturableFlatAdamW(net.named_parameters(), bucket, ema_decay=0.99)          # no model for the buffers


# ------------------------------------------------------------------------------------------------ GPU helpers
def _qm9_model(dev):
    from equiformer_b200.nets import model_entrypoint
    torch.manual_seed(0)
    model = model_entrypoint(QM9)(irreps_in="5x0e", radius=5.0, num_basis=128).to(dev).train()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return model


def _seeded_grads(model, step, nan_at=None, value=float("nan")):
    """Seeded gradients; ``nan_at``: index of an element of the largest parameter set to ``value``."""
    g = torch.Generator().manual_seed(100 + step)
    grads = [torch.randn(p.shape, generator=g) * (1.0 + (i % 7)) for i, p in enumerate(model.parameters())]
    if nan_at is not None:
        max(grads, key=lambda t: t.numel()).view(-1)[nan_at] = value
    return grads


class Float64Recipe:
    """The reference's step in float64: clip_grad_norm_, torch.optim.AdamW with the name-based decay groups, timm EMA."""

    def __init__(self, model, max_norm, ema_decay):
        from equiformer_b200.parallel import is_no_decay
        skip = model.no_weight_decay()
        self.named = [(n, p.detach().double().clone().requires_grad_(True)) for n, p in model.named_parameters()]
        self.params = [p for _, p in self.named]
        groups = [{"params": [p for n, p in self.named if not is_no_decay(n, skip)], "weight_decay": WD},
                  {"params": [p for n, p in self.named if is_no_decay(n, skip)], "weight_decay": 0.0}]
        self.opt = torch.optim.AdamW(groups, lr=LR, betas=BETAS, eps=EPS)
        self.max_norm, self.d = max_norm, ema_decay
        self.ema = [p.detach().clone() for p in self.params]
        self.norm = None

    def step(self, grads):
        for p, g in zip(self.params, grads):
            p.grad = g.to(p.device, torch.float64)
        if self.max_norm is not None:
            self.norm = float(torch.nn.utils.clip_grad_norm_(self.params, self.max_norm))
        self.opt.step()
        if self.d is not None:
            for e, p in zip(self.ema, self.params):
                e.copy_(self.d * e + (1.0 - self.d) * p.detach())


def _view(flat, bucket, i, p):
    off = bucket.offsets[i]
    return flat[off:off + p.numel()].view_as(p)


def _new_opt(model, max_norm=None, ema_decay=None, eps=EPS):
    from equiformer_b200.parallel import CapturableFlatAdamW, FlatGradAllReduce
    bucket = FlatGradAllReduce(model.parameters())
    opt = CapturableFlatAdamW(model.named_parameters(), bucket, lr=LR, betas=BETAS, eps=eps, weight_decay=WD,
                              no_decay=model.no_weight_decay(), max_grad_norm=max_norm, ema_decay=ema_decay, model=model)
    return bucket, opt


def _load_grads(bucket, grads):
    bucket.zero_grad()
    for p, g in zip(bucket.params, grads):
        p.grad.copy_(g)


# ------------------------------------------------------------------------------------------------ GPU: the recipe
@pytest.mark.gpu
@pytest.mark.parametrize("ema", [False, True])
@pytest.mark.parametrize("clip", ["active", "inactive", "off"])
def test_five_steps_match_the_float64_recipe(cuda_device, clip, ema):
    """Parameters, m, v, EMA, clipped gradients and ``grad_norm`` agree with the float64 statement to about 1e-6 (the
    parameters' displacement from their start to 2e-5); ``active`` clips every step, ``inactive`` never does."""
    model = _qm9_model(cuda_device)
    max_norm = {"active": 100.0, "inactive": 1e6, "off": None}[clip]
    d = 0.9 if ema else None
    ref = Float64Recipe(model, max_norm, d)
    p0 = [p.detach().double().clone() for p in model.parameters()]
    bucket, opt = _new_opt(model, max_norm, d)
    for step in range(5):
        grads = [g.to(cuda_device) for g in _seeded_grads(model, step)]
        _load_grads(bucket, grads)
        opt.step()
        ref.step(grads)
    assert int(opt.t) == 5
    if max_norm is not None:
        assert abs(float(opt.grad_norm) - ref.norm) <= 1e-6 * ref.norm
        assert (ref.norm > max_norm) == (clip == "active")
    worst = {}
    for i, ((name, r), p) in enumerate(zip(ref.named, model.parameters())):
        st = ref.opt.state[r]
        checks = {"p": (p, r), "dp": (p.double() - p0[i], r.detach() - p0[i]), "grad": (p.grad, r.grad),
                  "m": (_view(opt.m, bucket, i, p), st["exp_avg"]), "v": (_view(opt.v, bucket, i, p), st["exp_avg_sq"])}
        if ema:
            checks["ema"] = (_view(opt.ema, bucket, i, p), ref.ema[i])
        for k, (a, b) in checks.items():
            worst[k] = max(worst.get(k, 0.0), rel_err(a, b))
    bounds = {"p": 1e-6, "dp": 2e-5, "grad": 1e-6, "m": 1e-6, "v": 1e-6, "ema": 1e-6}
    assert all(worst[k] <= bounds[k] for k in worst), worst


@pytest.mark.gpu
def test_kernel_matches_flat_adamw_without_clip_and_ema(cuda_device):
    from equiformer_b200.parallel import FlatAdamW, FlatGradAllReduce
    a, b = _qm9_model(cuda_device), _qm9_model(cuda_device)
    bucket_a, opt_a = _new_opt(a)
    bucket_b = FlatGradAllReduce(b.parameters())
    opt_b = FlatAdamW(b.named_parameters(), bucket_b, lr=LR, betas=BETAS, eps=EPS, weight_decay=WD,
                      no_decay=b.no_weight_decay())
    p0 = opt_b.flat.clone()
    for step in range(5):
        grads = [g.to(cuda_device) for g in _seeded_grads(a, step)]
        _load_grads(bucket_a, grads)
        _load_grads(bucket_b, grads)
        opt_a.step()
        opt_b.step()
    assert torch.equal(bucket_a.flat, bucket_b.flat)                 # no clip: the gradient is left as it is
    assert rel_err(opt_a.flat, opt_b.flat) <= 3e-7
    assert rel_err(opt_a.flat - p0, opt_b.flat - p0) <= 1e-5
    assert rel_err(opt_a.m, opt_b.m) <= 1e-6 and rel_err(opt_a.v, opt_b.v) <= 1e-6


@pytest.mark.gpu
def test_runs_are_bitwise_identical(cuda_device):
    runs = []
    for _ in range(2):
        model = _qm9_model(cuda_device)
        bucket, opt = _new_opt(model, 100.0, 0.9)
        for step in range(3):
            _load_grads(bucket, [g.to(cuda_device) for g in _seeded_grads(model, step)])
            opt.step()
        runs.append([opt.flat.clone(), opt.m.clone(), opt.v.clone(), opt.ema.clone(), bucket.flat.clone(),
                     opt.grad_norm.clone(), opt.t.clone()])
    assert all(torch.equal(x, y) for x, y in zip(*runs))


# ------------------------------------------------------------------------------------------------ GPU: raw kernels
def _raw_lengths():
    from equiformer_b200 import _lib
    per_pass = 4 * _lib.EQF_OPTIM_THREADS * _lib.EQF_OPTIM_MAX_CTAS
    return [1, 3, 4 * 257 + 1, 2 * per_pass + 4 * 1000 + 3]      # odd, and past two full passes of the grid


@pytest.mark.gpu
@pytest.mark.parametrize("n", _raw_lengths())
def test_raw_kernels_at_odd_lengths_and_past_the_grid_cap(cuda_device, n):
    """Two steps of clip + AdamW on synthetic flat buffers against float64, the first with the EMA (every kernel of
    OPTIM_CLAIMS runs); the step count advances, and the completion tickets are back at zero."""
    from equiformer_b200 import _lib, optim_kernels
    dev = cuda_device
    gen = torch.Generator(device=dev).manual_seed(n)
    rnd = lambda: torch.randn(n, generator=gen, device=dev)
    state = {"p": rnd(), "m": 0.1 * rnd(), "v": 0.01 * rnd().abs(), "ema": rnd(),
             "decay": torch.where(rnd() > 0, 0.01, 0.0)}
    lr, t = torch.full((1,), 3e-3, device=dev), torch.full((1,), 7, dtype=torch.int64, device=dev)
    partials = torch.zeros(_lib.EQF_OPTIM_MAX_CTAS, dtype=torch.float64, device=dev)
    tickets = torch.zeros(2, dtype=torch.int32, device=dev)
    norm, coef = torch.zeros(1, device=dev), torch.zeros(1, device=dev)
    ref = {k: v.double().clone() for k, v in state.items()}
    grads = [3.0 * rnd() for _ in range(2)]
    max_norm = 0.5 * float(grads[0].double().norm())

    grads_in = [g.double().clone() for g in grads]
    for step, g in enumerate(grads):
        ema = state["ema"] if step == 0 else None
        optim_kernels.flat_sqnorm_raw(g, max_norm, partials, tickets[0:1], norm, coef)
        optim_kernels.flat_adamw_raw(g, state["p"], state["m"], state["v"], state["decay"], ema, coef, lr, t, BETAS,
                                     EPS, 0.99, tickets[1:2])
    b1, b2 = BETAS
    for step, g in enumerate(grads_in):
        tn = g.norm()
        c = min(1.0, max_norm / (float(tn) + 1e-6))
        g = g * c
        k = 8 + step
        ref["m"] = b1 * ref["m"] + (1 - b1) * g
        ref["v"] = b2 * ref["v"] + (1 - b2) * g * g
        ref["p"] = ref["p"] * (1 - 3e-3 * ref["decay"])
        ref["p"] = ref["p"] - 3e-3 / (1 - b1 ** k) * ref["m"] / (ref["v"].sqrt() / (1 - b2 ** k) ** 0.5 + EPS)
        if step == 0:
            ref["ema"] = 0.99 * ref["ema"] + 0.01 * ref["p"]
        assert rel_err(grads[step], g) <= 1e-6
    assert abs(float(norm) - float(tn)) <= 1e-6 * float(tn)
    for k in ("p", "m", "v", "ema"):
        assert rel_err(state[k], ref[k]) <= 1e-6, k
    assert int(t) == 9 and int(tickets.abs().sum()) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("value", [float("nan"), float("inf")])
def test_non_finite_gradient_propagates_as_in_clip_grad_norm(cuda_device, value):
    model = _qm9_model(cuda_device)
    twins = [p.detach().clone().requires_grad_(True) for p in model.parameters()]
    grads = [g.to(cuda_device) for g in _seeded_grads(model, 0, nan_at=12345, value=value)]
    for p, g in zip(twins, grads):
        p.grad = g.clone()
    ref_norm = torch.nn.utils.clip_grad_norm_(twins, 100.0)
    bucket, opt = _new_opt(model, 100.0)
    _load_grads(bucket, grads)
    opt.step()
    assert torch.equal(torch.isnan(opt.grad_norm), torch.isnan(ref_norm.view(1)))
    assert torch.equal(torch.isinf(opt.grad_norm), torch.isinf(ref_norm.view(1)))
    for p, r in zip(model.parameters(), twins):
        assert torch.equal(torch.isnan(p.grad), torch.isnan(r.grad))
        assert torch.equal(torch.nan_to_num(p.grad, nan=7.0), torch.nan_to_num(r.grad, nan=7.0))


# ------------------------------------------------------------------------------------------------ GPU: capture, EMA
@pytest.mark.gpu
def test_captured_step_with_optimiser_equals_eager_sequence(cuda_device):
    """Forward + loss + backward + clip + AdamW + EMA captured in one graph and replayed 5 times, against the same
    captured forward / backward with the optimiser stepping eagerly after each replay.  ``set_lr`` between replays
    changes the update without a new capture (a zero rate leaves the parameters exactly as they were).  eps = 1e-3 keeps
    the update Lipschitz in the gradient, so the run-to-run ulps of the float atomics of the weight-gradient kernels
    stay at the ulp level in the parameters."""
    from equiformer_b200.graphs import GraphedForwardBackward
    from equiformer_b200.synthetic import qm9_like_batch
    pos, batch, z = qm9_like_batch(32, seed=0)
    target = torch.randn(32, 1, generator=torch.Generator().manual_seed(1))
    inp = [t.to(cuda_device) for t in (pos, batch, z, target)]
    l1 = lambda out, tgt: (out - tgt).abs().mean()
    lrs = [5e-4, 2e-3, 0.0, 1e-3, 5e-4]
    runs = []
    for captured in (True, False):
        model = _qm9_model(cuda_device)
        bucket, opt = _new_opt(model, 0.5, 0.9, eps=1e-3)
        gfb = GraphedForwardBackward(model, l1, bucket, max_radius=5.0, after_backward=opt.step if captured else None)
        losses = []
        for step, lr in enumerate(lrs):
            opt.set_lr(lr)
            before = opt.flat.clone()
            losses.append(float(gfb(*inp)))
            if not captured:
                opt.step()
            assert torch.equal(opt.flat, before) == (lr == 0.0), step
        assert gfb.captures == 1 and int(opt.t) == 5
        runs.append((losses, opt.flat.clone(), opt.m.clone(), opt.v.clone(), opt.ema.clone(), opt.grad_norm.clone()))
    (lc, *tc), (le, *te) = runs
    assert all(abs(a - b) <= 1e-5 * abs(b) for a, b in zip(lc, le)), (lc, le)
    errs = [rel_err(a, b) for a, b in zip(tc, te)]
    assert max(errs) <= 1e-5, errs


@pytest.mark.gpu
def test_ema_state_dict_and_weight_swap(cuda_device):
    from equiformer_b200.nets import model_entrypoint
    from tests.reference_fixtures import load_state
    model = _qm9_model(cuda_device)
    bucket, opt = _new_opt(model, None, 0.5)
    for step in range(3):
        _load_grads(bucket, [g.to(cuda_device) for g in _seeded_grads(model, step)])
        opt.step()
    sd = opt.ema_state_dict()
    assert list(sd) == list(model.state_dict())
    fresh = load_state(model_entrypoint(QM9)(irreps_in="5x0e", radius=5.0, num_basis=128).to(cuda_device), sd)
    for (k, a), b in zip(fresh.state_dict().items(), sd.values()):
        assert torch.equal(a, b), k
    assert not torch.equal(opt.ema, opt.flat)
    live = copy.deepcopy(model.state_dict())
    with opt.ema_weights() as m:
        assert m is model
        for (k, a), b in zip(model.state_dict().items(), sd.values()):
            assert torch.equal(a, b), k
    for (k, a), b in zip(model.state_dict().items(), live.values()):
        assert torch.equal(a, b), k


@pytest.mark.gpu
def test_entry_points_refuse_misaligned_and_empty_device_buffers(cuda_device):
    """The entry points return their checks' errors on real device buffers 4 bytes off alignment and on n = 0, and
    leave the buffers untouched."""
    from equiformer_b200 import _lib
    lib = _lib.load_optim()
    buf = torch.ones(4096, device=cuda_device)
    part = torch.zeros(_lib.EQF_OPTIM_MAX_CTAS, dtype=torch.float64, device=cuda_device)
    ints = torch.zeros(4, dtype=torch.int64, device=cuda_device)
    ok, off = buf.data_ptr(), buf[1:].data_ptr()
    ticket, scal, step = ints.data_ptr(), buf[-4:].data_ptr(), ints[2:].data_ptr()
    stream = torch.cuda.current_stream().cuda_stream
    msg = lambda: lib.eqf_last_error().decode()
    assert lib.eqf_flat_sqnorm(off, 64, 1.0, part.data_ptr(), ticket, scal, scal, stream) != 0 and "aligned" in msg()
    assert lib.eqf_flat_sqnorm(ok, 0, 1.0, part.data_ptr(), ticket, scal, scal, stream) != 0 and "positive" in msg()
    for bad in range(6):
        ptrs = [off if i == bad else ok for i in range(6)]
        rc = lib.eqf_flat_adamw(*ptrs, 64, scal, scal, step, 0.9, 0.999, 1e-8, 0.9, ticket, stream)
        assert rc != 0 and "aligned" in msg(), bad
    assert lib.eqf_flat_adamw(ok, ok, ok, ok, ok, None, 0, scal, scal, step, 0.9, 0.999, 1e-8, 0.0, ticket, stream) != 0
    torch.cuda.synchronize()
    assert bool((buf == 1).all()) and int(ints.abs().sum()) == 0 and int(part.abs().sum()) == 0


def _hook_setup(dev):
    """QM9 model, bucket, optimiser (clip + EMA) and a 24-molecule batch on the device."""
    from equiformer_b200.synthetic import qm9_like_batch
    model = _qm9_model(dev)
    bucket, opt = _new_opt(model, 0.5, 0.9)
    pos, batch, z = qm9_like_batch(24, seed=3)
    target = torch.randn(24, 1, generator=torch.Generator().manual_seed(4))
    return model, bucket, opt, [t.to(dev) for t in (pos, batch, z, target)]


@pytest.mark.gpu
@pytest.mark.parametrize("capture", [True, False])
def test_bucketed_step_runs_the_hook_once_per_call(cuda_device, capture):
    """``BucketedForwardBackward``: the optimiser steps once per call, captured (never in the warm-up passes) or eager."""
    from equiformer_b200.graphs import BucketedForwardBackward
    model, bucket, opt, inp = _hook_setup(cuda_device)
    step = BucketedForwardBackward(model, lambda out, tgt: (out - tgt).abs().mean(), bucket, max_radius=5.0,
                                   capture=capture, after_backward=opt.step)
    for k in range(3):
        before = opt.flat.clone()
        assert bool(torch.isfinite(step(*inp)))
        assert int(opt.t) == k + 1 and not torch.equal(opt.flat, before)
    assert step.captures == (1 if capture else 0)


@pytest.mark.gpu
def test_graphed_step_runs_the_hook_once_per_replay(cuda_device):
    """``GraphedStep``: the optimiser steps once per replay and never in the warm-up passes before the capture."""
    from equiformer_b200.graph import radius_graph_csr
    from equiformer_b200.graphs import GraphedStep, csr_graph
    model, bucket, opt, (pos, batch, z, target) = _hook_setup(cuda_device)

    def fn(pos, batch, z, target, src, dst, row_ptr):
        out = model.forward_edges(pos, batch, z, src, dst, graph=csr_graph(src, dst, row_ptr, pos.shape[0]),
                                  n_graphs=target.shape[0])
        return (out - target).abs().mean()

    edge, row_ptr = radius_graph_csr(pos, 5.0, batch, max_num_neighbors=1000)
    tensors = [pos, batch, z, target, edge[0], edge[1], row_ptr]
    step = GraphedStep(fn, bucket, after_backward=opt.step)
    for k in range(3):
        before = opt.flat.clone()
        step((int(pos.shape[0]), int(edge.shape[1])), tensors)
        assert int(opt.t) == k + 1 and not torch.equal(opt.flat, before)
    assert step.captures == 1


@pytest.mark.gpu
@pytest.mark.parametrize("capture", [True, False])
def test_dens_step_runs_the_hook_once_per_call(cuda_device, capture):
    """``DensTrainStep``: the optimiser steps once per call, inside the captured graph or after the eager backward."""
    from equiformer_b200.graphs import DensTrainStep
    from equiformer_b200.nets.equiformer_md17_dens import Equiformer_MD17_DeNS
    from equiformer_b200.parallel import CapturableFlatAdamW, FlatGradAllReduce
    from tests.reference_fixtures import load
    case = load("reference_model_dens_small.npz")
    torch.manual_seed(0)
    model = Equiformer_MD17_DeNS(**case.cfg).to(cuda_device).eval()
    bucket = FlatGradAllReduce(model.parameters())
    opt = CapturableFlatAdamW(model.named_parameters(), bucket, lr=LR, weight_decay=1e-6, max_grad_norm=1.0,
                              ema_decay=0.9, model=model)
    pos, batch, z = case.t("pos", cuda_device).float(), case.t("batch", cuda_device), case.t("z", cuda_device)
    G = int(batch.max()) + 1
    gen = torch.Generator().manual_seed(2)
    y, dy = torch.randn(G, 1, generator=gen).to(cuda_device), torch.randn(pos.shape, generator=gen).to(cuda_device)
    step = DensTrainStep(model, bucket, capture=capture, after_backward=opt.step)
    noise = torch.Generator(device=cuda_device).manual_seed(4)
    for k in range(3):
        before = opt.flat.clone()
        assert bool(torch.isfinite(step(pos, batch, z, y, dy, G, 0.5, generator=noise)))
        assert int(opt.t) == k + 1 and not torch.equal(opt.flat, before)


@pytest.mark.gpu
def test_hook_and_captured_step_are_refused_across_processes(cuda_device, monkeypatch):
    """Across processes the optimiser must step after the all-reduce: the graphed steps refuse it as ``after_backward``
    and ``step()`` refuses to run inside a capture."""
    from equiformer_b200.graphs import BucketedForwardBackward, DensTrainStep, GraphedForwardBackward, GraphedStep
    model, bucket, opt, _inp = _hook_setup(cuda_device)
    monkeypatch.setattr(bucket, "world", 2)
    l1 = lambda out, tgt: (out - tgt).abs().mean()
    for make in (lambda: GraphedForwardBackward(model, l1, bucket, 5.0, after_backward=opt.step),
                 lambda: BucketedForwardBackward(model, l1, bucket, 5.0, capture=False, after_backward=opt.step),
                 lambda: GraphedStep(l1, bucket, after_backward=opt.step),
                 lambda: DensTrainStep(model, bucket, capture=False, after_backward=opt.step)):
        with pytest.raises(ValueError, match="bucket.reduce"):
            make()
    GraphedForwardBackward(model, l1, bucket, 5.0)                       # without the hook nothing changes
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    t0 = int(opt.t)
    with pytest.raises(RuntimeError, match="all-reduce"):
        opt.step()
    monkeypatch.undo()
    assert int(opt.t) == t0
