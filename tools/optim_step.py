#!/usr/bin/env python
"""Optimiser step with gradient clipping and a model EMA: the fused kernels beside the torch chain, and the captured QM9
step with the optimiser inside the graph beside AdamW stepping eagerly after it.

    python tools/optim_step.py [--steps K --warmup W --rounds R]

Optimiser step, on the flat parameter buffer of the ``bench.py`` QM9 model (``graph_attention_transformer_nonlinear_l2``)
and of the OC20 E(3) model (``OC20_L1_256_E3_NONLINEAR``), seeded gradients:
  a) ``FlatAdamW.step()``;
  b) a) plus ``torch.nn.utils.clip_grad_norm_`` over the flat gradient (one tensor whose ``.grad`` is the bucket) and an
     EMA ``lerp_`` of the flat parameters;
  c) ``CapturableFlatAdamW.step()`` with clipping and the EMA on (``eqf_flat_sqnorm`` + ``eqf_flat_adamw``);
  d) c) with the OC20 cosine schedule of ``l1_256_nonlinear`` attached (``eqf_flat_adamw_scheduled``: the same kernel
     instances, thread 0 of each CTA evaluating the rate).
Each is timed with CUDA events over 10 x ``--steps`` eager steps.  ``max_norm`` is half the seeded gradient's norm; b) and
c) share the gradient, so after the first clip its norm sits at ``max_norm`` and every later step scales it by
``max_norm / (norm + 1e-6)`` (the full clip arithmetic, a factor just below 1).

Training step, ``bench.py --workload qm9`` batch (128 molecules, radius 5, attention dropout off): neighbour list + replay
of ``GraphedForwardBackward`` (forward, L1 loss, backward), then
  eager:    ``FlatAdamW.step()`` after the replay;
  captured: clip (max norm 5) + AdamW + EMA (decay 0.9999) inside the replayed graph (``after_backward``);
  captured_scheduled: the same with the OC20 cosine schedule attached (no host write between replays).
Each step ends in a device synchronise.  The variants alternate for ``--rounds`` rounds in one process and the line reports
each one's best round, with the card's name, power limit and SM clock read before and after.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
from lmax4_step import _card, _no_dropout  # noqa: E402

LR, WD, EMA_DECAY = 5e-4, 5e-3, 0.9999
# the optim block of oc20/configs/is2re/all/graph_attention_transformer/l1_256_nonlinear_g@2_local.yml
OC20_OPTIM = {"lr_initial": 0.0002, "max_epochs": 20, "scheduler": "LambdaLR",
              "scheduler_params": {"lambda_type": "cosine", "warmup_factor": 0.2, "warmup_epochs": 2,
                                   "lr_min_factor": 1.e-2}}


def _oc20_schedule():
    from equiformer_b200.lr_schedule import LrSchedule
    return LrSchedule.from_oc20_optim(OC20_OPTIM, n_iter_per_epoch=1000)


def _model(name, dev):
    from equiformer_b200.nets import model_entrypoint
    from equiformer_b200.nets.graph_attention_transformer_oc20 import OC20_L1_256_E3_NONLINEAR
    torch.manual_seed(0)
    if name == "qm9":
        model = model_entrypoint(bench.WORKLOADS["qm9"]["model"])(irreps_in="5x0e", radius=5.0, num_basis=128)
    else:
        model = model_entrypoint("graph_attention_transformer_oc20")(**OC20_L1_256_E3_NONLINEAR)
    return _no_dropout(model.to(dev).train())


def optimiser_variants(name, dev):
    """-> (floats in the flat buffer, {variant: step function}) on one model's buffers."""
    from equiformer_b200.parallel import CapturableFlatAdamW, FlatAdamW, FlatGradAllReduce
    model = _model(name, dev)
    bucket = FlatGradAllReduce(model.parameters())
    bucket.flat.copy_(torch.randn(bucket.flat.shape, generator=torch.Generator(device=dev).manual_seed(1), device=dev))
    max_norm = 0.5 * float(bucket.flat.norm())
    skip = model.no_weight_decay()
    flat_adamw = FlatAdamW(model.named_parameters(), bucket, lr=LR, weight_decay=WD, no_decay=skip)
    ema = flat_adamw.flat.clone()
    # clip_grad_norm_ reads `.grad`: a holder whose gradient IS the flat bucket gives one norm over the whole buffer
    holder = torch.empty_like(bucket.flat, requires_grad=True)
    holder.grad = bucket.flat
    pre = float(torch.nn.utils.clip_grad_norm_([holder], max_norm))
    if not (pre > max_norm and float(bucket.flat.norm()) < 1.0001 * max_norm):
        raise RuntimeError(f"the torch clip chain did not clip the flat gradient (norm {pre}, max_norm {max_norm})")

    def torch_chain():
        torch.nn.utils.clip_grad_norm_([holder], max_norm)
        flat_adamw.step()
        ema.lerp_(flat_adamw.flat, 1.0 - EMA_DECAY)

    fused = CapturableFlatAdamW(model.named_parameters(), bucket, lr=LR, weight_decay=WD, no_decay=skip,
                                max_grad_norm=max_norm, ema_decay=EMA_DECAY, model=model)
    scheduled = CapturableFlatAdamW(model.named_parameters(), bucket, weight_decay=WD, no_decay=skip,
                                    max_grad_norm=max_norm, ema_decay=EMA_DECAY, model=model,
                                    lr_schedule=_oc20_schedule())
    return bucket.flat.numel(), {"flat_adamw": flat_adamw.step, "flat_adamw_torch_clip_ema": torch_chain,
                                 "fused_clip_adamw_ema": fused.step, "fused_clip_adamw_ema_scheduled": scheduled.step}


def _events(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / steps


def qm9_steps(dev, inp):
    from equiformer_b200.graphs import GraphedForwardBackward
    from equiformer_b200.parallel import CapturableFlatAdamW, FlatAdamW, FlatGradAllReduce
    l1 = lambda out, tgt: (out - tgt).abs().mean()
    steps = {}
    for variant in ("eager_adamw", "captured_clip_adamw_ema", "captured_clip_adamw_ema_scheduled"):
        model = _model("qm9", dev)
        bucket = FlatGradAllReduce(model.parameters())
        skip = model.no_weight_decay()
        if variant == "eager_adamw":
            opt = FlatAdamW(model.named_parameters(), bucket, lr=LR, weight_decay=WD, no_decay=skip)
            gfb = GraphedForwardBackward(model, l1, bucket, max_radius=5.0)
            steps[variant] = lambda gfb=gfb, opt=opt: (gfb(inp["pos"], inp["batch"], inp["z"], inp["target"]), opt.step())
        else:
            schedule = _oc20_schedule() if variant.endswith("_scheduled") else None
            opt = CapturableFlatAdamW(model.named_parameters(), bucket, lr=LR, weight_decay=WD, no_decay=skip,
                                      max_grad_norm=5.0, ema_decay=EMA_DECAY, model=model, lr_schedule=schedule)
            gfb = GraphedForwardBackward(model, l1, bucket, max_radius=5.0, after_backward=opt.step)
            steps[variant] = lambda gfb=gfb: gfb(inp["pos"], inp["batch"], inp["z"], inp["target"])
    return steps


def _host_timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("optim_step.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cuda.matmul.allow_tf32 = False
    res = {"card": _card()}
    opt_runs = {}
    for name in ("qm9", "oc20_e3"):
        n, fns = optimiser_variants(name, dev)
        res[f"{name}_flat_floats"] = n
        opt_runs[name] = fns
    inp = {k: v.to(dev) for k, v in bench.make_inputs("qm9", seed=0).items()}
    train = qm9_steps(dev, inp)
    best = {}
    for _ in range(args.rounds):
        for name, fns in opt_runs.items():
            for v, fn in fns.items():
                us = _events(fn, 10 * args.steps, args.warmup)
                best[f"{name}_{v}_us"] = min(best.get(f"{name}_{v}_us", us), us)
        for v, fn in train.items():
            ms = _host_timed(fn, args.steps, args.warmup)
            best[f"qm9_step_{v}_ms"] = min(best.get(f"qm9_step_{v}_ms", ms), ms)
    res.update({k: round(x, 3) for k, x in best.items()})
    res["card_after"] = _card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
