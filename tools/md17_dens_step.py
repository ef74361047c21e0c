#!/usr/bin/env python
"""Step time of MD17 DeNS training (the ``equiformer_dens`` configurations) on one GPU.

    python tools/md17_dens_step.py --workload dens_l2 [--steps K --warmup W --batches B]   # MD17_DENS_L2, 8 conformers
    python tools/md17_dens_step.py --workload dens_l3 [--eager]                           # MD17_DENS_L3, 5 conformers

Inputs are ``--batches`` seeded batches of aspirin-sized conformers (``synthetic.aspirin_like``, as ``bench.py --workload
md17_l3``) with seeded energy / force targets, cycled one per step.  One step (``graphs.DensTrainStep``):

1. ``add_masked_gaussian_noise`` with fresh draws every step (std 0.05, prob 0.25, corrupt ratio 0.25);
2. the neighbour list (``graph.radius_graph_csr``, eager);
3. padding to a bucket (``graphs.pad_to_bucket``, eager);
4. forward (energy, forces by a ``create_graph`` backward, denoising head), ``dens_loss`` (energy 1, force 80, denoising
   weight 5 decayed linearly over the epochs) and the backward - captured once per bucket and replayed;
5. AdamW (``parallel.FlatAdamW``: lr 5e-4 for L2, 2e-4 for L3, weight decay 1e-6 as in the scripts).

Batches and noise change the edge count from step to step; the JSON line reports how many captures the run needed.
``--eager`` times the same step without capture or padding.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

WORKLOADS = {
    # config dict, conformers per batch, learning rate, epochs (scripts/train/md17/equiformer_dens/se_l{2,3}/)
    "dens_l2": ("MD17_DENS_L2", 8, 5e-4, 1500),
    "dens_l3": ("MD17_DENS_L3", 5, 2e-4, 2000),
}
STD, PROB, CORRUPT_RATIO, DN_WEIGHT, W_E, W_F = 0.05, 0.25, 0.25, 5.0, 1.0, 80.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=sorted(WORKLOADS), default="dens_l3")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=8, help="untimed steps (they include the captures)")
    ap.add_argument("--batches", type=int, default=8, help="seeded conformer batches cycled over the steps")
    ap.add_argument("--eager", action="store_true", help="no CUDA graph")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("md17_dens_step.py needs a CUDA device")

    from equiformer_b200 import _lib
    from equiformer_b200.graphs import DensTrainStep
    from equiformer_b200.md17_dens_objective import denoising_pos_weight
    from equiformer_b200.nets import equiformer_md17_dens as M
    from equiformer_b200.parallel import FlatAdamW, FlatGradAllReduce
    from equiformer_b200.synthetic import aspirin_like

    _lib.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg_name, B, lr, epochs = WORKLOADS[args.workload]
    torch.manual_seed(0)
    model = M.Equiformer_MD17_DeNS(**getattr(M, cfg_name)).to(dev).train()
    bucket = FlatGradAllReduce(model.parameters())
    opt = FlatAdamW(model.named_parameters(), bucket, lr=lr, weight_decay=1e-6, no_decay=model.no_weight_decay())
    step_fn = DensTrainStep(model, bucket, task_mean=0.0, task_std=1.0, std=STD, prob=PROB, corrupt_ratio=CORRUPT_RATIO,
                            w_e=W_E, w_f=W_F, capture=not args.eager)

    batches = []
    for b in range(args.batches):
        confs = [aspirin_like(seed=b * 64 + s) for s in range(B)]
        g = torch.Generator().manual_seed(1000 + b)
        batches.append(tuple(t.to(dev) for t in (torch.cat([c[0] for c in confs]), torch.arange(B).repeat_interleave(21),
                                                 torch.cat([c[2] for c in confs]), torch.randn(B, 1, generator=g),
                                                 torch.randn(21 * B, 3, generator=g))))
    gen = torch.Generator(device=dev).manual_seed(7)
    w_dn = torch.full((1,), denoising_pos_weight(0, epochs, DN_WEIGHT, True), device=dev)
    edges = []

    def step(i):
        pos, batch, z, y, dy = batches[i % len(batches)]
        loss = step_fn(pos, batch, z, y, dy, B, w_dn, generator=gen)
        edges.append(step_fn.last_edges)
        bucket.reduce()
        opt.step()
        return loss

    for i in range(max(args.warmup, 1)):
        step(i)
    torch.cuda.synchronize()
    captures_before = step_fn.captures
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for i in range(args.steps):
        loss = step(args.warmup + i)
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end) / args.steps
    timed = edges[-args.steps:]
    e = sum(timed) / len(timed)
    print(json.dumps({
        "metric": f"edges/sec fwd+bwd, MD17 DeNS {cfg_name} (energy + force + denoising step)", "workload": args.workload,
        "value": e / (ms * 1e-3), "unit": "edges/s", "ms_per_step": ms, "steps": args.steps, "warmup": args.warmup,
        "batches": args.batches, "conformers": B, "atoms_per_step": 21 * B, "edges_per_step_mean": e,
        "edges_per_step_range": [min(timed), max(timed)],
        "launch": ("eager (no CUDA graph, no padding)" if args.eager else
                   "CUDA-graph replay of forward+loss+backward per bucket; noise, neighbour list, padding and AdamW eager"),
        "captures": None if args.eager else step_fn.captures,
        "captures_in_timed_steps": None if args.eager else step_fn.captures - captures_before,
        "std": STD, "prob": PROB, "corrupt_ratio": CORRUPT_RATIO, "lr": lr, "loss": loss.item(),
        "max_memory_gb": torch.cuda.max_memory_allocated(dev) / 1e9,
        "device": torch.cuda.get_device_name(dev), "power_limit_w": bench.power_limit(0),
    }), flush=True)


if __name__ == "__main__":
    main()
