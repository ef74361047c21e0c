#!/usr/bin/env python
"""Step time of OC20 IS2RE training with the IS2RS auxiliary task (the ``*_aux_*`` configurations) on one GPU.

    python tools/oc20_aux_step.py --workload aux6  [--steps K --warmup W]   # OC20_L1_256_NONLINEAR_AUX, 16 frames
    python tools/oc20_aux_step.py --workload aux18 [--eager]                # OC20_L1_256_BLOCKS18_NONLINEAR_AUX, 8 frames
    python tools/oc20_aux_step.py --workload aux6 --drop-path-rate 0 --alpha-drop 0    # regularisers off

Inputs are ``synthetic.oc20_like_frames`` (as ``bench.py --workload oc20_l1``) plus seeded relaxed positions.  One step:

1. ``interpolate_init_relaxed_pos`` (the augmentation of ``use_interpolate_init_relaxed_pos``);
2. the periodic neighbour list (``graph.radius_graph_pbc``, eager);
3. forward, ``L1(energy) + w * masked_l2mae(aux, relaxation_target)`` with ``w = auxiliary_task_weight(step)``, backward -
   captured once and replayed through ``graphs.GraphedStep``;
4. AdamW (``parallel.FlatAdamW``, lr 5e-4, weight decay 1e-3 as in the configurations).

The interpolation generator is re-seeded every step, so every step sees the same positions and edge count and the one
capture is replayed (a new edge count would need a new capture).  The regularisers run as configured (``drop_path_rate=0.05``,
``alpha_drop=0.2``) unless ``--drop-path-rate`` / ``--alpha-drop`` override them: stochastic depth draws its per-graph
factors from ``n_graphs`` and attention dropout draws its mask with torch's generator, so both are captured and every
replay draws afresh.  ``--eager`` times the same step without capture.  The JSON line says what was timed.
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
    # config dict, frames per GPU, positions_std of the configuration's dataset block
    "aux6": ("OC20_L1_256_NONLINEAR_AUX", 16, 0.9452036023139954),
    "aux18": ("OC20_L1_256_BLOCKS18_NONLINEAR_AUX", 8, 0.8771552443504333),
}
AUX_WEIGHT, TOTAL_STEPS = 15.0, 100_000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=sorted(WORKLOADS), default="aux6")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--eager", action="store_true", help="no CUDA graph")
    ap.add_argument("--drop-path-rate", type=float, default=None, help="stochastic depth rate (default: as configured)")
    ap.add_argument("--alpha-drop", type=float, default=None, help="attention-weight dropout (default: as configured)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("oc20_aux_step.py needs a CUDA device")

    from equiformer_b200 import _lib, ops
    from equiformer_b200.graph import radius_graph_pbc
    from equiformer_b200.graphs import GraphedStep
    from equiformer_b200.nets import graph_attention_transformer_oc20 as M
    from equiformer_b200.oc20_objective import (auxiliary_task_weight, interpolate_init_relaxed_pos, masked_l2mae,
                                                relaxation_target)
    from equiformer_b200.parallel import FlatAdamW, FlatGradAllReduce

    _lib.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg_name, n_frames, pos_std = WORKLOADS[args.workload]
    cfg = dict(getattr(M, cfg_name))
    if args.drop_path_rate is not None:
        cfg["drop_path_rate"] = args.drop_path_rate
    if args.alpha_drop is not None:
        cfg["alpha_drop"] = args.alpha_drop
    torch.manual_seed(0)
    model = M.GraphAttentionTransformerOC20(None, None, 1, **cfg).to(dev).train()
    bucket = FlatGradAllReduce(model.parameters())
    opt = FlatAdamW(model.named_parameters(), bucket, lr=5e-4, weight_decay=1e-3, no_decay=model.no_weight_decay())

    inp = {k: v.to(dev) for k, v in bench.make_inputs("oc20_l1", seed=0, n_graphs=n_frames).items()}
    g = torch.Generator().manual_seed(2024)
    relaxed = inp["pos"] + 0.3 * torch.randn(inp["pos"].shape, generator=g).to(dev)
    n = int(inp["pos"].shape[0])
    gen = torch.Generator(device=dev)

    def prepare(step):
        """Interpolation + periodic neighbour list + per-step scalars (eager)."""
        gen.manual_seed(7)
        pos = interpolate_init_relaxed_pos(inp["pos"], relaxed, inp["batch"], inp["tags"], n_frames, generator=gen)
        edge, offs, _ = radius_graph_pbc(pos, inp["batch"], inp["cell"], 5.0, cfg["max_neighbors"])
        src, dst = edge[0], edge[1]
        cells = inp["cell"].index_select(0, inp["batch"].index_select(0, dst))
        edge_vec = pos.index_select(0, src) - pos.index_select(0, dst) + torch.bmm(offs.to(pos.dtype).view(-1, 1, 3), cells).view(-1, 3)
        row_ptr = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        torch.cumsum(torch.zeros(n, dtype=torch.int64, device=dev).index_add_(0, dst, torch.ones_like(dst)), 0, out=row_ptr[1:])
        aux_target = relaxation_target(pos, relaxed, pos_std)
        w = torch.full((1,), auxiliary_task_weight(step, TOTAL_STEPS, AUX_WEIGHT), device=dev)
        return [edge_vec, inp["target"], aux_target, w, inp["batch"], inp["z"], inp["tags"], src, dst, row_ptr]

    def loss_fn(edge_vec, target, aux_target, w, batch, z, tags, src, dst, row_ptr, graph=None):
        energy, aux = model.forward_edges(edge_vec, batch, z, tags, src, dst, graph=graph, n_graphs=n_frames)
        return (energy - target).abs().mean() + w[0] * masked_l2mae(aux, aux_target, tags)

    def captured(edge_vec, target, aux_target, w, batch, z, tags, src, dst, row_ptr):
        csr = ops.Graph.__new__(ops.Graph)
        csr.n_nodes, csr.n_edges, csr.perm = n, int(src.numel()), None
        csr.src, csr.dst, csr.row_ptr = src, dst, row_ptr
        csr._src_perm = csr._src_row_ptr = None
        return loss_fn(edge_vec, target, aux_target, w, batch, z, tags, src, dst, row_ptr, graph=csr)

    graphed = None if args.eager else GraphedStep(captured, bucket)
    edges = []

    def step(i):
        t = prepare(i)
        edges.append(int(t[7].numel()))
        if graphed is None:
            bucket.zero_grad()
            loss = loss_fn(*t)
            loss.backward()
        else:
            loss = graphed((n, edges[-1], n_frames), t)
        bucket.reduce()
        opt.step()
        return loss

    for i in range(max(args.warmup, 1) + (0 if args.eager else 1)):     # the first graphed step includes the capture
        step(i)
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for i in range(args.steps):
        loss = step(args.warmup + i)
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end) / args.steps
    e = edges[-1]
    print(json.dumps({
        "metric": f"edges/sec fwd+bwd, OC20 IS2RE {cfg_name} + IS2RS auxiliary loss", "workload": args.workload,
        "value": e / (ms * 1e-3), "unit": "edges/s", "ms_per_step": ms, "steps": args.steps, "edges_per_step": e,
        "atoms_per_step": n, "frames": n_frames, "num_layers": cfg["num_layers"],
        "launch": ("eager (no CUDA graph)" if args.eager else
                   "CUDA-graph replay of forward+loss+backward; interpolation, neighbour list and AdamW eager"),
        "drop_path_rate": cfg["drop_path_rate"], "alpha_drop": cfg["alpha_drop"],
        "configured": {"drop_path_rate": getattr(M, cfg_name)["drop_path_rate"], "alpha_drop": getattr(M, cfg_name)["alpha_drop"]},
        "captures": getattr(graphed, "captures", None), "loss": loss.item(),
        "max_memory_gb": torch.cuda.max_memory_allocated(dev) / 1e9,
        "device": torch.cuda.get_device_name(dev), "power_limit_w": bench.power_limit(0),
    }), flush=True)


if __name__ == "__main__":
    main()
