#!/usr/bin/env python
"""Step time of OC20 IS2RE training of the E(3) graph-attention model (``OC20_L1_256_E3_NONLINEAR``) on one GPU.

    python tools/oc20_e3_step.py [--steps K --warmup W] [--eager] [--frames 16]

Inputs are ``synthetic.oc20_like_frames`` (as ``bench.py --workload oc20_l1``).  One step: the periodic neighbour list
(``graph.radius_graph_pbc``, eager; ``max_neighbors=500`` as configured), then forward, energy L1 loss and backward -
captured once and replayed through ``graphs.GraphedStep`` - then AdamW (``parallel.FlatAdamW``, lr 2e-4, weight decay
1e-3 as in the configuration).  Attention dropout runs as configured (``alpha_drop=0.2``); its mask is drawn with torch's
generator inside the capture, so every replay draws afresh.  ``--eager`` times the same step without capture.  The
model's depth-wise products all run the one plan ``256x0e+64x0o+64x1e+64x1o x 1x0e+1x1o``; the JSON line says whether the
library in use has a generated kernel for it (``dtp_generated``).
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--eager", action="store_true", help="no CUDA graph")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("oc20_e3_step.py needs a CUDA device")

    from equiformer_b200 import _lib, ops
    from equiformer_b200.graph import radius_graph_pbc
    from equiformer_b200.graphs import GraphedStep
    from equiformer_b200.nets import model_entrypoint
    from equiformer_b200.nets.graph_attention_transformer_oc20 import OC20_L1_256_E3_NONLINEAR as CFG
    from equiformer_b200.parallel import FlatAdamW, FlatGradAllReduce

    _lib.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    model = model_entrypoint("graph_attention_transformer_oc20")(**CFG).to(dev).train()
    bucket = FlatGradAllReduce(model.parameters())
    opt = FlatAdamW(model.named_parameters(), bucket, lr=2e-4, weight_decay=1e-3, no_decay=model.no_weight_decay())

    n_frames = args.frames
    inp = {k: v.to(dev) for k, v in bench.make_inputs("oc20_l1", seed=0, n_graphs=n_frames).items()}
    n = int(inp["pos"].shape[0])

    def prepare():
        pos = inp["pos"]
        edge, offs, _ = radius_graph_pbc(pos, inp["batch"], inp["cell"], CFG["max_radius"],
                                         CFG["max_neighbors"])
        src, dst = edge[0], edge[1]
        cells = inp["cell"].index_select(0, inp["batch"].index_select(0, dst))
        edge_vec = pos.index_select(0, src) - pos.index_select(0, dst) + torch.bmm(offs.to(pos.dtype).view(-1, 1, 3), cells).view(-1, 3)
        row_ptr = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        torch.cumsum(torch.zeros(n, dtype=torch.int64, device=dev).index_add_(0, dst, torch.ones_like(dst)), 0, out=row_ptr[1:])
        return [edge_vec, inp["target"], inp["batch"], inp["z"], inp["tags"], src, dst, row_ptr]

    def loss_fn(edge_vec, target, batch, z, tags, src, dst, row_ptr, graph=None):
        energy = model.forward_edges(edge_vec, batch, z, tags, src, dst, graph=graph, n_graphs=n_frames)
        return (energy - target).abs().mean()

    def captured(edge_vec, target, batch, z, tags, src, dst, row_ptr):
        csr = ops.Graph.__new__(ops.Graph)
        csr.n_nodes, csr.n_edges, csr.perm = n, int(src.numel()), None
        csr.src, csr.dst, csr.row_ptr = src, dst, row_ptr
        csr._src_perm = csr._src_row_ptr = None
        return loss_fn(edge_vec, target, batch, z, tags, src, dst, row_ptr, graph=csr)

    graphed = None if args.eager else GraphedStep(captured, bucket)
    edges = []

    def step():
        t = prepare()
        edges.append(int(t[5].numel()))
        if graphed is None:
            bucket.zero_grad()
            loss = loss_fn(*t)
            loss.backward()
        else:
            loss = graphed((n, edges[-1], n_frames), t)
        bucket.reduce()
        opt.step()
        return loss

    for _ in range(max(args.warmup, 1) + (0 if args.eager else 1)):     # the first graphed step includes the capture
        step()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(args.steps):
        loss = step()
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end) / args.steps
    e = edges[-1]
    print(json.dumps({
        "metric": "edges/sec fwd+bwd, OC20 IS2RE graph_attention_transformer l1_256_e3_nonlinear (OC20_L1_256_E3_NONLINEAR)",
        "value": e / (ms * 1e-3), "unit": "edges/s", "ms_per_step": ms, "steps": args.steps, "edges_per_step": e,
        "atoms_per_step": n, "frames": n_frames, "num_layers": CFG["num_layers"],
        "alpha_drop": CFG["alpha_drop"], "dtp_generated": bool(model.edge_deg_embed.dw.tp.plan.generated),
        "launch": ("eager (no CUDA graph)" if args.eager else
                   "CUDA-graph replay of forward+loss+backward; neighbour list and AdamW eager"),
        "captures": getattr(graphed, "captures", None), "loss": loss.item(),
        "max_memory_gb": torch.cuda.max_memory_allocated(dev) / 1e9,
        "device": torch.cuda.get_device_name(dev), "power_limit_w": bench.power_limit(0),
    }), flush=True)


if __name__ == "__main__":
    main()
