#!/usr/bin/env python
"""Captured QM9 training step with the layer, graph and instance norms, and the norm kernels beside the torch chain.

    python tools/norm_step.py [--steps K --warmup W --rounds R]

Step: ``graph_attention_transformer_nonlinear_l2`` (``bench.py --workload qm9``: 128 molecules, radius 5) with
``norm_layer`` set to ``layer``, ``graph`` and ``instance``, attention dropout off; one step = neighbour list + replay of
``GraphedForwardBackward`` (forward, L1 loss, backward), ending in a device synchronise.  The three models are timed in
turn, ``--rounds`` times, in one process; the line reports each one's best round (mean ms per step).

Norm: one ``EquivariantGraphNorm`` over the QM9 node irreps ``128x0e+64x1e+32x2e`` of the same batch, forward +
backward (the gradients of the input and the three parameters), on the kernels (``ops.SegmentNorm``) and on the
torch statement (``ops.segment_norm_planar_torch``).  Each is captured in a CUDA graph and the replays are timed with
CUDA events over 200 replays, so the figure is device time without the host's launch overhead (µs per forward +
backward).  The card's name, power limit and SM clocks are read in the same call.
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


def qm9_step(norm, dev, inp):
    from equiformer_b200.graphs import GraphedForwardBackward
    from equiformer_b200.nets.graph_attention_transformer import _qm9
    from equiformer_b200.parallel import FlatGradAllReduce
    torch.manual_seed(0)
    model = _no_dropout(_qm9("5x0e", 5.0, 128, None, None, None, nonlinear_message=True, norm_layer=norm).to(dev).train())
    bucket = FlatGradAllReduce(model.parameters())
    gfb = GraphedForwardBackward(model, lambda out, tgt: (out - tgt).abs().mean(), bucket, max_radius=5.0)
    return lambda: gfb(inp["pos"], inp["batch"], inp["z"], inp["target"])


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / steps


def norm_calls(dev, inp, steps, warmup):
    from equiformer_b200 import ops
    from equiformer_b200.nets.graph_norm import EquivariantGraphNorm
    m = EquivariantGraphNorm("128x0e+64x1e+32x2e").to(dev)
    batch = inp["batch"]
    G = int(inp["target"].shape[0])
    gen = torch.Generator(device=dev).manual_seed(1)
    xs = [torch.randn(batch.shape[0], ir.dim, mul, generator=gen, device=dev, requires_grad=True) for mul, ir in m.irreps]
    gys = [torch.randn(x.shape, generator=gen, device=dev) for x in xs]
    seg = ops.GraphSegments(batch, G)
    w, b, s = m.affine_weight, m.affine_bias, m.mean_shift
    wrt = [w, b, s, *xs]
    kern = lambda: torch.autograd.grad(ops.SegmentNorm.apply(m._layout, seg, w, b, s, *xs), wrt, gys)
    chain = lambda: torch.autograd.grad(tuple(ops.segment_norm_planar_torch(m._layout, xs, batch, G, w, b, s)), wrt, gys)
    out = {}
    for name, fn in (("kernels", kern), ("torch", chain)):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                fn()
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            fn()
        for _ in range(warmup):
            graph.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            graph.replay()
        e1.record()
        torch.cuda.synchronize()
        out[f"graph_norm_fwd_bwd_{name}_us"] = round(1e3 * e0.elapsed_time(e1) / steps, 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("norm_step.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cuda.matmul.allow_tf32 = False
    res = {"card": _card()}
    inp = {k: v.to(dev) for k, v in bench.make_inputs("qm9", seed=0).items()}
    steps = {n: qm9_step(n, dev, inp) for n in ("layer", "graph", "instance")}
    best = {}
    for _ in range(args.rounds):
        for n, fn in steps.items():
            ms = _time(fn, args.steps, args.warmup)
            best[n] = min(best.get(n, ms), ms)
    res.update({f"qm9_{n}_ms": round(ms, 3) for n, ms in best.items()})
    res.update(norm_calls(dev, inp, 200, 20))
    res["card_after"] = _card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
