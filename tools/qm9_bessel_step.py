#!/usr/bin/env python
"""Step time of the Bessel-basis QM9 configuration against the Gaussian one, on one GPU, in one process.

    python tools/qm9_bessel_step.py [--steps K --warmup W --rounds R]

Three models train on the headline QM9 batch (``bench.make_inputs('qm9', seed=0)``: 128 synthetic molecules, ~32.5 k
edges), each with the step ``bench.py`` times: CUDA-graph replay of forward + L1 loss + backward
(``graphs.GraphedForwardBackward``, neighbour search eager), then AdamW (lr 5e-4, weight decay 5e-3):

* ``bessel_k8``   - graph_attention_transformer_nonlinear_bessel_l2, num_basis 8 (the reference's scripts for targets 5-10);
* ``gaussian_k128`` - graph_attention_transformer_nonlinear_l2, num_basis 128 (the headline configuration);
* ``gaussian_k8``   - graph_attention_transformer_nonlinear_l2, num_basis 8: separates the basis from the width K of the
  radial MLPs' first layer.

The models alternate: every round times ``--steps`` steps of each, in turn, so that clock drift and other work on the
card spread over all three.  One JSON line per model gives the median and spread over rounds, with the card, its power
limit and the SM clock sampled during the timed rounds.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

MODELS = {
    "bessel_k8": ("graph_attention_transformer_nonlinear_bessel_l2", 8),
    "gaussian_k128": ("graph_attention_transformer_nonlinear_l2", 128),
    "gaussian_k8": ("graph_attention_transformer_nonlinear_l2", 8),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="timed steps per model per round")
    ap.add_argument("--warmup", type=int, default=8, help="untimed steps per model (they include the capture)")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("qm9_bessel_step.py needs a CUDA device")

    from equiformer_b200 import _lib
    from equiformer_b200.graphs import GraphedForwardBackward
    from equiformer_b200.nets import model_entrypoint
    from equiformer_b200.parallel import FlatAdamW, FlatGradAllReduce

    _lib.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cuda.matmul.allow_tf32 = False
    inp = {k: v.to(dev) for k, v in bench.make_inputs("qm9", seed=0).items()}
    edges = bench.count_edges("qm9", bench.make_inputs("qm9", seed=0))
    l1 = lambda out, tgt: (out - tgt).abs().mean()

    runs = {}
    for tag, (name, num_basis) in MODELS.items():
        torch.manual_seed(0)
        model = model_entrypoint(name)(irreps_in="5x0e", radius=5.0, num_basis=num_basis).to(dev).train()
        for m in model.modules():          # attention dropout off, as bench.py's default
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
        bucket = FlatGradAllReduce(model.parameters())
        opt = FlatAdamW(model.named_parameters(), bucket, lr=5e-4, weight_decay=5e-3, no_decay=model.no_weight_decay())
        graphed = GraphedForwardBackward(model, l1, bucket, max_radius=5.0)

        def step(graphed=graphed, bucket=bucket, opt=opt):
            loss = graphed(inp["pos"], inp["batch"], inp["z"], inp["target"])
            bucket.reduce()
            opt.step()
            return loss

        for _ in range(args.warmup):
            step()
        runs[tag] = dict(step=step, graphed=graphed, ms=[], loss=None)
    torch.cuda.synchronize()

    sampler = bench.ClockSampler(0)
    sampler.start()
    for _ in range(args.rounds):
        for tag, r in runs.items():
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(args.steps):
                loss = r["step"]()
            end.record()
            torch.cuda.synchronize()
            r["ms"].append(start.elapsed_time(end) / args.steps)
            r["loss"] = float(loss)
    clocks = sampler.stop()
    # read-only query right after the timed rounds; some cards report [N/A] for these fields, which is then what prints
    smi = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=10).stdout.strip()

    for tag, r in runs.items():
        name, num_basis = MODELS[tag]
        ms = statistics.median(r["ms"])
        print(json.dumps({
            "metric": "ms per QM9 training step (captured forward + loss + backward, AdamW)", "tag": tag, "model": name,
            "num_basis": num_basis, "ms_per_step": ms, "ms_per_round": r["ms"], "edges_per_step": edges,
            "edges_per_s": edges / (ms * 1e-3), "steps_per_round": args.steps, "rounds": args.rounds,
            "warmup": args.warmup, "captures": r["graphed"].captures, "loss": r["loss"],
            "device": torch.cuda.get_device_name(dev), "power_limit_w": bench.power_limit(0), "clocks": clocks,
            "nvidia_smi_sm_clock_max_clock_power_limit": smi,
        }), flush=True)


if __name__ == "__main__":
    main()
