#!/usr/bin/env python
"""Time of one validation pass: the reference-style eager loop against the captured ``evaluation.EvalPass``, on one GPU.

    python tools/eval_step.py --task qm9  [--batches K --rounds R]   # QM9 model, 96-128 molecules per batch
    python tools/eval_step.py --task md17                            # MD17 Lmax=3 (exp basis), 4-8 aspirin conformers
    python tools/eval_step.py --task oc20                            # OC20 l1_256_nonlinear (IS2RE), 8-16 frames

``--batches`` seeded synthetic batches of varying sizes (``synthetic.qm9_like_batch``, ``aspirin_like``,
``oc20_like_frames``, with seeded targets) go through two loops over the same model and data:

* the reference-style loop of ``engine.evaluate`` / ``main_md17.evaluate`` / the OC20 ``validate``: eager, under
  ``no_grad`` (the MD17 forces by the model's own ``enable_grad`` backward), one ``.item()`` per metric and batch into
  ``AverageMeter``s;
* ``EvalPass``: eager neighbour list and padding, then the captured forward and metric kernels per bucket, one host read
  at the end.

Both loops are warmed up once (the captures happen there), then timed ``--rounds`` times, alternating, each pass with
CUDA events and a synchronise at its end.  The JSON line gives the median ms per batch of each loop, graphs/s, the
captures, both loops' metrics, and the card's name, power limit and SM clock read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

MEAN, STD = 0.3, 1.7


def sm_clock(index: int):
    """(current, max) SM clock in MHz, read-only nvidia-smi query; None when unavailable."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                              str(index)], capture_output=True, text=True, timeout=10).stdout.strip()
        return [float(x) for x in out.split(",")]
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


class AverageMeter:
    def __init__(self):
        self.sum, self.count = 0.0, 0

    def update(self, val, n=1):
        self.sum += val * n
        self.count += n

    @property
    def avg(self):
        return self.sum / self.count


def setup(task: str, n_batches: int, dev):
    from equiformer_b200 import synthetic as S
    from equiformer_b200.nets import model_entrypoint
    torch.manual_seed(0)
    batches = []
    if task == "qm9":
        model = model_entrypoint("graph_attention_transformer_nonlinear_l2")(irreps_in="5x0e", radius=5.0, num_basis=128)
        for i in range(n_batches):
            n = (96, 112, 128)[i % 3]
            pos, batch, z = S.qm9_like_batch(n, seed=i)
            y = torch.randn(n, 19, generator=torch.Generator().manual_seed(i))
            batches.append(types.SimpleNamespace(pos=pos, batch=batch, z=z, y=y))
        kw = dict(target=7)
    elif task == "md17":
        model = model_entrypoint("graph_attention_transformer_nonlinear_exp_l3_md17")(irreps_in="64x0e", radius=5.0,
                                                                                    num_basis=32)
        for i in range(n_batches):
            B = (4, 6, 8)[i % 3]
            confs = [S.aspirin_like(seed=64 * i + s) for s in range(B)]
            g = torch.Generator().manual_seed(i)
            batches.append(types.SimpleNamespace(pos=torch.cat([c[0] for c in confs]),
                                                 batch=torch.arange(B).repeat_interleave(21),
                                                 z=torch.cat([c[2] for c in confs]), y=torch.randn(B, 1, generator=g),
                                                 dy=torch.randn(21 * B, 3, generator=g)))
        kw = dict(atom_quantum=32, edge_quantum=512)
    else:
        from equiformer_b200.nets.graph_attention_transformer_oc20 import (OC20_L1_256_NONLINEAR,
                                                                         GraphAttentionTransformerOC20)
        model = GraphAttentionTransformerOC20(None, None, 1, **OC20_L1_256_NONLINEAR)
        for i in range(n_batches):
            n = (8, 12, 16)[i % 3]
            pos, batch, z, tags, edge = S.oc20_like_frames(n, seed=i)
            batches.append(types.SimpleNamespace(pos=pos, batch=batch, atomic_numbers=z, tags=tags,
                                                 cell=torch.diag_embed(edge[:, None].expand(-1, 3)).float(),
                                                 y_relaxed=torch.randn(n, generator=torch.Generator().manual_seed(i))))
        kw = dict(edge_quantum=4096)                  # ~50 neighbours per atom: 4096 edges are under 10 % of a batch
    batches = [types.SimpleNamespace(**{k: v.to(dev) for k, v in vars(b).items()}) for b in batches]
    return model.to(dev).train(), batches, kw


def reference_loop(task: str, model, batches):
    """The reference drivers' evaluation loop, restated: eager, one ``.item()`` per metric and batch."""
    model.eval()
    meters = {}

    def upd(name, val, n):
        meters.setdefault(name, AverageMeter()).update(val, n)

    with torch.no_grad():
        for b in batches:
            if task == "qm9":
                pred = model(f_in=None, pos=b.pos, batch=b.batch, node_atom=b.z).squeeze()
                y = b.y[:, 7]
                upd("loss", torch.nn.functional.l1_loss(pred, (y - MEAN) / STD).item(), pred.shape[0])
                upd("mae", torch.mean(torch.abs(pred * STD + MEAN - y)).item(), pred.shape[0])
            elif task == "md17":
                pred_y, pred_dy = model(node_atom=b.z, pos=b.pos.clone(), batch=b.batch)
                l2mae = lambda a, t: torch.norm(a - t, p=2, dim=-1).mean()
                upd("energy_loss", l2mae(pred_y, (b.y - MEAN) / STD).item(), pred_y.shape[0])
                upd("force_loss", l2mae(pred_dy, b.dy / STD).item(), pred_dy.shape[0])
                upd("energy_mae", torch.mean(torch.abs(pred_y * STD + MEAN - b.y)).item(), pred_y.shape[0])
                upd("force_mae", torch.mean(torch.abs(pred_dy * STD - b.dy)).item(), pred_dy.shape[0])
            else:
                energy = model(b).view(-1)
                upd("loss", torch.nn.functional.l1_loss(energy, (b.y_relaxed - MEAN) / STD).item(), 1)
                err = torch.abs(b.y_relaxed - (energy * STD + MEAN))
                upd("energy_mae", torch.sum(err).item() / err.numel(), err.numel())
                upd("energy_mse", torch.sum(err * err).item() / err.numel(), err.numel())
                upd("energy_within_threshold", (err < 0.02).sum().item() / err.numel(), err.numel())
    model.train()
    return {k: m.avg for k, m in meters.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", choices=("qm9", "md17", "oc20"), default="qm9")
    ap.add_argument("--batches", type=int, default=24, help="seeded batches per pass")
    ap.add_argument("--rounds", type=int, default=3, help="timed passes of each loop, alternating")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("eval_step.py needs a CUDA device")
    from equiformer_b200 import _lib
    from equiformer_b200.evaluation import EvalPass
    _lib.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cuda.matmul.allow_tf32 = False
    model, batches, kw = setup(args.task, args.batches, dev)
    ev = EvalPass(model, "oc20_is2re" if args.task == "oc20" else args.task, 5.0, MEAN, STD, max_cached=32, **kw)
    graphs = sum(int((b.y_relaxed if args.task == "oc20" else b.y).shape[0]) for b in batches)

    def timed(fn):
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / len(batches), out

    ref = reference_loop(args.task, model, batches)          # warm-up of both loops; the captures happen here
    ours = ev.run(batches)
    captures = ev.captures
    t_ref, t_ours = [], []
    for _ in range(args.rounds):
        ms, ref = timed(lambda: reference_loop(args.task, model, batches))
        t_ref.append(ms)
        ms, ours = timed(lambda: ev.run(batches))
        t_ours.append(ms)
    ms_ref, ms_ours = statistics.median(t_ref), statistics.median(t_ours)
    print(json.dumps({
        "metric": f"validation pass, {args.task}: ms per batch", "task": args.task, "batches": args.batches,
        "graphs": graphs, "rounds": args.rounds,
        "eager_reference_loop": {"ms_per_batch": ms_ref, "graphs_per_s": graphs / (ms_ref * len(batches) * 1e-3),
                                 "runs_ms_per_batch": t_ref, "metrics": ref},
        "captured_eval_pass": {"ms_per_batch": ms_ours, "graphs_per_s": graphs / (ms_ours * len(batches) * 1e-3),
                               "runs_ms_per_batch": t_ours, "captures": captures,
                               "captures_in_timed_passes": ev.captures - captures,
                               "metrics": {k: v["metric"] for k, v in ours.items()}},
        "speedup": ms_ref / ms_ours,
        "device": torch.cuda.get_device_name(dev), "power_limit_w": bench.power_limit(0), "sm_clock_mhz": sm_clock(0),
    }), flush=True)


if __name__ == "__main__":
    main()
