#!/usr/bin/env python
"""Time of one OC20 IS2RE predict pass: the reference-style eager loop against the captured ``EvalPass.predict``.

    python tools/predict_step.py [--batches K --rounds R]

Two models, each over ``--batches`` seeded synthetic batches of 8-16 frames (``synthetic.oc20_like_frames``, no labels):

* ``l1_256_nonlinear_aux`` (``OC20_L1_256_NONLINEAR_AUX``) with ``write_pos``;
* ``l1_256_nonlinear`` (``OC20_L1_256_NONLINEAR``), energies only.

The reference-style loop is ``EnergyTrainerV2.predict`` restated: eager forward under ``no_grad``, de-normalised energy,
``sid.tolist()`` and ``energy.tolist()`` per batch, and with ``write_pos`` the moved atoms split per system onto the host.
``EvalPass.predict`` runs the eager neighbour list and padding, then the captured forward and prediction kernel per
bucket, and reads the results once at the end of the pass.

Both loops run once untimed (the captures happen there), then ``--rounds`` times each, alternating, each pass timed with
CUDA events and a synchronise at its end.  The JSON line per model gives the median ms per batch of each loop, the
captures, the largest difference between the two loops' predictions, and the card's name, power limit and SM clock read
in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
from eval_step import sm_clock  # noqa: E402

MEAN, STD, POS_STD = 0.3, 1.7, 0.9


def setup(cfg: dict, n_batches: int, dev):
    from equiformer_b200 import synthetic as S
    from equiformer_b200.nets.graph_attention_transformer_oc20 import GraphAttentionTransformerOC20
    torch.manual_seed(0)
    model = GraphAttentionTransformerOC20(None, None, 1, **cfg)
    batches, first = [], 0
    for i in range(n_batches):
        n = (8, 12, 16)[i % 3]
        pos, batch, z, tags, edge = S.oc20_like_frames(n, seed=i)
        batches.append(types.SimpleNamespace(pos=pos, batch=batch, atomic_numbers=z, tags=tags,
                                             cell=torch.diag_embed(edge[:, None].expand(-1, 3)).float(),
                                             natoms=torch.bincount(batch, minlength=n), sid=torch.arange(first, first + n)))
        first += n
    batches = [types.SimpleNamespace(**{k: v.to(dev) for k, v in vars(b).items()}) for b in batches]
    return model.to(dev).train(), batches


def reference_loop(model, batches, write_pos: bool):
    """``EnergyTrainerV2.predict(per_image=True)`` restated: eager, one ``.tolist()`` per batch."""
    model.eval()
    predictions, pos_preds = {"id": [], "energy": []}, {}
    with torch.no_grad():
        for b in batches:
            out = model(b)
            energy, aux = out if isinstance(out, tuple) else (out, None)
            energy = energy.view(-1) * STD + MEAN
            predictions["id"].extend([str(i) for i in b.sid.tolist()])
            predictions["energy"].extend(energy.tolist())
            if write_pos:
                delta_pos = aux * POS_STD + 0.0
                tag_mask = b.tags > 0
                pred_pos = b.pos.clone()
                pred_pos[tag_mask] = pred_pos[tag_mask] + delta_pos[tag_mask]
                sid_list = [str(sid) for sid in b.sid.tolist()]
                for sid, p in zip(sid_list, torch.split(pred_pos, b.natoms.tolist())):
                    pos_preds[sid] = p.detach().cpu()
    model.train()
    if write_pos:
        predictions["pos"] = pos_preds
    return predictions


def differences(a: dict, b: dict) -> dict:
    if a["id"] != b["id"]:
        raise AssertionError("the two loops give different ids")
    e = (torch.tensor(a["energy"], dtype=torch.float64) - torch.tensor(b["energy"], dtype=torch.float64)).abs()
    out = {"max_abs_energy": e.max().item(),
           "max_rel_energy": (e / torch.tensor(b["energy"], dtype=torch.float64).abs().clamp_min(1.0)).max().item()}
    if "pos" in a:
        if list(a["pos"]) != list(b["pos"]):
            raise AssertionError("the two loops give positions for different systems")
        out["max_abs_pos"] = max((a["pos"][k] - b["pos"][k]).abs().max().item() for k in a["pos"])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=24, help="seeded batches per pass")
    ap.add_argument("--rounds", type=int, default=3, help="timed passes of each loop, alternating")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("predict_step.py needs a CUDA device")
    from equiformer_b200 import _lib
    from equiformer_b200.evaluation import EvalPass
    from equiformer_b200.nets.graph_attention_transformer_oc20 import OC20_L1_256_NONLINEAR, OC20_L1_256_NONLINEAR_AUX
    _lib.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cuda.matmul.allow_tf32 = False
    for name, cfg, write_pos in (("l1_256_nonlinear_aux", OC20_L1_256_NONLINEAR_AUX, True),
                                 ("l1_256_nonlinear", OC20_L1_256_NONLINEAR, False)):
        model, batches = setup(cfg, args.batches, dev)
        # ~50 neighbours per atom: 4096 edges are under 10 % of a batch
        ev = EvalPass(model, "oc20_is2re", 5.0, MEAN, STD, positions_std=POS_STD, edge_quantum=4096, max_cached=32)
        frames = sum(int(b.natoms.numel()) for b in batches)

        def timed(fn):
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out = fn()
            e.record()
            torch.cuda.synchronize()
            return s.elapsed_time(e) / len(batches), out

        reference_loop(model, batches, write_pos)             # warm-up of both loops; the captures happen here
        ev.predict(batches, write_pos=write_pos)
        captures = ev.predict_captures
        t_ref, t_ours = [], []
        for _ in range(args.rounds):
            ms, ref = timed(lambda: reference_loop(model, batches, write_pos))
            t_ref.append(ms)
            ms, ours = timed(lambda: ev.predict(batches, write_pos=write_pos))
            t_ours.append(ms)
        ms_ref, ms_ours = statistics.median(t_ref), statistics.median(t_ours)
        print(json.dumps({
            "metric": f"OC20 IS2RE predict pass, {name}: ms per batch", "model": name, "write_pos": write_pos,
            "batches": args.batches, "frames": frames, "rounds": args.rounds,
            "eager_reference_loop": {"ms_per_batch": ms_ref, "frames_per_s": frames / (ms_ref * len(batches) * 1e-3),
                                     "runs_ms_per_batch": t_ref},
            "captured_predict": {"ms_per_batch": ms_ours, "frames_per_s": frames / (ms_ours * len(batches) * 1e-3),
                                 "runs_ms_per_batch": t_ours, "captures": captures,
                                 "captures_in_timed_passes": ev.predict_captures - captures},
            "speedup": ms_ref / ms_ours, "difference": differences(ours, ref),
            "device": torch.cuda.get_device_name(dev), "power_limit_w": bench.power_limit(0), "sm_clock_mhz": sm_clock(0),
        }), flush=True)
        del model, ev, batches
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
