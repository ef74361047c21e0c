#!/usr/bin/env python
"""Captured training-step time of the Lmax = 4 QM9 and MD17 models beside their Lmax = 3 counterparts, on one GPU.

    python tools/lmax4_step.py [--steps K --warmup W]

QM9: the QM9 configuration (``_qm9`` in nets/graph_attention_transformer.py, nonlinear messages, 6 blocks) with
``3e`` and ``4e`` blocks added (node ``128x0e+64x1e+32x2e+16x3e+16x4e``, harmonics ``0..4``), and the same model cut at
l = 3, on the ``bench.py --workload qm9`` batch; one step = neighbour list + replay of ``GraphedForwardBackward``
(forward, L1 loss, backward).  MD17: the ``graph_attention_transformer_nonlinear_exp_l3_md17`` configuration and the
same with ``32x4e`` node / ``8x4e`` head / ``96x4e`` MLP blocks and ``1x4e`` harmonics, on the ``md17_l3`` conformers;
one step = replay of ``GraphedStep`` (energy, forces through the double backward, energy + force loss, backward).
Attention dropout is off.  Every step ends in a device synchronise; the line reports the mean step time in ms over
``--steps`` steps, with the card name, power limit and SM clock read in the same call.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

QM9 = {3: dict(irreps_node_embedding="128x0e+64x1e+32x2e+16x3e", irreps_sh="1x0e+1x1e+1x2e+1x3e",
               irreps_head="32x0e+16x1e+8x2e+4x3e", irreps_mlp_mid="384x0e+192x1e+96x2e+48x3e"),
       4: dict(irreps_node_embedding="128x0e+64x1e+32x2e+16x3e+16x4e", irreps_sh="1x0e+1x1e+1x2e+1x3e+1x4e",
               irreps_head="32x0e+16x1e+8x2e+4x3e+4x4e", irreps_mlp_mid="384x0e+192x1e+96x2e+48x3e+48x4e")}
MD17_L4 = dict(irreps_node_embedding="128x0e+64x1e+64x2e+32x3e+32x4e", irreps_sh="1x0e+1x1e+1x2e+1x3e+1x4e",
               irreps_head="32x0e+16x1e+16x2e+8x3e+8x4e", irreps_mlp_mid="384x0e+192x1e+192x2e+96x3e+96x4e")


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _no_dropout(model):
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return model


def _time(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / steps


def qm9_step(lmax, dev, steps, warmup):
    from equiformer_b200.graphs import GraphedForwardBackward
    from equiformer_b200.nets.graph_attention_transformer import _qm9
    from equiformer_b200.parallel import FlatGradAllReduce
    torch.manual_seed(0)
    model = _no_dropout(_qm9("5x0e", 5.0, 128, None, None, None, nonlinear_message=True, **QM9[lmax]).to(dev).train())
    bucket = FlatGradAllReduce(model.parameters())
    gfb = GraphedForwardBackward(model, lambda out, tgt: (out - tgt).abs().mean(), bucket, max_radius=5.0)
    inp = {k: v.to(dev) for k, v in bench.make_inputs("qm9", seed=0).items()}
    return _time(lambda: gfb(inp["pos"], inp["batch"], inp["z"], inp["target"]), steps, warmup)


def md17_step(lmax, dev, steps, warmup):
    from equiformer_b200 import ops
    from equiformer_b200.graph import radius_graph_csr
    from equiformer_b200.graphs import GraphedStep
    from equiformer_b200.nets import model_entrypoint
    from equiformer_b200.nets.graph_attention_transformer_md17 import GraphAttentionTransformerMD17
    from equiformer_b200.parallel import FlatGradAllReduce
    torch.manual_seed(0)
    ref = model_entrypoint("graph_attention_transformer_nonlinear_exp_l3_md17")(irreps_in="64x0e", radius=5.0,
                                                                                 num_basis=32)
    # the registered factory's arguments (nets/graph_attention_transformer_md17.py, _make) with the degree-4 irreps
    cfg = dict(irreps_in="64x0e", num_layers=6, irreps_node_attr="1x0e", max_radius=5.0, number_of_basis=32,
               fc_neurons=[64, 64], irreps_feature="512x0e", num_heads=4, irreps_pre_attn=None, rescale_degree=False,
               nonlinear_message=True, norm_layer="layer", proj_drop=0.0, out_drop=0.0, drop_path_rate=0.0, mean=None,
               std=None, scale=None, atomref=None, basis_type="exp", alpha_drop=0.0, **MD17_L4)
    model = ref if lmax == 3 else GraphAttentionTransformerMD17(**cfg)
    model = _no_dropout(model.to(dev).train())
    bucket = FlatGradAllReduce(model.parameters())
    inp = {k: v.to(dev) for k, v in bench.make_inputs("md17_l3", seed=0).items()}
    n, n_graphs = int(inp["pos"].shape[0]), int(inp["target"].shape[0])

    def captured(pos, batch, z, target, ftarget, src, dst, row_ptr):
        csr = ops.Graph.__new__(ops.Graph)
        csr.n_nodes, csr.n_edges, csr.perm = n, int(src.numel()), None
        csr.src, csr.dst, csr.row_ptr = src, dst, row_ptr
        csr._src_perm = csr._src_row_ptr = None
        e, f = model.forward_edges(z, pos.detach().requires_grad_(True), batch, src, dst, graph=csr, n_graphs=n_graphs)
        return (e - target).norm(dim=-1).mean() + 100.0 * (f - ftarget).norm(dim=-1).mean()

    step = GraphedStep(captured, bucket)

    def one():
        edge, row_ptr = radius_graph_csr(inp["pos"], 5.0, inp["batch"], max_num_neighbors=1000)
        step((n, int(edge.shape[1]), n_graphs), [inp["pos"], inp["batch"], inp["z"], inp["target"], inp["ftarget"],
                                                 edge[0], edge[1], row_ptr])
    return _time(one, steps, warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("lmax4_step.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cuda.matmul.allow_tf32 = False
    res = {"card": _card()}
    for lmax in (3, 4):
        res[f"qm9_l{lmax}_ms"] = round(qm9_step(lmax, dev, args.steps, args.warmup), 3)
        res[f"md17_l{lmax}_ms"] = round(md17_step(lmax, dev, args.steps, args.warmup), 3)
    res["card_after"] = _card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
