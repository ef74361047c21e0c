"""Captured evaluation passes (``evaluation.EvalPass``) on the metric kernels of ``libeqf_b200_eval.so``.

CPU: the torch statement of the metric terms against restatements of the reference's evaluation loops
(``engine.evaluate``, ``main_md17.evaluate`` and ocpmodels' ``Evaluator`` for ``is2re``); the header's constants; the
library's kernel inventory; the exported argument checks and the launchers' refusals; the OC20 padding; the cross-process
reduction over two gloo processes.

GPU: the kernels against float64 at every length regime, with device-side atom counts, NaN and Inf; each task's captured
pass against the reference-style eager loop on the unpadded batches; no host synchronisation in a metric update; a pass
leaves no trace; the EMA and loaded weights through the same captures; the checkpoint round trip of the metrics.

ocpmodels is not part of the reference tree, so its evaluator's formulas are restated here from its source:
``energy_mae`` = ``abs(target - prediction)`` with total = its sum and numel = its length, ``energy_mse`` = the same of
``(target - prediction) ** 2``, ``energy_within_threshold`` = ``(abs(target - prediction) < 0.02).sum()`` over the frame
count, and ``Evaluator.update`` adds a dict's ``total`` / ``numel`` and counts a float as one element of ``total``.
"""
from __future__ import annotations

import os
import re
import socket
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

EVAL_CLAIMS = {"eqf::eval_graph_kernel", "eqf::eval_atom_kernel", "eqf::eval_batch_kernel"}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
QM9 = "graph_attention_transformer_nonlinear_l2"
MD17 = "graph_attention_transformer_nonlinear_exp_l2_md17"
MEAN, STD = 0.3, 1.7


# ------------------------------------------------------------------------------------------------ reference loops
class AverageMeter:
    """``engine.AverageMeter``: ``sum += val * n``, ``count += n``, ``avg = sum / count``."""

    def __init__(self):
        self.sum, self.count = 0.0, 0

    def update(self, val, n=1):
        self.sum += val * n
        self.count += n

    @property
    def avg(self):
        return self.sum / self.count


def reference_qm9(outputs, mean, std):
    """``engine.evaluate``: per batch ``(pred [G], y [G])``; ``L1Loss`` of the normalised target, MAE of the energy."""
    loss_m, mae_m = AverageMeter(), AverageMeter()
    for pred, y in outputs:
        loss = (pred - (y - mean) / std).abs().mean()
        loss_m.update(loss.item(), n=pred.shape[0])
        err = pred * std + mean - y
        mae_m.update(torch.mean(torch.abs(err)).item(), n=pred.shape[0])
    return {"mae": mae_m.avg, "loss": loss_m.avg}


def _l2mae(a, b):
    return torch.norm(a - b, p=2, dim=-1).mean()           # ocpmodels' L2MAELoss, the MD17 criterion


def reference_md17(outputs, mean, std):
    """``main_md17.evaluate`` / ``main_md17_dens.evaluate``: per batch ``(pred_y [G, 1], pred_dy [N, 3], y, dy)``."""
    loss = {"energy": AverageMeter(), "force": AverageMeter()}
    mae = {"energy": AverageMeter(), "force": AverageMeter()}
    for pred_y, pred_dy, y, dy in outputs:
        loss["energy"].update(_l2mae(pred_y, (y - mean) / std).item(), n=pred_y.shape[0])
        loss["force"].update(_l2mae(pred_dy, dy / std).item(), n=pred_dy.shape[0])
        mae["energy"].update(torch.mean(torch.abs(pred_y * std + mean - y)).item(), n=pred_y.shape[0])
        mae["force"].update(torch.mean(torch.abs(pred_dy * std - dy)).item(), n=pred_dy.shape[0])
    return {"energy_mae": mae["energy"].avg, "force_mae": mae["force"].avg, "energy_loss": loss["energy"].avg,
            "force_loss": loss["force"].avg}


def _ocp_update(key, stat, metrics):
    m = metrics.setdefault(key, {"metric": None, "total": 0, "numel": 0})
    if isinstance(stat, dict):
        m["total"] += stat["total"]
        m["numel"] += stat["numel"]
    else:
        m["total"] += stat
        m["numel"] += 1
    m["metric"] = m["total"] / m["numel"]
    return metrics


def reference_oc20(outputs, mean, std):
    """``base_trainer_v2.validate`` with ``Evaluator(task='is2re')``: per batch ``(energy [G] normalised, y [G], loss)``."""
    metrics = {}
    for energy, y, loss in outputs:
        pred = energy * std + mean                          # normalizers["target"].denorm
        err = torch.abs(y - pred)
        _ocp_update("energy_mae", {"total": torch.sum(err).item(), "numel": err.numel()}, metrics)
        sq = (y - pred) ** 2
        _ocp_update("energy_mse", {"total": torch.sum(sq).item(), "numel": sq.numel()}, metrics)
        _ocp_update("energy_within_threshold", {"total": (err < 0.02).sum().item(), "numel": y.size(0)}, metrics)
        _ocp_update("loss", loss.item(), metrics)
    return {k: v["metric"] for k, v in metrics.items()}


def oc20_reference_loss(energy, y, mean, std, aux=None, delta=None, tags=None, w=0.0):
    """``energy_trainer_v2._compute_loss``: L1 of the normalised energy, plus ``w`` times the L2MAE of the auxiliary head
    over the atoms with ``tag > 0`` (``_mask_input`` selects them)."""
    loss = torch.nn.functional.l1_loss(energy, (y - mean) / std)
    if aux is not None:
        m = tags > 0
        loss = loss + _l2mae(aux[m], delta[m]) * w
    return loss


def _close(got: dict, ref: dict, tol: float):
    assert set(got) == set(ref), (sorted(got), sorted(ref))
    for k, v in ref.items():
        g = got[k]["metric"] if isinstance(got[k], dict) else got[k]
        assert abs(g - v) <= tol * max(abs(v), 1e-30), (k, g, v)


# ------------------------------------------------------------------------------------------------ CPU
def _fake_batches(seed, sizes, atoms_per_graph=7):
    g = torch.Generator().manual_seed(seed)
    out = []
    for G in sizes:
        N = G * atoms_per_graph
        out.append((torch.randn(G, 1, generator=g, dtype=torch.float64), torch.randn(N, 3, generator=g, dtype=torch.float64),
                    torch.randn(G, 1, generator=g, dtype=torch.float64) * 2, torch.randn(N, 3, generator=g, dtype=torch.float64),
                    torch.randn(N, 3, generator=g, dtype=torch.float64), torch.randint(0, 3, (N,), generator=g)))
    return out


SIZES = (8, 8, 13, 8, 3)                 # the last batch is short


def test_torch_statement_matches_the_reference_loops():
    from equiformer_b200 import evaluation as E
    from equiformer_b200.eval_kernels import eval_atom_torch, eval_batch_torch, eval_graph_torch
    from equiformer_b200.oc20_objective import masked_l2mae
    batches = _fake_batches(0, SIZES)
    sl = lambda acc, a, b: acc[a:b]
    # QM9
    acc = torch.zeros(E.SLOTS["qm9"], dtype=torch.float64)
    for pred_y, _f, y, *_ in batches:
        eval_graph_torch(pred_y, y, y.shape[0], MEAN, STD, 0.02, sl(acc, 0, 5))
    ref = reference_qm9([(p.reshape(-1), y.reshape(-1)) for p, _f, y, *_ in batches], MEAN, STD)
    _close(E.metrics_from_accumulator("qm9", acc), ref, 1e-12)
    # MD17
    acc = torch.zeros(E.SLOTS["md17"], dtype=torch.float64)
    for pred_y, pred_dy, y, dy, *_ in batches:
        eval_graph_torch(pred_y, y, y.shape[0], MEAN, STD, 0.02, sl(acc, 0, 5))
        eval_atom_torch(pred_dy, dy, dy.shape[0], STD, sl(acc, 5, 8))
    ref = reference_md17([b[:4] for b in batches], MEAN, STD)
    _close(E.metrics_from_accumulator("md17", acc), ref, 1e-12)
    # OC20, without and with the auxiliary loss (w = 3)
    for w in (None, 3.0):
        acc = torch.zeros(E.SLOTS["oc20_is2re"], dtype=torch.float64)
        outs = []
        for pred_y, aux, y, delta, _dy, tags in batches:
            e, t = pred_y.reshape(-1), y.reshape(-1)
            ref_loss = oc20_reference_loss(e, t, MEAN, STD, *((aux, delta, tags, w) if w else ()))
            loss = (e - (t - MEAN) / STD).abs().mean()
            if w:
                loss = loss + w * masked_l2mae(aux, delta, tags)
            eval_graph_torch(pred_y, y, y.shape[0], MEAN, STD, 0.02, sl(acc, 0, 5))
            eval_batch_torch(loss, sl(acc, 5, 7))
            outs.append((e, t, ref_loss))
        got = E.metrics_from_accumulator("oc20_is2re", acc)
        _close(got, reference_oc20(outs, MEAN, STD), 1e-12)
        assert got["energy_mae"]["numel"] == sum(SIZES) and got["loss"]["numel"] == len(SIZES)


def test_threshold_counts_strictly_and_not_nan():
    from equiformer_b200.eval_kernels import eval_graph_torch
    acc = torch.zeros(5, dtype=torch.float64)
    pred = torch.tensor([0.0, 0.02, 0.0199, float("nan")], dtype=torch.float64)
    eval_graph_torch(pred, torch.zeros(4, dtype=torch.float64), 4, 0.0, 1.0, 0.02, acc)
    assert acc[2].item() == 2.0 and torch.isnan(acc[0]) and acc[4].item() == 4.0


def test_header_constants_match():
    from equiformer_b200 import _lib
    header = open(os.path.join(ROOT, "include", "eqf_b200_eval.h")).read()
    for name in ("EQF_EVAL_THREADS", "EQF_EVAL_MAX_CTAS", "EQF_EVAL_SCRATCH", "EQF_EVAL_GRAPH_SLOTS", "EQF_EVAL_ATOM_SLOTS",
                 "EQF_EVAL_BATCH_SLOTS"):
        assert int(re.search(rf"#define {name} (\d+)", header).group(1)) == getattr(_lib, name), name
    terms = int(re.search(r"#define EQF_EVAL_MAX_TERMS (\d+)", header).group(1))
    assert _lib.EQF_EVAL_SCRATCH == _lib.EQF_EVAL_MAX_CTAS * terms


def test_eval_library_inventory_is_claimed(built_lib):
    """Every kernel of the library is launched by test_kernels_against_float64 (graph, atom) and the task passes
    (batch)."""
    from equiformer_b200 import _lib
    from tests.test_gpu_kernel_instances import inventory
    inv = inventory(_lib.EVAL_LIB_PATH)
    assert inv == EVAL_CLAIMS, (sorted(inv - EVAL_CLAIMS), sorted(EVAL_CLAIMS - inv))
    assert "eqf_eval.cu" not in _lib.SOURCES and "eqf_eval.cu" not in _lib.OPTIM_SOURCES
    assert not {n for n in inventory(_lib.LIB_PATH) if n.startswith("eqf::eval_")}


def test_argument_checks_refuse_lengths_and_null_pointers(built_lib):
    """The exported checks, called on their own: host code that launches and dereferences nothing."""
    from equiformer_b200 import _lib
    lib = _lib.load_eval()
    ok = 1 << 20
    msg = lambda: lib.eqf_last_error().decode()
    assert lib.eqf_eval_graph_check(ok, ok, 1, ok, ok, ok) == 0
    assert lib.eqf_eval_graph_check(ok, ok, 0, ok, ok, ok) != 0 and "positive" in msg()
    for bad in range(5):
        ptrs = [None if i == bad else ok for i in range(5)]
        assert lib.eqf_eval_graph_check(ptrs[0], ptrs[1], 4, *ptrs[2:]) != 0 and "null" in msg(), bad
    assert lib.eqf_eval_atom_check(ok, ok, 1, ok, ok, ok, ok) == 0
    assert lib.eqf_eval_atom_check(ok, ok, -3, ok, ok, ok, ok) != 0 and "positive" in msg()
    for bad in range(6):
        ptrs = [None if i == bad else ok for i in range(6)]
        assert lib.eqf_eval_atom_check(ptrs[0], ptrs[1], 4, *ptrs[2:]) != 0 and "null" in msg(), bad
    assert lib.eqf_eval_batch_check(None, ok) == 0 and lib.eqf_eval_batch_check(ok, ok) == 0
    assert lib.eqf_eval_batch_check(ok, None) != 0 and "null" in msg()


def test_launchers_refuse_cpu_wrong_dtypes_and_lengths():
    from equiformer_b200 import _lib
    from equiformer_b200.eval_kernels import eval_atom_raw, eval_batch_raw, eval_graph_raw, new_scratch
    scratch = new_scratch("cpu")
    f = torch.zeros(8)
    with pytest.raises(_lib.EqfError, match="CUDA-only"):
        eval_graph_raw(f, f, 8, 0.0, 1.0, 0.02, torch.zeros(5, dtype=torch.float64), scratch)
    with pytest.raises(_lib.EqfError, match="float32"):
        eval_graph_raw(f.double(), f, 8, 0.0, 1.0, 0.02, torch.zeros(5, dtype=torch.float64), scratch)
    with pytest.raises(_lib.EqfError, match="float64"):
        eval_graph_raw(f, f, 8, 0.0, 1.0, 0.02, torch.zeros(5), scratch)
    with pytest.raises(_lib.EqfError, match="elements"):
        eval_graph_raw(f[:4], f, 8, 0.0, 1.0, 0.02, torch.zeros(5, dtype=torch.float64), scratch)
    with pytest.raises(_lib.EqfError, match=r"\[rows, 3\]"):
        eval_atom_raw(torch.zeros(4, 3), torch.zeros(4, 2), torch.zeros(1, dtype=torch.int64), 1.0,
                      torch.zeros(3, dtype=torch.float64), scratch)
    with pytest.raises(_lib.EqfError, match="int64"):
        eval_atom_raw(torch.zeros(4, 3), torch.zeros(4, 3), torch.zeros(1, dtype=torch.int32), 1.0,
                      torch.zeros(3, dtype=torch.float64), scratch)
    with pytest.raises(_lib.EqfError, match="CUDA-only"):
        eval_batch_raw(torch.zeros(1), torch.zeros(2, dtype=torch.float64))


def test_oc20_padding_keeps_the_real_frames():
    from equiformer_b200.evaluation import pad_oc20
    from equiformer_b200.graph import radius_graph_pbc
    from equiformer_b200.synthetic import oc20_like_frames
    pos, batch, z, tags, edge = oc20_like_frames(3, seed=4, mean_atoms=24, neighbours=20)
    cell = torch.diag_embed(edge[:, None].expand(-1, 3)).float()
    e, offs, _ = radius_graph_pbc(pos, batch, cell, 5.0, 500)
    src, dst = e[0], e[1]
    ev = pos[src] - pos[dst] + torch.bmm(offs.float().view(-1, 1, 3), cell[batch[dst]]).view(-1, 3)
    (ev_p, batch_p, z_p, tags_p, src_p, dst_p, row_ptr), (Nb, Eb) = pad_oc20(pos, batch, z, tags, src, dst, ev, 3, 32, 512)
    N, E = pos.shape[0], src.numel()
    assert Nb % 32 == 0 and Eb % 512 == 0 and Nb >= N + 2 and ev_p.shape == (Eb, 3) and tags_p.shape == (Nb,)
    assert torch.equal(ev_p[:E], ev) and torch.equal(tags_p[:N], tags) and torch.equal(z_p[:N], z)
    assert not tags_p[N:].any() and bool((batch_p[N:] == 3).all())
    assert bool((src_p[E:] >= N).all() and (dst_p[E:] >= N).all())
    assert bool((ev_p[E:].norm(dim=-1) > 0).all())                     # dummy edges join distinct dummy atoms
    assert int(row_ptr[-1]) == Eb and bool((dst_p[1:] >= dst_p[:-1]).all())


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _fill(acc, batches):
    from equiformer_b200.eval_kernels import eval_atom_torch, eval_graph_torch
    for pred_y, pred_dy, y, dy, *_ in batches:
        eval_graph_torch(pred_y, y, y.shape[0], MEAN, STD, 0.02, acc[0:5])
        eval_atom_torch(pred_dy, dy, dy.shape[0], STD, acc[5:8])


def _shard_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    from equiformer_b200 import evaluation as E
    from equiformer_b200.parallel import init_distributed
    init_distributed("gloo")
    batches = _fake_batches(1, SIZES)
    acc = torch.zeros(E.SLOTS["md17"], dtype=torch.float64)
    _fill(acc, batches[rank::world])                          # each rank evaluates its shard
    E.reduce_accumulator(acc)
    ret[rank] = E.metrics_from_accumulator("md17", acc)
    dist.destroy_process_group()


def test_sharded_accumulators_reduce_to_the_whole_loader():
    from equiformer_b200 import evaluation as E
    world = 2
    with mp.Manager() as mgr:
        ret = mgr.dict()
        mp.spawn(_shard_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
        got = dict(ret)
    acc = torch.zeros(E.SLOTS["md17"], dtype=torch.float64)
    _fill(acc, _fake_batches(1, SIZES))
    whole = E.metrics_from_accumulator("md17", acc)
    ref = reference_md17([b[:4] for b in _fake_batches(1, SIZES)], MEAN, STD)
    for r in range(world):
        assert got[r].keys() == whole.keys()
        for k in whole:
            assert got[r][k]["numel"] == whole[k]["numel"]
            assert abs(got[r][k]["total"] - whole[k]["total"]) <= 1e-12 * abs(whole[k]["total"])
        _close(got[r], ref, 1e-12)


# ------------------------------------------------------------------------------------------------ GPU: kernels
def _graph_ref(pred, y, n, mean, std, thr):
    from equiformer_b200.eval_kernels import eval_graph_torch
    acc = torch.zeros(5, dtype=torch.float64)
    eval_graph_torch(pred.cpu(), y.cpu(), n, mean, std, thr, acc)
    return acc


def _atom_ref(pred, dy, n, std):
    from equiformer_b200.eval_kernels import eval_atom_torch
    acc = torch.zeros(3, dtype=torch.float64)
    eval_atom_torch(pred.cpu(), dy.cpu(), n, std, acc)
    return acc


def _assert_acc(got, ref, tol=1e-6):
    got = got.cpu()
    assert torch.equal(torch.isnan(got), torch.isnan(ref)), (got, ref)
    fin = ~torch.isnan(ref)
    assert torch.equal(torch.isinf(got[fin]), torch.isinf(ref[fin])), (got, ref)
    fin &= ~torch.isinf(ref)
    assert ((got[fin] - ref[fin]).abs() <= tol * ref[fin].abs().clamp_min(1e-300)).all(), (got, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [1, 200, 5000, 100_000])     # one row, one CTA, many CTAs, past the 128-CTA cap
def test_kernels_against_float64(cuda_device, rows):
    from equiformer_b200.eval_kernels import eval_atom_raw, eval_graph_raw, new_scratch
    dev = cuda_device
    g = torch.Generator().manual_seed(rows)
    scratch = new_scratch(dev)
    # graph level: 3 padding rows after the real ones, which must not count
    pred = torch.randn(rows + 3, generator=g).to(dev)
    pred[rows:] = float("nan")
    y = (torch.randn(rows, generator=g) * 1.5 + 0.2).to(dev)
    y[: rows // 3] = (pred[: rows // 3] * STD + MEAN + 0.01 * torch.randn(rows // 3, generator=g).to(dev))   # near 0
    acc = torch.zeros(5, dtype=torch.float64, device=dev)
    eval_graph_raw(pred, y, rows, MEAN, STD, 0.02, acc, scratch)
    ref = _graph_ref(pred, y, rows, MEAN, STD, 0.02)
    _assert_acc(acc, ref)
    assert acc[2].item() == ref[2].item() and acc[4].item() == rows
    again = torch.zeros_like(acc)
    eval_graph_raw(pred, y, rows, MEAN, STD, 0.02, again, scratch)
    assert torch.equal(acc, again)                                       # fixed-order: bitwise repeatable
    eval_graph_raw(pred, y, rows, MEAN, STD, 0.02, again, scratch)
    _assert_acc(again, 2 * ref)                                          # it accumulates
    # atom level: the real count read from the device, NaN in the padding rows
    n_real = max(1, rows - 7)
    pd, dy = torch.randn(rows, 3, generator=g).to(dev), torch.randn(rows, 3, generator=g).to(dev)
    pd[n_real:] = float("nan")
    n_dev = torch.full((1,), n_real, dtype=torch.int64, device=dev)
    acc = torch.zeros(3, dtype=torch.float64, device=dev)
    eval_atom_raw(pd, dy, n_dev, STD, acc, scratch)
    _assert_acc(acc, _atom_ref(pd, dy, n_real, STD))
    assert acc[2].item() == n_real
    again = torch.zeros_like(acc)
    eval_atom_raw(pd, dy, n_dev, STD, again, scratch)
    assert torch.equal(acc, again)
    # a count past the rows is clamped to them, a negative one to zero
    for n, expect in ((rows + 50, rows), (-4, 0)):
        acc = torch.zeros(3, dtype=torch.float64, device=dev)
        eval_atom_raw(pd.nan_to_num(0.0), dy, torch.full((1,), n, dtype=torch.int64, device=dev), STD, acc, scratch)
        assert acc[2].item() == expect


@pytest.mark.gpu
def test_kernels_propagate_nan_and_inf(cuda_device):
    from equiformer_b200.eval_kernels import eval_atom_raw, eval_batch_raw, eval_graph_raw, new_scratch
    dev, scratch = cuda_device, new_scratch(cuda_device)
    for bad in (float("nan"), float("inf"), -float("inf")):
        pred = torch.randn(600, generator=torch.Generator().manual_seed(3)).to(dev)
        pred[417] = bad
        y = torch.zeros(600, device=dev)
        acc = torch.zeros(5, dtype=torch.float64, device=dev)
        eval_graph_raw(pred, y, 600, MEAN, STD, 0.02, acc, scratch)
        _assert_acc(acc, _graph_ref(pred, y, 600, MEAN, STD, 0.02))
        pd = torch.randn(300, 3, generator=torch.Generator().manual_seed(4)).to(dev)
        pd[123, 1] = bad
        acc = torch.zeros(3, dtype=torch.float64, device=dev)
        eval_atom_raw(pd, torch.zeros_like(pd), torch.full((1,), 300, dtype=torch.int64, device=dev), STD, acc, scratch)
        _assert_acc(acc, _atom_ref(pd, torch.zeros_like(pd), 300, STD))
        acc = torch.zeros(2, dtype=torch.float64, device=dev)
        eval_batch_raw(torch.full((1,), bad, device=dev), acc)
        eval_batch_raw(None, acc)
        ref = torch.tensor([bad, 2.0], dtype=torch.float64)
        _assert_acc(acc, ref)


@pytest.mark.gpu
def test_metric_update_does_not_synchronise(cuda_device):
    from equiformer_b200.eval_kernels import eval_atom_raw, eval_batch_raw, eval_graph_raw, new_scratch
    dev, scratch = cuda_device, new_scratch(cuda_device)
    pred, y = torch.randn(40, device=dev), torch.randn(32, device=dev)
    pd, n = torch.randn(50, 3, device=dev), torch.full((1,), 45, dtype=torch.int64, device=dev)
    loss, acc = torch.ones(1, device=dev), torch.zeros(10, dtype=torch.float64, device=dev)
    eval_graph_raw(pred, y, 32, MEAN, STD, 0.02, acc[0:5], scratch)      # loads the library
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        eval_graph_raw(pred, y, 32, MEAN, STD, 0.02, acc[0:5], scratch)
        eval_atom_raw(pd, pd, n, STD, acc[5:8], scratch)
        eval_batch_raw(loss, acc[8:10])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert acc[4].item() == 64 and acc[7].item() == 45 and acc[9].item() == 1


# ------------------------------------------------------------------------------------------------ GPU: task passes
def _qm9_model(dev, alpha_drop=0.0, drop_path_rate=0.0):
    from equiformer_b200.nets import model_entrypoint
    from equiformer_b200.nets.drop import GraphDropPath
    torch.manual_seed(0)
    model = model_entrypoint(QM9)(irreps_in="5x0e", radius=5.0, num_basis=128)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = alpha_drop
    if drop_path_rate > 0.0:
        for blk in model.blocks:
            blk.drop_path = GraphDropPath(drop_path_rate)
    return model.to(dev).train()


def _qm9_loader(dev, sizes=(8, 8, 12, 8, 12, 5)):
    from equiformer_b200.synthetic import qm9_like_batch
    out = []
    for i, n in enumerate(sizes):
        pos, batch, z = qm9_like_batch(n, seed=50 + i)
        y = torch.randn(n, 19, generator=torch.Generator().manual_seed(i)) * 2
        out.append(types.SimpleNamespace(pos=pos.to(dev), batch=batch.to(dev), z=z.to(dev), y=y.to(dev)))
    return out


def _qm9_eager(model, loader, target=7):
    """The reference-style loop: eager, no_grad, unpadded, one .item() per batch."""
    was = model.training
    model.eval()
    outs = []
    with torch.no_grad():
        for b in loader:
            pred = model(f_in=None, pos=b.pos, batch=b.batch, node_atom=b.z).squeeze()
            outs.append((pred, b.y[:, target]))
    model.train(was)
    return reference_qm9(outs, MEAN, STD)


def _buckets(loader, r, aq, eq, pbc=None):
    from equiformer_b200.graph import radius_graph_csr, radius_graph_pbc
    from equiformer_b200.graphs import pad_to_bucket
    keys = set()
    for b in loader:
        if pbc:
            e = radius_graph_pbc(b.pos, b.batch, b.cell, r, pbc)[0]
            G, z = b.y_relaxed.shape[0], b.atomic_numbers
        else:
            e = radius_graph_csr(b.pos, r, b.batch, max_num_neighbors=1000)[0]
            G, z = b.y.shape[0], b.z
        keys.add((pad_to_bucket(b.pos, b.batch, z, e[0], e[1], G, aq, eq)[1], G))
    return len(keys)


# Two replays of the same captures on the same inputs give model outputs that differ in the last bits (the model's own
# forward kernels are not bitwise reproducible; the metric kernels are, see test_kernels_against_float64), so repeated
# passes agree to REPEAT relative, far below what a dropout or stochastic-depth draw would change.
REPEAT = 1e-7


def _same(a: dict, b: dict, tol: float = REPEAT):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k]["numel"] == b[k]["numel"], k
        assert abs(a[k]["total"] - b[k]["total"]) <= tol * abs(b[k]["total"]), (k, a[k], b[k])


def _check_pass(ev, loader, ref, tol, n_buckets):
    got = ev.run(loader)
    _close(got, ref, tol)
    assert ev.captures == n_buckets and n_buckets >= 3
    again = ev.run(loader)
    assert ev.captures == n_buckets                                      # no new capture
    _same(again, got)
    return got


@pytest.mark.gpu
def test_qm9_pass_matches_the_reference_loop(cuda_device):
    from equiformer_b200.evaluation import EvalPass
    model, loader = _qm9_model(cuda_device), _qm9_loader(cuda_device)
    ref = _qm9_eager(model, loader)
    ev = EvalPass(model, "qm9", 5.0, MEAN, STD, target=7)
    got = _check_pass(ev, loader, ref, 1e-5, _buckets(loader, 5.0, 128, 2048))
    assert got["mae"]["numel"] == sum(b.y.shape[0] for b in loader)
    eager = EvalPass(model, "qm9", 5.0, MEAN, STD, target=7, capture=False).run(loader)      # padded, not captured
    _close(eager, ref, 1e-5)


def _md17_loader(dev, sizes=(4, 4, 6, 4, 6, 3)):
    from equiformer_b200.synthetic import aspirin_like
    out = []
    for i, B in enumerate(sizes):
        confs = [aspirin_like(seed=100 * i + s) for s in range(B)]
        g = torch.Generator().manual_seed(i)
        out.append(types.SimpleNamespace(pos=torch.cat([c[0] for c in confs]).to(dev),
                                         batch=torch.arange(B).repeat_interleave(21).to(dev),
                                         z=torch.cat([c[2] for c in confs]).to(dev),
                                         y=(torch.randn(B, 1, generator=g) * 2).to(dev),
                                         dy=torch.randn(21 * B, 3, generator=g).to(dev)))
    return out


def _md17_eager(model, loader, dens: bool):
    was = model.training
    model.eval()
    outs = []
    with torch.no_grad():
        for b in loader:
            if dens:
                pred_y, pred_dy = model(types.SimpleNamespace(z=b.z, pos=b.pos.clone(), batch=b.batch))
            else:
                pred_y, pred_dy = model(node_atom=b.z, pos=b.pos.clone(), batch=b.batch)
            outs.append((pred_y.detach(), pred_dy.detach(), b.y, b.dy))
    model.train(was)
    return reference_md17(outs, MEAN, STD)


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["md17", "dens"])
def test_md17_pass_matches_the_reference_loop(cuda_device, family):
    from equiformer_b200.evaluation import EvalPass
    torch.manual_seed(0)
    if family == "dens":
        from equiformer_b200.nets.equiformer_md17_dens import MD17_DENS_L2, Equiformer_MD17_DeNS
        model = Equiformer_MD17_DeNS(**dict(MD17_DENS_L2, num_layers=2)).to(cuda_device).train()
    else:
        from equiformer_b200.nets import model_entrypoint
        model = model_entrypoint(MD17)(irreps_in="64x0e", radius=5.0, num_basis=32).to(cuda_device).train()
    loader = _md17_loader(cuda_device)
    ref = _md17_eager(model, loader, family == "dens")
    ev = EvalPass(model, "md17", 5.0, MEAN, STD, atom_quantum=32, edge_quantum=512)
    got = _check_pass(ev, loader, ref, 1e-4, _buckets(loader, 5.0, 32, 512))
    assert got["force_mae"]["numel"] == 3 * sum(b.dy.shape[0] for b in loader)


def _oc20_loader(dev, sizes=(2, 2, 3, 2, 3, 1)):
    from equiformer_b200.synthetic import oc20_like_frames
    out = []
    for i, n in enumerate(sizes):
        pos, batch, z, tags, edge = oc20_like_frames(n, seed=30 + i)
        g = torch.Generator().manual_seed(i)
        out.append(types.SimpleNamespace(pos=pos.to(dev), batch=batch.to(dev), atomic_numbers=z.to(dev),
                                         tags=tags.to(dev), cell=torch.diag_embed(edge[:, None].expand(-1, 3)).float().to(dev),
                                         y_relaxed=(torch.randn(n, generator=g) * 2).to(dev),
                                         pos_relaxed=(pos + 0.3 * torch.randn(pos.shape, generator=g)).to(dev)))
    return out


def _oc20_eager(model, loader, w, pos_std):
    was = model.training
    model.eval()
    outs = []
    with torch.no_grad():
        for b in loader:
            out = model(b)
            energy, aux = out if isinstance(out, tuple) else (out, None)
            energy = energy.view(-1)
            extra = (aux, (b.pos_relaxed - b.pos) / pos_std, b.tags, w) if aux is not None else ()
            outs.append((energy, b.y_relaxed, oc20_reference_loss(energy, b.y_relaxed, MEAN, STD, *extra)))
    model.train(was)
    return reference_oc20(outs, MEAN, STD)


@pytest.mark.gpu
@pytest.mark.parametrize("aux", [False, True])
def test_oc20_pass_matches_the_reference_loop(cuda_device, aux):
    from equiformer_b200.evaluation import EvalPass
    from equiformer_b200.nets import graph_attention_transformer_oc20 as M
    torch.manual_seed(0)
    cfg = dict(M.OC20_L1_256_NONLINEAR_AUX if aux else M.OC20_L1_256_NONLINEAR, num_layers=2)
    model = M.GraphAttentionTransformerOC20(None, None, 1, **cfg).to(cuda_device).train()
    loader = _oc20_loader(cuda_device)
    ref = _oc20_eager(model, loader, 3.0, 0.9)
    ev = EvalPass(model, "oc20_is2re", 5.0, MEAN, STD, positions_std=0.9, aux_weight=1.0)
    ev.set_aux_weight(3.0)
    got = _check_pass(ev, loader, ref, 1e-5, _buckets(loader, 5.0, 128, 2048, pbc=500))
    assert got["loss"]["numel"] == len(loader)
    if aux:                                              # a new weight reaches the captures without a new capture
        n = ev.captures
        ev.set_aux_weight(0.5)
        _close(ev.run(loader), _oc20_eager(model, loader, 0.5, 0.9), 1e-5)
        assert ev.captures == n


@pytest.mark.gpu
def test_pass_leaves_no_trace(cuda_device):
    from equiformer_b200.evaluation import EvalPass
    from equiformer_b200.parallel import FlatGradAllReduce
    model = _qm9_model(cuda_device, alpha_drop=0.2, drop_path_rate=0.1)
    bucket = FlatGradAllReduce(model.parameters())
    bucket.flat.normal_(generator=torch.Generator(device=cuda_device).manual_seed(5))
    loader = _qm9_loader(cuda_device, sizes=(8, 12, 5))
    before = {k: v.clone() for k, v in model.state_dict().items()}
    flat, cpu_rng, cuda_rng = bucket.flat.clone(), torch.get_rng_state(), torch.cuda.get_rng_state()
    ev = EvalPass(model, "qm9", 5.0, MEAN, STD, target=7)
    first = ev.run(loader)                                   # captures
    assert ev.captures == 3 and model.training
    second = ev.run(loader)
    _same(second, first)
    for k, v in model.state_dict().items():
        assert torch.equal(v, before[k]), k
    assert torch.equal(bucket.flat, flat)
    assert torch.equal(torch.get_rng_state(), cpu_rng) and torch.equal(torch.cuda.get_rng_state(), cuda_rng)
    model.eval()
    _same(ev.run(loader), first)
    assert not model.training and ev.captures == 3             # an eval-mode caller stays in eval mode


@pytest.mark.gpu
def test_ema_and_loaded_weights_through_the_same_captures(cuda_device, tmp_path):
    from equiformer_b200.checkpoint import load_training_state, save_training_state
    from equiformer_b200.evaluation import EvalPass
    from equiformer_b200.parallel import CapturableFlatAdamW, FlatGradAllReduce
    model = _qm9_model(cuda_device)
    bucket = FlatGradAllReduce(model.parameters())
    opt = CapturableFlatAdamW(model.named_parameters(), bucket, lr=2e-3, ema_decay=0.8, model=model,
                              no_decay=model.no_weight_decay())
    g = torch.Generator(device=cuda_device).manual_seed(9)

    def steps(k):
        for _ in range(k):
            for p in bucket.params:                          # gradients of the parameters; the bucket's padding stays 0
                p.grad.normal_(generator=g)
            opt.step()

    steps(4)
    loader = _qm9_loader(cuda_device, sizes=(8, 12, 5))
    ev = EvalPass(model, "qm9", 5.0, MEAN, STD, target=7)
    live = ev.run(loader)
    _close(live, _qm9_eager(model, loader), 1e-5)
    n = ev.captures
    weights = opt.flat.clone()
    with opt.ema_weights():
        ema = ev.run(loader)
    assert ev.captures == n and torch.equal(opt.flat, weights)           # the live weights come back bitwise
    fresh = _qm9_model(cuda_device)
    fresh.load_state_dict(opt.ema_state_dict())
    _close(ema, _qm9_eager(fresh, loader), 1e-5)
    assert abs(ema["mae"]["metric"] - live["mae"]["metric"]) > 1e-6 * live["mae"]["metric"]
    # the metrics go into the checkpoint and come back; a load into the live objects reaches the captures
    path = tmp_path / "checkpoint.pt"
    save_training_state(path, model, opt, epoch=1, step=4, val_metrics=live)
    assert torch.load(path, weights_only=False)["val_metrics"] == live
    steps(3)
    assert ev.run(loader) != live
    load_training_state(path, model, opt)
    assert torch.equal(opt.flat, weights)
    loaded = ev.run(loader)
    assert ev.captures == n
    _same(loaded, live)
    _close(loaded, _qm9_eager(model, loader), 1e-5)
    with opt.ema_weights():
        _same(ev.run(loader), ema)
