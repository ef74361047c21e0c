"""OC20 IS2RE predictions on the device (``evaluation.EvalPass.predict``, ``libeqf_b200_predict.so``) and the results
files (``evaluation.save_predictions`` / ``save_pos_predictions``).

CPU: the header's constants; the library's kernel inventory; the exported argument checks; the results files against a
restatement of the reference trainer's ``save_results`` and ``write_pos`` gather, in one process and in two gloo
processes whose shards overlap; the refusals of ``predict``.

GPU: the kernel against its torch statement, bitwise, at every length regime, with sentinel rows, NaN and Inf; the
captured pass against the reference-style eager predict loop on the unpadded, unlabelled batches; no synchronisation in
the captured function; a pass leaves no trace; the EMA and loaded weights through the same captures.
"""
from __future__ import annotations

import os
import re
import types
from collections import defaultdict

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_evaluation import _buckets, _free_port, _oc20_loader

PREDICT_CLAIMS = {"eqf::predict_is2re_kernel"}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEAN, STD, POS_STD = 0.3, 1.7, 0.9
# Two replays of one capture on the same batch differ in the model's last bits (see test_evaluation.REPEAT, which bounds
# the summed metrics); one frame's energy repeats to REPEAT relative, or absolute below 1
REPEAT = 1e-6


# ------------------------------------------------------------------------------------------------ reference restatements
def reference_save_results(per_rank: list, results_dir, results_file="predictions", name="is2re", keys=("energy",)):
    """``BaseTrainer.save_results`` (``oc20/trainer/base_trainer_oc20.py:707-757``), each rank's write run in turn, then
    rank 0's gather.  ocpmodels' ``distutils`` is not in the tree: ``synchronize`` is the point between the two."""
    for rank, predictions in enumerate(per_rank):
        results_file_path = os.path.join(results_dir, f"{name}_{results_file}_{rank}.npz")
        np.savez_compressed(results_file_path, ids=predictions["id"], **{key: predictions[key] for key in keys})
    gather_results = defaultdict(list)
    full_path = os.path.join(results_dir, f"{name}_{results_file}.npz")
    for i in range(len(per_rank)):
        rank_path = os.path.join(results_dir, f"{name}_{results_file}_{i}.npz")
        rank_results = np.load(rank_path, allow_pickle=True)
        gather_results["ids"].extend(rank_results["ids"])
        for key in keys:
            gather_results[key].extend(rank_results[key])
        os.remove(rank_path)
    _, idx = np.unique(gather_results["ids"], return_index=True)
    gather_results["ids"] = np.array(gather_results["ids"])[idx]
    for k in keys:
        gather_results[k] = np.array(gather_results[k])[idx]
    np.savez_compressed(full_path, **gather_results)
    return full_path


def reference_gather_pos(per_rank: list, run_dir):
    """The ``write_pos`` block of ``EnergyTrainerV2.predict`` (``oc20/trainer/energy_trainer_v2.py:208-222``)."""
    for rank, pos_preds in enumerate(per_rank):
        torch.save(pos_preds, os.path.join(run_dir, "pos_pred_{}.pt".format(rank)))
    gather_pos_preds = {}
    for i in range(len(per_rank)):
        rank_pos_preds = torch.load(os.path.join(run_dir, "pos_pred_{}.pt".format(i)))
        for k, v in rank_pos_preds.items():
            if k not in gather_pos_preds.keys():
                gather_pos_preds[k] = v
    torch.save(gather_pos_preds, os.path.join(run_dir, "pos_pred.pt"))
    return os.path.join(run_dir, "pos_pred.pt")


def reference_predict(model, loader, mean, std, pos_std=None):
    """``EnergyTrainerV2.predict(per_image=True)`` restated on the unpadded batches: eager, ``no_grad``, one ``.tolist()``
    per batch, and with ``pos_std`` the ``write_pos`` positions split per system."""
    was = model.training
    model.eval()
    predictions, pos_preds = {"id": [], "energy": []}, {}
    with torch.no_grad():
        for b in loader:
            out = model(b)
            energy, aux = out if isinstance(out, tuple) else (out, None)
            energy = energy.view(-1) * std + mean                         # normalizers["target"].denorm
            predictions["id"].extend([str(i) for i in b.sid.tolist()])
            predictions["energy"].extend(energy.tolist())
            if pos_std is not None:
                delta_pos = aux * pos_std + 0.0                           # normalizers["positions"].denorm, mean 0
                tag_mask = b.tags > 0
                pred_pos = b.pos.clone()
                pred_pos[tag_mask] = pred_pos[tag_mask] + delta_pos[tag_mask]
                for sid, p in zip([str(s) for s in b.sid.tolist()], torch.split(pred_pos, b.natoms.tolist())):
                    pos_preds[sid] = p.detach().cpu()
    model.train(was)
    return predictions, pos_preds


def _same_npz(a_path, b_path):
    with np.load(a_path, allow_pickle=True) as a, np.load(b_path, allow_pickle=True) as b:
        assert a.files == b.files, (a.files, b.files)
        for k in a.files:
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, (k, a[k].dtype, b[k].dtype)
            assert a[k].tobytes() == b[k].tobytes(), k


def _same_pos_file(a_path, b_path):
    a, b = torch.load(a_path), torch.load(b_path)
    assert list(a) == list(b)
    for k in a:
        assert a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), k


# ------------------------------------------------------------------------------------------------ CPU
def test_header_constants_match():
    from equiformer_b200 import _lib
    header = open(os.path.join(ROOT, "include", "eqf_b200_predict.h")).read()
    for name in ("EQF_PREDICT_THREADS", "EQF_PREDICT_MAX_CTAS"):
        assert int(re.search(rf"#define {name} (\d+)", header).group(1)) == getattr(_lib, name), name


def test_predict_library_inventory_is_claimed(built_lib):
    """The one kernel of the library is launched by test_kernel_matches_the_torch_statement; no other library holds a
    prediction kernel or compiles eqf_predict.cu."""
    from equiformer_b200 import _lib
    from tests.test_gpu_kernel_instances import inventory
    inv = inventory(_lib.PREDICT_LIB_PATH)
    assert inv == PREDICT_CLAIMS, (sorted(inv - PREDICT_CLAIMS), sorted(PREDICT_CLAIMS - inv))
    for sources in (_lib.SOURCES, _lib.L4_SOURCES, _lib.NORM_SOURCES, _lib.OPTIM_SOURCES, _lib.EVAL_SOURCES):
        assert "eqf_predict.cu" not in sources
    for path in (_lib.LIB_PATH, _lib.NORM_LIB_PATH, _lib.OPTIM_LIB_PATH, _lib.EVAL_LIB_PATH):
        assert not {n for n in inventory(path) if n.startswith("eqf::predict_")}, path.name


def test_argument_checks_refuse_null_pointers_partial_sets_and_negative_sizes(built_lib):
    """The exported check, called on its own: host code that launches and dereferences nothing."""
    from equiformer_b200 import _lib
    lib = _lib.load_predict()
    ok = 1 << 20
    msg = lambda: lib.eqf_last_error().decode()
    # energy, n_graphs, pos, delta, tags, n_rows, energy_out, pos_out
    assert lib.eqf_predict_is2re_check(ok, 4, ok, ok, ok, 9, ok, ok) == 0
    assert lib.eqf_predict_is2re_check(ok, 4, None, None, None, 0, ok, None) == 0            # energies only
    assert lib.eqf_predict_is2re_check(ok, 0, ok, ok, ok, 0, ok, ok) == 0                    # empty is allowed
    assert lib.eqf_predict_is2re_check(None, 4, None, None, None, 0, ok, None) != 0 and "null" in msg()
    assert lib.eqf_predict_is2re_check(ok, 4, None, None, None, 0, None, None) != 0 and "null" in msg()
    for bad in range(4):                                                     # a partly NULL position set
        ptrs = [None if i == bad else ok for i in range(4)]
        assert lib.eqf_predict_is2re_check(ok, 4, ptrs[0], ptrs[1], ptrs[2], 9, ok, ptrs[3]) != 0, bad
        assert "all given or all NULL" in msg()
    for only in range(4):
        ptrs = [ok if i == only else None for i in range(4)]
        assert lib.eqf_predict_is2re_check(ok, 4, ptrs[0], ptrs[1], ptrs[2], 9, ok, ptrs[3]) != 0, only
        assert "all given or all NULL" in msg()
    assert lib.eqf_predict_is2re_check(ok, -1, ok, ok, ok, 9, ok, ok) != 0 and "n_graphs" in msg()
    assert lib.eqf_predict_is2re_check(ok, 4, ok, ok, ok, -2, ok, ok) != 0 and "n_rows" in msg()


def test_launcher_refuses_cpu_wrong_dtypes_shapes_and_partial_sets():
    from equiformer_b200 import _lib
    from equiformer_b200.eval_kernels import predict_is2re_raw
    e, out, p, t = torch.zeros(4), torch.zeros(4), torch.zeros(6, 3), torch.zeros(6, dtype=torch.int64)
    with pytest.raises(_lib.EqfError, match="CUDA-only"):
        predict_is2re_raw(e, 4, MEAN, STD, out)
    with pytest.raises(_lib.EqfError, match="float32"):
        predict_is2re_raw(e.double(), 4, MEAN, STD, out)
    with pytest.raises(_lib.EqfError, match="elements"):
        predict_is2re_raw(e, 5, MEAN, STD, out)
    with pytest.raises(_lib.EqfError, match="together"):
        predict_is2re_raw(e, 4, MEAN, STD, out, pos=p, delta=p, tags=t)
    with pytest.raises(_lib.EqfError, match=r"\[rows, 3\]"):
        predict_is2re_raw(e, 4, MEAN, STD, out, pos=p, delta=p[:5], tags=t, pos_out=p)
    with pytest.raises(_lib.EqfError, match="int64"):
        predict_is2re_raw(e, 4, MEAN, STD, out, pos=p, delta=p, tags=t.int(), pos_out=p)


def _rank_predictions(rank, world, n=7):
    """What rank ``rank`` of ``world`` predicts for a dataset of ``n`` systems under a padding ``DistributedSampler``
    (the last rank repeats system 0).  The sids have different digit counts, so their string order is not numeric; a
    repeated system is predicted with other values than its first copy, so the tests see which copy is kept."""
    sampler = torch.utils.data.DistributedSampler(range(n), num_replicas=world, rank=rank, shuffle=False)
    sids = [7, 120, 33, 5, 1000, 64, 2]
    pred, pos = {"id": [], "energy": []}, {}
    for j, i in enumerate(sampler):
        g = torch.Generator().manual_seed(1000 * rank + j)
        pred["id"].append(str(sids[i]))
        pred["energy"].append(float(torch.randn((), generator=g, dtype=torch.float64)) * 3.0 + i)
        pos[str(sids[i])] = torch.randn(3 + i, 3, generator=g)
    return pred, pos


def test_results_files_match_the_reference_in_one_process(tmp_path):
    from equiformer_b200.evaluation import save_pos_predictions, save_predictions
    ours, ref = tmp_path / "ours", tmp_path / "ref"
    ours.mkdir(), ref.mkdir()
    pred, pos = _rank_predictions(0, 1)
    path = save_predictions(pred, ours)
    assert path == os.path.join(str(ours), "is2re_predictions.npz")
    _same_npz(path, reference_save_results([pred], ref))
    assert not (ours / "is2re_predictions_0.npz").exists()
    full = save_pos_predictions(pos, ours)
    _same_pos_file(full, reference_gather_pos([pos], ref))
    assert (ours / "pos_pred_0.pt").exists()
    _same_pos_file(ours / "pos_pred_0.pt", ref / "pos_pred_0.pt")
    path = save_predictions(pred, ours, results_file="best", name="s2ef")          # the names follow the arguments
    assert os.path.basename(path) == "s2ef_best.npz" and os.path.exists(path)


def _results_worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    from equiformer_b200.evaluation import save_pos_predictions, save_predictions
    from equiformer_b200.parallel import init_distributed
    init_distributed("gloo")
    pred, pos = _rank_predictions(rank, world)
    path = save_predictions(pred, out_dir)
    assert os.path.exists(path)                                    # every rank returns once the gathered file is there
    full = save_pos_predictions(pos, out_dir)
    assert os.path.exists(full)
    dist.destroy_process_group()


def test_results_files_match_the_reference_over_two_processes(tmp_path):
    world = 2
    ours, ref = tmp_path / "ours", tmp_path / "ref"
    ours.mkdir(), ref.mkdir()
    mp.spawn(_results_worker, args=(world, _free_port(), str(ours)), nprocs=world, join=True)
    per_rank = [_rank_predictions(r, world) for r in range(world)]
    assert sum(len(p["id"]) for p, _ in per_rank) == 8                 # 7 systems, one repeated
    _same_npz(ours / "is2re_predictions.npz", reference_save_results([p for p, _ in per_rank], ref))
    assert not any((ours / f"is2re_predictions_{r}.npz").exists() for r in range(world))
    with np.load(ours / "is2re_predictions.npz") as r:
        ids = list(r["ids"])
        assert ids == sorted(set(ids)) and len(ids) == 7                   # de-duplicated, sorted as strings
        assert ids[:3] == ["1000", "120", "2"]
        first = per_rank[0][0]
        assert r["energy"][ids.index("7")] == first["energy"][first["id"].index("7")]     # the first copy is kept
    _same_pos_file(ours / "pos_pred.pt", reference_gather_pos([p for _, p in per_rank], ref))
    for r in range(world):
        _same_pos_file(ours / f"pos_pred_{r}.pt", ref / f"pos_pred_{r}.pt")                # kept, as the reference does
    assert torch.equal(torch.load(ours / "pos_pred.pt")["7"], per_rank[0][1]["7"])


def test_predict_refuses_other_tasks_and_positions_without_the_auxiliary_head():
    from equiformer_b200.evaluation import EvalPass
    model = torch.nn.Linear(1, 1)
    for task in ("qm9", "md17"):
        with pytest.raises(ValueError, match="OC20 IS2RE"):
            EvalPass(model, task, 5.0, capture=False).predict([])
    with pytest.raises(ValueError, match="auxiliary head"):
        EvalPass(model, "oc20_is2re", 5.0, capture=False).predict([], write_pos=True)
    assert EvalPass(model, "oc20_is2re", 5.0, capture=False).predict([]) == {"id": [], "energy": []}


# ------------------------------------------------------------------------------------------------ GPU: kernel
def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [1, 200, 5000, 100_000])     # one row, one CTA, several CTAs, past the 128-CTA cap
def test_kernel_matches_the_torch_statement(cuda_device, rows):
    from equiformer_b200.eval_kernels import predict_is2re_raw, predict_is2re_torch
    dev = cuda_device
    g = torch.Generator().manual_seed(rows)
    sentinel = -12345.0
    for n_graphs in sorted({max(1, rows // 3), rows}):
        energy = (torch.randn(n_graphs + 4, generator=g) * 3).to(dev)                  # padded rows after the real ones
        pos = (torch.rand(rows, 3, generator=g) * 20).to(dev)
        delta = torch.randn(rows, 3, generator=g).to(dev)
        tags = torch.randint(0, 3, (rows,), generator=g).to(dev)
        if rows > 3:                                                                     # NaN and Inf on moving atoms
            energy[1], energy[n_graphs - 1] = float("nan"), float("inf")
            tags[:3] = 1
            delta[0, 1], delta[1, 2], pos[2, 0] = float("nan"), -float("inf"), float("inf")
        e_buf = torch.full((n_graphs + 5,), sentinel, device=dev)
        p_buf = torch.full((rows + 7, 3), sentinel, device=dev)
        predict_is2re_raw(energy, n_graphs, MEAN, STD, e_buf, pos, delta, tags, POS_STD, p_buf[:rows])
        e_ref, p_ref = predict_is2re_torch(energy, n_graphs, MEAN, STD, pos, delta, tags, POS_STD)
        assert torch.equal(_bits(e_buf[:n_graphs]), _bits(e_ref))
        assert torch.equal(_bits(p_buf[:rows]), _bits(p_ref))
        moving = tags > 0
        assert torch.equal(_bits(p_buf[:rows][moving]), _bits(pos[moving] + (delta[moving] * POS_STD + 0.0)))
        assert torch.equal(_bits(p_buf[:rows][~moving]), _bits(pos[~moving]))
        assert bool((e_buf[n_graphs:] == sentinel).all()) and bool((p_buf[rows:] == sentinel).all())
        if rows > 3:
            assert torch.isnan(e_buf[1]) and torch.isinf(e_buf[n_graphs - 1]) and e_buf[n_graphs - 1] > 0
            assert torch.isnan(p_buf[0, 1]) and torch.isinf(p_buf[1, 2]) and torch.isinf(p_buf[2, 0])
        again_e, again_p = torch.full_like(e_buf, sentinel), torch.full_like(p_buf, sentinel)
        predict_is2re_raw(energy, n_graphs, MEAN, STD, again_e, pos, delta, tags, POS_STD, again_p[:rows])
        assert torch.equal(_bits(again_e), _bits(e_buf)) and torch.equal(_bits(again_p), _bits(p_buf))
        only = torch.full_like(e_buf, sentinel)                                          # energies only
        predict_is2re_raw(energy, n_graphs, MEAN, STD, only)
        assert torch.equal(_bits(only), _bits(e_buf))


# ------------------------------------------------------------------------------------------------ GPU: the pass
def _oc20_model(dev, aux, **over):
    from equiformer_b200.nets import graph_attention_transformer_oc20 as M
    torch.manual_seed(0)
    cfg = dict(M.OC20_L1_256_NONLINEAR_AUX if aux else M.OC20_L1_256_NONLINEAR, num_layers=2, **over)
    return M.GraphAttentionTransformerOC20(None, None, 1, **cfg).to(dev).train()


def _test_split(dev, sizes=(2, 2, 3, 2, 3, 1)):
    """The batches of test_evaluation's OC20 loader without their labels, with ``natoms`` and ``sid`` (not in order)."""
    labelled = _oc20_loader(dev, sizes)
    out, first = [], 0
    for b in labelled:
        G = int(b.cell.shape[0])
        natoms = torch.bincount(b.batch, minlength=G)
        sid = torch.arange(first, first + G, device=dev) * 37 % 101 + 1000 * (first % 2)
        first += G
        out.append(types.SimpleNamespace(pos=b.pos, batch=b.batch, atomic_numbers=b.atomic_numbers, tags=b.tags,
                                         cell=b.cell, natoms=natoms, sid=sid))
    return out, _buckets(labelled, 5.0, 128, 2048, pbc=500)


def _close_predictions(got, ref, ref_pos=None, e_tol=1e-5, p_tol=1e-5):
    assert got["id"] == ref["id"]
    e, r = torch.tensor(got["energy"], dtype=torch.float64), torch.tensor(ref["energy"], dtype=torch.float64)
    assert ((e - r).abs() <= e_tol * r.abs().clamp_min(1.0)).all(), ((e - r).abs().max().item(), e, r)
    if ref_pos is not None:
        assert list(got["pos"]) == list(ref_pos)
        for k, v in ref_pos.items():
            assert got["pos"][k].dtype == torch.float32 and got["pos"][k].device.type == "cpu"
            assert got["pos"][k].shape == v.shape, k
            assert (got["pos"][k] - v).abs().max() <= p_tol, (k, (got["pos"][k] - v).abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("aux", [False, True])
def test_predict_matches_the_reference_loop(cuda_device, aux):
    from equiformer_b200.evaluation import EvalPass
    model = _oc20_model(cuda_device, aux)
    loader, n_buckets = _test_split(cuda_device)
    assert n_buckets >= 3 and not hasattr(loader[0], "y_relaxed") and not hasattr(loader[0], "pos_relaxed")
    ref, ref_pos = reference_predict(model, loader, MEAN, STD, POS_STD if aux else None)
    ev = EvalPass(model, "oc20_is2re", 5.0, MEAN, STD, positions_std=POS_STD)
    got = ev.predict(loader, write_pos=aux)
    _close_predictions(got, ref, ref_pos if aux else None)
    assert ("pos" in got) == aux and len(got["id"]) == sum(int(b.natoms.numel()) for b in loader)
    assert ev.predict_captures == n_buckets and ev.captures == 0
    again = ev.predict(loader, write_pos=aux)
    assert ev.predict_captures == n_buckets                                      # no new capture
    _close_predictions(again, got, got.get("pos"), e_tol=REPEAT, p_tol=1e-6)
    if aux:                                                                      # energies only, on captures of their own
        _close_predictions(ev.predict(loader), ref)
        assert ev.predict_captures == 2 * n_buckets
    eager = EvalPass(model, "oc20_is2re", 5.0, MEAN, STD, positions_std=POS_STD, capture=False)
    _close_predictions(eager.predict(loader, write_pos=aux), ref, ref_pos if aux else None)


@pytest.mark.gpu
def test_captured_function_does_not_synchronise(cuda_device):
    from equiformer_b200.evaluation import EvalPass
    model = _oc20_model(cuda_device, True).eval()
    ev = EvalPass(model, "oc20_is2re", 5.0, MEAN, STD, positions_std=POS_STD)
    b = _test_split(cuda_device, sizes=(3,))[0][0]
    pos, padded, (Nb, _Eb) = ev._oc20_inputs(b, 3)
    tensors = [*padded, b.natoms, torch.cat([pos, pos.new_zeros(Nb - pos.shape[0], 3)])]
    ev._oc20_predict(*tensors)                                                   # loads the libraries, builds the plans
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        energy, pos_out = ev._oc20_predict(*tensors)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert energy.shape == (3,) and pos_out.shape == (Nb, 3) and bool(torch.isfinite(energy).all())


@pytest.mark.gpu
def test_predict_leaves_no_trace(cuda_device):
    from equiformer_b200.evaluation import EvalPass
    from equiformer_b200.parallel import FlatGradAllReduce
    model = _oc20_model(cuda_device, True, alpha_drop=0.2, drop_path_rate=0.05)
    bucket = FlatGradAllReduce(model.parameters())
    bucket.flat.normal_(generator=torch.Generator(device=cuda_device).manual_seed(5))
    loader, n_buckets = _test_split(cuda_device, sizes=(2, 3, 1))
    before = {k: v.clone() for k, v in model.state_dict().items()}
    flat, cpu_rng, cuda_rng = bucket.flat.clone(), torch.get_rng_state(), torch.cuda.get_rng_state()
    ev = EvalPass(model, "oc20_is2re", 5.0, MEAN, STD, positions_std=POS_STD)
    first = ev.predict(loader, write_pos=True)                                   # captures
    assert ev.predict_captures == n_buckets and model.training
    second = ev.predict(loader, write_pos=True)
    _close_predictions(second, first, first["pos"], e_tol=REPEAT, p_tol=1e-6)
    for k, v in model.state_dict().items():
        assert torch.equal(v, before[k]), k
    assert torch.equal(bucket.flat, flat)
    assert torch.equal(torch.get_rng_state(), cpu_rng) and torch.equal(torch.cuda.get_rng_state(), cuda_rng)
    model.eval()
    _close_predictions(ev.predict(loader, write_pos=True), first, first["pos"], e_tol=REPEAT, p_tol=1e-6)
    assert not model.training and ev.predict_captures == n_buckets


@pytest.mark.gpu
def test_ema_and_loaded_weights_through_the_same_captures(cuda_device, tmp_path):
    from equiformer_b200.checkpoint import load_training_state, save_training_state
    from equiformer_b200.evaluation import EvalPass
    from equiformer_b200.parallel import CapturableFlatAdamW, FlatGradAllReduce
    model = _oc20_model(cuda_device, True)
    bucket = FlatGradAllReduce(model.parameters())
    opt = CapturableFlatAdamW(model.named_parameters(), bucket, lr=2e-3, ema_decay=0.8, model=model,
                              no_decay=model.no_weight_decay())
    g = torch.Generator(device=cuda_device).manual_seed(9)

    def steps(k):
        for _ in range(k):
            for p in bucket.params:
                p.grad.normal_(generator=g)
            opt.step()

    steps(4)
    loader, _ = _test_split(cuda_device, sizes=(2, 3, 1))
    ev = EvalPass(model, "oc20_is2re", 5.0, MEAN, STD, positions_std=POS_STD)
    live = ev.predict(loader, write_pos=True)
    _close_predictions(live, *reference_predict(model, loader, MEAN, STD, POS_STD))
    n = ev.predict_captures
    weights = opt.flat.clone()
    with opt.ema_weights():
        ema = ev.predict(loader, write_pos=True)
    assert ev.predict_captures == n and torch.equal(opt.flat, weights)        # the live weights come back bitwise
    fresh = _oc20_model(cuda_device, True)
    fresh.load_state_dict(opt.ema_state_dict())
    _close_predictions(ema, *reference_predict(fresh, loader, MEAN, STD, POS_STD))
    assert max(abs(a - b) for a, b in zip(ema["energy"], live["energy"])) > 1e-5
    path = tmp_path / "checkpoint.pt"
    save_training_state(path, model, opt, epoch=1, step=4)
    steps(3)
    moved = ev.predict(loader, write_pos=True)
    assert max(abs(a - b) for a, b in zip(moved["energy"], live["energy"])) > 1e-5
    load_training_state(path, model, opt)
    loaded = ev.predict(loader, write_pos=True)
    assert ev.predict_captures == n
    _close_predictions(loaded, live, live["pos"], e_tol=REPEAT, p_tol=1e-6)
    _close_predictions(loaded, *reference_predict(model, loader, MEAN, STD, POS_STD))
