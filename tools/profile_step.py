"""torch.profiler breakdown of one training step of bench.py's workload: GPU-busy time vs wall time, top kernels."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from equiformer_b200.nets import model_entrypoint  # noqa: E402


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else "profile_out"
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model = model_entrypoint(bench.WORKLOADS["qm9"]["model"])(irreps_in="5x0e", radius=5.0, num_basis=128, alpha_drop=0.0).to(dev).train()
    opt = torch.optim.AdamW(model.parameters(), lr=5e-4)
    inp = bench.make_inputs("qm9", 0)
    pos, batch, z, target = [inp[k].to(dev) for k in ("pos", "batch", "z", "target")]

    def step():
        opt.zero_grad(set_to_none=True)
        out = model(f_in=None, pos=pos, batch=batch, node_atom=z)
        loss = (out - target).abs().mean()
        loss.backward()
        opt.step()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    n = 3
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], record_shapes=True) as prof:
        for _ in range(n):
            step()
        torch.cuda.synchronize()
    ev = prof.key_averages()
    rows = []
    total_cuda = 0.0
    for e in ev:
        t = getattr(e, "self_device_time_total", None)
        if t is None:
            t = getattr(e, "self_cuda_time_total", 0.0)
        if e.device_type is not None and str(e.device_type).endswith("CUDA") or t > 0:
            rows.append((e.key, e.count, t))
    kern = [(k, c, t) for k, c, t in rows if t > 0]
    kern.sort(key=lambda r: -r[2])
    total_cuda = sum(t for _, _, t in kern)
    lines = [f"steps={n} total_gpu_kernel_time_per_step={total_cuda / n / 1e3:.2f} ms  distinct={len(kern)} "
             f"launches_per_step={sum(c for _, c, _ in kern) / n:.0f}"]
    for k, c, t in kern[:45]:
        lines.append(f"{t / n / 1e3:9.3f} ms/step  n/step={c / n:7.1f}  {k[:110]}")
    text = "\n".join(lines)
    print(text)
    with open(os.path.join(out_dir, "profile_step.txt"), "w") as f:
        f.write(text + "\n")
    # which torch ops (by input shape) hold the device time that is not in our kernels
    shaped = []
    for e in prof.key_averages(group_by_input_shape=True):
        t = getattr(e, "self_device_time_total", None)
        if t is None:
            t = getattr(e, "self_cuda_time_total", 0.0)
        if t > 0 and e.key.startswith("aten::"):
            shaped.append((t / n / 1e3, e.count / n, e.key, str(e.input_shapes)[:150]))
    shaped.sort(reverse=True)
    with open(os.path.join(out_dir, "profile_step_shapes.txt"), "w") as f:
        for t, c, k, sh in shaped[:120]:
            f.write(f"{t:8.3f} ms/step n/step={c:6.1f} {k:28s} {sh}\n")
    # the same rows by LAUNCH COUNT: inside the graph replay every launch costs ~2 us of dependent-launch latency
    shaped.sort(key=lambda r: -r[1])
    with open(os.path.join(out_dir, "profile_step_shapes_by_count.txt"), "w") as f:
        for t, c, k, sh in shaped[:160]:
            f.write(f"n/step={c:6.1f} {t:8.3f} ms/step {k:28s} {sh}\n")


if __name__ == "__main__":
    main()
