"""Timing of the MNIST solve (mbd_mnist_step_launch) at the reference's shape (N = 256, Ndiffuse = 500) on synthetic data of MNIST's
shapes, against the same step in eager torch fp32.

  - per-kernel times: torch.profiler (CUDA activity) over PROF_STEPS graph replays, in a run of its own;
  - the per-step time: CUDA events around STEP_REPS graph replays (the step counter is re-armed between the blocks);
  - the whole solve: wall clock of run_mnist (schedule upload, minibatch table, capture, 499 steps, accuracy every step);
  - the forward kernel's rate: 3.29 GFLOP useful (2 * 256 * 256 * 784 * 32 for layer 1) and 6.58 GFLOP issued (hi + lo), set
    against 495 TF32 dense TFLOP/s, and its compulsory bytes (Y0s read once, 27.1 MB, plus the minibatch pixels) against 3.35 TB/s;
  - the eager baseline: the same step in torch fp32 with TF32 off (randn / rand noise and masks, gather, bmm layer 1, the
    remaining layers, log_softmax, the weights and the weighted mean, plus the accuracy of the new mean), CUDA events over
    STEP_REPS steps after a warm-up.  Its noise is torch's, not JAX's: it is a cost baseline, not a port.
The GPU name, power limit and SM clocks are read in the same run.
    python scripts/gpu_mnist_timing.py [out.json]     (default profiles/h100_mnist.json)"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from mbd_b200.blackbox import mbd_mnist as mm  # noqa: E402
from mbd_b200.planners.engine import make_schedule  # noqa: E402
from tests import mnist_synth as ms  # noqa: E402

N, ND = 256, 500
STEP_REPS = 200
PROF_STEPS = 50
TF32_PEAK, HBM_PEAK = 495.0, 3.35   # TFLOP/s (dense), TB/s: H100 SXM data sheet


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")])) if out.strip() else {}


def engine(data):
    e = mm.MnistEngine(data, N, 0.3, ND)
    e.load_schedule(0, make_schedule(3e-5, 1e-3, ND)[3], mm.params_to_row(mm.init_params(0)))
    e.set_step(ND - 1)
    e.capture()
    return e


def timed_steps(e):
    """ms per step: CUDA events around blocks of graph replays, counter re-armed before each block"""
    out = []
    for _ in range(3):
        e.set_step(ND - 1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(STEP_REPS):
            e.step()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) / STEP_REPS)
    return out


def kernel_times(e):
    """mean device time per launch of every kernel of the step (torch.profiler, CUDA activity)"""
    from torch.profiler import ProfilerActivity, profile
    e.set_step(ND - 1)
    e.step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(PROF_STEPS):
            e.step()
        torch.cuda.synchronize()
    res = {}
    for ev in prof.key_averages():
        if ev.device_type.name == "CUDA" and ev.count > 0:
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            res[ev.key] = {"count": int(ev.count), "us_per_launch": t / ev.count}
    return res


def eager_step(data_t, mean, sigma, gen):
    """one step in torch fp32 (TF32 off) with the same work as the device step"""
    trx, trY, tex, teY = data_t
    Y = mean[None].expand(N, -1).clone()
    noise = torch.randn(Y.shape, device=Y.device, generator=gen) * sigma
    noise[:, :mm.OFF_B1] *= 0.1
    Y += noise * (torch.rand(Y.shape, device=Y.device, generator=gen) < 0.2)
    idx = torch.randperm(trx.shape[0], device=Y.device, generator=gen)[:N]
    x, lab = trx[idx].float() / 255.0, trY[idx].long()

    def mlp(P, xx):
        W1 = P[:, :mm.OFF_B1].view(-1, 32, 784).transpose(1, 2)
        h = torch.relu(torch.matmul(xx, W1) + P[:, None, mm.OFF_B1:mm.OFF_W2])
        h = torch.relu(torch.matmul(h, P[:, mm.OFF_W2:mm.OFF_B2].view(-1, 32, 32)) + P[:, None, mm.OFF_B2:mm.OFF_W3])
        return torch.log_softmax(torch.matmul(h, P[:, mm.OFF_W3:mm.OFF_B3].view(-1, 32, 10)) + P[:, None, mm.OFF_B3:], -1)

    lp = mlp(Y, x[None].expand(N, -1, -1))
    J = lp.gather(2, lab[None, :, None].expand(N, -1, 1))[..., 0].mean(1)
    std = J.std(unbiased=False)
    w = torch.softmax((J - J.mean()) / torch.where(std < 1e-4, torch.ones_like(std), std) / 0.3, 0)
    new = (w[:, None] * Y).sum(0)
    acc_tr = (mlp(new[None], trx.float()[None] / 255.0)[0].argmax(1) == trY.long()).sum()
    acc_te = (mlp(new[None], tex.float()[None] / 255.0)[0].argmax(1) == teY.long()).sum()
    return new, J.mean(), acc_tr, acc_te


def eager_times(data, mean0):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    d = torch.device("cuda")
    data_t = tuple(torch.from_numpy(np.array(a)).to(d) for a in data)
    gen = torch.Generator(device=d)
    gen.manual_seed(0)
    mean = torch.from_numpy(mean0).to(d)
    for _ in range(3):
        eager_step(data_t, mean, 0.01, gen)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 20
    a.record()
    for _ in range(reps):
        mean = eager_step(data_t, mean, 0.01, gen)[0]
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "profiles",
                                                                  "h100_mnist.json")
    torch.cuda.set_device(0)
    info0 = gpu_info()
    data = ms.make()
    e = engine(data)
    step_ms = timed_steps(e)
    kern = kernel_times(e)
    with tempfile.TemporaryDirectory() as td:
        ms.write_dir(td, data)
        torch.cuda.synchronize()
        t0 = time.time()
        res = mm.run_mnist(mm.Args(data_dir=td))
        torch.cuda.synchronize()
        solve_s = time.time() - t0
    eager_ms = eager_times(data, mm.params_to_row(mm.init_params(0)))
    fwd = [v["us_per_launch"] for k, v in kern.items() if "k_mnist_fwd<false>" in k or "k_mnist_fwdILb0E" in k]
    fwd_us = fwd[0] if fwd else float("nan")
    flop_useful = 2.0 * N * N * 784 * 32
    flop_issued = 2 * flop_useful
    bytes_fwd = N * mm.HNU * 4 + N * 784
    rec = {
        "gpu": info0, "gpu_end": gpu_info(), "shape": {"N": N, "Ndiffuse": ND, "HNu": mm.HNU},
        "step_ms_graph_replay": step_ms, "kernels_us": kern,
        "forward": {
            "us": fwd_us,
            "useful_gflop": flop_useful / 1e9, "issued_gflop": flop_issued / 1e9,
            "useful_tflops": flop_useful / (fwd_us * 1e-6) / 1e12, "issued_tflops": flop_issued / (fwd_us * 1e-6) / 1e12,
            "tf32_peak_tflops": TF32_PEAK, "share_of_tf32_peak_issued": flop_issued / (fwd_us * 1e-6) / 1e12 / TF32_PEAK,
            "compulsory_bytes": bytes_fwd, "share_of_hbm_peak": bytes_fwd / (fwd_us * 1e-6) / (HBM_PEAK * 1e12),
            "least_time_us": max(flop_issued / (TF32_PEAK * 1e12), bytes_fwd / (HBM_PEAK * 1e12)) * 1e6,
        },
        "solve_wall_s": solve_s, "solve_final_test_acc_synthetic": float(res["test_acc"][-1]),
        "eager_torch_fp32_step_ms": eager_ms,
    }
    rec["speedup_vs_eager"] = eager_ms / float(np.median(step_ms))
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps({k: rec[k] for k in ("gpu", "step_ms_graph_replay", "forward", "solve_wall_s", "eager_torch_fp32_step_ms",
                                          "speedup_vs_eager")}, indent=1))
    for k, v in sorted(kern.items(), key=lambda kv: -kv[1]["us_per_launch"] * kv[1]["count"])[:12]:
        print(f"{v['us_per_launch']:10.2f} us x {v['count']:4d}  {k[:120]}")


if __name__ == "__main__":
    main()
