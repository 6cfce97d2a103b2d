"""The black-box optimiser's seed sweep, sequential against batched, and launch (1)'s kernel time.

For Ackley, Rastrigin and Levy at mbd_opt.py's shape (6 seeds x 64 samples x 800 dims, Ndiffuse 100): the wall clock of ONE
run_exp_batch over seeds 0..5 against 6 sequential run_exp calls (B = 1 each), alternated REPEATS times in this process after one
warm-up of each; medians reported.  Then launch (1) (k_bbo, B = 1) at N in {64, 2048, 8192} x dim in {800, 6912}, on the first
step (which also draws the per-sample mean) and on a later one: CUDA events around KERNEL_REPS whole steps and around KERNEL_REPS
tail-only MPPI steps (mbd_pi_batch_step_launch with tail_only) on the same buffers; launch (1) is the difference per step.
The GPU name, power limit and SM clocks are read in the same run.
    python scripts/gpu_bbo_sweep.py [out.json]     (default profiles/h100_bbo_sweep.json)"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from mbd_b200 import _lib, ops  # noqa: E402
from mbd_b200.blackbox import mbd_opt  # noqa: E402

FNS = ("Ackley", "Rastrigin", "Levy")
REPEATS = 3
KERNEL_REPS = 200
KERNEL_SHAPES = [(n, d) for n in (64, 2048, 8192) for d in (800, 6912)]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")])) if out.strip() else {}


def sweep(fn):
    a = mbd_opt.Args(fn_name=fn)
    seeds = list(range(a.Nexp))

    def sequential():
        t0 = time.time()
        ys = [mbd_opt.run_exp(a, s)[1] for s in seeds]
        torch.cuda.synchronize()
        return time.time() - t0, np.stack(ys)

    def batched():
        t0 = time.time()
        ys = mbd_opt.run_exp_batch(a, seeds)[1]
        torch.cuda.synchronize()
        return time.time() - t0, ys

    sequential(); batched()   # warm-up
    seq, bat = [], []
    for _ in range(REPEATS):
        seq.append(sequential())
        bat.append(batched())
    same = all(np.array_equal(s[1].view(np.uint32), b[1].view(np.uint32)) for s, b in zip(seq, bat))
    ts, tb = float(np.median([s[0] for s in seq])), float(np.median([b[0] for b in bat]))
    return dict(fn=fn, B=a.Nexp, N=a.Nsample, dim=a.dim, Ndiffuse=a.Ndiffuse, sequential_s=ts, batched_s=tb, speedup=ts / tb,
                sequential_runs_s=[s[0] for s in seq], batched_runs_s=[b[0] for b in bat], bit_identical=bool(same),
                ys_first=float(bat[0][1].mean(0)[0]), ys_last=float(bat[0][1].mean(0)[-1]))


def kernel_time(fn, N, dim, first):
    """launch (1) at step i (the first step draws the per-sample mean as well): CUDA events around KERNEL_REPS full steps and
    KERNEL_REPS tail-only MPPI steps on the same buffers; the difference per step is launch (1)"""
    Nd = KERNEL_REPS + 2
    e = mbd_opt.BboEngine(fn, dim, N, [1.0], Nd)
    sig = np.full(Nd, 0.5, np.float32)
    keys, k0 = mbd_opt.problem_keys(0, Nd)
    e.load_schedule([keys], sig, [k0])
    pibufs = _lib.PiBufs(None, None, None)

    def timed(tail_only):
        e.set_step(Nd - 1)
        e.Ybars.uniform_(-0.5, 0.5)
        if first:
            launch = (lambda: (e.set_step(Nd - 1), e._launch())) if not tail_only else \
                (lambda: (e.set_step(Nd - 1), ops.pi_batch_step_launch(e._plan_c, 1, Nd, 1, e.temps, pibufs, True)))
        else:
            launch = e._launch if not tail_only else (lambda: ops.pi_batch_step_launch(e._plan_c, 1, Nd, 1, e.temps, pibufs, True))
        launch()   # warm-up
        e.set_step(Nd - 1)
        torch.cuda.synchronize()
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(KERNEL_REPS):
            launch()
        t.record()
        torch.cuda.synchronize()
        return s.elapsed_time(t) / KERNEL_REPS

    full, tail = timed(False), timed(True)
    return dict(fn=fn, N=N, dim=dim, step="first" if first else "later", step_ms=full, tail_ms=tail, launch1_ms=full - tail)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "profiles",
                                                             "h100_bbo_sweep.json")
    torch.cuda.set_device(0)
    res = dict(gpu=gpu_info(), torch=torch.__version__, repeats=REPEATS, kernel_reps=KERNEL_REPS, sweep=[], kernel=[])
    for fn in FNS:
        r = sweep(fn)
        print(json.dumps(r), flush=True)
        res["sweep"].append(r)
    for fn in FNS:
        for N, dim in KERNEL_SHAPES:
            for first in (True, False):
                r = kernel_time(fn, N, dim, first)
                print(json.dumps(r), flush=True)
                res["kernel"].append(r)
    res["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", out)


if __name__ == "__main__":
    main()
