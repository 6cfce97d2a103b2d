"""The path-integral baselines' 8-seed sweep, host-stepped against batched, on the reference's shapes.

For MPPI, CMA-ES and CEM and every shape of SHAPES (the reference's recommended parameters: hopper and ant 2048 x 50 with
Nrefine 100, pushT 2048 x 40 with Nrefine 200, humanoidrun 8192 x 50 with Nrefine 300): the wall clock of 8 sequential
run_path_integral calls (seeds 0..7, what `run_mbd --algo path_integral` runs) against ONE run_path_integral_batch of the same
8 Args (`--pi_batch`), alternated REPEATS times in this process after one warm-up of each; medians reported.  Then the tail of
one step (launches 2 and 3 together: weights, then the update) from CUDA events over TAIL_REPS tail-only launches, for MBD
(mbd_step_tail_launch) and each baseline (mbd_pi_batch_step_launch with tail_only), B = 1, at N = 2048 and 8192, H * Nu = 850.
The GPU name, power limit and SM clocks are read in the same run.
    python scripts/gpu_pi_sweep.py [out.json]     (default profiles/h100_pi_sweep.json)"""
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from mbd_b200 import ops  # noqa: E402
from mbd_b200.planners import engine as eng  # noqa: E402
from mbd_b200.planners import path_integral as pi  # noqa: E402
from mbd_b200.scripts import run_mbd  # noqa: E402

SHAPES = ("hopper", "ant", "pushT", "humanoidrun")   # shapes come from the recommended-parameter table
METHODS = ("mppi", "cma-es", "cem")
REPEATS = 3
TAIL_REPS = 200


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")])) if out.strip() else {}


def sweep(env_name, method):
    args = lambda: run_mbd.pi_seed_args(run_mbd.Args(env_name=env_name, update_method=method))   # noqa: E731

    def sequential():
        t0 = time.time()
        r = [pi.run_path_integral(a) for a in args()]
        torch.cuda.synchronize()
        return time.time() - t0, r

    def batched():
        t0 = time.time()
        r = pi.run_path_integral_batch(args())
        torch.cuda.synchronize()
        return time.time() - t0, list(r)

    with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
        sequential(); batched()   # warm-up
        seq, bat = [], []
        for _ in range(REPEATS):
            seq.append(sequential())
            bat.append(batched())
    a = args()[0]
    with contextlib.redirect_stdout(io.StringIO()):
        pi.apply_recommended_params(a)
    return dict(env=env_name, method=method, shape=f"{a.Nsample}x{a.Hsample}, Nrefine {a.Nrefine}",
                sequential_8_s=[s[0] for s in seq], batch_of_8_s=[b[0] for b in bat],
                sequential_median_s=float(np.median([s[0] for s in seq])), batch_median_s=float(np.median([b[0] for b in bat])),
                speedup_median=float(np.median([s[0] for s in seq]) / np.median([b[0] for b in bat])),
                rew_final_sequential=[float(x) for x in seq[-1][1]], rew_final_batch=[float(x) for x in bat[-1][1]])


def tail_ms(method, Ns, HNu=850):
    """ms per tail (launches 2 + 3) of one problem, CUDA events over TAIL_REPS launches after 20 warm-up launches, on an engine
    without an env (Nu = 1, H * Nu = any column count)"""
    Nd = TAIL_REPS + 22
    rng = np.random.default_rng(0)
    none = eng.LaunchInputs.none()
    if method == "mbd":
        e = eng.DiffusionEngine(None, Ns, HNu, 0.1, False, None, Ndiffuse=Nd, inputs=none, nu=1)
        _, al, ab, sig = eng.make_schedule(1e-4, 1e-2, Nd)
        e.load_schedule(eng.key_chain(np.uint32([1, 2]), Nd), sig, al, ab)
        rews, Y = e.rews_local, e.Y0s
        launch = lambda: ops.step_tail_launch(e._plan_c)   # noqa: E731
    else:
        e = pi.BatchedPathIntegralEngine(None, Ns, HNu, [0.1], [None], Nd, method, inputs=none, nu=1)
        e.load_schedule([eng.key_chain(np.uint32([1, 2]), Nd)])
        rews, Y = e.rews[0], e.Y0s[0]
        launch = e.tail_step
    rews.copy_(torch.from_numpy(rng.normal(size=Ns).astype(np.float32)))
    Y.copy_(torch.from_numpy(np.clip(rng.normal(size=(Ns, HNu)) * 0.5, -1, 1).astype(np.float32)))
    e.set_step(Nd - 1)
    for _ in range(20):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(TAIL_REPS):
        launch()
    e1.record()
    torch.cuda.synchronize()
    e.check_exchange()
    return e0.elapsed_time(e1) / TAIL_REPS


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(__file__), "..", "profiles", "h100_pi_sweep.json")
    torch.cuda.set_device(0)
    res = dict(gpu_before=gpu_info(),
               method=f"wall clock (synchronised) of 8 sequential run_path_integral calls vs one run_path_integral_batch of the same "
                      f"8 seeds, alternated {REPEATS}x after one warm-up each; tail = launches 2 + 3 of one step, CUDA events over "
                      f"{TAIL_REPS} tail-only launches, B = 1, H * Nu = 850",
               sweeps=[], tail_ms=[])
    for m in ("mbd",) + METHODS:
        for Ns in (2048, 8192):
            res["tail_ms"].append(dict(rule=m, N=Ns, ms=tail_ms(m, Ns)))
            print(res["tail_ms"][-1], flush=True)
    for env_name in SHAPES:
        for m in METHODS:
            res["sweeps"].append(sweep(env_name, m))
            r = res["sweeps"][-1]
            print(r["env"], r["method"], r["shape"], r["sequential_median_s"], r["batch_median_s"], r["speedup_median"], flush=True)
    res["gpu_after"] = gpu_info()
    with open(out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
