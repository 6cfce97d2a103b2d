"""Batch-size sweep of the batched diffusion step (BatchedDiffusionEngine, mbd_batch_step_launch) on the reference's shapes.

For every shape and B in {1, 2, 4, 8, 16}: the step time of the captured three-launch graph (CUDA events over >= 50 replays
after warm-up) and the solve throughput B * N * H / step time (sample-steps per second).  End to end: the wall clock of
`run_mbd --mode seed --algo mbd --env_name hopper` (one batch of 8 seeds) against 8 sequential run_diffusion calls of the
same Args, in the same process, alternated.  The GPU name, power limit and SM clocks are read in the same run.
    python scripts/gpu_batch_sweep.py [out.json]     (default profiles/h100_batch_sweep.json)"""
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
import mbd_b200  # noqa: E402
from mbd_b200 import prng  # noqa: E402
from mbd_b200.planners import engine as eng  # noqa: E402
from mbd_b200.planners.mbd_planner import Args, run_diffusion  # noqa: E402
from mbd_b200.scripts import run_mbd  # noqa: E402

SHAPES = [("car2d", 64, 40), ("hopper", 1024, 50), ("ant", 2048, 50), ("pushT", 2048, 40), ("humanoidrun", 1024, 50),
          ("humanoidrun", 8192, 50)]
BATCHES = (1, 2, 4, 8, 16)
WARMUP, REPLAYS = 10, 60


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")])) if out.strip() else {}


def step_time(env_name, Ns, H, B):
    """ms per batched step: one captured graph replayed REPLAYS times after WARMUP replays"""
    env = mbd_b200.envs.get_env(env_name)
    Nd = WARMUP + REPLAYS + 2
    st = env.reset(prng.split(prng.PRNGKey(0))[1])
    _, alphas, alphas_bar, sigmas = eng.make_schedule(1e-4, 1e-2, Nd)
    keys = [eng.key_chain(np.uint32([b, 7]), Nd) for b in range(B)]
    be = eng.BatchedDiffusionEngine(env, Ns, H, [0.1] * B, False, [st] * B, Nd)
    be.load_schedule(keys, [sigmas] * B, [alphas] * B, [alphas_bar] * B)
    be.set_step(Nd - 1)
    be.capture()
    for _ in range(WARMUP):
        be.step()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(REPLAYS):
        be.step()
    e1.record()
    torch.cuda.synchronize()
    be.check_exchange()
    return e0.elapsed_time(e1) / REPLAYS


def end_to_end():
    """seconds: one run_mbd seed batch (8 seeds) vs 8 sequential run_diffusion calls, hopper defaults; alternated, 3 each"""
    def sequential():
        t0 = time.time()
        for s in run_mbd.SEEDS:
            run_diffusion(Args(seed=s, env_name="hopper", not_render=True))
        torch.cuda.synchronize()
        return time.time() - t0

    def batched():
        t0 = time.time()
        run_mbd.run_multiple_seed(run_mbd.Args(algo="mbd", mode="seed", env_name="hopper"))
        return time.time() - t0

    quiet = contextlib.redirect_stdout(io.StringIO())
    with quiet:
        sequential(); batched()   # warm-up (module load, graph capture paths)
    seq, bat = [], []
    for _ in range(3):
        with contextlib.redirect_stdout(io.StringIO()):
            seq.append(sequential())
            bat.append(batched())
    a = Args(env_name="hopper")
    from mbd_b200.planners.mbd_planner import apply_recommended_params
    with contextlib.redirect_stdout(io.StringIO()):
        apply_recommended_params(a)
    return dict(command="run_mbd --mode seed --algo mbd --env_name hopper", shape=f"{a.Nsample}x{a.Hsample}, Ndiffuse {a.Ndiffuse}",
                sequential_8_run_diffusion_s=seq, run_mbd_batch_of_8_s=bat,
                speedup_median=float(np.median(seq) / np.median(bat)))


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(__file__), "..", "profiles", "h100_batch_sweep.json")
    torch.cuda.set_device(0)
    res = dict(gpu_before=gpu_info(), method=f"CUDA events over {REPLAYS} graph replays of one batched step after {WARMUP} warm-up "
               "replays; throughput = B * N * H / step time (sample-steps per second)", shapes=[])
    for env_name, Ns, H in SHAPES:
        rows = []
        for B in BATCHES:
            with contextlib.redirect_stdout(io.StringIO()):
                ms = step_time(env_name, Ns, H, B)
            rows.append(dict(B=B, step_ms=ms, sample_steps_per_s=B * Ns * H / (ms * 1e-3)))
            print(env_name, Ns, H, rows[-1], flush=True)
        base = rows[0]["step_ms"]
        for r in rows:
            r["step_ms_vs_B1"] = r["step_ms"] / base
            r["throughput_vs_B1"] = r["B"] * base / r["step_ms"]
        res["shapes"].append(dict(env=env_name, N=Ns, H=H, rows=rows))
    res["end_to_end"] = end_to_end()
    print(res["end_to_end"], flush=True)
    res["gpu_after"] = gpu_info()
    with open(out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
