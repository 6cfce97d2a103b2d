"""Model factors of the vector env (DESIGN.md §5k) on the current GPU: what a per-env plant costs, and what a mismatched plant does to
the closed-loop controllers.

  - step: one captured VecEnv step replayed from a CUDA graph without factors (nominal kernels) and with a [B, 2] factor table (the
    per-env-model kernels), for hopper and humanoidrun at B in {1, 256, 4096, 16384}; CUDA events over REPS replays, the two
    alternated and the best of 3 kept for each;
  - closed loop on hopper: mbd, mppi, cma-es, cem (1024 samples x 50, Nsolve 100, Nwarm 10, Nstep 50, seeds 0..7, the planners'
    recommended temperatures) and zero actions, against plants with friction in {0.5, 1.0, 1.5} x gear in {0.7, 1.0, 1.3}; each
    algorithm's 72 problems (9 plants x 8 seeds) run as one batch, the planners keep the nominal model.
The GPU name and power limit are read in the same run.
    python scripts/gpu_mismatch_timing.py [out.json]     (default profiles/h100_mismatch.json)"""
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mbd_b200 import prng  # noqa: E402
from mbd_b200.envs import get_env  # noqa: E402
from mbd_b200.envs.vec import VecEnv  # noqa: E402
from mbd_b200.planners import mbd_mpc, pi_mpc  # noqa: E402
from mbd_b200.scripts import run_mpc  # noqa: E402
from scripts.gpu_vecenv_timing import gpu_info, timed  # noqa: E402

ENVS = ["hopper", "humanoidrun"]
SIZES = [1, 256, 4096, 16384]
FRICTION = [0.5, 1.0, 1.5]
GEAR = [0.7, 1.0, 1.3]


def captured_step(env, B, factors: bool):
    venv = VecEnv(env, B)
    if factors:
        rng = np.random.default_rng(B)
        venv.set_model_factors(friction=rng.uniform(0.5, 1.5, B), gear=rng.uniform(0.7, 1.3, B))
    venv.reset(prng.split(prng.PRNGKey(0), B))
    venv.actions.uniform_(-1, 1)
    venv.step()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        venv.step()
    torch.cuda.current_stream().wait_stream(s)
    return venv, g


def step_rows():
    rows = []
    for name in ENVS:
        env = get_env(name)
        for B in SIZES:
            (v0, g0), (v1, g1) = captured_step(env, B, False), captured_step(env, B, True)
            t0, t1 = [], []
            for _ in range(3):   # alternated, best of 3
                t0.append(timed(g0.replay))
                t1.append(timed(g1.replay))
            row = dict(env=name, B=B, nominal_us=round(min(t0), 2), factors_us=round(min(t1), 2),
                       ratio=round(min(t1) / min(t0), 3))
            print(row, flush=True)
            rows.append(row)
            del v0, v1, g0, g1
    return rows


def closed_loop():
    base = run_mpc.Args(env_name="hopper", Nsample=1024, Hsample=50, Nsolve=100, Nwarm=10, Nstep=50)
    plants = [(f, g) for f in FRICTION for g in GEAR]
    seeds = run_mpc.SEEDS
    out = dict(shape=dict(Nsample=1024, Hsample=50, Nsolve=100, Nwarm=10, Nstep=50, seeds=list(seeds)),
               plants=[dict(friction=f, gear=g) for f, g in plants], algos={})
    states0 = None
    for algo in ("mbd",) + run_mpc.BASELINES:
        al = []
        for f, g in plants:
            a = run_mpc.Args(**{**base.__dict__, "plant_friction": f, "plant_gear": g})
            al += run_mpc.mbd_args(a, seeds) if algo == "mbd" else run_mpc.pi_args(a, algo, seeds)
        mod = mbd_mpc if algo == "mbd" else pi_mpc
        t = time.perf_counter()
        ctl = mod.Controller(mod._prepare(al, batch=True), al)
        res = ctl.run()
        wall = time.perf_counter() - t
        rew = res.reward.reshape(len(plants), len(seeds))
        states0 = res.states[:, 0]
        out["algos"][algo] = dict(mean=[round(float(r.mean()), 4) for r in rew], std=[round(float(r.std()), 4) for r in rew],
                                  per_seed=rew.round(5).tolist(), ms_per_warm_control_step=round(ctl.warm_seconds / 49 * 1e3, 2),
                                  wall_s=round(wall, 1))
        print(algo, out["algos"][algo]["mean"], flush=True)
        del ctl
    fr = np.repeat([f for f, _ in plants], len(seeds))
    gr = np.repeat([g for _, g in plants], len(seeds))
    zero = run_mpc.zero_action_rewards(get_env("hopper"), states0, 50, fr, gr).reshape(len(plants), len(seeds))
    out["algos"]["zero"] = dict(mean=[round(float(r.mean()), 4) for r in zero], std=[round(float(r.std()), 4) for r in zero],
                                per_seed=zero.round(5).tolist())
    print("zero", out["algos"]["zero"]["mean"], flush=True)
    return out


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join("profiles", "h100_mismatch.json")
    res = dict(gpu=gpu_info(), timed="graph-replayed VecEnv step, CUDA events over 50 replays, nominal and factors alternated, "
                                     "best of 3", steps=step_rows())
    res["closed_loop_hopper"] = closed_loop()
    os.makedirs(os.path.dirname(out_path) or ".", exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
