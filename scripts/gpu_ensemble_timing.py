"""Planner ensembles (DESIGN.md §5l) on the current GPU: what planning against K models costs, and what it does in closed loop.

  - step: one graph-replayed batched MBD step (one problem) without an ensemble at N samples, with an ensemble of K in {1, 3, 9}
    members at the same N, and without one at N * K (the same rollout count); hopper at N = 1024, humanoidrun at N = 1024 and 8192.
    CUDA events over REPS replays, the arms alternated and the best of 3 kept for each;
  - closed loop on hopper with the settings of §5k (1024 samples x 50, Nsolve 100, Nwarm 10, Nstep 50, seeds 0..7, the 9 plants
    friction {0.5, 1.0, 1.5} x gear {0.7, 1.0, 1.3}), every algorithm planning three ways: nominal (re-run here), with the gear
    ensemble {(1, 0.7), (1, 1), (1, 1.3)}, and nominal at 3072 samples (the ensemble's rollout budget).
The GPU name and power limit are read in the same run.
    python scripts/gpu_ensemble_timing.py [out.json]     (default profiles/h100_ensemble.json)"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mbd_b200 import prng  # noqa: E402
from mbd_b200.envs import get_env  # noqa: E402
from mbd_b200.planners import mbd_mpc, pi_mpc  # noqa: E402
from mbd_b200.planners.engine import BatchedDiffusionEngine, key_chain, make_schedule  # noqa: E402
from mbd_b200.scripts import run_mpc  # noqa: E402
from scripts.gpu_vecenv_timing import REPS, gpu_info, timed  # noqa: E402

STEP_CASES = [("hopper", 1024), ("humanoidrun", 1024), ("humanoidrun", 8192)]
KS = [1, 3, 9]
H = 50
ND = 3 * (5 + REPS) + 2          # every replay of the three timed rounds runs a real step (the counter never reaches 0)
FRICTION = [0.5, 1.0, 1.5]
GEAR = [0.7, 1.0, 1.3]
GEAR_ENSEMBLE = dict(plan_friction=(1.0, 1.0, 1.0), plan_gear=(0.7, 1.0, 1.3))


def captured_engine(env, N, K=0):
    """a one-problem batched MBD engine (K members with factors in [0.7, 1.3], or none) with one step captured"""
    rng, rng_reset = prng.split(prng.PRNGKey(0))
    ens = None if K == 0 else np.random.default_rng(K).uniform(0.7, 1.3, (1, K, 2)).astype(np.float32)
    e = BatchedDiffusionEngine(env, N, H, [0.1], False, [env.reset(rng_reset)], ND, ensemble=ens)
    _, al, ab, sg = make_schedule(1e-4, 1e-2, ND)
    e.load_schedule([key_chain(prng.split(rng)[0], ND)], [sg], [al], [ab])
    e.set_step(ND - 1)
    e.capture()
    return e


def step_rows():
    rows = []
    for name, N in STEP_CASES:
        env = get_env(name)
        arms = {"nominal": captured_engine(env, N)}
        for K in KS:
            arms[f"ens{K}"] = captured_engine(env, N, K)
            if K > 1:
                arms[f"nominal_x{K}"] = captured_engine(env, N * K)
        t = {k: [] for k in arms}
        for _ in range(3):   # alternated, best of 3
            for k, e in arms.items():
                t[k].append(timed(e.graph.replay))
        for e in arms.values():
            e.check_exchange()
        best = {k: min(v) for k, v in t.items()}
        row = dict(env=name, N=N, H=H, us={k: round(v, 2) for k, v in best.items()},
                   ratio_to_nominal={k: round(v / best["nominal"], 3) for k, v in best.items()})
        print(row, flush=True)
        rows.append(row)
        del arms
    return rows


def dump(res, out_path):
    os.makedirs(os.path.dirname(out_path) or ".", exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1)


def closed_loop(res, out_path):
    """fills res["closed_loop_hopper"], written after every algorithm"""
    base = run_mpc.Args(env_name="hopper", Nsample=1024, Hsample=50, Nsolve=100, Nwarm=10, Nstep=50)
    plants = [(f, g) for f in FRICTION for g in GEAR]
    seeds = run_mpc.SEEDS
    ways = {"nominal": dict(), "gear_ensemble": GEAR_ENSEMBLE, "nominal_3072": dict(Nsample=3072)}
    out = dict(shape=dict(Nsample=1024, Hsample=50, Nsolve=100, Nwarm=10, Nstep=50, seeds=list(seeds)),
               plants=[dict(friction=f, gear=g) for f, g in plants],
               ways=dict(nominal="planner on the nominal model, 1024 samples",
                         gear_ensemble="planner on the members (1, 0.7), (1, 1), (1, 1.3), 1024 samples (3072 rollouts)",
                         nominal_3072="planner on the nominal model, 3072 samples"),
               algos={})
    res["closed_loop_hopper"] = out
    for algo in ("mbd",) + run_mpc.BASELINES:
        out["algos"][algo] = {}
        for way, kw in ways.items():
            al = []
            for f, g in plants:
                a = run_mpc.Args(**{**base.__dict__, "plant_friction": f, "plant_gear": g, **kw})
                al += run_mpc.mbd_args(a, seeds) if algo == "mbd" else run_mpc.pi_args(a, algo, seeds)
            mod = mbd_mpc if algo == "mbd" else pi_mpc
            t = time.perf_counter()
            ctl = mod.Controller(mod._prepare(al, batch=True), al)
            r = ctl.run()
            wall = time.perf_counter() - t
            rew = r.reward.reshape(len(plants), len(seeds))
            out["algos"][algo][way] = dict(mean=[round(float(r.mean()), 4) for r in rew], std=[round(float(r.std()), 4) for r in rew],
                                           per_seed=rew.round(5).tolist(),
                                           ms_per_warm_control_step=round(ctl.warm_seconds / 49 * 1e3, 2), wall_s=round(wall, 1))
            print(algo, way, out["algos"][algo][way]["mean"], out["algos"][algo][way]["ms_per_warm_control_step"], flush=True)
            del ctl
        dump(res, out_path)


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join("profiles", "h100_ensemble.json")
    res = dict(gpu=gpu_info(), timed=f"graph-replayed batched MBD step (B = 1, H = {H}), CUDA events over {REPS} replays, arms "
                                     "alternated, best of 3", steps=step_rows())
    dump(res, out_path)
    closed_loop(res, out_path)
    res["gpu_after"] = gpu_info()
    dump(res, out_path)


if __name__ == "__main__":
    main()
