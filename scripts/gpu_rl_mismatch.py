"""Domain randomisation for the RL baselines (DESIGN.md §5n) on the current GPU: hopper SAC trained on the nominal model and with
domain randomisation over friction [0.5, 1.5] x gear [0.7, 1.3] (same seed, learner and budget), each scored on §5k's 9 plants x
seeds 0..7 by run_mpc's policy row (50 steps from each controller's s_0, act keys split(PRNGKey(3 * 2^32 | seed), 50)), printed
beside §5k's MBD and MPPI columns read from profiles/h100_mismatch.json.  The settings are checked to match: the same shape, and the
zero-action rewards from these s_0 equal §5k's zero row.  The GPU name and power limit are read in the same run.
    python scripts/gpu_rl_mismatch.py [out.json] [--num_timesteps N] [--learner torch|fused]   (default profiles/h100_rl_mismatch.json)"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mbd_b200.envs import get_env  # noqa: E402
from mbd_b200.rl import sac  # noqa: E402
from mbd_b200.rl.train_sac import sac_config  # noqa: E402
from mbd_b200.scripts import run_mpc  # noqa: E402
from scripts.gpu_vecenv_timing import gpu_info  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DR = dict(friction_range=(0.5, 1.5), gear_range=(0.7, 1.3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?", default=os.path.join("profiles", "h100_rl_mismatch.json"))
    ap.add_argument("--num_timesteps", type=int, default=None, help="the budget of both arms (default: the reference's 6 553 600)")
    ap.add_argument("--learner", default="fused", choices=sac.LEARNERS)
    a = ap.parse_args()
    with open(os.path.join(ROOT, "profiles", "h100_mismatch.json")) as f:
        ref = json.load(f)["closed_loop_hopper"]
    Nstep, seeds = 50, list(run_mpc.SEEDS)
    assert ref["shape"]["Nstep"] == Nstep and ref["shape"]["seeds"] == seeds, ref["shape"]
    plants = [(p["friction"], p["gear"]) for p in ref["plants"]]
    env = get_env("hopper")
    states0 = run_mpc.initial_states(env, seeds)
    fr = np.repeat([f for f, _ in plants], len(seeds))
    gr = np.repeat([g for _, g in plants], len(seeds))
    zero = run_mpc.zero_action_rewards(env, np.tile(states0, (len(plants), 1)), Nstep, fr, gr).reshape(len(plants), len(seeds))
    zero_gap = float(np.abs(zero.round(5) - np.array(ref["algos"]["zero"]["per_seed"])).max())
    print(f"zero-action rows against §5k's: max |diff| {zero_gap:.2e}", flush=True)
    assert zero_gap <= 1e-5, "the s_0 here are not the controllers' s_0"
    cfg = sac_config("hopper")
    if a.num_timesteps is not None:
        cfg["num_timesteps"] = a.num_timesteps
    out = dict(gpu=gpu_info(), learner=a.learner, num_timesteps=cfg["num_timesteps"], seed=cfg["seed"], randomization=DR,
               shape=dict(Nstep=Nstep, seeds=seeds), plants=ref["plants"], zero_gap=zero_gap, arms={})
    for arm, rnd in (("nominal", None), ("dr", DR)):
        curve = []
        t = time.perf_counter()
        _, params, _ = sac.train(environment=env, learner=a.learner, randomization=rnd,
                                 progress_fn=lambda n, m: curve.append((n, round(m["eval/episode_reward"], 2))), **cfg)
        train_s = time.perf_counter() - t
        rew = np.stack([run_mpc.policy_rewards(env, "sac", params, states0, seeds, Nstep, f, g) for f, g in plants])
        out["arms"][arm] = dict(mean=[round(float(r.mean()), 4) for r in rew], std=[round(float(r.std()), 4) for r in rew],
                                per_seed=rew.round(5).tolist(), train_s=round(train_s, 1), eval_curve=curve)
        print(arm, f"trained in {train_s:.0f} s, last eval {curve[-1][1] if curve else None}", flush=True)
    print(f"{'plant (f, g)':>14} | {'SAC nominal':>16} | {'SAC DR':>16} | {'MBD (§5k)':>16} | {'MPPI (§5k)':>16}")
    for i, (f, g) in enumerate(plants):
        cols = (out["arms"]["nominal"], out["arms"]["dr"], ref["algos"]["mbd"], ref["algos"]["mppi"])
        print(f"{f:>6} , {g:<5} | " + " | ".join(f"{c['mean'][i]:7.3f} ± {c['std'][i]:6.3f}" for c in cols))
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
