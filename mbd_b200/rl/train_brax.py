"""python -m mbd_b200.rl.train_brax --env_name halfcheetah — the counterpart of the reference's mbd/rl/train_brax.py.

Trains PPO (mbd_b200.rl.ppo) with the reference's per-env hyperparameters, prints `step: N, episode return: X` at every evaluation,
`time to jit`, `time to train`, saves the parameters to results/{env}/params.npz (Brax's pickle format is not reproduced), runs the
reference's final evaluation (8 episodes of 50 steps, 40 for pushT, one env, the reference's key chain) and writes results/{env}/RL.html.
Extensions: --num_timesteps and --seed override the table for short runs; --dr_friction lo hi / --dr_gear lo hi train with domain
randomisation (DESIGN.md §5n: every episode of every training env draws its friction and actuator-gear factors from those ranges, an
omitted one is 1 1; evaluation stays on the nominal model) and write params_dr.npz / RL_dr.html instead.  hopper, which the reference trains with SAC, has its own
script (python -m mbd_b200.rl.train_sac --env_name hopper); pusher fails in get_env as in the reference.  ant trains without Brax's
unhealthy termination: the host Ant and the vector env never terminate.
"""
from __future__ import annotations

import argparse
import os

import numpy as np

# the reference's table (mbd/rl/train_brax.py), restated as data; every entry also has normalize_observations=True, action_repeat=1
PPO_TABLE = {
    #                num_timesteps, evals, reward_scaling, episode_length, unroll, minibatches, updates, discounting, lr, entropy, envs, batch, seed
    "ant":             (100_000_000, 10, 10.0, 1000, 5, 32, 4, 0.97, 3e-4, 1e-2, 4096, 2048, 0),
    "walker2d":        (50_000_000, 20, 1.0, 1000, 20, 32, 8, 0.95, 3e-4, 1e-3, 2048, 512, 3),
    "halfcheetah":     (50_000_000, 20, 1.0, 1000, 20, 32, 8, 0.95, 3e-4, 1e-3, 2048, 512, 3),
    "pusher":          (50_000_000, 20, 5.0, 1000, 30, 16, 8, 0.95, 3e-4, 1e-2, 2048, 512, 3),
    "pushT":           (100_000_000, 10, 1.0, 100, 20, 16, 8, 0.99, 3e-4, 1e-2, 2048, 1024, 2),
    "humanoidrun":     (100_000_000, 10, 0.1, 100, 10, 32, 8, 0.97, 3e-4, 1e-3, 2048, 1024, 1),
    "humanoidstandup": (100_000_000, 20, 0.1, 1000, 15, 32, 8, 0.97, 6e-4, 1e-2, 2048, 1024, 1),
}
_FIELDS = ("num_timesteps", "num_evals", "reward_scaling", "episode_length", "unroll_length", "num_minibatches", "num_updates_per_batch",
           "discounting", "learning_rate", "entropy_cost", "num_envs", "batch_size", "seed")
SAC_ENVS = ("hopper",)


def ppo_config(env_name: str) -> dict:
    cfg = dict(zip(_FIELDS, PPO_TABLE[env_name]))
    cfg.update(normalize_observations=True, action_repeat=1)
    return cfg


def add_dr_flags(ap: argparse.ArgumentParser) -> None:
    ap.add_argument("--dr_friction", type=float, nargs=2, default=None, metavar=("LO", "HI"),
                    help="domain randomisation: the range of every training episode's friction factor")
    ap.add_argument("--dr_gear", type=float, nargs=2, default=None, metavar=("LO", "HI"),
                    help="domain randomisation: the range of every training episode's actuator-gear factor")


def randomization(a: argparse.Namespace):
    """the trainers' `randomization` from --dr_friction / --dr_gear (None without either; an omitted one is (1, 1))"""
    if a.dr_friction is None and a.dr_gear is None:
        return None
    return dict(friction_range=tuple(a.dr_friction or (1.0, 1.0)), gear_range=tuple(a.dr_gear or (1.0, 1.0)))


def parse_args(argv=None) -> argparse.Namespace:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--env_name", default="halfcheetah")
    ap.add_argument("--num_timesteps", type=int, default=None, help="override the table's num_timesteps")
    ap.add_argument("--seed", type=int, default=None, help="override the table's seed")
    add_dr_flags(ap)
    return ap.parse_args(argv)


def main(argv=None):
    a = parse_args(argv)
    if a.env_name in SAC_ENVS:
        raise SystemExit(f"{a.env_name}: the reference trains it with Brax SAC, not PPO: run python -m mbd_b200.rl.train_sac --env_name {a.env_name}")

    from ..envs import get_env
    from . import ppo

    env = get_env(a.env_name)       # pusher raises here, as in the reference
    if a.env_name not in PPO_TABLE:
        raise SystemExit(f"no PPO configuration for {a.env_name}")
    cfg = ppo_config(a.env_name)
    if a.num_timesteps is not None:
        cfg["num_timesteps"] = a.num_timesteps
    if a.seed is not None:
        cfg["seed"] = a.seed
    dr = randomization(a)
    ppo.check_randomization(dr, env)
    progress, times = progress_printer()
    make_inference_fn, params, _ = ppo.train(environment=env, progress_fn=progress, randomization=dr, **cfg)
    post_training(a.env_name, env, make_inference_fn, params, times, tag="_dr" if dr else "")


def progress_printer():
    """the reference's progress_fn: prints `step: N, episode return: X` and records the time of every evaluation"""
    from datetime import datetime
    times = [datetime.now()]

    def progress(num_steps, metrics):
        times.append(datetime.now())
        print(f"step: {num_steps}, episode return: {metrics['eval/episode_reward']:.2f}", flush=True)

    return progress, times


def post_training(env_name, env, make_inference_fn, params, times, tag: str = ""):
    """the reference script's tail after training: the times, results/{env}/params{tag}.npz, the mean reward of 8 episodes of 50
    steps (40 for pushT) on one env of the nominal model with the reference's key chain, and results/{env}/RL{tag}.html of one more
    rollout"""
    import torch

    import mbd_b200
    from .. import prng
    from ..envs.vec import VecEnv
    from ..io import brax_json

    rng = prng.PRNGKey(0)
    rng, rng_reset = prng.split2(rng)
    print(f"time to jit: {times[1] - times[0]}")
    print(f"time to train: {times[-1] - times[1]}")

    path = f"{mbd_b200.__path__[0]}/../results/{env_name}"
    os.makedirs(path, exist_ok=True)
    np.savez(f"{path}/params{tag}.npz", **params)

    venv = VecEnv(env, 1)
    actor = make_inference_fn(params)(venv)
    nstep = 40 if env_name == "pushT" else 50
    rew = []
    for _ in range(8):
        rng, rng_i = prng.split2(rng)
        venv.reset(rng_i.reshape(1, 2))
        rews = []
        for _ in range(nstep):
            act_rng, rng = prng.split2(rng)
            actor.act(act_rng)
            venv.step()
            rews.append(float(venv.reward[0].item()))
        rew.append(np.mean(np.float32(rews)))
    rew = np.float32(rew)
    print(f"mean reward: {rew.mean():.2f}, std: {rew.std():.2f}")

    venv.reset(rng_reset.reshape(1, 2))
    rollout = []
    for _ in range(nstep):
        rollout.append(venv.pipeline_state(0))
        act_rng, rng = prng.split2(rng)
        actor.act(act_rng)
        venv.step()
    torch.cuda.synchronize()
    with open(f"{path}/RL{tag}.html", "w") as f:
        f.write(brax_json.render(env.sys, rollout, env.dt))


if __name__ == "__main__":
    main()
