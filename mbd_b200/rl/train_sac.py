"""python -m mbd_b200.rl.train_sac --env_name hopper — the SAC row of the reference's mbd/rl/train_brax.py.

Trains SAC (mbd_b200.rl.sac) with the reference's hopper hyperparameters and then runs the same tail as train_brax: the
`step: N, episode return: X` lines, `time to jit`, `time to train`, results/{env}/params.npz, the mean reward of 8 episodes of 50
steps and results/{env}/RL.html.  --num_timesteps and --seed override the table for short runs; --learner fused runs the gradient
update as the fused CUDA kernels (sac.FusedLearner) instead of the torch learner; --dr_friction lo hi / --dr_gear lo hi train with
domain randomisation as train_brax's flags do and write params_dr.npz / RL_dr.html.  The PPO envs are trained by
python -m mbd_b200.rl.train_brax.
"""
from __future__ import annotations

import argparse

# the reference's table (mbd/rl/train_brax.py), restated as data
SAC_TABLE = {
    "hopper": dict(num_timesteps=6_553_600, num_evals=20, reward_scaling=30.0, episode_length=1000, normalize_observations=True,
                   action_repeat=1, discounting=0.997, learning_rate=6e-4, num_envs=128, batch_size=512, grad_updates_per_step=64,
                   max_devices_per_host=1, max_replay_size=1048576, min_replay_size=8192, seed=1),
}


def sac_config(env_name: str) -> dict:
    return dict(SAC_TABLE[env_name])


def parse_args(argv=None) -> argparse.Namespace:
    from .train_brax import add_dr_flags
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--env_name", default="hopper")
    ap.add_argument("--num_timesteps", type=int, default=None, help="override the table's num_timesteps")
    ap.add_argument("--seed", type=int, default=None, help="override the table's seed")
    ap.add_argument("--learner", default="torch", choices=("torch", "fused"),
                    help="the gradient update: torch ops (default) or the fused CUDA update")
    add_dr_flags(ap)
    return ap.parse_args(argv)


def main(argv=None):
    a = parse_args(argv)
    if a.env_name not in SAC_TABLE:
        raise SystemExit(f"{a.env_name}: the reference trains it with Brax PPO: run python -m mbd_b200.rl.train_brax --env_name {a.env_name}")

    from ..envs import get_env
    from . import sac
    from .common import check_randomization
    from .train_brax import post_training, progress_printer, randomization

    env = get_env(a.env_name)
    cfg = sac_config(a.env_name)
    if a.num_timesteps is not None:
        cfg["num_timesteps"] = a.num_timesteps
    if a.seed is not None:
        cfg["seed"] = a.seed
    dr = randomization(a)
    check_randomization(dr, env)
    progress, times = progress_printer()
    make_inference_fn, params, _ = sac.train(environment=env, progress_fn=progress, learner=a.learner, randomization=dr, **cfg)
    post_training(a.env_name, env, make_inference_fn, params, times, tag="_dr" if dr else "")


if __name__ == "__main__":
    main()
