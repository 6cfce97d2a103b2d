"""Seed and temperature sweeps — counterpart of upstream mbd/scripts/run_mbd.py, same `Args` and stdout lines.

    python -m mbd_b200.scripts.run_mbd --algo mbd --mode seed --env_name hopper

algo=mbd runs the eight problems of a sweep as ONE batch (run_diffusion_batch): one three-launch step advances all of them,
and each problem's result equals its stand-alone run_diffusion bit for bit.  The `time:` line then reports the batch's wall
clock divided by the batch size (the problems are not timed one by one).  algo=path_integral calls run_path_integral once per
seed or temperature, as the reference does; with --pi_batch it runs the eight as ONE batch (run_path_integral_batch) and reports
the batch's wall clock divided by B, like algo=mbd.

The path_integral temperature sweep keeps the reference's quirk: it builds Args(seed=0, env_name, temp_sample=t) without
disable_recommended_params and without update_method, so for an env of the recommended-parameter table every problem runs at the
recommended temperature, and every temperature runs MPPI.  The batch builds the same eight Args.
"""
from __future__ import annotations

from dataclasses import dataclass
from time import time

import numpy as np

from mbd_b200.planners import mbd_planner, path_integral

SEEDS = tuple(range(8))
TEMPS = (0.01, 0.03, 0.06, 0.1, 0.2, 0.4, 0.6, 0.8)   # run_mbd.py:43


@dataclass
class Args:
    algo: str = "mbd"  # path_integral, mbd
    update_method: str = "mppi"  # softmax, cma-es, cem
    mode: str = "seed"  # temp
    env_name: str = "ant"
    pi_batch: bool = False  # algo=path_integral: run the sweep as one batch (run_path_integral_batch)


def seed_args(args: Args):
    return [mbd_planner.Args(seed=s, env_name=args.env_name, not_render=True) for s in SEEDS]


def temp_args(args: Args):
    return [mbd_planner.Args(seed=0, env_name=args.env_name, temp_sample=t, not_render=True, disable_recommended_params=True)
            for t in TEMPS]


def pi_seed_args(args: Args):
    return [path_integral.Args(seed=s, env_name=args.env_name, update_method=args.update_method) for s in SEEDS]


def pi_temp_args(args: Args):
    """the reference's quirk: no disable_recommended_params, no update_method (see the module docstring)"""
    return [path_integral.Args(seed=0, env_name=args.env_name, temp_sample=float(t)) for t in TEMPS]


def _run_batch(run, args_list):
    """(rews [B], seconds per problem): the batch's wall clock, synchronised, divided by B"""
    import torch
    t0 = time()
    rews = run(args_list)
    torch.cuda.synchronize()
    return np.asarray(rews), (time() - t0) / len(args_list)


def _run_mbd_batch(args_list):
    return _run_batch(mbd_planner.run_diffusion_batch, args_list)


def run_multiple_seed(args: Args):
    if args.algo == "mbd":
        rews, per = _run_mbd_batch(seed_args(args))
        print(f"rew: {rews.mean():.2f} \\pm {rews.std():.2f}")
        print(f"time: {per:.2f} \\pm {0.0:.2f} (wall clock of one batch of {len(rews)} / {len(rews)})")
        return rews
    if args.algo != "path_integral":
        raise NotImplementedError(args.algo)
    if args.pi_batch:
        rews, per = _run_batch(path_integral.run_path_integral_batch, pi_seed_args(args))
        print(f"rew: {rews.mean():.2f} \\pm {rews.std():.2f}")
        print(f"time: {per:.2f} \\pm {0.0:.2f} (wall clock of one batch of {len(rews)} / {len(rews)})")
        return rews
    rews, times = [], []
    for pa in pi_seed_args(args):
        t0 = time()
        rews.append(path_integral.run_path_integral(pa))
        times.append(time() - t0)
    rews, times = np.array(rews), np.array(times)
    print(f"rew: {rews.mean():.2f} \\pm {rews.std():.2f}")
    print(f"time: {times.mean():.2f} \\pm {times.std():.2f}")
    return rews


def run_multiple_temp(args: Args):
    temps = np.array(TEMPS)
    if args.algo == "mbd":
        rews, _ = _run_mbd_batch(temp_args(args))
    elif args.algo == "path_integral" and args.pi_batch:
        rews, _ = _run_batch(path_integral.run_path_integral_batch, pi_temp_args(args))
    elif args.algo == "path_integral":
        rews = np.array([path_integral.run_path_integral(pa) for pa in pi_temp_args(args)])
    else:
        raise NotImplementedError(args.algo)
    best_temp = temps[np.argmax(rews)]
    print(f"rews: {rews}")
    print(f"best_temp: {best_temp:.2f}")
    return rews


def main(argv=None):
    import tyro
    args = tyro.cli(Args, args=argv)
    if args.mode == "seed":
        return run_multiple_seed(args)
    if args.mode == "temp":
        return run_multiple_temp(args)
    raise ValueError(f"mode must be seed or temp, got {args.mode!r}")


if __name__ == "__main__":
    main()
