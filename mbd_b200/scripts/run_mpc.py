"""Model-based diffusion against the path-integral baselines in closed loop (this project's own comparison: the reference compares
them open loop only, DESIGN.md §5j).

    python -m mbd_b200.scripts.run_mpc --env_name hopper

For each of mbd, mppi, cma-es and cem the eight seeds run as ONE batch of receding-horizon controllers (run_mpc_batch /
run_pi_mpc_batch) at the same Nsample, Hsample, Nwarm and Nstep, the cold solve at Nsolve steps (Ndiffuse = Nrefine) and each
planner's recommended temperature for the env.  `zero` is the plant under zero actions from the same reset states.  Per algorithm
one line: the closed-loop mean reward over the seeds and the wall time of one warm control step of the whole batch.
`--plant_friction` / `--plant_gear` run every algorithm and the zero-action baseline against a plant whose contact friction and
actuator gear are scaled by those factors, while the planners keep the nominal model (DESIGN.md §5k).  `--plan_friction` /
`--plan_gear` (K values each) let every algorithm plan against the ensemble of the K models (DESIGN.md §5l).  `--plan_members K`
with `--plan_friction_range lo hi` / `--plan_gear_range lo hi` draws the K members afresh at every control step instead, and
`--plan_worst m` scores a sample by its m worst members rather than the mean of all K (DESIGN.md §5m).  `--policy PATH` with
`--policy_algo {ppo,sac}` adds a `policy` line: the trained policy of params.npz / params_dr.npz (python -m mbd_b200.rl.train_brax /
train_sac) acting on each seed's s_0 against the same plant for Nstep steps, with act key c = split(PRNGKey(3 * 2^32 | seed),
Nstep)[c] and the controllers' score, the mean reward (DESIGN.md §5n).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

import mbd_b200
from mbd_b200 import prng
from mbd_b200.planners import mbd_mpc, mbd_planner, path_integral, pi_mpc

SEEDS = tuple(range(8))
BASELINES = ("mppi", "cma-es", "cem")


@dataclass
class Args:
    env_name: str = "hopper"
    Nsample: int = 1024  # samples of every planner
    Hsample: int = 50  # horizon
    Nsolve: int = 100  # steps of the cold solve at control step 0 (Ndiffuse of mbd, Nrefine of the baselines)
    Nwarm: int = 10  # steps of every later control step
    Nstep: int = 50  # control steps
    sigma_warm: float = 1.0  # the baselines' sampling sigma at the start of every warm control step
    plant_friction: float = 1.0  # the plant's contact friction over the planners' model (xpbd envs)
    plant_gear: float = 1.0  # the plant's actuator gear over the planners' model (xpbd envs)
    plan_friction: tuple[float, ...] = ()  # the planners' ensemble: member k's friction factor (xpbd envs; empty = nominal)
    plan_gear: tuple[float, ...] = ()  # member k's actuator-gear factor (as many as plan_friction)
    plan_members: int = 0  # members drawn afresh at every control step (excludes plan_friction / plan_gear; 0 = none)
    plan_friction_range: tuple[float, ...] = ()  # (lo, hi) of the drawn members' friction factors
    plan_gear_range: tuple[float, ...] = ()  # (lo, hi) of the drawn members' actuator-gear factors
    plan_worst: int = 0  # score a sample by the mean of its plan_worst worst member returns (0 = the mean of all)
    policy: str = ""  # params.npz of a trained policy: adds the `policy` line (needs policy_algo)
    policy_algo: str = ""  # the algorithm that trained it: ppo or sac


POLICY_ALGOS = ("ppo", "sac")


def check_policy_args(args: Args) -> None:
    """--policy and --policy_algo, checked before anything runs"""
    if args.policy and args.policy_algo not in POLICY_ALGOS:
        raise ValueError(f"--policy needs --policy_algo in {POLICY_ALGOS} (got {args.policy_algo!r})")
    if args.policy_algo and not args.policy:
        raise ValueError("--policy_algo needs --policy")


def policy_keys(seed: int, Nstep: int) -> np.ndarray:
    """[Nstep, 2] the policy row's act keys of `seed` (0 <= seed < 2^32): split(PRNGKey(3 * 2^32 | seed), Nstep).  The root [3, seed]
    differs from the controllers' [0, seed], the member keys' [1, seed] and the trainers' DR keys' [2, seed]."""
    if not 0 <= int(seed) < 1 << 32:
        raise ValueError(f"the policy row needs a seed in 0 .. 2^32 - 1 (got {seed})")
    return prng.split(prng.PRNGKey((3 << 32) | int(seed)), Nstep)


def make_actor(algo: str, params: dict, venv):
    """the stochastic Actor of `algo` (ppo / sac) with a trained policy's params on venv"""
    from mbd_b200.rl import ppo, sac
    d = venv.device
    t = [torch.as_tensor(np.asarray(params[k], np.float32)).to(d) for k in ("policy", "mean", "std")]
    return {"ppo": ppo.Actor, "sac": sac.Actor}[algo](venv, *t)


def policy_rewards(env, algo: str, params: dict, states0: np.ndarray, seeds, Nstep: int, friction=1.0, gear=1.0) -> np.ndarray:
    """[len(seeds)] the policy row: for seed seeds[i], the policy acts on a VecEnv of one env (no episode wrapper) from states0[i]
    against the plant (friction, gear) for Nstep steps with act keys policy_keys(seed, Nstep); the score is the mean reward"""
    from mbd_b200.envs.vec import VecEnv
    out = []
    for i, s in enumerate(seeds):
        venv = VecEnv(env, 1)
        if friction != 1.0 or gear != 1.0:
            venv.set_model_factors(friction=friction, gear=gear)
        venv.set_state(np.asarray(states0[i])[None])
        actor = make_actor(algo, params, venv)
        rews = []
        for key in policy_keys(s, Nstep):
            actor.act(key)
            rews.append(venv.step().reward.clone())
        out.append(torch.cat(rews).cpu().numpy().astype(np.float64).mean())
    return np.array(out)


def initial_states(env, seeds=SEEDS) -> np.ndarray:
    """[len(seeds), S] s_0 of every seed's controller (env.reset(rng_reset) of mbd_mpc.mpc_keys), without running one"""
    from mbd_b200.planners.engine import LaunchInputs
    d = torch.device("cuda", torch.cuda.current_device())
    return np.stack([LaunchInputs.of_env(env, env.reset(mbd_mpc.mpc_keys(s, 1, 1, 1)[0]), False, d).state_init.reshape(-1).cpu().numpy()
                     for s in seeds])


def plan_risk(args: Args) -> dict:
    """the drawn-ensemble and risk-measure fields every algorithm's Args takes as they are"""
    return dict(plan_members=args.plan_members, plan_friction_range=tuple(args.plan_friction_range),
                plan_gear_range=tuple(args.plan_gear_range), plan_worst=args.plan_worst)


def mbd_args(args: Args, seeds=SEEDS):
    temp = mbd_planner.TEMP_RECOMMEND.get(args.env_name, mbd_planner.Args.temp_sample)
    return [mbd_mpc.Args(seed=s, env_name=args.env_name, Nsample=args.Nsample, Hsample=args.Hsample, Ndiffuse=args.Nsolve,
                         Nwarm=args.Nwarm, Nstep=args.Nstep, temp_sample=temp, plant_friction=args.plant_friction,
                         plant_gear=args.plant_gear, plan_friction=tuple(args.plan_friction), plan_gear=tuple(args.plan_gear),
                         **plan_risk(args), not_render=True, disable_recommended_params=True)
            for s in seeds]


def pi_args(args: Args, method: str, seeds=SEEDS):
    temp = path_integral.TEMP_RECOMMEND.get(args.env_name, path_integral.Args.temp_sample)
    return [pi_mpc.Args(seed=s, env_name=args.env_name, update_method=method, Nsample=args.Nsample, Hsample=args.Hsample,
                        Nrefine=args.Nsolve, Nwarm=args.Nwarm, Nstep=args.Nstep, sigma_warm=args.sigma_warm, temp_sample=temp,
                        plant_friction=args.plant_friction, plant_gear=args.plant_gear, plan_friction=tuple(args.plan_friction),
                        plan_gear=tuple(args.plan_gear), **plan_risk(args), not_render=True, disable_recommended_params=True)
            for s in seeds]


def zero_action_rewards(env, states0: np.ndarray, Nstep: int, friction=1.0, gear=1.0) -> np.ndarray:
    """[B] mean reward of Nstep env steps under zero actions from states0 [B, S] (the controller's plant: no episode wrapper, model
    factors friction / gear, scalars or [B])"""
    from mbd_b200.envs.vec import VecEnv
    venv = VecEnv(env, len(states0))
    if np.any(np.asarray(friction) != 1.0) or np.any(np.asarray(gear) != 1.0):
        venv.set_model_factors(friction=friction, gear=gear)
    venv.set_state(states0)
    zeros = torch.zeros_like(venv.actions)
    rews = torch.stack([venv.step(zeros).reward.clone() for _ in range(Nstep)], dim=1)
    return rews.cpu().numpy().astype(np.float64).mean(axis=1)


def run_controllers(algo: str, args: Args, seeds=SEEDS):
    """(MpcResult, seconds per warm control step of the batch) of one algorithm"""
    if algo == "mbd":
        al = mbd_args(args, seeds)
        ctl = mbd_mpc.Controller(mbd_mpc._prepare(al, batch=True), al)
    else:
        al = pi_args(args, algo, seeds)
        ctl = pi_mpc.Controller(pi_mpc._prepare(al, batch=True), al)
    res = ctl.run()
    return res, ctl.warm_seconds / max(args.Nstep - 1, 1)


def main(argv=None):
    import tyro
    args = tyro.cli(Args, args=argv)
    check_policy_args(args)
    params = dict(np.load(args.policy)) if args.policy else None
    out = {}
    for algo in ("mbd",) + BASELINES:
        res, per = run_controllers(algo, args)
        out[algo] = res.reward
        print(f"{algo}: rew: {res.reward.mean():.2f} \\pm {res.reward.std():.2f}  time per control step: {per * 1e3:.2f} ms "
              f"(batch of {len(res.reward)})")
    zero = zero_action_rewards(mbd_b200.envs.get_env(args.env_name), res.states[:, 0], args.Nstep,   # s_0 is every algorithm's
                               args.plant_friction, args.plant_gear)
    out["zero"] = zero
    print(f"zero: rew: {zero.mean():.2f} \\pm {zero.std():.2f}")
    if params is not None:
        pol = policy_rewards(mbd_b200.envs.get_env(args.env_name), args.policy_algo, params, res.states[:, 0], SEEDS, args.Nstep,
                             args.plant_friction, args.plant_gear)
        out["policy"] = pol
        print(f"policy: rew: {pol.mean():.2f} \\pm {pol.std():.2f}")
    return out


if __name__ == "__main__":
    main()
