"""MBD planner — drop-in for upstream mbd/planners/mbd_planner.py.

Same `Args` fields, same recommended-parameter override, same `run_diffusion(args) -> rew_final`
signature, stdout lines and `results/{env}/mu_0ts.npy` artefact; the jitted `reverse_once` is
replaced by `DiffusionEngine.reverse_once` (hand-written sm_90a CUDA behind the C ABI).
Under torchrun (WORLD_SIZE > 1) the Nsample axis is sharded over ranks.
"""
from __future__ import annotations

import os
from dataclasses import dataclass

import numpy as np
import torch
import torch.distributed as dist

import mbd_b200
from mbd_b200 import ops, prng
from mbd_b200.planners.engine import BatchedDiffusionEngine, DiffusionEngine, key_chain, make_schedule

## load config
@dataclass
class Args:
    # exp
    seed: int = 0
    disable_recommended_params: bool = False
    not_render: bool = False
    # env
    env_name: str = (
        "ant"  # "humanoidstandup", "ant", "halfcheetah", "hopper", "walker2d", "car2d"
    )
    # diffusion
    Nsample: int = 2048  # number of samples
    Hsample: int = 50  # horizon
    Ndiffuse: int = 100  # number of diffusion steps
    temp_sample: float = 0.1  # temperature for sampling
    beta0: float = 1e-4  # initial beta
    betaT: float = 1e-2  # final beta
    enable_demo: bool = False


# recommended parameters (mbd_planner.py:45-63)
TEMP_RECOMMEND = {"ant": 0.1, "halfcheetah": 0.4, "hopper": 0.1, "humanoidstandup": 0.1, "humanoidrun": 0.1, "walker2d": 0.1,
                  "pushT": 0.2}
NDIFFUSE_RECOMMEND = {"pushT": 200, "humanoidrun": 300}
NSAMPLE_RECOMMEND = {"humanoidrun": 8192}
HSAMPLE_RECOMMEND = {"pushT": 40}


def apply_recommended_params(args: Args) -> Args:
    """mbd_planner.py:64-69 — mutates args in place exactly like the reference."""
    if not args.disable_recommended_params:
        args.temp_sample = TEMP_RECOMMEND.get(args.env_name, args.temp_sample)
        args.Ndiffuse = NDIFFUSE_RECOMMEND.get(args.env_name, args.Ndiffuse)
        args.Nsample = NSAMPLE_RECOMMEND.get(args.env_name, args.Nsample)
        args.Hsample = HSAMPLE_RECOMMEND.get(args.env_name, args.Hsample)
        if _is_main():   # one line per job, as in the single-process reference (every rank of a torchrun job runs this)
            print(f"override temp_sample to {args.temp_sample}")
    return args


def _is_main() -> bool:
    return not (dist.is_available() and dist.is_initialized()) or dist.get_rank() == 0


def run_diffusion(args: Args, log_every: int = 10, return_trajectory: bool = False):
    rng = prng.PRNGKey(seed=args.seed)

    ## setup env
    apply_recommended_params(args)
    env = mbd_b200.envs.get_env(args.env_name)
    Nu = env.action_size

    rng, rng_reset = prng.split(rng)  # NOTE: rng_reset should never be changed.
    state_init = env.reset(rng_reset)

    ## run diffusion
    betas, alphas, alphas_bar, sigmas = make_schedule(args.beta0, args.betaT, args.Ndiffuse)
    if _is_main():
        print(f"init sigma = {sigmas[-1]:.2e}")

    engine = DiffusionEngine(env, args.Nsample, args.Hsample, args.temp_sample, args.enable_demo, state_init, Ndiffuse=args.Ndiffuse)
    # Everything the loop of mbd_planner.py:138-148 feeds into reverse_once is uploaded ONCE: the Y0s_rng chain
    # (rng, Y0s_rng = split(rng) per step, :103), sigmas[i] and the schedule scalars.  engine.Ybars row N-1 = YN = 0 and
    # row i-1 receives Ybar_{i-1}; one step is captured in a CUDA graph and replayed, nothing is copied to the host inside
    # the loop.
    rng_exp, rng = prng.split(rng)
    engine.load_schedule(key_chain(rng_exp, args.Ndiffuse), sigmas, alphas, alphas_bar)

    def log(i):
        # the reference formats rew every step (a device->host sync each step, mbd_planner.py:147);
        # here the sync is paid every `log_every` steps only
        rew = f"{engine.rew_hist[i].item():.2e}"
        engine.check_exchange()
        return {"rew": rew}
    engine.solve(log if _is_main() else None, log_every, "Diffusing" if _is_main() else None)
    Ybars = engine.Ybars
    Yi = Ybars[: args.Ndiffuse - 1].flip(0).reshape(args.Ndiffuse - 1, args.Hsample, Nu)  # jnp.array(Ybars) order

    if not args.not_render and _is_main():
        path = f"{mbd_b200.__path__[0]}/../results/{args.env_name}"
        if not os.path.exists(path):
            os.makedirs(path)
        np.save(f"{path}/mu_0ts.npy", Yi.cpu().numpy())
        if args.env_name == "car2d":
            _render_car2d(env, state_init, Yi[-1].cpu().numpy(), args, path)
        elif env.kind in ("xpbd", "pusht"):
            # mbd_planner.py:168-178: rollout.html = brax.io.html.render(sys with opt.timestep = env.dt, rollout).  The same
            # page (and the JSON document inside it, which vis_diffusion.py / brax.io.html.render_from_json consume) is written
            # by mbd_b200.io.brax_json; rollout_states.npz keeps the plain arrays
            from ..io import brax_json
            from ..utils import rollout_states, trajectory_arrays
            rollout = rollout_states(env.step, state_init, Yi[-1].cpu().numpy())
            with open(f"{path}/rollout.html", "w") as f:
                f.write(brax_json.render(env.sys, rollout, env.dt))
            with open(f"{path}/rollout.json", "w") as f:
                f.write(brax_json.dumps(env.sys, rollout, env.dt))
            np.savez(f"{path}/rollout_states.npz", **trajectory_arrays(env, rollout))
    rew_final = final_reward(env, engine, Yi[-1])
    if return_trajectory:
        return rew_final, Yi
    return rew_final


# fields every problem of one run_diffusion_batch call must share (one env and shape); seed, temp_sample, beta0 and betaT may differ
BATCH_SHARED_FIELDS = ("env_name", "Nsample", "Hsample", "Ndiffuse", "enable_demo")


def check_batch_args(args_list) -> None:
    """The argument checks of run_diffusion_batch, before anything touches the device: raises ValueError naming the field.
    Expects the recommended parameters already applied."""
    if len(args_list) < 1:
        raise ValueError("run_diffusion_batch needs at least one Args")
    for a in args_list:
        if not a.not_render:
            raise ValueError("run_diffusion_batch requires not_render=True (it writes no artefacts)")
    for f in BATCH_SHARED_FIELDS:
        vals = [getattr(a, f) for a in args_list]
        if any(v != vals[0] for v in vals):
            raise ValueError(f"run_diffusion_batch: every problem must have the same {f} (got {vals})")
    if int(os.environ.get("WORLD_SIZE", "1")) > 1 or (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        raise ValueError("run_diffusion_batch runs on one GPU; it cannot run under WORLD_SIZE > 1")


def run_diffusion_batch(args_list, log_every: int = 10, return_trajectory: bool = False):
    """run_diffusion for B problems of one env and shape at once: ONE three-launch step advances all of them
    (BatchedDiffusionEngine).  Each problem's reset, key chain and schedule come from its own Args exactly as in
    run_diffusion, so problem b returns the rew_final of run_diffusion(args_list[b]) bit for bit.  Returns np.ndarray[B] of
    rew_final (and with return_trajectory the list of every problem's Yi).  Requires not_render=True; one GPU only."""
    for a in args_list:
        apply_recommended_params(a)
    check_batch_args(args_list)
    a0 = args_list[0]
    env = mbd_b200.envs.get_env(a0.env_name)
    Nu = env.action_size
    state_inits, keys, scheds = [], [], []
    for a in args_list:
        rng = prng.PRNGKey(seed=a.seed)
        rng, rng_reset = prng.split(rng)  # NOTE: rng_reset should never be changed.
        state_inits.append(env.reset(rng_reset))
        betas, alphas, alphas_bar, sigmas = make_schedule(a.beta0, a.betaT, a.Ndiffuse)
        print(f"init sigma = {sigmas[-1]:.2e}")
        rng_exp, rng = prng.split(rng)
        keys.append(key_chain(rng_exp, a.Ndiffuse))
        scheds.append((sigmas, alphas, alphas_bar))
    engine = BatchedDiffusionEngine(env, a0.Nsample, a0.Hsample, [a.temp_sample for a in args_list], a0.enable_demo, state_inits,
                                    a0.Ndiffuse)
    engine.load_schedule(keys, [s[0] for s in scheds], [s[1] for s in scheds], [s[2] for s in scheds])

    def log(i):
        rew = f"{engine.rew_hist[:, i].mean().item():.2e}"   # mean over the problems
        engine.check_exchange()
        return {"rew": rew}
    engine.solve(log, log_every, f"Diffusing x{engine.B}")
    Yis = [engine.Ybars[b, : a0.Ndiffuse - 1].flip(0).reshape(a0.Ndiffuse - 1, a0.Hsample, Nu) for b in range(engine.B)]
    rew_final = np.array([final_reward(env, engine.problem(b), Yis[b][-1]) for b in range(engine.B)])
    if return_trajectory:
        return rew_final, Yis
    return rew_final


def final_reward(env, engine: DiffusionEngine, us: torch.Tensor) -> float:
    """rollout_us(state_init, Yi[-1])[0].mean()  (mbd_planner.py:179-180) — one n=1 launch."""
    us = us.reshape(1, engine.H, engine.Nu).contiguous()
    if env.kind == "xpbd":
        out = ops.rollout(engine.model, engine.state_init, us)
    elif env.kind == "pusht":
        out = ops.pusht_rollout(engine.params_car, engine.state_init, us)
    else:
        out = ops.car2d_rollout(engine.params_car, engine.state_init, us)
    return float(out["rews"][0].item())


def _render_car2d(env, state_init, us, args, path):
    try:
        import matplotlib
        matplotlib.use("Agg")
        from matplotlib import pyplot as plt
    except Exception:  # noqa: BLE001
        return
    fig, ax = plt.subplots(1, 1, figsize=(3, 3))
    xs = [np.asarray(state_init.pipeline_state)]
    state = state_init
    for t in range(us.shape[0]):
        state = env.step(state, us[t])
        xs.append(np.asarray(state.pipeline_state))
    env.render(ax, np.stack(xs))
    if args.enable_demo:
        ax.plot(env.xref[:, 0], env.xref[:, 1], "g--", label="RRT path")
    ax.legend()
    plt.savefig(f"{path}/rollout.png")


def _maybe_init_distributed():
    if int(os.environ.get("WORLD_SIZE", "1")) > 1 and not dist.is_initialized():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl")


if __name__ == "__main__":
    import tyro

    _maybe_init_distributed()
    rew_final = run_diffusion(args=tyro.cli(Args))
    if _is_main():
        print(f"final reward = {rew_final:.2e}")
