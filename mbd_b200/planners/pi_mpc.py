"""The path-integral baselines (MPPI, CMA-ES, CEM) as receding-horizon controllers: the closed loop of mbd_mpc.py with the planner
exchanged, so that the diffusion controller has something to be compared with.

The definition is this project's own (DESIGN.md §5j).  Control step 0 is `run_path_integral`'s refinement unchanged (mu = 0,
sigma = 1, steps Nrefine - 1 ... 1), so its plan is `run_path_integral_batch`'s `mu_0ts[-1]` bit for bit.  Every later control step
c warm-starts from the previous plan shifted by one row, `mu_{Nwarm} = shift(P_{c-1})`, and runs steps Nwarm ... 1 of the method's
unchanged update with the keys of `key_chain(rng_c, Nwarm + 1)`, `rng, rng_c = split(rng)` (`mbd_mpc.mpc_keys` with Nrefine in the
place of Ndiffuse).  Execute, shift and the result are mbd_mpc.py's.

The sampling sigma is **reset, not carried**: every control step c >= 1 starts from `sigma_warm`.  MPPI and CEM keep it; CMA-ES
adapts it inside the control step as the reference's update does, and the sigma each control step ends with is logged
(`MpcResult.sigmas`).  A carried CMA-ES sigma would sit at the reference's 1e-3 floor after the first solve and could not re-plan.
With `sigma_warm = 1.0` a warm step is the reference's update verbatim.  `plant_friction` / `plant_gear` give every problem its
own plant, `plan_friction` / `plan_gear` a planner ensemble, `plan_members` with its two ranges members drawn at every control step
and `plan_worst` a worst-m score, as in mbd_mpc.py.

Everything runs on the device: the B loops share one `BatchedPathIntegralEngine` that plans from the state buffer of a `VecEnv`,
`mbd_mpc_pi_advance` executes the plan, re-arms the next control step and resets its sigma rows, and a warm control step (Nwarm
batched baseline steps, ACT, the env step, RECORD) is one captured CUDA graph:

    python -m mbd_b200.planners.pi_mpc --env_name hopper --update_method mppi --Nwarm 10 --Nstep 50
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass

import numpy as np
import torch

import mbd_b200
from mbd_b200 import _lib, ops
from mbd_b200.planners import mbd_mpc, path_integral
from mbd_b200.planners.path_integral import PI_BATCH_SHARED_FIELDS, BatchedPathIntegralEngine, apply_recommended_params


@dataclass
class Args(path_integral.Args):
    not_render: bool = False
    # receding horizon
    Nwarm: int = 10  # refinement steps of every control step after the first (1 <= Nwarm <= Nrefine - 1)
    Nstep: int = 50  # control steps
    sigma_warm: float = 1.0  # the sampling sigma every control step after the first starts from
    # model mismatch (mbd_mpc.Args): the plant's friction and actuator gear over the planner's (xpbd envs; per problem)
    plant_friction: float = 1.0
    plant_gear: float = 1.0
    # planner ensemble (mbd_mpc.Args): member k plans with (plan_friction[k], plan_gear[k]); empty = the nominal model
    plan_friction: tuple[float, ...] = ()
    plan_gear: tuple[float, ...] = ()
    # drawn planner ensemble and its risk measure (mbd_mpc.Args): K = plan_members members drawn at every control step from the
    # two (lo, hi) ranges; plan_worst = m scores a sample by its m worst members (0 = the mean)
    plan_members: int = 0
    plan_friction_range: tuple[float, ...] = ()
    plan_gear_range: tuple[float, ...] = ()
    plan_worst: int = 0


# fields every problem of one run_pi_mpc_batch call must share; seed and temp_sample may differ
PI_MPC_SHARED_FIELDS = PI_BATCH_SHARED_FIELDS + ("Nwarm", "Nstep", "sigma_warm")


def check_args(args_list, batch: bool) -> None:
    """The argument checks of run_pi_mpc / run_pi_mpc_batch, before anything touches the device: ValueError, and KeyError for an
    unknown update_method (as run_path_integral raises).  Expects the recommended parameters already applied."""
    if len(args_list) < 1:
        raise ValueError("run_pi_mpc_batch needs at least one Args")
    for a in args_list:
        if a.update_method not in _lib.PI_METHODS:
            raise KeyError(a.update_method)
        if not 1 <= a.Nwarm <= a.Nrefine - 1:
            raise ValueError(f"Nwarm must be in 1..Nrefine - 1 = {a.Nrefine - 1} (got {a.Nwarm})")
        if a.Nstep < 1:
            raise ValueError(f"Nstep must be at least 1 (got {a.Nstep})")
        if not (math.isfinite(a.sigma_warm) and a.sigma_warm > 0):
            raise ValueError(f"sigma_warm must be finite and above 0 (got {a.sigma_warm})")
        if batch and not a.not_render:
            raise ValueError("run_pi_mpc_batch requires not_render=True (it writes no artefacts)")
    for f in PI_MPC_SHARED_FIELDS:
        vals = [getattr(a, f) for a in args_list]
        if any(v != vals[0] for v in vals):
            raise ValueError(f"run_pi_mpc_batch: every problem must have the same {f} (got {vals})")
    mbd_mpc.check_plant(args_list)
    mbd_mpc.check_plan(args_list)
    import torch.distributed as dist
    if int(os.environ.get("WORLD_SIZE", "1")) > 1 or (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        raise ValueError("the controller runs on one GPU; it cannot run under WORLD_SIZE > 1")


class Controller(mbd_mpc.Controller):
    """mbd_mpc.Controller planning with a path-integral baseline: the same loops around a `BatchedPathIntegralEngine`, with
    `mbd_mpc_pi_advance` in the place of `mbd_mpc_advance`.  `sigmas` [B, Nstep] is the sigma log on the device."""

    steps_field = "Nrefine"

    def __init__(self, env, args_list, host: bool = False):
        self.sigma_warm = float(args_list[0].sigma_warm)
        super().__init__(env, args_list, host)

    def _make_engine(self, colds, state_buffer):
        a0 = self.args[0]
        self.sigmas = torch.zeros((self.B, self.Nstep), device=self.device, dtype=torch.float32)
        e = BatchedPathIntegralEngine(self.env, a0.Nsample, a0.Hsample, [a.temp_sample for a in self.args], self.host_states,
                                      a0.Nrefine, a0.update_method, device=self.device, state_buffer=state_buffer,
                                      ensemble=mbd_mpc.plan_ensemble(self.args), ens_worst=a0.plan_worst)
        e.load_schedule(colds)   # sigma = 1.0 in every row (path_integral.py:140)
        return e

    def _make_plan(self) -> "_lib.MpcPiPlan":
        p = _lib.MpcPiPlan()
        p.base = super()._make_plan()
        p.sigma_warm, p.sigma_log_dev = self.sigma_warm, self.sigmas.data_ptr()
        return p

    def _advance(self, mode: int):
        ops.mpc_pi_advance(self.plan, mode)

    def _sigma_log(self) -> np.ndarray:
        return self.sigmas.cpu().numpy()

    def _host_sigma(self, c: int, more: bool):
        sig = self.engine.params[:, :, 2]          # the sigma word of every row, as int32 bits
        self.sigmas[:, c] = sig[:, 0].view(torch.float32)
        if more:
            sig[:, 0:self.Nwarm + 1] = int(np.float32(self.sigma_warm).view(np.int32))


def _prepare(args_list, batch: bool):
    for a in args_list:
        apply_recommended_params(a)
    check_args(args_list, batch)
    return mbd_b200.envs.get_env(args_list[0].env_name)


def run_pi_mpc_batch(args_list, log_every: int = 10, return_result: bool = False):
    """run_pi_mpc for B closed loops of one env, shape and update_method at once (seed and temp_sample may differ): problem b
    returns run_pi_mpc(args_list[b]) bit for bit.  Returns np.ndarray[B] of closed-loop mean rewards (and with return_result the
    MpcResult, whose `sigmas` [B, Nstep] is the sigma every control step ended with).  Requires not_render=True; one GPU only."""
    env = _prepare(args_list, batch=True)
    res = Controller(env, args_list).run(log_every=log_every)
    return (res.reward, res) if return_result else res.reward


def run_pi_mpc(args: Args, log_every: int = 10, return_result: bool = False):
    """the closed loop of one seed: returns its mean reward over the Nstep control steps (and with return_result the MpcResult of a
    batch of one).  Unless not_render is set it writes results/{env}/mpc_{update_method}.npz (actions, rewards, states, sigmas)
    and the executed rollout (mpc_{update_method}_rollout.html, car2d .png)."""
    env = _prepare([args], batch=False)
    res = Controller(env, [args]).run(log_every=log_every)
    if not args.not_render:
        path = f"{mbd_b200.__path__[0]}/../results/{args.env_name}"
        os.makedirs(path, exist_ok=True)
        np.savez(f"{path}/mpc_{args.update_method}.npz", actions=res.actions[0], rewards=res.rewards[0], states=res.states[0],
                 sigmas=res.sigmas[0])
        mbd_mpc._render(env, res.states[0], path, name=f"mpc_{args.update_method}_rollout")
    rew = float(res.reward[0])
    return (rew, res) if return_result else rew


if __name__ == "__main__":
    import tyro

    rew = run_pi_mpc(args=tyro.cli(Args))
    print(f"closed-loop reward = {rew:.2e}")
