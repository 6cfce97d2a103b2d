"""Path-integral baselines (MPPI / CMA-ES / CEM) — drop-in for
upstream mbd/planners/path_integral.py: same `Args`, same recommended-parameter table, same
`run_path_integral(args) -> rew`.  The sample -> rollout -> softmax skeleton reuses the MBD kernels
unchanged (SURVEY section 8f.1); only the update rules differ:
    mppi   mu = einsum(w, Y0s)                                      (path_integral.py:33-36)
    cma-es mu as mppi; sigma = sqrt(einsum(w, (Y0s-mu_0t)^2)).mean() * sigma, floored at 1e-3 (:39-45)
    cem    mu = mean of the 10 best samples, idx = argsort(w)[::-1][:10]  (:48-52, bit-exact index work)
One deviation: the shared statistics kernel keeps MBD's guard `std < 1e-4 -> 1` (mbd_planner.py:112),
which path_integral.py:121 lacks (there a zero std turns every weight into NaN).
Single-GPU (the reference is single-device; mppi alone would shard like MBD).

Two implementations of the same solve:
    run_path_integral        PathIntegralEngine.update_once: the round-1 per-operator kernels driven step by step from the host
                             (CMA-ES reads sigma back every step, CEM selects with torch.sort)
    run_path_integral_batch  BatchedPathIntegralEngine: B problems stepped by ONE three-launch device step
                             (mbd_pi_batch_step_launch) captured in a CUDA graph; sigma stays on the device in fp32
They agree to the statistics' rounding, not bit for bit: the weights come from different softmax reduction orders.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

import mbd_b200
from mbd_b200 import _lib, ops, prng
from mbd_b200.planners.engine import BatchedDiffusionEngine, DiffusionEngine, key_chain, pack_step_params

try:
    from tqdm import tqdm
except Exception:  # noqa: BLE001
    tqdm = None


@dataclass
class Args:
    # exp
    seed: int = 0
    disable_recommended_params: bool = False
    update_method: str = "mppi"  # mppi, cma-es, cem
    # env
    env_name: str = (
        "ant"  # "humanoidstandup", "ant", "halfcheetah", "hopper", "walker2d"
    )
    # diffusion
    Nsample: int = 2048  # number of samples
    Hsample: int = 50  # horizon
    Nrefine: int = 100  # number of repeat steps
    temp_sample: float = 0.1  # temperature for sampling


TEMP_RECOMMEND = {"ant": 0.1, "halfcheetah": 0.4, "hopper": 0.1, "humanoidstandup": 0.1, "humanoidrun": 0.1, "walker2d": 0.1,
                  "pushT": 0.2}
NREFINE_RECOMMEND = {"pushT": 200, "humanoidrun": 300}
NSAMPLE_RECOMMEND = {"humanoidrun": 8192}
HSAMPLE_RECOMMEND = {"pushT": 40}


def apply_recommended_params(args: Args) -> Args:
    """path_integral.py:86-91."""
    if not args.disable_recommended_params:
        args.temp_sample = TEMP_RECOMMEND.get(args.env_name, args.temp_sample)
        args.Nrefine = NREFINE_RECOMMEND.get(args.env_name, args.Nrefine)
        args.Nsample = NSAMPLE_RECOMMEND.get(args.env_name, args.Nsample)
        args.Hsample = HSAMPLE_RECOMMEND.get(args.env_name, args.Hsample)
        print(f"override temp_sample to {args.temp_sample}")
    return args


class PathIntegralEngine(DiffusionEngine):
    """update_once (path_integral.py:111-127) on the device."""

    def __init__(self, env, Nsample, Hsample, temp_sample, state_init, update_method: str):
        super().__init__(env, Nsample, Hsample, temp_sample, False, state_init)
        if self.P != 1:
            raise NotImplementedError("path-integral baselines are single-GPU")
        if update_method not in ("mppi", "cma-es", "cem"):
            raise KeyError(update_method)
        self.update_method = update_method
        self.zeros = torch.zeros(self.HNu, device=self.device)
        self.sq = torch.empty(self.HNu, device=self.device)

    def update_once(self, key, mu_0t: torch.Tensor, sigma: float, out: torch.Tensor):
        """returns (mu_0tm1 [device], sigma [host float], rews.mean() [device scalar])"""
        self.rollout_phase(key, sigma, mu_0t)                       # eps*sigma + mu_0t, clip, eval_us
        ops.softmax_weights(self.rews_local, None, 0, self.n_local, self.temp, 0.0, self.weights, self.scalars, self.logp_scratch)
        if self.update_method == "cem":
            order = torch.sort(self.weights, stable=True).indices   # jnp.argsort (stable, ascending)
            idx = order.flip(0)[:10]                                # [::-1][:10]
            out.copy_(self.Y0s[idx].mean(dim=0))
            return out, sigma, self.scalars[0]
        ops.weighted_sum(self.weights, self.Y0s, self.HNu, self.run_scratch, self.partial)
        ops.update(self.partial, 1, self.HNu, self.zeros, [1.0, 1.0, 1.0, 1.0, 1.0], out)   # out = einsum(w, Y0s) exactly
        if self.update_method == "cma-es":
            ops.weighted_sqerr_sum(self.weights, self.Y0s, mu_0t, self.HNu, self.run_scratch, self.sq)
            sigma = float(torch.sqrt(self.sq).mean().item()) * sigma
            sigma = max(sigma, 1e-3)
        return out, sigma, self.scalars[0]


def run_path_integral(args: Args, log_every: int = 10, return_trajectory: bool = False):
    rng = prng.PRNGKey(seed=args.seed)
    apply_recommended_params(args)
    env = mbd_b200.envs.get_env(args.env_name)
    Nu = env.action_size
    rng, rng_reset = prng.split(rng)  # NOTE: rng_reset should never be changed.
    state_init = env.reset(rng_reset)
    eng = PathIntegralEngine(env, args.Nsample, args.Hsample, args.temp_sample, state_init, args.update_method)
    HNu = args.Hsample * Nu
    mus = torch.zeros((args.Nrefine, HNu), device=eng.device)
    rews = torch.zeros(args.Nrefine, device=eng.device)
    rng_exp, rng = prng.split(rng)
    r = rng_exp
    sigma = 1.0
    steps = range(args.Nrefine - 1, 0, -1)
    pbar = tqdm(steps, desc="Path Integrating") if tqdm is not None else None
    for n_done, t in enumerate(pbar if pbar is not None else steps):
        r, k = prng.split(r)
        _, sigma, rew = eng.update_once(k, mus[t], sigma, mus[t - 1])
        rews[t].copy_(rew, non_blocking=True)
        if pbar is not None and (n_done % log_every == log_every - 1 or t == 1):
            pbar.set_postfix({"rew": f"{rews[t].item():.2e}"})
    mu_0ts = mus[: args.Nrefine - 1].flip(0).reshape(args.Nrefine - 1, args.Hsample, Nu)
    from mbd_b200.planners.mbd_planner import final_reward
    rew_final = final_reward(env, eng, mu_0ts[-1])
    if return_trajectory:
        return rew_final, mu_0ts
    return rew_final


class BatchedPathIntegralEngine(BatchedDiffusionEngine):
    """B independent refinements of one env and shape (N, H, Nrefine, update_method) stepped in lockstep by ONE three-launch
    step (`mbd_pi_batch_step_launch`); the solve-level surface of BatchedDiffusionEngine (load_schedule, set_step, step,
    capture, check_exchange, problem).  Ybars[b] holds problem b's means: row t = mu_0t of step t, row t-1 its result; launch (1)
    reads sigma_t from params[b][t].sigma.  CMA-ES writes sigma' to params[b][t-1].sigma and sigma_hist[b][t-1] on the device.
    Problem b draws the noise of a stand-alone solve with its own key and reduces in the same order, so it reproduces the B = 1
    solve of the same inputs bit for bit.  state_buffer and ensemble: as in BatchedDiffusionEngine (the receding-horizon controller
    of pi_mpc.py passes `VecEnv.state`)."""

    def __init__(self, env, Nsample: int, Hsample: int, temps, state_inits, Nrefine: int, update_method: str,
                 device: Optional[torch.device] = None, state_buffer: Optional[torch.Tensor] = None, ensemble=None):
        if update_method not in _lib.PI_METHODS:
            raise KeyError(update_method)
        super().__init__(env, Nsample, Hsample, temps, False, state_inits, Nrefine, device, state_buffer, ensemble)
        self.update_method = update_method
        self.method = _lib.PI_METHODS[update_method]
        d, f = self.device, dict(device=self.device, dtype=torch.float32)
        nruns = (self.N + ops.RUN - 1) // ops.RUN
        self.sigma_hist = torch.ones((self.B, self.Nd), **f)          # row t = sigma_t (constant 1 for MPPI / CEM)
        self.cma_scratch = torch.empty((self.B, nruns + 1, self.HNu), **f) if update_method == "cma-es" else None
        self.cem_idx = torch.zeros((self.B, _lib.PI_IDX_STRIDE), device=d, dtype=torch.int32) if update_method == "cem" else None
        vp = lambda t: None if t is None else t.data_ptr()   # noqa: E731
        self._bufs = _lib.PiBufs(vp(self.sigma_hist), vp(self.cma_scratch), vp(self.cem_idx))

    def load_schedule(self, keys, sigma0: float = 1.0):
        """uploads every problem's key chain keys[b] [Nrefine, 2] (engine.key_chain); sigma_t = sigma0 in every row
        (path_integral.py:140, sigma = 1.0)"""
        if len(keys) != self.B:
            raise ops.MbdError(f"need {self.B} key chains, one per problem")
        sig = np.full(self.Nd, sigma0, np.float32)
        tab = np.stack([pack_step_params(np.asarray(k, np.uint32), sig, None, None) for k in keys])
        self.params.copy_(torch.from_numpy(tab))
        self.sigma_hist.fill_(float(np.float32(sigma0)))

    def _launch(self, tail_only: bool = False):
        ops.pi_batch_step_launch(self._plan_c, self.B, self.Nd, self.method, self.temps, self._bufs, tail_only)

    def tail_step(self):
        """launches 2 and 3 only (weights + update) on whatever Y0s / rews / Ybars[:, t] / params[:, t] hold (tests)"""
        self._launch(tail_only=True)

    def cem_indices(self, b: int) -> np.ndarray:
        """the rows CEM averaged in the last step of problem b, in rank order"""
        row = self.cem_idx[b].cpu().numpy()
        return row[: int(row[_lib.PI_TOPK])]


# fields every problem of one run_path_integral_batch call must share; seed and temp_sample may differ
PI_BATCH_SHARED_FIELDS = ("env_name", "Nsample", "Hsample", "Nrefine", "update_method")


def check_pi_batch_args(args_list) -> None:
    """The argument checks of run_path_integral_batch, before anything touches the device (recommended parameters already
    applied): ValueError naming the field, KeyError for an unknown update_method (as run_path_integral raises)."""
    if len(args_list) < 1:
        raise ValueError("run_path_integral_batch needs at least one Args")
    for f in PI_BATCH_SHARED_FIELDS:
        vals = [getattr(a, f) for a in args_list]
        if any(v != vals[0] for v in vals):
            raise ValueError(f"run_path_integral_batch: every problem must have the same {f} (got {vals})")
    if args_list[0].update_method not in _lib.PI_METHODS:
        raise KeyError(args_list[0].update_method)
    if args_list[0].Nrefine < 2:
        raise ValueError(f"run_path_integral_batch: Nrefine must be at least 2 (got {args_list[0].Nrefine}); the reference "
                         "would run no step and index an empty trajectory")
    import torch.distributed as dist
    if int(os.environ.get("WORLD_SIZE", "1")) > 1 or (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        raise ValueError("run_path_integral_batch runs on one GPU; it cannot run under WORLD_SIZE > 1")


def run_path_integral_batch(args_list, log_every: int = 10, return_trajectory: bool = False):
    """run_path_integral for B problems of one env and shape at once: ONE three-launch device step advances all of them
    (BatchedPathIntegralEngine).  Each problem's recommended parameters, reset and key chain come from its own Args exactly as
    in run_path_integral.  Returns np.ndarray[B] of rew_final (and with return_trajectory the list of every problem's
    (Nrefine-1, H, Nu) mu trajectory, laid out as run_path_integral returns it).  One GPU only."""
    for a in args_list:
        apply_recommended_params(a)
    check_pi_batch_args(args_list)
    a0 = args_list[0]
    env = mbd_b200.envs.get_env(a0.env_name)
    Nu = env.action_size
    state_inits, keys = [], []
    for a in args_list:
        rng = prng.PRNGKey(seed=a.seed)
        rng, rng_reset = prng.split(rng)  # NOTE: rng_reset should never be changed.
        state_inits.append(env.reset(rng_reset))
        rng_exp, rng = prng.split(rng)
        keys.append(key_chain(rng_exp, a.Nrefine))
    eng = BatchedPathIntegralEngine(env, a0.Nsample, a0.Hsample, [a.temp_sample for a in args_list], state_inits, a0.Nrefine,
                                    a0.update_method)
    eng.load_schedule(keys)
    eng.set_step(a0.Nrefine - 1)
    if os.environ.get("MBD_GRAPH", "1") != "0":
        eng.capture()
    steps = range(a0.Nrefine - 1, 0, -1)
    pbar = tqdm(steps, desc=f"Path Integrating x{eng.B}") if tqdm is not None else None
    for n_done, t in enumerate(pbar if pbar is not None else steps):
        eng.step()
        if pbar is not None and (n_done % log_every == log_every - 1 or t == 1):
            pbar.set_postfix({"rew": f"{eng.rew_hist[:, t].mean().item():.2e}"})   # mean over the problems
            eng.check_exchange()
    eng.check_exchange()
    from mbd_b200.planners.mbd_planner import final_reward
    mu_0ts = [eng.Ybars[b, : a0.Nrefine - 1].flip(0).reshape(a0.Nrefine - 1, a0.Hsample, Nu) for b in range(eng.B)]
    rew_final = np.array([final_reward(env, eng.problem(b), mu_0ts[b][-1]) for b in range(eng.B)])
    if return_trajectory:
        return rew_final, mu_0ts
    return rew_final


if __name__ == "__main__":
    import tyro

    rew = run_path_integral(args=tyro.cli(Args))
    print(f"rew: {rew:.2e}")
