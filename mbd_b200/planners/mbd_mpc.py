"""Model-based diffusion as a receding-horizon controller: plan, execute the plan's first action, shift, plan again.

The reference has no controller; the definition is this project's own (DESIGN.md §5i).  Control step 0 is `run_diffusion`
unchanged (cold start from YN = 0 over all Ndiffuse steps), so its plan is `run_diffusion`'s `Yi[-1]` bit for bit.  Every later
control step c warm-starts from the previous plan shifted by one row, `Ybar_{Nwarm} = shift(P_{c-1})`, and runs diffusion steps
Nwarm ... 1 on the same schedule rows as the Ndiffuse-step solve, with the keys of `key_chain(rng_c, Nwarm + 1)` where
`rng, rng_c = split(rng)`.  The first row of the plan, unclipped, is applied to the plant with `env.step` (no episode wrapper,
`done` ignored).

The plant may differ from the model the planner plans with (DESIGN.md §5k): `plant_friction` and `plant_gear` scale every contact
friction and every actuator gear of the plant of one problem (`envs.vec.scaled_env`), while the planner keeps the nominal model.
The planner may plan against an ensemble of models instead (DESIGN.md §5l): with `plan_friction` / `plan_gear` of length K every
sample is rolled out under the K models (plan_friction[k], plan_gear[k]) and scored by the mean of the K returns.  With
`plan_members = K` the K members are drawn afresh at every control step from `plan_friction_range` x `plan_gear_range` with a key
chain of the problem's own (DESIGN.md §5m, `member_keys`), and `plan_worst = m >= 1` scores a sample by the mean of its m worst
member returns instead of all K (1 = the minimum).

Everything runs on the device: B closed loops (one per seed) share one `BatchedDiffusionEngine` that plans from the state buffer of
a `VecEnv`, and `mbd_mpc_advance` executes the plan and re-arms the next control step.  A warm control step (the member draw when
members are drawn, Nwarm batched diffusion steps, ACT, the env step, RECORD) is one captured CUDA graph:

    python -m mbd_b200.planners.mbd_mpc --env_name hopper --Nwarm 10 --Nstep 50
"""
from __future__ import annotations

import math
import os
import time
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch
import torch.distributed as dist

import mbd_b200
from mbd_b200 import _lib, ops, prng
from mbd_b200.planners import mbd_planner
from mbd_b200.planners.engine import BatchedDiffusionEngine, LaunchInputs, key_chain, make_schedule
from mbd_b200.planners.mbd_planner import BATCH_SHARED_FIELDS, apply_recommended_params

try:  # tqdm is cosmetic
    from tqdm import tqdm
except Exception:  # noqa: BLE001
    tqdm = None


@dataclass
class Args(mbd_planner.Args):
    # receding horizon
    Nwarm: int = 10  # diffusion steps of every control step after the first (1 <= Nwarm <= Ndiffuse - 1)
    Nstep: int = 50  # control steps
    # model mismatch: the plant's friction and actuator gear over the planner's (xpbd envs; per problem)
    plant_friction: float = 1.0
    plant_gear: float = 1.0
    # planner ensemble: member k plans with friction plan_friction[k] and gear plan_gear[k] (xpbd envs; equal lengths K, the same K
    # for every problem of a batch, values per problem); empty = the nominal model
    plan_friction: tuple[float, ...] = ()
    plan_gear: tuple[float, ...] = ()
    # drawn planner ensemble: plan_members = K members drawn afresh at every control step, friction uniform in plan_friction_range
    # and gear uniform in plan_gear_range ((lo, hi) with 0 <= lo <= hi, per problem); 0 = none.  Excludes plan_friction / plan_gear
    plan_members: int = 0
    plan_friction_range: tuple[float, ...] = ()
    plan_gear_range: tuple[float, ...] = ()
    # risk measure of either ensemble: score a sample by the mean of its plan_worst worst member returns (1 .. K); 0 = the mean
    plan_worst: int = 0


# fields every problem of one run_mpc_batch call must share; seed, temp_sample, beta0 and betaT may differ
MPC_SHARED_FIELDS = BATCH_SHARED_FIELDS + ("Nwarm", "Nstep")


def check_args(args_list, batch: bool) -> None:
    """The argument checks of run_mpc / run_mpc_batch, before anything touches the device: raises ValueError.  Expects the
    recommended parameters already applied."""
    if len(args_list) < 1:
        raise ValueError("run_mpc_batch needs at least one Args")
    for a in args_list:
        if a.enable_demo:
            raise ValueError("the controller does not take enable_demo: the demo log-density reads the demonstration from the start "
                             "of the horizon, which a closed loop moves")
        if not 1 <= a.Nwarm <= a.Ndiffuse - 1:
            raise ValueError(f"Nwarm must be in 1..Ndiffuse - 1 = {a.Ndiffuse - 1} (got {a.Nwarm})")
        if a.Nstep < 1:
            raise ValueError(f"Nstep must be at least 1 (got {a.Nstep})")
        if batch and not a.not_render:
            raise ValueError("run_mpc_batch requires not_render=True (it writes no artefacts)")
    for f in MPC_SHARED_FIELDS:
        vals = [getattr(a, f) for a in args_list]
        if any(v != vals[0] for v in vals):
            raise ValueError(f"run_mpc_batch: every problem must have the same {f} (got {vals})")
    check_plant(args_list)
    check_plan(args_list)
    if int(os.environ.get("WORLD_SIZE", "1")) > 1 or (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        raise ValueError("the controller runs on one GPU; it cannot run under WORLD_SIZE > 1")


def check_plant(args_list) -> None:
    """plant_friction / plant_gear: finite and >= 0, and 1 on car2d and pushT (ValueError)"""
    for a in args_list:
        for f in ("plant_friction", "plant_gear"):
            v = getattr(a, f)
            if not (math.isfinite(v) and v >= 0):
                raise ValueError(f"{f} must be finite and >= 0 (got {v})")
            if v != 1.0 and a.env_name in ("car2d", "pushT"):
                raise ValueError(f"{f} != 1: model factors exist for the positional (xpbd) envs only, not {a.env_name}")


def check_plan(args_list) -> None:
    """plan_friction / plan_gear: equal lengths K <= ENS_MAXK, values finite and >= 0.  plan_members: 0 .. ENS_MAXK, not together
    with plan_friction / plan_gear, with both ranges (lo, hi) finite in float32 and 0 <= lo <= hi, and a seed in 0 .. 2^32 - 1;
    ranges without plan_members are refused.  plan_worst: 0 .. K, 0 without an ensemble.  K, plan_worst and whether members are
    drawn are the same for every problem; car2d and pushT plan with the nominal model (ValueError)"""
    ks, worsts, drawn = set(), set(), set()
    for a in args_list:
        fr, gr = tuple(a.plan_friction), tuple(a.plan_gear)
        if len(fr) != len(gr):
            raise ValueError(f"plan_friction and plan_gear must have the same length (got {len(fr)} and {len(gr)})")
        if len(fr) > _lib.ENS_MAXK:
            raise ValueError(f"a planner ensemble has at most {_lib.ENS_MAXK} members (got {len(fr)})")
        for f, vals in (("plan_friction", fr), ("plan_gear", gr)):
            with np.errstate(over="ignore"):
                v32 = np.asarray(vals, dtype=np.float64).astype(np.float32)
            if not (np.isfinite(v32).all() and (v32 >= 0).all()):
                raise ValueError(f"{f} must be finite and >= 0 in float32 (got {vals})")
        M = a.plan_members
        if isinstance(M, bool) or not isinstance(M, (int, np.integer)) or not 0 <= M <= _lib.ENS_MAXK:
            raise ValueError(f"plan_members must be an int in 0 .. {_lib.ENS_MAXK} (got {M!r})")
        if M and fr:
            raise ValueError("plan_members draws the ensemble: it excludes plan_friction / plan_gear")
        for f in ("plan_friction_range", "plan_gear_range"):
            rng = tuple(getattr(a, f))
            if not M:
                if rng:
                    raise ValueError(f"{f} needs plan_members >= 1 (the members it draws)")
                continue
            if len(rng) != 2:
                raise ValueError(f"{f} must be (lo, hi) when plan_members >= 1 (got {rng})")
            with np.errstate(over="ignore"):
                lo, hi = (float(np.float32(v)) for v in rng)
            if not (math.isfinite(lo) and math.isfinite(hi) and 0 <= lo <= hi):
                raise ValueError(f"{f} must be (lo, hi) with 0 <= lo <= hi, finite in float32 (got {rng})")
        if M and not 0 <= a.seed < 1 << 32:
            raise ValueError(f"drawn members need a seed in 0 .. 2^32 - 1 (got {a.seed})")
        K = M or len(fr)
        if K and a.env_name in ("car2d", "pushT"):
            raise ValueError(f"planner ensembles exist for the positional (xpbd) envs only, not {a.env_name}")
        w = a.plan_worst
        if isinstance(w, bool) or not isinstance(w, (int, np.integer)):
            raise ValueError(f"plan_worst must be an int (got {w!r})")
        if w and not K:
            raise ValueError(f"plan_worst = {w} needs a planner ensemble (plan_friction / plan_gear or plan_members)")
        if not 0 <= w <= K:
            raise ValueError(f"plan_worst must be in 0 .. K = {K} (got {w})")
        ks.add(K)
        worsts.add(int(w))
        drawn.add(bool(M))
    if len(ks) > 1:
        raise ValueError(f"every problem of a batch must plan with the same number of ensemble members (got {sorted(ks)})")
    if len(drawn) > 1:
        raise ValueError("every problem of a batch must draw its members (plan_members) or none may")
    if len(worsts) > 1:
        raise ValueError(f"every problem of a batch must plan with the same plan_worst (got {sorted(worsts)})")


def plan_ensemble(args_list):
    """the [B, K, 2] planner ensemble of the problems (member k of problem b = (plan_friction[k], plan_gear[k])), or None when
    they plan with the nominal model.  Drawn members start as the ones of (1, 1): the draw of control step 0 replaces them before
    the first diffusion step."""
    if args_list[0].plan_members:
        return np.ones((len(args_list), args_list[0].plan_members, 2), np.float32)
    if not args_list[0].plan_friction:
        return None
    return np.array([[(f, g) for f, g in zip(a.plan_friction, a.plan_gear)] for a in args_list], dtype=np.float32)


def member_keys(seed: int, Nstep: int) -> np.ndarray:
    """[Nstep, 2] the member key of every control step of the loop of `seed` (0 <= seed < 2^32): split(PRNGKey(2^32 | seed), Nstep).
    The root key [1, seed] differs from the controller's [0, seed] (mpc_keys), so the two chains share no key."""
    return prng.split(prng.PRNGKey((1 << 32) | int(seed)), Nstep)


def draw_members(key, K: int, friction_range, gear_range) -> np.ndarray:
    """[K, 2] the members drawn with one control step's member key: kf, kg = split(key); member k = (uniform(kf, (K,), flo, fhi)[k],
    uniform(kg, (K,), glo, ghi)[k]).  The specification of mbd_ens_draw."""
    kf, kg = prng.split(key)
    f = prng.uniform(kf, (K,), friction_range[0], friction_range[1])
    g = prng.uniform(kg, (K,), gear_range[0], gear_range[1])
    return np.stack([f, g], axis=1).astype(np.float32)


def plant_factors(args_list):
    """([B] friction, [B] gear) of the problems' plants, or None when every plant is the nominal model"""
    fr = [float(a.plant_friction) for a in args_list]
    gr = [float(a.plant_gear) for a in args_list]
    return None if all(v == 1.0 for v in fr + gr) else (fr, gr)


def mpc_keys(seed: int, Ndiffuse: int, Nwarm: int, Nstep: int):
    """(rng_reset, cold [Ndiffuse, 2], warm [Nstep, Nwarm, 2]) of one closed loop.  cold is run_diffusion's key chain; warm[c][j - 1]
    is the key of diffusion step j of control step c >= 1, row j of key_chain(rng_c, Nwarm + 1) with rng, rng_c = split(rng).
    warm[0] is zero (control step 0 is the cold solve)."""
    rng = prng.PRNGKey(seed=seed)
    rng, rng_reset = prng.split(rng)
    rng_exp, rng = prng.split(rng)
    cold = key_chain(rng_exp, Ndiffuse)
    warm = np.zeros((Nstep, Nwarm, 2), np.uint32)
    for c in range(1, Nstep):
        rng, rng_c = prng.split(rng)
        warm[c] = key_chain(rng_c, Nwarm + 1)[1:]
    return rng_reset, cold, warm


def shift(P):
    """the warm start of the next control step: row h takes row h + 1, the last row is 0 (the cold start's prior mean).
    P [..., H, Nu] (numpy or torch)"""
    out = np.zeros_like(P) if isinstance(P, np.ndarray) else torch.zeros_like(P)
    out[..., :-1, :] = P[..., 1:, :]
    return out


@dataclass
class MpcResult:
    actions: np.ndarray     # [B, Nstep, Nu] executed actions a_c
    rewards: np.ndarray     # [B, Nstep] r_c
    states: np.ndarray      # [B, Nstep + 1, S] s_0 ... s_Nstep (the vector env's layout)
    rew_hist: np.ndarray    # [B, Nstep] rews.mean() of every control step's last diffusion step
    sigmas: Optional[np.ndarray] = None   # [B, Nstep] the sampling sigma every control step ended with (pi_mpc only)

    @property
    def reward(self) -> np.ndarray:
        """the closed-loop mean reward of every problem, mean_c r_c"""
        return self.rewards.astype(np.float64).mean(axis=-1)


class Controller:
    """B closed loops of one env and shape.  `run()` replays the captured control step; `run_host_driven()` runs the same
    arithmetic with the host in the loop (eager steps, a device->host synchronisation and a host `env.step` per control step), the
    baseline the graph-replayed loop is measured and tested against.  Each instance runs once.

    The planner is model-based diffusion.  `pi_mpc.Controller` plans with the path-integral baselines instead by overriding what
    differs: `steps_field`, `_make_engine`, `_make_plan`, `_advance` and the two sigma hooks."""

    steps_field = "Ndiffuse"   # the Args field holding the steps of the cold solve

    def __init__(self, env, args_list, host: bool = False):
        a0 = args_list[0]
        self.env, self.args, self.host = env, args_list, bool(host)
        self.B, self.Nd, self.Nwarm, self.Nstep = len(args_list), getattr(a0, self.steps_field), a0.Nwarm, a0.Nstep
        self.H, self.Nu = a0.Hsample, env.action_size
        self.device = d = torch.device("cuda", torch.cuda.current_device())
        self.host_states, colds, warms = [], [], []
        for a in args_list:
            rng_reset, cold, warm = mpc_keys(a.seed, self.Nd, a.Nwarm, a.Nstep)
            self.host_states.append(env.reset(rng_reset))   # NOTE: rng_reset as in run_diffusion
            colds.append(cold), warms.append(warm)
        s0 = torch.stack([LaunchInputs.of_env(env, s, False, d).state_init.reshape(-1) for s in self.host_states]).contiguous()
        self.S = s0.shape[1]
        self.venv = None
        factors = plant_factors(args_list)
        if self.host:
            from mbd_b200.envs.vec import scaled_env
            state_buffer = s0
            # every problem's plant as a host env: the specification of the vector env's per-env model
            self.plants = [env] * self.B if factors is None else [scaled_env(env, fr, gr) for fr, gr in zip(*factors)]
        else:
            from mbd_b200.envs.vec import VecEnv
            self.venv = VecEnv(env, self.B, device=d)
            if self.venv.state.shape[1] != self.S:
                raise ValueError(f"the vector env's state has {self.venv.state.shape[1]} words, the planner's {self.S}")
            if factors is not None:
                self.venv.set_model_factors(friction=factors[0], gear=factors[1])
            self.venv.set_state(s0)
            state_buffer = self.venv.state
        self.engine = self._make_engine(colds, state_buffer)
        self.engine.set_step(self.Nd - 1)
        self.warm_keys = np.stack(warms)                                   # [B, Nstep, Nwarm, 2] uint32
        f = dict(device=d, dtype=torch.float32)
        self.keys = torch.as_tensor(self.warm_keys.view(np.int32), device=d).contiguous()
        self.mpc_ctl = torch.zeros(self.B, device=d, dtype=torch.int32)
        self.actions = torch.zeros((self.B, self.Nstep, self.Nu), **f)
        self.rewards = torch.zeros((self.B, self.Nstep), **f)
        self.states = torch.zeros((self.B, self.Nstep + 1, self.S), **f)
        self.rew_hist = torch.zeros((self.B, self.Nstep), **f)
        self.draws = None      # [B, Nstep, K, 2] the host's drawn members (host-driven loop)
        self.draw_plan = None  # mbd_ens_draw's plan (device loop)
        if a0.plan_members:
            mk = np.stack([member_keys(a.seed, self.Nstep) for a in args_list])                  # [B, Nstep, 2] uint32
            ranges = np.array([tuple(a.plan_friction_range) + tuple(a.plan_gear_range) for a in args_list], np.float32)
            if self.host:
                self.draws = np.stack([np.stack([draw_members(mk[b, c], a0.plan_members, ranges[b, :2], ranges[b, 2:])
                                                 for c in range(self.Nstep)]) for b in range(self.B)])
            else:
                self.member_keys = torch.as_tensor(mk.view(np.int32), device=d).contiguous()
                self.ranges = torch.as_tensor(ranges, device=d).contiguous()
                dp = self.draw_plan = _lib.EnsDrawPlan()
                dp.B, dp.K, dp.Nstep = self.B, a0.plan_members, self.Nstep
                dp.keys_dev, dp.ranges_dev = self.member_keys.data_ptr(), self.ranges.data_ptr()
                dp.mpc_ctl_dev, dp.ens_factors_dev = self.mpc_ctl.data_ptr(), self.engine.ens_factors.data_ptr()
        self.graph = None
        self.warm_seconds = 0.0    # wall time of control steps 1 ... Nstep - 1 of the last run (synchronised at both ends)
        self.plan = self._make_plan() if not self.host else None

    def _make_engine(self, colds, state_buffer):
        """the planner of all B loops, reading its initial states from state_buffer, with the cold solve's schedule loaded"""
        a0, scheds = self.args[0], []
        for a in self.args:
            _, alphas, alphas_bar, sigmas = make_schedule(a.beta0, a.betaT, a.Ndiffuse)
            print(f"init sigma = {sigmas[-1]:.2e}")
            scheds.append((sigmas, alphas, alphas_bar))
        e = BatchedDiffusionEngine(self.env, a0.Nsample, a0.Hsample, [a.temp_sample for a in self.args], False, self.host_states,
                                   a0.Ndiffuse, device=self.device, state_buffer=state_buffer, ensemble=plan_ensemble(self.args),
                                   ens_worst=a0.plan_worst)
        e.load_schedule(colds, [s[0] for s in scheds], [s[1] for s in scheds], [s[2] for s in scheds])
        return e

    def _make_plan(self) -> "_lib.MpcPlan":
        p = _lib.MpcPlan()
        e, v = self.engine, self.venv
        p.B, p.H, p.nu, p.Ndiffuse, p.Nwarm, p.Nstep, p.state_words = self.B, self.H, self.Nu, self.Nd, self.Nwarm, self.Nstep, self.S
        p.params_dev, p.ctl_dev, p.Ybars_dev, p.rew_hist_dev = e.params.data_ptr(), e.ctl.data_ptr(), e.Ybars.data_ptr(), e.rew_hist.data_ptr()
        p.keys_dev, p.mpc_ctl_dev = self.keys.data_ptr(), self.mpc_ctl.data_ptr()
        p.env_actions_dev, p.env_state_dev, p.env_reward_dev = v.actions.data_ptr(), v.state.data_ptr(), v.reward.data_ptr()
        p.actions_dev, p.rewards_dev, p.states_dev = self.actions.data_ptr(), self.rewards.data_ptr(), self.states.data_ptr()
        p.rew_hist_log_dev = self.rew_hist.data_ptr()
        return p

    # ---- the device loop --------------------------------------------------------------------------------------------------
    def _execute(self):
        """ACT, the env step and RECORD: a_c into the plant, s_{c+1} and r_c into the logs, the next control step re-armed"""
        self._advance(_lib.MPC_ACT)
        ops.vec_step(self.venv.plan)
        self._advance(_lib.MPC_RECORD)

    def _advance(self, mode: int):
        ops.mpc_advance(self.plan, mode)

    def _sigma_log(self) -> Optional[np.ndarray]:
        """MpcResult.sigmas: model-based diffusion's sigmas are its schedule's, so it logs none"""
        return None

    def _host_sigma(self, c: int, more: bool):
        """the host-driven loop's share of what ACT does to the sampling sigmas at control step c (nothing for this planner)"""

    def _draw(self):
        """the members of every problem's current control step (mbd_ens_draw), when members are drawn"""
        if self.draw_plan is not None:
            ops.ens_draw(self.draw_plan)

    def _warm_step(self):
        self._draw()
        for _ in range(self.Nwarm):
            self.engine._launch()
        self._execute()

    def control_step(self):
        """one warm control step (one graph replay once `run` has captured it)"""
        if self.graph is not None:
            self.graph.replay()
        else:
            self._warm_step()

    def run(self, log_every: int = 10, graph: Optional[bool] = None) -> MpcResult:
        """the closed loops on the device.  graph None: MBD_GRAPH (default on) decides whether the steps are replayed graphs"""
        if self.host:
            raise ValueError("this controller was built for the host-driven loop")
        graph = os.environ.get("MBD_GRAPH", "1") != "0" if graph is None else graph
        e = self.engine
        with torch.cuda.device(self.device):
            self._draw()                        # control step 0's members, before the cold solve
            if graph:
                e.capture()
            for _ in range(self.Nd - 1):        # control step 0: run_diffusion's solve
                e.step()
            e.graph = None
            self._execute()
            if graph and self.Nstep > 1:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._warm_step()
                self.graph = g
            steps = range(1, self.Nstep)
            pbar = tqdm(steps, desc=f"Controlling x{self.B}") if tqdm is not None else None
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for c in (pbar if pbar is not None else steps):
                self.control_step()
                if pbar is not None and (c % log_every == 0 or c == self.Nstep - 1):
                    pbar.set_postfix({"rew": f"{self.rewards[:, c].mean().item():.2e}"})   # mean over the problems
            torch.cuda.synchronize()
            self.warm_seconds = time.perf_counter() - t0
            e.check_exchange()
            done = self.mpc_ctl.cpu().numpy()
            if not (done == self.Nstep).all():
                raise ops.MbdError(f"control counters {done.tolist()} after {self.Nstep} control steps")
        return self.result()

    def result(self) -> MpcResult:
        n = lambda t: t.detach().cpu().numpy()   # noqa: E731
        return MpcResult(n(self.actions), n(self.rewards), n(self.states), n(self.rew_hist), self._sigma_log())

    # ---- the host-driven loop ---------------------------------------------------------------------------------------------
    def run_host_driven(self) -> MpcResult:
        """the same arithmetic with the host in the loop: eager batched steps, then per control step the plan is copied to the
        host, every plant is stepped by the host `env.step`, and the warm start, keys and step counters are written with torch.  Drawn
        members are drawn on the host (`draw_members`) and written with `set_ensemble` before each control step's diffusion steps"""
        if not self.host:
            raise ValueError("this controller was built for the device loop")
        e, B, Nu, nw, env = self.engine, self.B, self.Nu, self.Nwarm, self.env
        acts = np.zeros((B, self.Nstep, Nu), np.float32)
        rews = np.zeros((B, self.Nstep), np.float32)
        sts = np.zeros((B, self.Nstep + 1, self.S), np.float32)
        rh = np.zeros((B, self.Nstep), np.float32)
        st = list(self.host_states)
        sts[:, 0] = e.state_init.cpu().numpy()
        with torch.cuda.device(self.device):
            for c in range(self.Nstep):
                if c == 1:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                if self.draws is not None:
                    e.set_ensemble(self.draws[:, c])
                for _ in range(self.Nd - 1 if c == 0 else nw):
                    e.step()
                P = e.Ybars[:, 0].reshape(B, self.H, Nu)
                a = P[:, 0].cpu().numpy()
                rh[:, c] = e.rew_hist[:, 1].cpu().numpy()
                for b in range(B):
                    st[b] = self.plants[b].step(st[b], a[b])
                    sts[b, c + 1] = host_raw(env, st[b])
                    rews[b, c] = np.float32(st[b].reward)
                acts[:, c] = a
                self._host_sigma(c, c + 1 < self.Nstep)
                if c + 1 < self.Nstep:
                    e.state_init.copy_(torch.as_tensor(sts[:, c + 1], device=self.device))
                    e.Ybars[:, nw].copy_(shift(P).reshape(B, -1))
                    e.params[:, 1:nw + 1, 0:2].copy_(self.keys[:, c + 1])
                    e.set_step(nw)
            torch.cuda.synchronize()
            self.warm_seconds = time.perf_counter() - t0 if self.Nstep > 1 else 0.0
            e.check_exchange()
        return MpcResult(acts, rews, sts, rh, self._sigma_log())


def host_raw(env, state) -> np.ndarray:
    """the flat float32 state of a host env state in the vector env's layout"""
    ps = state.pipeline_state
    raw = ps if env.kind == "car2d" else ps.raw
    return np.ascontiguousarray(raw, dtype=np.float32).reshape(-1)


def _prepare(args_list, batch: bool):
    for a in args_list:
        apply_recommended_params(a)
    check_args(args_list, batch)
    return mbd_b200.envs.get_env(args_list[0].env_name)


def run_mpc_batch(args_list, log_every: int = 10, return_result: bool = False):
    """run_mpc for B closed loops of one env and shape at once (seed, temp_sample, beta0 and betaT may differ): problem b returns
    run_mpc(args_list[b]) bit for bit.  Returns np.ndarray[B] of closed-loop mean rewards (and with return_result the MpcResult).
    Requires not_render=True; one GPU only."""
    env = _prepare(args_list, batch=True)
    res = Controller(env, args_list).run(log_every=log_every)
    return (res.reward, res) if return_result else res.reward


def run_mpc(args: Args, log_every: int = 10, return_result: bool = False):
    """the closed loop of one seed: returns its mean reward over the Nstep control steps (and with return_result the MpcResult of
    a batch of one).  Unless not_render is set it writes results/{env}/mpc.npz and the executed rollout (mpc_rollout.html, car2d
    mpc_rollout.png)."""
    env = _prepare([args], batch=False)
    res = Controller(env, [args]).run(log_every=log_every)
    if not args.not_render:
        path = f"{mbd_b200.__path__[0]}/../results/{args.env_name}"
        os.makedirs(path, exist_ok=True)
        np.savez(f"{path}/mpc.npz", actions=res.actions[0], rewards=res.rewards[0], states=res.states[0])
        _render(env, res.states[0], path)
    rew = float(res.reward[0])
    return (rew, res) if return_result else rew


def _render(env, states: np.ndarray, path: str, name: str = "mpc_rollout"):
    """the executed states s_0 ... s_Nstep: the Brax-visualizer page {name}.html (positional envs, pushT) or car2d's plot {name}.png"""
    if env.kind == "car2d":
        try:
            import matplotlib
            matplotlib.use("Agg")
            from matplotlib import pyplot as plt
        except Exception:  # noqa: BLE001
            return
        fig, ax = plt.subplots(1, 1, figsize=(3, 3))
        env.render(ax, states)
        ax.legend()
        plt.savefig(f"{path}/{name}.png")
        plt.close(fig)
        return
    from ..io import brax_json
    if env.kind == "xpbd":
        rollout = [env._make_pipeline_state(s.reshape(-1, 13)) for s in states]
    else:
        rollout = [env.pipeline_init(s[:8], s[8:]) for s in states]
    with open(f"{path}/{name}.html", "w") as f:
        f.write(brax_json.render(env.sys, rollout, env.dt))


if __name__ == "__main__":
    import tyro

    rew = run_mpc(args=tyro.cli(Args))
    print(f"closed-loop reward = {rew:.2e}")
