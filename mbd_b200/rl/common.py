"""What the PPO and SAC trainers share: the acting actor's key-table protocol, the acting fields of their plans, Brax's Evaluator
(its keys, the evaluation loop and its graph), the trainer's set-up around the algorithm, the warm-up before a torch update is
captured, the outer training loop, and the host side of domain randomisation (DESIGN.md §5n).

`ppo.py` and `sac.py` supply what differs: the plan type and launch of their actor, their key chains, buffers and plans, and the
pieces of a training step.
"""
from __future__ import annotations

import time
from typing import Callable, Optional

import numpy as np
import torch

from .. import _lib, ops, prng
from ..envs.base import PipelineEnv
from ..envs.vec import VecEnv, dr_range


def _i32(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a, np.uint32).view(np.int32)).to(dev)


def dr_keys(seed: int, num_envs: int) -> np.ndarray:
    """[num_envs, 2] the DR keys of the training envs (DESIGN.md §5n): split(PRNGKey(2^33 | seed), num_envs).  The root [2, seed]
    differs from the trainer's [0, seed] and from the controllers' member keys [1, seed], so no chain shares a key with them."""
    if not 0 <= int(seed) < 1 << 32:
        raise ValueError(f"domain randomisation needs a seed in 0 .. 2^32 - 1 (got {seed})")
    return prng.split(prng.PRNGKey((2 << 32) | int(seed)), num_envs)


def check_randomization(randomization: Optional[dict], env) -> Optional[tuple]:
    """the trainers' `randomization` argument checked on the host: None, or dict(friction_range=(lo, hi), gear_range=(lo, hi)) on an
    xpbd env (either range may be omitted: (1, 1)).  Returns None or (friction_range, gear_range) as float32 pairs."""
    if randomization is None:
        return None
    if not isinstance(randomization, dict) or set(randomization) - {"friction_range", "gear_range"}:
        raise ValueError(f"randomization must be None or dict(friction_range=(lo, hi), gear_range=(lo, hi)) (got {randomization!r})")
    if not isinstance(env, PipelineEnv):
        raise ValueError(f"domain randomisation exists for the positional (xpbd) envs only, not {type(env).__name__}")
    r = dr_range(randomization.get("friction_range", (1.0, 1.0)), randomization.get("gear_range", (1.0, 1.0)))
    return (r[0], r[1]), (r[2], r[3])


def eval_keys(eval_key, n_eval: int, num_eval_envs: int, episode_length: int):
    """the Evaluator's keys, (eval_reset [n_eval, num_eval_envs, 2], eval_act [n_eval, episode_length, 2]): per evaluation
    `eval_key, unroll_key = split(eval_key)`, reset keys split(unroll_key, num_eval_envs) and act keys from unroll_key as an unroll"""
    eval_reset = np.zeros((n_eval, num_eval_envs, 2), np.uint32)
    eval_act = np.zeros((n_eval, episode_length, 2), np.uint32)
    for i in range(n_eval):
        eval_key, uk = prng.split2(eval_key)
        eval_reset[i] = prng.split(uk, num_eval_envs)
        cur = uk
        for t in range(episode_length):
            eval_act[i, t], cur = prng.split2(cur)
    return eval_reset, eval_act


def acting_plan(P, venv: VecEnv, policy: torch.Tensor, mean: torch.Tensor, std: torch.Tensor, keys: torch.Tensor, ctl: torch.Tensor):
    """fills the acting fields a PpoPlan and a SacPlan share (the sizes, the policy and its statistics, the act key table and its
    control block, the VecEnv's buffers) and returns P"""
    P.B, P.O, P.nu, P.act_key_rows = venv.num_envs, venv.spec.obs_size, venv.spec.nu, keys.shape[0]
    P.policy_dev, P.mean_dev, P.std_dev = policy.data_ptr(), mean.data_ptr(), std.data_ptr()
    P.act_keys_dev, P.act_ctl_dev = keys.data_ptr(), ctl.data_ptr()
    P.env_obs_dev, P.env_reward_dev, P.env_done_dev = venv.obs.data_ptr(), venv.reward.data_ptr(), venv.done.data_ptr()
    P.env_trunc_dev, P.env_actions_dev = venv.truncation.data_ptr(), venv.actions.data_ptr()
    return P


def graph(step: Callable[[], None]) -> torch.cuda.CUDAGraph:
    """`step` captured as a CUDA graph"""
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    return g


# ---- acting ------------------------------------------------------------------------------------------------------------------------
class Actor:
    """The stochastic policy on a VecEnv: `act(key)` writes tanh(raw) for every env into the VecEnv's actions (one acting launch,
    make_inference_fn(params)(obs, key) of Brax); start_eval / finish_eval accumulate the return of every env's first episode.
    policy: flat fp32 cuda tensor; mean / std: [O] cuda tensors.  A subclass names its plan (`_plan(B)`: the empty plan with its
    size field set), its launch (`_launch(mode)` on self.plan) and its two evaluation modes (EVAL, EVAL_RECORD)."""

    def __init__(self, venv: VecEnv, policy: torch.Tensor, mean: torch.Tensor, std: torch.Tensor, keys: Optional[torch.Tensor] = None):
        d = venv.device
        self.own_key = keys is None       # no table: every act() is given its key
        self.venv, self.keys = venv, (torch.zeros((1, 2), device=d, dtype=torch.int32) if keys is None else keys)
        self.ctl = torch.zeros(4, device=d, dtype=torch.int32)
        self.ret, self.active = torch.zeros(venv.num_envs, device=d), torch.ones(venv.num_envs, device=d)
        self.policy, self.mean, self.std = policy, mean, std
        P = acting_plan(self._plan(venv.num_envs), venv, policy, mean, std, self.keys, self.ctl)
        P.ret_dev, P.active_dev = self.ret.data_ptr(), self.active.data_ptr()
        self.plan = P

    def start_eval(self):
        """zero the episode returns, mark every env active and restart the key table"""
        self.ret.zero_()
        self.active.fill_(1.0)
        self.ctl.zero_()

    def act(self, key=None):
        """one acting launch; `key` (uint32 [2]) replaces the table with that single key.  An actor built without a key table must be
        given a key at every call (its one-row table is used up by the previous launch)."""
        if key is None and self.own_key:
            raise ValueError("this actor has no key table: pass the key of every act() call")
        if key is not None:
            self.keys[0].copy_(_i32(np.asarray(key).reshape(2), self.keys.device))
            self.ctl.zero_()
        with torch.cuda.device(self.venv.device):
            self._launch(self.EVAL)

    def finish_eval(self) -> torch.Tensor:
        """folds in the last step's reward; returns the episode returns [B]"""
        with torch.cuda.device(self.venv.device):
            self._launch(self.EVAL_RECORD)
        return self.ret


# ---- the trainer -------------------------------------------------------------------------------------------------------------------
class Trainer:
    """The set-up, evaluation and capture both trainers share.  A subclass names its `actor_cls`, builds its key chain (`keys`, with
    the Keys fields env, eval_reset and eval_act) and counts (`c`), and its `_setup` opens with `_make_envs` and ends with
    `_finish_setup`; it supplies `_capture_training`, `training_step` and `params`."""
    actor_cls: type

    def __init__(self, env, episode_length: int, num_envs: int, seed: int, device, randomization: Optional[dict]):
        self.dr = check_randomization(randomization, env)
        _lib.require_gpu()
        self.dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.env, self.B, self.episode_length = env, num_envs, episode_length
        self.dr_keys = dr_keys(seed, num_envs) if self.dr is not None else None

    def _make_envs(self, num_eval_envs: int):
        """the training and evaluation VecEnvs, and the sizes the acting kernels take"""
        d = self.dev
        self.venv = VecEnv(self.env, self.B, self.episode_length, device=d)
        self.evenv = VecEnv(self.env, num_eval_envs, self.episode_length, device=d)
        O, nu = self.venv.spec.obs_size, self.venv.spec.nu
        if O > _lib.PPO_MAX_OBS or nu > _lib.PPO_MAX_NU:
            raise ValueError(f"observation size {O} / action size {nu} above {_lib.PPO_MAX_OBS} / {_lib.PPO_MAX_NU}")
        self.O, self.nu = O, nu

    def _finish_setup(self, policy: torch.Tensor):
        """the evaluator's keys and actor (on `policy`, self.mean and self.std), domain randomisation, the reset of the training envs
        and the counters"""
        K, d = self.keys, self.dev
        self.eval_keys = _i32(K.eval_act.reshape(-1, 2), d)
        self.eval_reset = _i32(K.eval_reset, d)
        self.actor = self.actor_cls(self.evenv, policy, self.mean, self.std, self.eval_keys)
        if self.dr is not None:          # the training envs only: evaluation stays on the nominal model
            self.venv.set_domain_randomization(*self.dr, self.dr_keys)
        self.venv.reset(_i32(K.env, d))
        self.step_index = 0
        self.eval_index = 0
        self._eval_graph = None

    def _warm_up(self, step: Callable[[], None], kept, zeroed: Callable[[], list]):
        """runs `step` twice on a side stream, then restores every tensor of `kept` and zeroes every tensor `zeroed()` returns.
        `zeroed` is called after the warm-up because torch's optimisers create their state at their first step."""
        snap = [t.detach().clone() for t in kept]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                step()
        torch.cuda.current_stream().wait_stream(s)
        with torch.no_grad():
            for t, v in zip(kept, snap):
                t.copy_(v)
            for t in zeroed():
                t.zero_()

    def capture(self):
        """captures the algorithm's training graphs (`_capture_training`) and the evaluation step as CUDA graphs"""
        with torch.cuda.device(self.dev):
            self._capture_training()
            self._eval_graph = graph(self._eval_step)

    def _eval_step(self):
        self.actor.act()
        ops.vec_step(self.evenv.plan)

    def evaluate(self) -> float:
        """Evaluator.run_evaluation: num_eval_envs envs from split(unroll_key, num_eval_envs), episode_length stochastic steps, the
        mean return of every env's first episode (synchronises)"""
        with torch.cuda.device(self.dev):
            self.evenv.reset(self.eval_reset[self.eval_index])
            self.actor.start_eval()
            self.actor.ctl[1:2].fill_(self.eval_index * self.episode_length)
            for _ in range(self.episode_length):
                self._eval_graph.replay() if self._eval_graph is not None else self._eval_step()
            ret = self.actor.finish_eval()
            out = float(ret.mean().item())
        self.eval_index += 1
        return out

    def prefill(self):
        """what runs before the first training step (nothing, unless the algorithm has a replay buffer to fill)"""

    def env_steps(self) -> int:
        """the env steps run so far, as Brax reports them"""
        return self.step_index * self.c.env_steps_per_training_step


def run_training(tr: Trainer, num_evals: int, progress_fn: Callable[[int, dict], None], capture: bool):
    """Brax's outer loop on a built trainer: the capture, the initial evaluation when num_evals > 1, the prefill, then per epoch
    steps_per_epoch training steps, an evaluation and progress_fn(env steps, metrics).  Returns (make_inference_fn, params,
    metrics): make_inference_fn(params) gives a factory of the trainer's Actor for a VecEnv."""
    if capture:
        tr.capture()
    c = tr.c
    metrics = {}
    if num_evals > 1:
        metrics = {"eval/episode_reward": tr.evaluate()}
        progress_fn(0, metrics)
    tr.prefill()
    for _ in range(c.num_evals_after_init):
        t0 = time.perf_counter()
        for _ in range(c.steps_per_epoch):
            tr.training_step()
        torch.cuda.synchronize(tr.dev)
        sps = c.steps_per_epoch * c.env_steps_per_training_step / (time.perf_counter() - t0)
        metrics = {"eval/episode_reward": tr.evaluate(), "training/sps": sps}
        progress_fn(tr.env_steps(), metrics)
    params = tr.params()
    actor_cls = tr.actor_cls          # not the trainer: the factory must not keep its buffers alive

    def make_inference_fn(p):
        def make(venv: VecEnv) -> Actor:
            d = venv.device
            return actor_cls(venv, torch.from_numpy(p["policy"]).to(d), torch.from_numpy(p["mean"]).to(d), torch.from_numpy(p["std"]).to(d))
        return make

    return make_inference_fn, params, metrics
