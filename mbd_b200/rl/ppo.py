"""PPO (Brax's `brax.training.agents.ppo.train`, v0.10.x line **[brax-recalled]**) on the device vector env.

Acting is one CUDA launch per env step (`mbd_ppo_act`, csrc/ppo.cuh) followed by the two launches of the vector env's step; the
observation statistics and GAE are device kernels too (`mbd_ppo_obs_stats`, `mbd_ppo_gae`).  The networks, the PPO loss and Adam are
torch fp32.  One unroll (T x (act + env step)) and one SGD minibatch step (gather, forward, GAE, loss, backward, Adam) are each a
CUDA graph; every key of a run is computed on the host up front (`key_chain`) and read on the device through counters, so between
two evaluations the host only replays graphs and launches the statistics and the minibatch permutations.

Step accounting as Brax: env_steps_per_training_step = batch_size * num_minibatches * unroll_length; U = batch_size * num_minibatches
/ num_envs unrolls per training step; num_evals_after_init = max(num_evals - 1, 1); training steps per epoch =
ceil(num_timesteps / (num_evals_after_init * env_steps_per_training_step)).  Declared deviations: the initial parameters (networks.py),
the float64 observation statistics, and the permutation's two sort rounds at every size (JAX takes one round below 1626 trajectories).
"""
from __future__ import annotations

import ctypes
import dataclasses
import math
from typing import Callable, Optional

import numpy as np
import torch

from .. import _lib, ops, prng
from ..envs import get_env
from ..prng import fold_in
from . import common
from . import networks as nets
from .common import _i32, check_randomization, dr_keys  # noqa: F401  (ppo.check_randomization and ppo.dr_keys are public)


# ---- step accounting and the key chain (host only) -------------------------------------------------------------------------------
@dataclasses.dataclass
class Counts:
    U: int                       # unrolls per training step
    env_steps_per_training_step: int
    num_evals_after_init: int
    steps_per_epoch: int         # training steps between two evaluations


def counts(num_timesteps: int, num_envs: int, batch_size: int, num_minibatches: int, unroll_length: int, num_evals: int) -> Counts:
    if (batch_size * num_minibatches) % num_envs:
        raise ValueError("batch_size * num_minibatches must be a multiple of num_envs")
    per_step = batch_size * num_minibatches * unroll_length
    after = max(num_evals - 1, 1)
    return Counts(batch_size * num_minibatches // num_envs, per_step, after, int(math.ceil(num_timesteps / (after * per_step))))


@dataclasses.dataclass
class Keys:
    policy: np.ndarray           # init keys of the two networks
    value: np.ndarray
    env: np.ndarray              # [num_envs, 2] reset keys of the training envs
    act: np.ndarray              # [steps, U * T, 2] act keys of every training step
    perm: np.ndarray             # [steps, E + 1, 2, 2] two sort-round keys of every epoch's permutation (row 0 unused)
    loss: np.ndarray             # [steps, E * num_minibatches, 2]
    eval_reset: np.ndarray       # [num_evals_after_init + 1, num_eval_envs, 2]
    eval_act: np.ndarray         # [num_evals_after_init + 1, episode_length, 2]


def key_chain(seed: int, c: Counts, num_envs: int, unroll_length: int, num_updates_per_batch: int, num_minibatches: int,
              num_eval_envs: int, episode_length: int) -> Keys:
    """ppo.train's keys: PRNGKey(seed) -> global, local; local = fold_in(local, 0); local, key_env, eval_key = split(local, 3);
    policy, value = split(global).  Per epoch `epoch_key, local = split(local)` and key = split(epoch_key, 1)[0]; per training step
    `key_sgd, key_unroll, key = split(key, 3)`; per unroll `cur, next = split(k)` and per unroll step `act, next = split(cur)`; per
    SGD epoch `key, key_perm, key_grad = split(key, 3)`, the permutation's rounds `k, sub = split(k)` and per minibatch
    `k, key_loss = split(k)`.  The evaluator's keys are common.eval_keys of eval_key."""
    T, U, E = unroll_length, c.U, num_updates_per_batch
    gk, lk = prng.split(prng.PRNGKey(seed))
    lk = fold_in(lk, 0)
    lk, key_env, eval_key = prng.split(lk, 3)
    kp, kv = prng.split(gk)
    steps = c.num_evals_after_init * c.steps_per_epoch
    act = np.zeros((steps, U * T, 2), np.uint32)
    perm = np.zeros((steps, E + 1, 2, 2), np.uint32)
    loss = np.zeros((steps, E * num_minibatches, 2), np.uint32)
    s = 0
    for _ in range(c.num_evals_after_init):
        epoch_key, lk = prng.split2(lk)
        key = prng.split(epoch_key, 1)[0]
        for _ in range(c.steps_per_epoch):
            key_sgd, key_unroll, key = prng.split(key, 3)
            ku = key_unroll
            for u in range(U):
                cur, ku = prng.split2(ku)
                for t in range(T):
                    act[s, u * T + t], cur = prng.split2(cur)
            ks = key_sgd
            for e in range(E):
                ks, kperm, kgrad = prng.split(ks, 3)
                for r in range(2):
                    kperm, perm[s, e + 1, r] = prng.split2(kperm)
                for m in range(num_minibatches):
                    kgrad, loss[s, e * num_minibatches + m] = prng.split2(kgrad)
            s += 1
    eval_reset, eval_act = common.eval_keys(eval_key, c.num_evals_after_init + 1, num_eval_envs, episode_length)
    return Keys(kp, kv, prng.split(key_env, num_envs), act, perm, loss, eval_reset, eval_act)


# ---- acting ------------------------------------------------------------------------------------------------------------------------
class Actor(common.Actor):
    """PPO's stochastic policy on a VecEnv (common.Actor): one mbd_ppo_act launch per act()."""
    EVAL, EVAL_RECORD = _lib.PPO_EVAL, _lib.PPO_EVAL_RECORD

    def _plan(self, B):
        return _lib.PpoPlan(slots=1)

    def _launch(self, mode):
        ops.ppo_act(self.plan, mode)


# ---- the trainer -------------------------------------------------------------------------------------------------------------------
class PPOTrainer(common.Trainer):
    actor_cls = Actor

    def __init__(self, env, num_timesteps: int, episode_length: int, num_envs: int, num_eval_envs: int, learning_rate: float,
                 entropy_cost: float, discounting: float, seed: int, unroll_length: int, batch_size: int, num_minibatches: int,
                 num_updates_per_batch: int, num_evals: int, normalize_observations: bool, reward_scaling: float,
                 clipping_epsilon: float, gae_lambda: float, device=None, randomization: Optional[dict] = None):
        super().__init__(env, episode_length, num_envs, seed, device, randomization)
        if batch_size > _lib.PPO_MAX_MB:
            raise ValueError(f"batch_size (trajectories per minibatch) must be at most {_lib.PPO_MAX_MB}")
        self.c = c = counts(num_timesteps, num_envs, batch_size, num_minibatches, unroll_length, num_evals)
        self.T, self.U, self.mb, self.nmb, self.E = unroll_length, c.U, batch_size, num_minibatches, num_updates_per_batch
        self.entropy_cost, self.clip = entropy_cost, clipping_epsilon
        self.normalize_observations = normalize_observations
        self.keys = key_chain(seed, c, num_envs, unroll_length, num_updates_per_batch, num_minibatches, num_eval_envs, episode_length)
        with torch.cuda.device(self.dev):
            self._setup(num_eval_envs, learning_rate, discounting, reward_scaling, gae_lambda)

    def _setup(self, num_eval_envs, learning_rate, discounting, reward_scaling, gae_lambda):
        d, B, T, U, mb = self.dev, self.B, self.T, self.U, self.mb
        self._make_envs(num_eval_envs)
        O, nu = self.O, self.nu
        self.psizes, self.vsizes = nets.policy_sizes(O, nu), nets.value_sizes(O)
        self.Np = nets.num_params(self.psizes)
        K = self.keys
        flat = np.concatenate([nets.init_params(K.policy, self.psizes), nets.init_params(K.value, self.vsizes)])
        self.theta = torch.from_numpy(flat).to(d).requires_grad_(True)
        self.theta.grad = torch.zeros_like(self.theta)
        self.opt = torch.optim.Adam([self.theta], lr=learning_rate, capturable=True)
        S = U * T
        f32 = dict(device=d, dtype=torch.float32)
        self.obs = torch.zeros((S + 1, B, O), **f32)
        self.raw = torch.zeros((S, B, nu), **f32)
        self.logp, self.reward, self.disc, self.trunc = (torch.zeros((S, B), **f32) for _ in range(4))
        self.mean, self.std = torch.zeros(O, **f32), torch.ones(O, **f32)
        self.stat = torch.zeros(1 + 2 * O, device=d, dtype=torch.float64)
        self.stat_scratch = torch.zeros(((S * B + _lib.PPO_STAT_ROWS - 1) // _lib.PPO_STAT_ROWS) * 2 * O, device=d, dtype=torch.float64)
        self.act_keys = _i32(K.act.reshape(-1, 2), d)
        self.act_ctl = torch.zeros(4, device=d, dtype=torch.int32)
        self.loss_keys = _i32(K.loss.reshape(-1, 2), d)
        self.mb_ctl = torch.zeros(2, device=d, dtype=torch.int32)     # {perm row, loss key row}
        self.perm = torch.zeros(((self.E + 1) * U * B,), device=d, dtype=torch.int32)
        self.perm2d = self.perm.view(-1, mb)
        self.sel = torch.zeros((1, mb), device=d, dtype=torch.int32)
        self.tau = torch.arange(T + 1, device=d, dtype=torch.int64)
        self.vs, self.adv = torch.zeros((T, mb), **f32), torch.zeros((T, mb), **f32)
        self.ent_eps = torch.zeros((T, mb, nu), **f32)
        nbytes = ctypes.c_size_t(0)
        _lib.check(_lib.lib().mbd_mnist_batch_indices(None, self.E + 1, U * B, U * B, None, None, ctypes.byref(nbytes), None),
                   "mbd_mnist_batch_indices")
        self.perm_scratch = torch.empty(int(nbytes.value), device=d, dtype=torch.uint8)
        self.perm_bytes = nbytes
        P = common.acting_plan(_lib.PpoPlan(), self.venv, self.theta, self.mean, self.std, self.act_keys, self.act_ctl)
        P.slots, P.unroll, P.mb = S, T, mb
        P.reward_scaling, P.discount, P.gae_lambda = reward_scaling, discounting, gae_lambda
        P.loss_key_rows = self.loss_keys.shape[0]
        P.obs_dev, P.raw_dev, P.logp_dev = self.obs.data_ptr(), self.raw.data_ptr(), self.logp.data_ptr()
        P.reward_dev, P.disc_dev, P.trunc_dev = self.reward.data_ptr(), self.disc.data_ptr(), self.trunc.data_ptr()
        P.stat_dev, P.stat_scratch_dev = self.stat.data_ptr(), self.stat_scratch.data_ptr()
        P.loss_keys_dev, P.loss_ctl_dev = self.loss_keys.data_ptr(), self.mb_ctl.data_ptr() + 4
        P.traj_dev, P.vs_dev, P.adv_dev, P.ent_eps_dev = self.sel.data_ptr(), self.vs.data_ptr(), self.adv.data_ptr(), self.ent_eps.data_ptr()
        self.plan = P
        self._finish_setup(self.theta.detach()[:self.Np])
        self._unroll_graph = self._sgd_graph = None

    # -- the pieces ------------------------------------------------------------------------------------------------------------------
    def unroll(self):
        """T x (act, env step): one of Brax's generate_unroll calls"""
        for _ in range(self.T):
            ops.ppo_act(self.plan, _lib.PPO_ACT)
            ops.vec_step(self.venv.plan, self.venv.dr)

    def sgd_step(self):
        """one minibatch: gather (outside autograd), forward, GAE, loss, backward, Adam"""
        T, B, O, nu, mb = self.T, self.B, self.O, self.nu, self.mb
        with torch.no_grad():
            torch.index_select(self.perm2d, 0, self.mb_ctl[0:1], out=self.sel)
            n = self.sel[0].long()
            u = torch.div(n, B, rounding_mode="floor")
            rows = (u * T).unsqueeze(0) + self.tau.unsqueeze(1)
            rows = rows * B + (n - u * B).unsqueeze(0)                        # [T + 1, mb] flat (slot, env) rows
            obs = self.obs.view(-1, O).index_select(0, rows.reshape(-1)).view(T + 1, mb, O)
            ra = rows[:T].reshape(-1)
            raw = self.raw.view(-1, nu).index_select(0, ra).view(T, mb, nu)
            blp = self.logp.view(-1).index_select(0, ra).view(T, mb)
        x = nets.normalize(obs, self.mean, self.std)
        logits = nets.mlp(x[:T].reshape(-1, O), nets.unflatten(self.theta[:self.Np], self.psizes)).view(T, mb, 2 * nu)
        values = nets.mlp(x.reshape(-1, O), nets.unflatten(self.theta[self.Np:], self.vsizes)).view(T + 1, mb)
        vd = values.detach()
        self.plan.values_dev = vd.data_ptr()
        ops.ppo_gae(self.plan)
        rho = torch.exp(nets.log_prob(logits, raw) - blp)
        adv = self.adv
        policy_loss = -torch.mean(torch.minimum(rho * adv, torch.clamp(rho, 1 - self.clip, 1 + self.clip) * adv))
        err = self.vs - values[:T]
        v_loss = torch.mean(err * err) * 0.5 * 0.5
        ent = torch.mean(nets.entropy(logits, self.ent_eps))
        loss = policy_loss + v_loss - self.entropy_cost * ent
        self.theta.grad.zero_()
        loss.backward()
        self.opt.step()
        with torch.no_grad():
            self.mb_ctl.add_(1)

    def _permutations(self):
        sub = np.ascontiguousarray(self.keys.perm[self.step_index], np.uint32)
        n = self.U * self.B
        _lib.check(_lib.lib().mbd_mnist_batch_indices(sub.ctypes.data_as(_lib.c_u32p), self.E + 1, n, n, ctypes.c_void_p(self.perm.data_ptr()),
                                                      ctypes.c_void_p(self.perm_scratch.data_ptr()), ctypes.byref(self.perm_bytes),
                                                      ops._stream()), "mbd_mnist_batch_indices")

    def _capture_training(self):
        """captures the unroll and the SGD minibatch step as CUDA graphs.  The SGD step is warmed up on a side stream first and every
        state it touched is restored, so capturing changes no result."""
        self._unroll_graph = common.graph(self.unroll)
        self._warm_up(self.sgd_step, (self.theta, self.mb_ctl, self.vs, self.adv, self.ent_eps, self.sel),
                      lambda: [*self.opt.state[self.theta].values(), self.theta.grad])
        self._sgd_graph = common.graph(self.sgd_step)

    def training_step(self):
        """Brax's training_step: U unrolls, the record of the last step, the statistics, E epochs of minibatch steps"""
        if self.step_index >= self.keys.act.shape[0]:
            raise RuntimeError("every training step of the key chain has run")
        with torch.cuda.device(self.dev):
            for _ in range(self.U):
                self._unroll_graph.replay() if self._unroll_graph is not None else self.unroll()
            ops.ppo_act(self.plan, _lib.PPO_RECORD)
            if self.normalize_observations:
                ops.ppo_obs_stats(self.plan)
            self._permutations()
            self.mb_ctl[0:1].fill_(self.nmb)
            for _ in range(self.E * self.nmb):
                self._sgd_graph.replay() if self._sgd_graph is not None else self.sgd_step()
        self.step_index += 1

    def params(self) -> dict:
        th = self.theta.detach().cpu().numpy()
        return dict(policy=th[:self.Np].copy(), value=th[self.Np:].copy(), mean=self.mean.cpu().numpy(), std=self.std.cpu().numpy(),
                    stat=self.stat.cpu().numpy())


def train(environment, num_timesteps: int, episode_length: int, action_repeat: int = 1, num_envs: int = 1,
          max_devices_per_host: Optional[int] = None, num_eval_envs: int = 128, learning_rate: float = 1e-4,
          entropy_cost: float = 1e-4, discounting: float = 0.9, seed: int = 0, unroll_length: int = 10, batch_size: int = 32,
          num_minibatches: int = 16, num_updates_per_batch: int = 2, num_evals: int = 1, num_resets_per_eval: int = 0,
          normalize_observations: bool = False, reward_scaling: float = 1.0, clipping_epsilon: float = 0.3, gae_lambda: float = 0.95,
          deterministic_eval: bool = False, normalize_advantage: bool = True,
          progress_fn: Callable[[int, dict], None] = lambda *a: None, capture: bool = True, randomization: Optional[dict] = None):
    """ppo.train with Brax's signature and defaults for the arguments the reference passes.  Returns (make_inference_fn, params,
    metrics): make_inference_fn(params) gives an `Actor` factory for a VecEnv; params is a dict of numpy arrays (policy, value, the
    observation statistics).  randomization = dict(friction_range=(lo, hi), gear_range=(lo, hi)) trains with domain randomisation
    (DESIGN.md §5n): every episode of every training env draws its own model factors; the evaluation envs stay nominal."""
    if action_repeat != 1:
        raise NotImplementedError("action_repeat != 1 is not built (the vector env steps once per action)")
    if num_resets_per_eval != 0:
        raise NotImplementedError("num_resets_per_eval > 0 is not built")
    if deterministic_eval or not normalize_advantage:
        raise NotImplementedError("only the stochastic evaluation and normalised advantages of the reference's configs are built")
    env = get_env(environment) if isinstance(environment, str) else environment
    tr = PPOTrainer(env, num_timesteps, episode_length, num_envs, num_eval_envs, learning_rate, entropy_cost, discounting, seed,
                    unroll_length, batch_size, num_minibatches, num_updates_per_batch, num_evals, normalize_observations,
                    reward_scaling, clipping_epsilon, gae_lambda, randomization=randomization)
    return common.run_training(tr, num_evals, progress_fn, capture)
