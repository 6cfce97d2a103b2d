"""SAC (Brax's `brax.training.agents.sac.train`, v0.10.x line **[brax-recalled]**) on the device vector env.

Acting is one CUDA launch per env step (`mbd_sac_act`, csrc/sac.cuh) followed by the two launches of the vector env's step, the
replay record (`mbd_sac_record`) and PPO's observation statistics (`mbd_ppo_obs_stats` over the B acting observations).  The replay
buffer is a device ring with Brax's queue semantics, and one `mbd_sac_sample` launch per training step draws the batch of every
gradient update and the noise of its three losses.  The losses and the three Adam optimisers are torch fp32 (`Learner`, the
default) or two CUDA launches per update (`FusedLearner`, learner="fused").  Every key of a run is
computed on the host up front (`key_chain`) and read on the device through counters: a training step is the acting graph, the
sampling graph and 64 replays of the update graph, with no host synchronisation.

Step accounting as Brax: num_prefill_actor_steps = ceil(min_replay_size / num_envs); num_evals_after_init = max(num_evals - 1, 1);
training steps per epoch = ceil((num_timesteps - prefill env steps) / (num_evals_after_init * num_envs)); the reported env-step count
includes the prefill.  Declared deviations: the initial parameters (networks.py), the float64 observation statistics, the Polyak
update as target + tau (q - target) (torch's lerp; Brax writes target (1 - tau) + q tau), and the project's fp32 transcendentals.
"""
from __future__ import annotations

import dataclasses
from typing import Callable, Optional

import numpy as np
import torch
import torch.nn.functional as F

from .. import _lib, ops, prng
from ..envs import get_env
from ..prng import fold_in
from . import common
from . import networks as nets
from .common import _i32, dr_keys  # noqa: F401  (sac.dr_keys is public)

ALPHA_LEARNING_RATE = 3e-4      # Brax's alpha optimiser is adam(3e-4) whatever learning_rate is


# ---- step accounting and the key chain (host only) -------------------------------------------------------------------------------
@dataclasses.dataclass
class Counts:
    prefill_steps: int           # num_prefill_actor_steps
    prefill_env_steps: int
    num_evals_after_init: int
    steps_per_epoch: int         # training steps between two evaluations
    env_steps_per_training_step: int


def counts(num_timesteps: int, num_envs: int, min_replay_size: int, num_evals: int) -> Counts:
    prefill = -(-min_replay_size // num_envs)
    prefill_env = prefill * num_envs
    if num_timesteps < prefill_env:
        raise ValueError("num_timesteps must cover the replay prefill (ceil(min_replay_size / num_envs) * num_envs env steps)")
    after = max(num_evals - 1, 1)
    return Counts(prefill, prefill_env, after, -(-(num_timesteps - prefill_env) // (after * num_envs)), num_envs)


def split_many(keys, num: int) -> np.ndarray:
    """prng.split(k, num) of every row of keys [n, 2] at once: [n, num, 2] (the current threefry layout)"""
    keys = np.ascontiguousarray(keys, np.uint32).reshape(-1, 2)
    k = (keys[:, 0:1], keys[:, 1:2])
    idx = np.arange(num, dtype=np.uint32)[None, :]
    if prng._PARTITIONABLE:
        o0, o1 = prng.threefry2x32(k, np.zeros_like(idx), idx)
        return np.stack([o0, o1], -1).astype(np.uint32)
    o0, o1 = prng.threefry2x32(k, idx, idx + np.uint32(num))      # bits(key, 2 num): blocks (i, i + num)
    return np.concatenate([o0, o1], 1).reshape(-1, num, 2).astype(np.uint32)


@dataclasses.dataclass
class Keys:
    policy: np.ndarray           # init keys of the policy and of the two critics
    q: np.ndarray
    env: np.ndarray              # [num_envs, 2] reset keys of the training envs
    buffer: np.ndarray           # [2] the replay buffer's initial key
    act: np.ndarray              # [prefill_steps + steps, 2] act keys: the prefill steps, then every training step's experience key
    noise: np.ndarray            # [steps, updates, 3, 2] key_alpha, key_critic, key_actor of every update
    eval_reset: np.ndarray       # [num_evals_after_init + 1, num_eval_envs, 2]
    eval_act: np.ndarray         # [num_evals_after_init + 1, episode_length, 2]


def key_chain(seed: int, c: Counts, num_envs: int, updates: int, num_eval_envs: int, episode_length: int) -> Keys:
    """sac.train's keys: PRNGKey(seed) -> global, local; local = fold_in(local, 0); local, rb_key, env_key, eval_key = split(local, 4);
    policy, q = split(global); the buffer key split(rb_key, 1)[0].  Prefill: `prefill_key, local = split(local)`, k = split(prefill_key,
    1)[0], per step `k, next = split(k)` and act with k.  Per epoch `epoch_key, local = split(local)`, k = split(epoch_key, 1)[0]; per
    training step `k, next = split(k)`, `experience_key, training_key = split(k)`; per update `key, key_alpha, key_critic, key_actor =
    split(key, 4)` from training_key.  The evaluator's keys are common.eval_keys of eval_key.  The training steps of all epochs and the update chains run as array
    operations (split_many): a Python loop over the 3.3 M splits of the reference's hopper run takes about a minute."""
    gk, lk = prng.split(prng.PRNGKey(seed))
    lk = fold_in(lk, 0)
    lk, rb_key, env_key, eval_key = prng.split(lk, 4)
    kp, kq = prng.split(gk)
    prefill_key, lk = prng.split2(lk)
    k = prng.split(prefill_key, 1)[0]
    pre = np.zeros((c.prefill_steps, 2), np.uint32)
    for i in range(c.prefill_steps):
        pre[i], k = prng.split2(k)
    E, S = c.num_evals_after_init, c.steps_per_epoch
    k = np.zeros((E, 2), np.uint32)
    for e in range(E):
        epoch_key, lk = prng.split2(lk)
        k[e] = prng.split(epoch_key, 1)[0]
    step = np.zeros((E, S, 2), np.uint32)
    for s in range(S):
        kk = split_many(k, 2)
        step[:, s], k = kk[:, 0], kk[:, 1]
    et = split_many(step.reshape(-1, 2), 2)
    key = et[:, 1]
    noise = np.zeros((E * S, updates, 3, 2), np.uint32)
    for g in range(updates):
        k4 = split_many(key, 4)
        key, noise[:, g] = k4[:, 0], k4[:, 1:]
    eval_reset, eval_act = common.eval_keys(eval_key, E + 1, num_eval_envs, episode_length)
    return Keys(kp, kq, prng.split(env_key, num_envs), prng.split(rb_key, 1)[0], np.concatenate([pre, et[:, 0]]), noise,
                eval_reset, eval_act)


# ---- the learner (torch; runs on any device) --------------------------------------------------------------------------------------
def unpack_rows(rows: torch.Tensor, O: int, nu: int):
    """(obs, action, reward, discount, next_obs, truncation) of replay rows [n, 2 O + Nu + 3] (include/mbd_sac.h)"""
    return (rows[:, :O], rows[:, O:O + nu], rows[:, O + nu], rows[:, O + nu + 1], rows[:, O + nu + 2:2 * O + nu + 2],
            rows[:, 2 * O + nu + 2])


def losses(policy, q, target_q, log_alpha, mean, std, rows, eps, O: int, nu: int, reward_scaling: float, discounting: float):
    """Brax's alpha, critic and actor losses on one batch: eps [3, n, Nu] = the normal noise of key_alpha, key_critic, key_actor.
    Every loss sees the parameters from before the update: the critic and the actor use alpha = exp(old log_alpha), the actor the old
    Q.  The gradient of each loss reaches only its own parameters, so one backward of the sum gives the three gradients."""
    psizes, qsizes = nets.sac_policy_sizes(O, nu), nets.sac_q_sizes(O, nu)
    obs, action, reward, discount, next_obs, trunc = unpack_rows(rows, O, nu)
    x, xn = nets.normalize(obs, mean, std), nets.normalize(next_obs, mean, std)
    players = nets.unflatten(policy, psizes)
    logits = nets.relu_mlp(x, players)
    loc, s = logits.chunk(2, dim=-1)
    scale = F.softplus(s) + nets.MIN_STD
    target_entropy = -0.5 * nu
    raw_a = eps[0] * scale + loc
    lp_a = nets.log_prob(logits, raw_a)
    alpha_loss = torch.mean(torch.exp(log_alpha) * (-lp_a - target_entropy).detach())
    alpha = torch.exp(log_alpha).detach()
    with torch.no_grad():
        ln = nets.relu_mlp(xn, nets.unflatten(policy.detach(), psizes))
        locn, sn = ln.chunk(2, dim=-1)
        raw_c = eps[1] * (F.softplus(sn) + nets.MIN_STD) + locn
        next_v = torch.min(nets.sac_q(nets.sac_q_unflatten(target_q, qsizes), xn, torch.tanh(raw_c)), 0).values - alpha * nets.log_prob(ln, raw_c)
        target = reward * reward_scaling + discount * discounting * next_v
    qv = nets.sac_q(nets.sac_q_unflatten(q, qsizes), x, action)
    err = (qv - target) * (1.0 - trunc)
    critic_loss = 0.5 * torch.mean(err * err)
    raw_p = eps[2] * scale + loc
    qa = nets.sac_q(nets.sac_q_unflatten(q.detach(), qsizes), x, torch.tanh(raw_p))
    actor_loss = torch.mean(alpha * nets.log_prob(logits, raw_p) - torch.min(qa, 0).values)
    return alpha_loss, critic_loss, actor_loss


class Learner:
    """the parameters (policy, Q, target Q, log_alpha: flat fp32 tensors), their three Adam optimisers (capturable) and Brax's
    sgd_step: the three losses with the old parameters, the three Adam steps, then target = lerp(target, new Q, tau)"""

    def __init__(self, policy: np.ndarray, q: np.ndarray, O: int, nu: int, learning_rate: float, reward_scaling: float,
                 discounting: float, tau: float, device):
        d = torch.device(device)
        self.O, self.nu, self.reward_scaling, self.discounting, self.tau = O, nu, reward_scaling, discounting, tau
        self.policy = torch.tensor(np.asarray(policy, np.float32), device=d).requires_grad_(True)    # copies: the caller's arrays stay
        self.q = torch.tensor(np.asarray(q, np.float32), device=d).requires_grad_(True)
        self.target_q = self.q.detach().clone()
        self.log_alpha = torch.zeros(1, device=d, requires_grad=True)
        cap = d.type == "cuda"
        for t in (self.policy, self.q, self.log_alpha):
            t.grad = torch.zeros_like(t)
        self.opt_alpha = torch.optim.Adam([self.log_alpha], lr=ALPHA_LEARNING_RATE, capturable=cap)
        self.opt_q = torch.optim.Adam([self.q], lr=learning_rate, capturable=cap)
        self.opt_policy = torch.optim.Adam([self.policy], lr=learning_rate, capturable=cap)

    def update(self, rows, eps, mean, std):
        la, lc, lp = losses(self.policy, self.q, self.target_q, self.log_alpha, mean, std, rows, eps, self.O, self.nu,
                            self.reward_scaling, self.discounting)
        for t in (self.policy, self.q, self.log_alpha):
            t.grad.zero_()
        (la + lc + lp).backward()
        self.opt_alpha.step()
        self.opt_q.step()
        self.opt_policy.step()
        with torch.no_grad():
            self.target_q.lerp_(self.q, self.tau)

    def state(self):
        return [self.policy, self.q, self.target_q, self.log_alpha] + [s for o in (self.opt_alpha, self.opt_q, self.opt_policy)
                                                                       for st in o.state.values() for s in st.values()]


class FusedLearner:
    """The same sgd_step as `Learner` as two CUDA launches (mbd_sac_update, include/mbd_sac_learn.h): the three losses with the old
    parameters, the three Adam steps and the Polyak step.  The parameters, the Adam moments and the step count live on the device;
    the policy is updated in place, so an acting plan that holds its pointer sees every update.  `bind` points the learner at the
    sampler's batch [updates, batch, row] and noise [3, updates, batch, Nu] buffers, the update counter (int64 [1]) and the
    observation statistics; each `update()` then runs update *upd_ctl and advances it."""

    def __init__(self, policy: np.ndarray, q: np.ndarray, O: int, nu: int, learning_rate: float, reward_scaling: float,
                 discounting: float, tau: float, device, batch_size: int):
        d = torch.device(device)
        if d.type != "cuda":
            raise ValueError("the fused learner runs on a CUDA device")
        if not 1 <= batch_size <= _lib.SAC_LEARN_MAX_BATCH:
            raise ValueError(f"batch_size must be in 1..{_lib.SAC_LEARN_MAX_BATCH}")
        self.O, self.nu, self.batch_size = O, nu, batch_size
        self.learning_rate, self.reward_scaling, self.discounting, self.tau = learning_rate, reward_scaling, discounting, tau
        f32 = dict(device=d, dtype=torch.float32)
        self.policy = torch.tensor(np.asarray(policy, np.float32), device=d)
        self.q = torch.tensor(np.asarray(q, np.float32), device=d)
        self.target_q = self.q.clone()
        self.log_alpha = torch.zeros(1, **f32)
        self.policy_m, self.policy_v = torch.zeros_like(self.policy), torch.zeros_like(self.policy)
        self.q_m, self.q_v = torch.zeros_like(self.q), torch.zeros_like(self.q)
        self.alpha_mv = torch.zeros(2, **f32)
        self.ctl = torch.zeros(2, device=d, dtype=torch.int64)     # Adam step count, ticket
        self.losses = torch.zeros(3, **f32)                         # alpha, critic, actor loss of the last update
        self.scratch = torch.zeros(ops.sac_learn_scratch(O, nu, batch_size), **f32)
        self.plan = None

    def bind(self, batch: torch.Tensor, eps: torch.Tensor, upd_ctl: torch.Tensor, mean: torch.Tensor, std: torch.Tensor):
        G = batch.shape[0]
        if tuple(batch.shape) != (G, self.batch_size, 2 * self.O + self.nu + 3) or tuple(eps.shape) != (3, G, self.batch_size, self.nu):
            raise ValueError("batch must be [updates, batch_size, row] and eps [3, updates, batch_size, nu]")
        if upd_ctl.dtype != torch.int64 or upd_ctl.numel() < 1:
            raise ValueError("upd_ctl must be an int64 tensor")
        self._bound = (batch, eps, upd_ctl, mean, std)      # keeps the buffers alive as long as the plan points at them
        P = _lib.SacLearnPlan()
        P.O, P.nu, P.batch, P.updates = self.O, self.nu, self.batch_size, G
        P.learning_rate, P.reward_scaling, P.discounting, P.tau = self.learning_rate, self.reward_scaling, self.discounting, self.tau
        P.policy_dev, P.q_dev, P.target_q_dev, P.log_alpha_dev = (t.data_ptr() for t in (self.policy, self.q, self.target_q,
                                                                                         self.log_alpha))
        P.policy_m_dev, P.policy_v_dev, P.q_m_dev, P.q_v_dev, P.alpha_mv_dev = (t.data_ptr() for t in (
            self.policy_m, self.policy_v, self.q_m, self.q_v, self.alpha_mv))
        P.ctl_dev, P.mean_dev, P.std_dev = self.ctl.data_ptr(), mean.data_ptr(), std.data_ptr()
        P.batch_dev, P.eps_dev, P.upd_ctl_dev = batch.data_ptr(), eps.data_ptr(), upd_ctl.data_ptr()
        P.scratch_dev, P.scratch_floats, P.losses_dev = self.scratch.data_ptr(), self.scratch.numel(), self.losses.data_ptr()
        self.plan = P

    def update(self):
        if self.plan is None:
            raise RuntimeError("bind the learner to its batch, noise and counter first")
        with torch.cuda.device(self.policy.device):
            ops.sac_update(self.plan)

    def state(self):
        return [self.policy, self.q, self.target_q, self.log_alpha, self.policy_m, self.policy_v, self.q_m, self.q_v, self.alpha_mv,
                self.ctl]


LEARNERS = ("torch", "fused")


# ---- acting ------------------------------------------------------------------------------------------------------------------------
class Actor(common.Actor):
    """SAC's stochastic policy on a VecEnv (common.Actor): one mbd_sac_act launch per act()."""
    EVAL, EVAL_RECORD = _lib.SAC_EVAL, _lib.SAC_EVAL_RECORD

    def _plan(self, B):
        return _lib.SacPlan(capacity=B)

    def _launch(self, mode):
        ops.sac_act(self.plan, mode)


# ---- the trainer -------------------------------------------------------------------------------------------------------------------
class SACTrainer(common.Trainer):
    actor_cls = Actor

    def __init__(self, env, num_timesteps: int, episode_length: int, num_envs: int, num_eval_envs: int, learning_rate: float,
                 discounting: float, seed: int, batch_size: int, num_evals: int, normalize_observations: bool, reward_scaling: float,
                 tau: float, min_replay_size: int, max_replay_size: int, grad_updates_per_step: int, device=None,
                 learner: str = "torch", randomization: Optional[dict] = None):
        if learner not in LEARNERS:
            raise ValueError(f"learner must be one of {LEARNERS}, not {learner!r}")
        super().__init__(env, episode_length, num_envs, seed, device, randomization)
        self.learner_kind = learner
        if not num_envs <= max_replay_size <= _lib.SAC_MAX_CAPACITY:
            raise ValueError(f"max_replay_size must be in num_envs..{_lib.SAC_MAX_CAPACITY}")
        self.c = c = counts(num_timesteps, num_envs, min_replay_size, num_evals)
        self.mb, self.G, self.cap = batch_size, grad_updates_per_step, max_replay_size
        self.normalize_observations = normalize_observations
        self.keys = key_chain(seed, c, num_envs, grad_updates_per_step, num_eval_envs, episode_length)
        with torch.cuda.device(self.dev):
            self._setup(num_eval_envs, learning_rate, discounting, reward_scaling, tau)

    def _setup(self, num_eval_envs, learning_rate, discounting, reward_scaling, tau):
        d, B, G, mb, K = self.dev, self.B, self.G, self.mb, self.keys
        self._make_envs(num_eval_envs)
        O, nu = self.O, self.nu
        self.R = 2 * O + nu + 3
        psizes, qsizes = nets.sac_policy_sizes(O, nu), nets.sac_q_sizes(O, nu)
        if self.learner_kind == "fused":
            self.learner = FusedLearner(nets.init_params(K.policy, psizes), nets.sac_q_init(K.q, qsizes), O, nu, learning_rate,
                                        reward_scaling, discounting, tau, d, mb)
        else:
            self.learner = Learner(nets.init_params(K.policy, psizes), nets.sac_q_init(K.q, qsizes), O, nu, learning_rate,
                                   reward_scaling, discounting, tau, d)
        f32 = dict(device=d, dtype=torch.float32)
        self.mean, self.std = torch.zeros(O, **f32), torch.ones(O, **f32)
        self.stat = torch.zeros(1 + 2 * O, device=d, dtype=torch.float64)
        self.stat_scratch = torch.zeros(((B + _lib.PPO_STAT_ROWS - 1) // _lib.PPO_STAT_ROWS) * 2 * O, device=d, dtype=torch.float64)
        self.stage = torch.zeros((B, O), **f32)
        self.ring = torch.zeros((self.cap, self.R), **f32)
        self.ring_ctl = torch.zeros(4, device=d, dtype=torch.int32)
        self.sample_ctl = torch.zeros(4, device=d, dtype=torch.int32)
        self.sample_ctl[2:4].copy_(_i32(K.buffer, d))
        self.act_keys = _i32(K.act, d)
        self.act_ctl = torch.zeros(4, device=d, dtype=torch.int32)
        self.noise_keys = _i32(K.noise.reshape(-1), d)
        self.idx = torch.zeros(G * mb, device=d, dtype=torch.int32)
        self.batch = torch.zeros((G, mb, self.R), **f32)
        self.eps = torch.zeros((3, G, mb, nu), **f32)
        self.upd_ctl = torch.zeros(1, device=d, dtype=torch.int64)
        if self.learner_kind == "fused":
            self.learner.bind(self.batch, self.eps, self.upd_ctl, self.mean, self.std)
        P = common.acting_plan(_lib.SacPlan(), self.venv, self.learner.policy, self.mean, self.std, self.act_keys, self.act_ctl)
        P.capacity, P.batch, P.updates, P.noise_key_rows = self.cap, mb, G, K.noise.shape[0]
        P.stage_obs_dev, P.ring_dev, P.ring_ctl_dev, P.sample_ctl_dev = (t.data_ptr() for t in (self.stage, self.ring, self.ring_ctl,
                                                                                                  self.sample_ctl))
        P.noise_keys_dev, P.idx_dev, P.batch_dev, P.eps_dev = (t.data_ptr() for t in (self.noise_keys, self.idx, self.batch, self.eps))
        self.plan = P
        S = _lib.PpoPlan()         # running_statistics.update over the B acting observations: PPO's launch with one slot
        S.B, S.O, S.nu, S.slots = B, O, nu, 1
        S.obs_dev, S.stat_dev, S.stat_scratch_dev = self.stage.data_ptr(), self.stat.data_ptr(), self.stat_scratch.data_ptr()
        S.mean_dev, S.std_dev = self.mean.data_ptr(), self.std.data_ptr()
        self.stat_plan = S
        self._finish_setup(self.learner.policy.detach())
        self._act_graph = self._sample_graph = self._sgd_graph = None

    # -- the pieces ------------------------------------------------------------------------------------------------------------------
    def actor_step(self):
        """acting.actor_step + running_statistics.update + insert: act, env step, record, statistics"""
        ops.sac_act(self.plan, _lib.SAC_ACT)
        ops.vec_step(self.venv.plan, self.venv.dr)
        ops.sac_record(self.plan)
        if self.normalize_observations:
            ops.ppo_obs_stats(self.stat_plan)

    def sample(self):
        ops.sac_sample(self.plan)
        self.upd_ctl.zero_()

    def sgd_step(self):
        """update upd_ctl of the training step: its batch and noise, Brax's sgd_step, then upd_ctl += 1"""
        if self.learner_kind == "fused":
            self.learner.update()         # reads the batch and noise at upd_ctl and advances it on the device
            return
        with torch.no_grad():
            rows = torch.index_select(self.batch.view(self.G, -1), 0, self.upd_ctl).view(self.mb, self.R)
            eps = torch.index_select(self.eps.view(3, self.G, -1), 1, self.upd_ctl).view(3, self.mb, self.nu)
        self.learner.update(rows, eps, self.mean, self.std)
        with torch.no_grad():
            self.upd_ctl.add_(1)

    def prefill(self):
        """prefill_replay_buffer: num_prefill_actor_steps acting steps with the initial policy"""
        with torch.cuda.device(self.dev):
            for _ in range(self.c.prefill_steps):
                self._act_graph.replay() if self._act_graph is not None else self.actor_step()

    def _capture_training(self):
        """captures the acting step, the sampling and one update as CUDA graphs.  The torch update is warmed up on a side stream
        first and every state it touched is restored, so capturing changes no result; the fused update is two kernel launches and is
        captured without running."""
        self._act_graph = common.graph(self.actor_step)
        self._sample_graph = common.graph(self.sample)
        if self.learner_kind == "torch":
            L = self.learner              # L.state()[4:]: the optimisers' moments and step counts
            self._warm_up(self.sgd_step, (L.policy, L.q, L.target_q, L.log_alpha, self.upd_ctl),
                          lambda: [*L.state()[4:], L.policy.grad, L.q.grad, L.log_alpha.grad])
        self._sgd_graph = common.graph(self.sgd_step)

    def training_step(self):
        """Brax's training_step: an actor step, the replay sample, grad_updates_per_step updates"""
        if self.step_index >= self.keys.noise.shape[0]:
            raise RuntimeError("every training step of the key chain has run")
        with torch.cuda.device(self.dev):
            self._act_graph.replay() if self._act_graph is not None else self.actor_step()
            self._sample_graph.replay() if self._sample_graph is not None else self.sample()
            for _ in range(self.G):
                self._sgd_graph.replay() if self._sgd_graph is not None else self.sgd_step()
        self.step_index += 1

    def env_steps(self) -> int:
        """Brax's count includes the prefill"""
        return self.c.prefill_env_steps + self.step_index * self.B

    def params(self) -> dict:
        L = self.learner
        return dict(policy=L.policy.detach().cpu().numpy(), q=L.q.detach().cpu().numpy(), target_q=L.target_q.cpu().numpy(),
                    log_alpha=L.log_alpha.detach().cpu().numpy(), mean=self.mean.cpu().numpy(), std=self.std.cpu().numpy(),
                    stat=self.stat.cpu().numpy())


def train(environment, num_timesteps: int, episode_length: int, action_repeat: int = 1, num_envs: int = 1, num_eval_envs: int = 128,
          learning_rate: float = 1e-4, discounting: float = 0.9, seed: int = 0, batch_size: int = 256, num_evals: int = 1,
          normalize_observations: bool = False, max_devices_per_host: Optional[int] = None, reward_scaling: float = 1.0,
          tau: float = 0.005, min_replay_size: int = 0, max_replay_size: Optional[int] = None, grad_updates_per_step: int = 1,
          deterministic_eval: bool = False, progress_fn: Callable[[int, dict], None] = lambda *a: None, capture: bool = True,
          learner: str = "torch", randomization: Optional[dict] = None):
    """sac.train with Brax's signature and defaults for the arguments the reference passes.  Returns (make_inference_fn, params,
    metrics): make_inference_fn(params) gives an `Actor` factory for a VecEnv; params is a dict of numpy arrays (policy, q, target_q,
    log_alpha, the observation statistics).  One device: max_devices_per_host is accepted and has nothing to choose.  learner:
    "torch" (`Learner`, the default) or "fused" (`FusedLearner`, the update as two CUDA launches).  randomization: as ppo.train's
    (domain randomisation of the training envs, DESIGN.md §5n)."""
    if learner not in LEARNERS:
        raise ValueError(f"learner must be one of {LEARNERS}, not {learner!r}")
    if action_repeat != 1:
        raise NotImplementedError("action_repeat != 1 is not built (the vector env steps once per action)")
    if deterministic_eval:
        raise NotImplementedError("only the stochastic evaluation of the reference's config is built")
    if max_replay_size is None:
        max_replay_size = num_timesteps
    env = get_env(environment) if isinstance(environment, str) else environment
    tr = SACTrainer(env, num_timesteps, episode_length, num_envs, num_eval_envs, learning_rate, discounting, seed, batch_size, num_evals,
                    normalize_observations, reward_scaling, tau, min_replay_size, max_replay_size, grad_updates_per_step,
                    learner=learner, randomization=randomization)
    return common.run_training(tr, num_evals, progress_fn, capture)
