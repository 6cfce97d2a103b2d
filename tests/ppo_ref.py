"""numpy restatements of Brax's PPO formulas **[brax-recalled]** (v0.10.x): compute_gae, the advantage normalisation,
running_statistics.update, NormalTanhDistribution and the policy MLP — in float64, and the GAE kernel's float32 order."""
import numpy as np

from mbd_b200.rl import networks as nets
from mbd_b200.rl import train_brax

f = np.float32

# The learning check of tests/test_ppo_gpu.py and its calibration in scripts/gpu_ppo_timing.py (one definition for both): halfcheetah
# at the reference's configuration for three training steps (983 040 env steps), with an evaluation before and after.
LEARN_ENV = "halfcheetah"
LEARN_STEPS = 3


def learn_config(seed: int) -> dict:
    cfg = train_brax.ppo_config(LEARN_ENV)
    per_step = cfg["batch_size"] * cfg["num_minibatches"] * cfg["unroll_length"]
    cfg.update(num_timesteps=LEARN_STEPS * per_step, num_evals=2, seed=seed)
    return cfg


def compute_gae(truncation, termination, rewards, values, bootstrap_value, lambda_, discount):
    """brax.training.agents.ppo.losses.compute_gae, float64, time-major [T, n]"""
    truncation_mask = 1 - truncation
    v_tp1 = np.concatenate([values[1:], bootstrap_value[None]], 0)
    deltas = (rewards + discount * (1 - termination) * v_tp1 - values) * truncation_mask
    acc = np.zeros_like(bootstrap_value)
    out = np.zeros_like(values)
    for t in range(values.shape[0] - 1, -1, -1):
        acc = deltas[t] + discount * (1 - termination[t]) * truncation_mask[t] * lambda_ * acc
        out[t] = acc
    vs = out + values
    vs_tp1 = np.concatenate([vs[1:], bootstrap_value[None]], 0)
    adv = (rewards + discount * (1 - termination) * vs_tp1 - values) * truncation_mask
    return vs, adv


def normalize_advantage(adv):
    return (adv - adv.mean()) / (adv.std() + 1e-8)


def _block_sum(v, P):
    s = np.zeros(P, f)
    s[:len(v)] = v
    k = P // 2
    while k > 0:
        s[:k] = s[:k] + s[k:2 * k]
        k //= 2
    return s[0]


def gae_kernel_f32(reward, disc, trunc, values, traj, B, T, reward_scaling, discount, lam):
    """k_ppo_gae in its float32 order: reward / disc / trunc [slots, B] rollout buffers, values [T + 1, mb], traj [mb]"""
    mb = len(traj)
    g, lam, rs = f(discount), f(lam), f(reward_scaling)
    u, b = traj // B, traj % B
    rows = (u * T)[None, :] + np.arange(T)[:, None]
    r = (reward[rows, b[None, :]] * rs).astype(f)
    tr = trunc[rows, b[None, :]].astype(f)
    term = ((f(1) - disc[rows, b[None, :]]) * (f(1) - tr)).astype(f)
    tm = (f(1) - tr).astype(f)
    v, boot = values[:T].astype(f), values[T].astype(f)
    vs = np.zeros((T, mb), f)
    acc, vnext = np.zeros(mb, f), boot.copy()
    for t in range(T - 1, -1, -1):
        delta = (r[t] + g * (f(1) - term[t]) * vnext - v[t]) * tm[t]
        acc = delta + g * (f(1) - term[t]) * tm[t] * lam * acc
        vs[t] = acc + v[t]
        vnext = v[t]
    vsn = np.concatenate([vs[1:], boot[None]], 0)
    adv = ((r + g * (f(1) - term) * vsn - v) * tm).astype(f)
    P = 32
    while P < mb and P < 1024:
        P *= 2
    s, q = np.zeros(P, f), np.zeros(P, f)
    for i in range(mb):                 # thread i % P takes trajectories in ascending order
        for t in range(T):
            s[i % P] = s[i % P] + adv[t, i]
    mean = f(_block_sum(s, P) / f(T * mb))
    for i in range(mb):
        for t in range(T):
            d = adv[t, i] - mean
            q[i % P] = q[i % P] + d * d
    sd = np.sqrt(f(_block_sum(q, P) / f(T * mb))).astype(f)
    return vs, ((adv - mean) / (sd + f(1e-8))).astype(f)


def running_update(state, batch, std_min=1e-6, std_max=1e6):
    """running_statistics.update (count, mean, summed_variance) -> (new state, std), float64"""
    count, mean, sv = state
    batch = np.asarray(batch, np.float64).reshape(-1, len(mean))
    count = count + batch.shape[0]
    d_old = batch - mean
    mean = mean + d_old.sum(0) / count
    sv = sv + (d_old * (batch - mean)).sum(0)
    return (count, mean, sv), np.clip(np.sqrt(sv / count), std_min, std_max)


def softplus(x):
    return np.logaddexp(x, 0.0)


def normal_tanh(loc, s, raw):
    """(log_prob summed over the last axis, scale) of NormalTanhDistribution, float64"""
    scale = softplus(s) + 0.001
    lp = -0.5 * np.square(raw / scale - loc / scale) - (0.5 * np.log(2 * np.pi) + np.log(scale))
    lp = lp - 2.0 * (np.log(2.0) - raw - softplus(-2.0 * raw))
    return lp.sum(-1), scale


def entropy(loc, s, eps):
    scale = softplus(s) + 0.001
    x = eps * scale + loc
    ent = 0.5 + 0.5 * np.log(2 * np.pi) + np.log(scale) + 2.0 * (np.log(2.0) - x - softplus(-2.0 * x))
    return ent.sum(-1)


def policy_act64(policy, mean, std, obs, eps, O, nu):
    """the acting step in float64: (act, raw, logp)"""
    x = (np.asarray(obs, np.float64) - mean) / std
    layers = nets.unflatten(np.asarray(policy, np.float64), nets.policy_sizes(O, nu))
    for l, (W, b) in enumerate(layers):
        x = x @ W + b
        if l + 1 < len(layers):
            x = x / (1.0 + np.exp(-x))
    loc, s = x[:, :nu], x[:, nu:]
    scale = softplus(s) + 0.001
    raw = eps * scale + loc
    lp, _ = normal_tanh(loc, s, raw)
    return np.tanh(raw), raw, lp
