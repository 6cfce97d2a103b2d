"""Restatements of Brax's SAC pieces **[brax-recalled]** / **[jax-recalled]** (v0.10.x), written from the formulas and independent of
mbd_b200/rl/sac.py: jax.random.randint's arithmetic, QueueBase.insert with np.roll, the device ring, the sampler, the acting step and
the three losses with one sgd_step in float64."""
import numpy as np
import torch

from mbd_b200 import prng
from mbd_b200.blackbox.mbd_mnist import normal_host
from mbd_b200.rl import networks as nets

M32 = 0xFFFFFFFF

# The learning check of tests/test_sac_gpu.py and its calibration in scripts/gpu_sac_timing.py (one definition for both): hopper at
# the reference's configuration, the prefill and LEARN_STEPS training steps, with an evaluation before and after.
LEARN_ENV = "hopper"
LEARN_STEPS = 600


def learn_config(seed: int) -> dict:
    from mbd_b200.rl import train_sac
    cfg = train_sac.sac_config(LEARN_ENV)
    prefill = -(-cfg["min_replay_size"] // cfg["num_envs"]) * cfg["num_envs"]
    cfg.update(num_timesteps=prefill + LEARN_STEPS * cfg["num_envs"], num_evals=2, seed=seed)
    return cfg


# ---- randint ---------------------------------------------------------------------------------------------------------------------
def randint_int(hi: int, lo: int, span: int) -> int:
    """one offset, Python ints with every uint32 wrap written out"""
    span = span & M32
    m = (65536 % span) & M32
    mult = ((m * m) & M32) % span
    prod = ((hi % span) * mult) & M32
    return ((prod + lo % span) & M32) % span


def randint_np(hi, lo, span: int) -> np.ndarray:
    """the same in numpy uint32 arithmetic"""
    with np.errstate(over="ignore"):
        s = np.uint32(span)
        m = np.uint32(65536) % s
        mult = (m * m) % s
        return ((np.asarray(hi, np.uint32) % s) * mult + np.asarray(lo, np.uint32) % s) % s


def randint(key, n: int, minval: int, maxval: int) -> np.ndarray:
    """jax.random.randint(key, (n,), minval, maxval) for 0 <= minval, maxval < 2^31 (the current threefry layout)"""
    k1, k2 = prng.split(key)
    span = 1 if maxval <= minval else maxval - minval
    return minval + randint_np(prng.random_bits(k1, n), prng.random_bits(k2, n), span).astype(np.int64)


# ---- the replay queue ------------------------------------------------------------------------------------------------------------
class QueueRef:
    """QueueBase.insert / UniformSamplingQueue.sample's view of Brax's replay buffer: roll left when an insert would overflow"""

    def __init__(self, cap: int, width: int):
        self.data = np.zeros((cap, width), np.float32)
        self.insert_position = 0
        self.sample_position = 0

    def insert(self, update):
        cap, n = len(self.data), len(update)
        roll = min(0, cap - self.insert_position - n)
        if roll:
            self.data = np.roll(self.data, roll, axis=0)
        pos = self.insert_position + roll
        self.data[pos:pos + n] = update
        self.insert_position = (pos + n) % (cap + 1)
        self.sample_position = max(0, self.sample_position + roll)

    def content(self):
        return self.data[self.sample_position:self.insert_position]

    def take(self, idx):
        """jnp.take(data, sample_position + idx)"""
        return self.data[self.sample_position + np.asarray(idx)]


class RingRef:
    """the device ring: pos = the next write row, size = min(inserted, cap); logical i -> (pos - size + i) mod cap"""

    def __init__(self, cap: int, width: int):
        self.data = np.zeros((cap, width), np.float32)
        self.pos = self.size = 0

    def insert(self, update):
        cap = len(self.data)
        for b, row in enumerate(update):
            self.data[(self.pos + b) % cap] = row
        self.pos = (self.pos + len(update)) % cap
        self.size = min(self.size + len(update), cap)

    def rows(self, idx):
        cap = len(self.data)
        return self.data[(self.pos - self.size + np.asarray(idx)) % cap]


def sample_host(ring_rows, pos, size, buffer_key, noise_keys, updates, batch, nu):
    """one mbd_sac_sample: (next buffer key, indices [updates * batch], rows [updates, batch, R], eps [3, updates, batch, nu]) with
    ring_rows the physical ring [cap, R] and noise_keys [updates, 3, 2] of this training step"""
    buffer_key, sample_key = prng.split(buffer_key)
    idx = randint(sample_key, updates * batch, 0, size)
    cap = len(ring_rows)
    rows = ring_rows[(pos - size + idx) % cap].reshape(updates, batch, -1)
    eps = np.stack([np.stack([normal_host(noise_keys[g, w], (batch, nu)) for g in range(updates)]) for w in range(3)])
    return buffer_key, idx, rows, eps


# ---- networks and losses in float64 ----------------------------------------------------------------------------------------------
def softplus(x):
    return np.logaddexp(x, 0.0)


def policy_act64(policy, mean, std, obs, eps, O, nu):
    """the acting step in float64: (act, raw, logp)"""
    x = (np.asarray(obs, np.float64) - mean) / std
    layers = nets.unflatten(np.asarray(policy, np.float64), nets.sac_policy_sizes(O, nu))
    for l, (W, b) in enumerate(layers):
        x = x @ W + b
        if l + 1 < len(layers):
            x = np.maximum(x, 0.0)
    loc, s = x[:, :nu], x[:, nu:]
    scale = softplus(s) + 0.001
    raw = eps * scale + loc
    lp = -0.5 * np.square((raw - loc) / scale) - (0.5 * np.log(2 * np.pi) + np.log(scale)) - 2.0 * (np.log(2.0) - raw - softplus(-2.0 * raw))
    return np.tanh(raw), raw, lp.sum(-1)


def _mlp64(x, flat, sizes):
    k = 0
    for l, (i, o) in enumerate(sizes):
        W = flat[k:k + i * o].reshape(i, o)
        k += i * o
        x = x @ W + flat[k:k + o]
        k += o
        if l + 1 < len(sizes):
            x = torch.relu(x)
    return x


def _critics64(q, O, nu):
    """critic c's own flat buffer from the layer-major Q buffer"""
    sizes = nets.sac_q_sizes(O, nu)
    parts = [[] for _ in range(2)]
    k = 0
    for i, o in sizes:
        for c in range(2):
            parts[c].append(q[k + c * i * o:k + (c + 1) * i * o])
        k += 2 * i * o
        for c in range(2):
            parts[c].append(q[k + c * o:k + (c + 1) * o])
        k += 2 * o
    return [torch.cat(p) for p in parts], sizes


def _dist(logits, nu, eps):
    loc, s = logits[:, :nu], logits[:, nu:]
    scale = torch.nn.functional.softplus(s) + 0.001
    raw = eps * scale + loc
    lp = -0.5 * ((raw - loc) / scale) ** 2 - (0.5 * np.log(2 * np.pi) + torch.log(scale)) \
        - 2.0 * (np.log(2.0) - raw - torch.nn.functional.softplus(-2.0 * raw))
    return raw, lp.sum(-1)


def losses64(policy, q, target_q, log_alpha, mean, std, rows, eps, O, nu, reward_scaling, discounting):
    """alpha_loss, critic_loss, actor_loss of sac/losses.py in float64 torch (tensors may require grad)"""
    rows = torch.as_tensor(rows, dtype=torch.float64)
    eps = torch.as_tensor(eps, dtype=torch.float64)
    obs, action = rows[:, :O], rows[:, O:O + nu]
    reward, discount = rows[:, O + nu], rows[:, O + nu + 1]
    next_obs, trunc = rows[:, O + nu + 2:2 * O + nu + 2], rows[:, 2 * O + nu + 2]
    x, xn = (obs - mean) / std, (next_obs - mean) / std
    psizes = nets.sac_policy_sizes(O, nu)
    crit, qsizes = _critics64(q, O, nu)
    tcrit, _ = _critics64(target_q, O, nu)
    # alpha
    _, lp = _dist(_mlp64(x, policy, psizes), nu, eps[0])
    alpha_loss = (torch.exp(log_alpha) * (-lp - (-0.5 * nu)).detach()).mean()
    alpha = torch.exp(log_alpha).detach()
    # critic
    q_old = torch.stack([_mlp64(torch.cat([x, action], -1), c, qsizes)[:, 0] for c in crit], -1)
    raw_n, lp_n = _dist(_mlp64(xn, policy, psizes), nu, eps[1])
    next_q = torch.stack([_mlp64(torch.cat([xn, torch.tanh(raw_n)], -1), c, qsizes)[:, 0] for c in tcrit], -1)
    next_v = next_q.min(-1).values - alpha * lp_n
    target = (reward * reward_scaling + discount * discounting * next_v).detach()
    q_error = (q_old - target[:, None]) * (1 - trunc)[:, None]
    critic_loss = 0.5 * (q_error ** 2).mean()
    # actor, with the old Q
    raw_p, lp_p = _dist(_mlp64(x, policy, psizes), nu, eps[2])
    q_act = torch.stack([_mlp64(torch.cat([x, torch.tanh(raw_p)], -1), c.detach(), qsizes)[:, 0] for c in crit], -1)
    actor_loss = (alpha * lp_p - q_act.min(-1).values).mean()
    return alpha_loss, critic_loss, actor_loss


def grads64(policy, q, target_q, log_alpha, mean, std, rows, eps, O, nu, reward_scaling, discounting):
    """(losses, d alpha_loss / d log_alpha, d critic_loss / d q, d actor_loss / d policy) in float64"""
    t = lambda a, g=False: torch.tensor(np.asarray(a, np.float64), requires_grad=g)   # noqa: E731
    pol, qq, la = t(policy, True), t(q, True), t(log_alpha, True)
    ls = losses64(pol, qq, t(target_q), la, t(mean), t(std), rows, eps, O, nu, reward_scaling, discounting)
    ga = torch.autograd.grad(ls[0], la)[0]
    gq = torch.autograd.grad(ls[1], qq)[0]
    gp = torch.autograd.grad(ls[2], pol)[0]
    return [float(v.detach()) for v in ls], ga.numpy(), gq.numpy(), gp.numpy()


def first_sgd_step64(policy, q, target_q, log_alpha, g_alpha, g_q, g_policy, lr, alpha_lr, tau):
    """sgd_step's parameters after Adam's first step (lr * sign(g) where |g| >> eps) and target (1 - tau) + new q tau"""
    policy_new = np.asarray(policy, np.float64) - lr * np.sign(g_policy)
    q_new = np.asarray(q, np.float64) - lr * np.sign(g_q)
    la_new = np.asarray(log_alpha, np.float64) - alpha_lr * np.sign(g_alpha)
    return policy_new, q_new, np.asarray(target_q, np.float64) * (1 - tau) + q_new * tau, la_new
