"""Input families of the fused SAC update's contract (tests/sac_learn_ref.py), in the style of tests/rl_families.py: every family is
(policy, q, target_q, log_alpha, mean, std, rows [n, row], eps [3, n, Nu], O, Nu, reward_scaling, discounting) as fp32 arrays."""
from __future__ import annotations

import numpy as np

from mbd_b200 import prng
from mbd_b200.rl import networks as nets

f32 = np.float32
MILD = [(O, nu, n) for O in (1, 11, 31, 33, 128) for nu in (1, 3, 17, 32) for n in (1, 37, 512)]


def base(O: int, nu: int, n: int, seed: int = 0, reward_scaling: float = 1.0, discounting: float = 0.97) -> dict:
    rng = np.random.default_rng(seed)
    key = prng.PRNGKey(seed)
    kp, kq = prng.split(key)
    policy = nets.init_params(kp, nets.sac_policy_sizes(O, nu))
    q = nets.sac_q_init(kq, nets.sac_q_sizes(O, nu))
    target_q = (q + f32(0.01) * rng.standard_normal(q.shape).astype(f32)).astype(f32)
    R = 2 * O + nu + 3
    rows = np.zeros((n, R), f32)
    rows[:, :O] = rng.standard_normal((n, O))
    rows[:, O:O + nu] = np.tanh(rng.standard_normal((n, nu)))
    rows[:, O + nu] = rng.standard_normal(n)
    rows[:, O + nu + 1] = (rng.random(n) > 0.1).astype(f32)
    rows[:, O + nu + 2:2 * O + nu + 2] = rows[:, :O] + 0.1 * rng.standard_normal((n, O))
    rows[:, 2 * O + nu + 2] = (rng.random(n) < 0.1).astype(f32)
    return dict(policy=policy, q=q, target_q=target_q, log_alpha=np.array([0.1 * rng.standard_normal()], f32),
                mean=(0.1 * rng.standard_normal(O)).astype(f32), std=(1.0 + 0.2 * rng.random(O)).astype(f32), rows=rows,
                eps=rng.standard_normal((3, n, nu)).astype(f32), O=O, nu=nu, reward_scaling=reward_scaling, discounting=discounting)


def _trunc(f, v):
    O, nu = f["O"], f["nu"]
    f["rows"][:, 2 * O + nu + 2] = v
    return f


def _last_bias(f, v):
    """the policy's output bias (loc: first Nu, scale logit: the rest)"""
    nu = f["nu"]
    k = len(f["policy"]) - 2 * nu
    f["policy"][k:k + nu] += v[0]
    f["policy"][k + nu:] += v[1]
    return f


def families(O: int = 11, nu: int = 3, n: int = 64) -> dict:
    """the special families at one shape (the mild shapes are MILD)"""
    out = {}
    out["all_truncated"] = _trunc(base(O, nu, n, 1), 1.0)
    out["none_truncated"] = _trunc(base(O, nu, n, 2), 0.0)
    out["discount_0"] = base(O, nu, n, 3, discounting=0.0)
    f = base(O, nu, n, 4)
    qs = nets.sac_q_unflatten(f["q"], nets.sac_q_sizes(O, nu))
    for W, b in qs:                       # critic 1 = critic 0: every Q ties in min
        W[1] = W[0]
        b[1] = b[0]
    out["critics_equal"] = f
    f = base(O, nu, n, 5)
    f["policy"][O * 256:O * 256 + 256] = -(f["rows"][0, :O] - f["mean"]) / f["std"] @ nets.unflatten(
        f["policy"], nets.sac_policy_sizes(O, nu))[0][0]     # row 0's first-layer pre-activations at 0
    out["preact_zero"] = f
    out["scale_floor"] = _last_bias(base(O, nu, n, 6), (0.0, -40.0))
    out["raw_beyond_cap"] = _last_bias(base(O, nu, n, 7), (25.0, 0.0))
    out["reward_scaling_30"] = base(O, nu, n, 8, reward_scaling=30.0, discounting=0.997)
    f = base(O, nu, n, 9)
    f["std"][:] = f32(1e-6)
    f["rows"][:, O + nu + 2:2 * O + nu + 2] = f["rows"][:, :O] = f["mean"][None, :] + f32(1e-6) * np.round(
        np.random.default_rng(9).standard_normal((n, O)))
    out["std_floor"] = f
    return out
