"""Constructed inputs for the float64 contract of the RL acting step, GAE and the observation statistics (tests/rl_ref.py).

Acting families (`act_cases`), each a list of launches (O, Nu, policy, mean, std, obs, key); eps = normal(key, (B, Nu)) as the
kernels draw it:
  mild        the inputs of the harness tests: Flax-initialised weights, biases N(0, 0.3), std in [0.2, 3], obs within ~1.5 std;
              at O in {1, 31, 32, 33, 127, 128} and Nu in {1, 17, 32}
  std_floor   half the columns with std at the 1e-6 floor and obs ~1 from the mean: normalised inputs ~1e6 (their first-layer
              weights scaled by 1e-6)
  obs_mean    obs exactly equal to the mean: the first layer sees exact zeros
  floor       last-layer biases putting s at -30, -12 and -8 (scale at or near its 0.001 floor), loc 0
  loc         loc at +-1e3 with s in {-30, -8, 0, 20}: r / scale and loc / scale cancel
  wide        s at 0 and 20, loc 0
  raw         loc placing raw near 0 (scale 0.001), in (2, 20), beyond +-20, and at +-20 within 0.003 (both sides of the tanh cap)
  cap         hidden biases putting pre-activations below -80 and within +-0.5 of it (both sides of the swish cap; ReLU's
              negative side for SAC)
GAE families (`gae_cases`): rollout rows [T][B] with B = mb, trajectory i = env traj[i], values [T + 1][mb]:
  mild, the done / truncation patterns (none, all done, all truncated, first step, last step, alternating, both on one step),
  offset (rewards and values 1e3 + 1e-2 z), constant (every advantage equal), each at several (gamma, lambda, reward_scaling).
Statistics families (`stat_cases`): sequences of fp32 batches [n][O]: mild, offset (1e4 + 1e-3 z), constant, wide (spread
above 1e6: the 1e6 clip), and a count past 2^24 (O = 1)."""
import numpy as np

from mbd_b200 import prng
from mbd_b200.rl import networks as nets

f32 = np.float32
ACT_FAMILIES = ("mild", "std_floor", "obs_mean", "floor", "loc", "wide", "raw", "cap")
GAE_FAMILIES = ("mild", "none", "all_done", "all_trunc", "first", "last", "alternating", "both", "offset", "constant")
STAT_FAMILIES = ("mild", "offset", "constant", "wide", "count")
MILD_SHAPES = [(O, nu) for O in (1, 31, 32, 33, 127, 128) for nu in (1, 17, 32)]


def _sizes(kind, O, nu):
    return nets.policy_sizes(O, nu) if kind == "ppo" else nets.sac_policy_sizes(O, nu)


def _base(kind, O, nu, B, seed):
    """the mild family: (policy layers, mean, std, obs)"""
    rng = np.random.default_rng(seed)
    layers = nets.unflatten(nets.init_params(prng.PRNGKey(seed), _sizes(kind, O, nu)).copy(), _sizes(kind, O, nu))
    for W, b in layers:
        b[:] = rng.normal(0, 0.3, b.shape)
    mean = rng.normal(0, 1, O).astype(f32)
    std = rng.uniform(0.2, 3.0, O).astype(f32)
    obs = (mean + std * rng.normal(0, 1.5, (B, O))).astype(f32)
    return layers, mean, std, obs, rng


def _head_bias(layers, nu, loc, s):
    W, b = layers[-1]
    W *= 1e-3
    b[:nu], b[nu:] = loc, s


def _case(kind, O, nu, B, seed, family, **kw):
    layers, mean, std, obs, rng = _base(kind, O, nu, B, seed)
    if family == "std_floor":
        cols = np.arange(O) % 2 == 0
        std[cols] = f32(1e-6)
        obs[:, cols] = (mean[cols] + rng.choice([-1.0, 1.0], (B, int(cols.sum()))) * rng.uniform(0.5, 1.5, (B, int(cols.sum())))).astype(f32)
        layers[0][0][cols] *= 1e-6   # the first layer takes the ~1e6 inputs to O(1) pre-activations, as a trained policy would
    elif family == "obs_mean":
        obs[:] = mean
    elif family in ("floor", "loc", "wide", "raw"):
        _head_bias(layers, nu, kw["loc"], kw["s"])
    elif family == "cap":
        for W, b in layers[:-1]:
            W *= 0.05
            half = np.arange(b.size) % 2 == 0
            b[half] = rng.uniform(-120, -81, int(half.sum()))
            b[~half] = -80 + rng.uniform(-0.5, 0.5, int((~half).sum()))
    key = prng.PRNGKey(seed + 1)
    return (O, nu, nets.flatten(layers).astype(f32), mean, std, obs.astype(f32), key)


def act_cases(kind: str, B: int, shapes=None, seed: int = 0) -> dict:
    """{family: [(O, nu, policy, mean, std, obs, key)]}; `shapes` overrides the mild family's (O, nu) list"""
    out = {f: [] for f in ACT_FAMILIES}
    shapes = MILD_SHAPES if shapes is None else shapes
    for i, (O, nu) in enumerate(shapes):
        out["mild"].append(_case(kind, O, nu, B, seed + 10 * i, "mild"))
    O, nu = 17, 6
    out["std_floor"] = [_case(kind, 33, 5, B, seed + 1, "std_floor"), _case(kind, 128, 17, B, seed + 2, "std_floor")]
    out["obs_mean"] = [_case(kind, O, nu, B, seed + 3, "obs_mean"), _case(kind, 128, 32, B, seed + 4, "obs_mean")]
    out["floor"] = [_case(kind, O, nu, B, seed + 5 + k, "floor", loc=0.0, s=s) for k, s in enumerate((-30.0, -12.0, -8.0))]
    out["loc"] = [_case(kind, O, nu, B, seed + 9 + k, "loc", loc=sg * 1e3, s=s)
                  for k, (sg, s) in enumerate((g, s) for g in (1.0, -1.0) for s in (-30.0, -8.0, 0.0, 20.0))]
    out["wide"] = [_case(kind, O, nu, B, seed + 20 + k, "wide", loc=0.0, s=s) for k, s in enumerate((0.0, 20.0))]
    out["raw"] = [_case(kind, O, nu, B, seed + 25 + k, "raw", loc=loc, s=s)
                  for k, (loc, s) in enumerate(((0.0, -30.0), (1e-6, -30.0), (8.0, 0.0), (-8.0, 0.0), (25.0, 0.0), (-25.0, 0.0),
                                                (20.0, -30.0), (-20.0, -30.0), (10.0, -30.0), (-10.0, -30.0)))]
    out["cap"] = [_case(kind, O, nu, B, seed + 40, "cap"), _case(kind, 128, 3, B, seed + 41, "cap")]
    return out


# ---- GAE --------------------------------------------------------------------------------------------------------------------------
GAE_PARAMS = [(0.97, 0.95, 1.0), (0.99, 1.0, 0.1), (1.0, 0.95, 30.0), (1.0, 1.0, 1.0)]   # (discount, lambda, reward_scaling)


def gae_case(family: str, T: int, mb: int, seed: int = 0, params=(0.97, 0.95, 1.0)) -> dict:
    """one minibatch: reward / disc / trunc rollout rows [T][B = mb], values [T + 1][mb], traj [mb], and the three scalars"""
    rng = np.random.default_rng(seed * 7919 + T * 131 + mb + GAE_FAMILIES.index(family))
    B = mb
    reward = rng.normal(size=(T, B))
    values = rng.normal(size=(T + 1, mb))
    done = np.zeros((T, B))
    trunc = np.zeros((T, B))
    if family == "mild":
        done = (rng.uniform(size=(T, B)) < 0.1).astype(float)
        trunc = done * (rng.uniform(size=(T, B)) < 0.5)
    elif family == "all_done":
        done[:] = 1
    elif family == "all_trunc":
        done[:] = 1
        trunc[:] = 1
    elif family == "first":
        done[0] = 1
        trunc[0] = rng.uniform(size=B) < 0.5
    elif family == "last":
        done[T - 1] = 1
        trunc[T - 1] = rng.uniform(size=B) < 0.5
    elif family == "alternating":
        done[::2] = 1
        trunc[::4] = 1
    elif family == "both":
        k = rng.integers(0, T, B)
        done[k, np.arange(B)] = 1
        trunc[k, np.arange(B)] = 1
    elif family == "offset":
        reward = 1e3 + 1e-2 * rng.normal(size=(T, B))
        values = 1e3 + 1e-2 * rng.normal(size=(T + 1, mb))
    elif family == "constant":
        done[:] = 1
        reward[:] = 0.37
        values[:] = 0.0
    traj = rng.permutation(B)[:mb].astype(np.int32)
    g, lam, rs = params
    return dict(T=T, mb=mb, B=B, reward=reward.astype(f32), disc=(1 - done).astype(f32), trunc=trunc.astype(f32),
                values=values.astype(f32), traj=traj, discount=g, lam=lam, reward_scaling=rs)


def gae_rows(c: dict):
    """the minibatch's time-major rows [T][mb] of a case (trajectory i = env traj[i] of the single unroll)"""
    t = c["traj"]
    return c["reward"][:, t], c["disc"][:, t], c["trunc"][:, t]


# ---- statistics -------------------------------------------------------------------------------------------------------------------
def stat_batches(family: str, O: int, rows: int, updates: int = 3, seed: int = 0):
    """fp32 batches [rows][O] of one family"""
    rng = np.random.default_rng(seed * 31 + O + STAT_FAMILIES.index(family))
    out = []
    for k in range(updates):
        if family == "mild":
            x = rng.normal(k, 1.0 + k, (rows, O))
        elif family == "offset":
            x = 1e4 + 1e-3 * rng.normal(size=(rows, O))
        elif family == "constant":
            x = np.full((rows, O), 0.3 + k)
        elif family == "wide":
            x = rng.normal(0, 3e6, (rows, O))
        else:
            x = rng.normal(2.0, 0.5, (rows, O))
        out.append(x.astype(f32))
    return out
