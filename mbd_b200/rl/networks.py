"""The PPO networks of Brax's `ppo_networks.make_ppo_networks` **[brax-recalled]** as views into flat fp32 parameter buffers.

policy: O -> 32 -> 32 -> 32 -> 32 -> 2 Nu; value: O -> 256 x 5 -> 1; swish between layers, none after the last; the observation is
normalised first, (obs - mean) / std.  Flat layout, layer by layer: W [in][out] (Flax's kernel), then b [out].  The policy buffer is
what the acting kernel reads (include/mbd_ppo.h).  Init: lecun_uniform weights (U(-sqrt(3 / fan_in), +sqrt(3 / fan_in))) and zero biases,
one key per layer from `key, layer_key = split(key)`; Flax derives its per-layer keys differently, so the initial bits differ from
Brax's (a declared deviation).
"""
from __future__ import annotations

import math
from typing import List, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from .. import prng

POLICY_HIDDEN = (32, 32, 32, 32)
VALUE_HIDDEN = (256, 256, 256, 256, 256)
MIN_STD = 0.001
HALF_LOG_2PI = 0.5 * math.log(2.0 * math.pi)
LOG2 = math.log(2.0)


def layer_sizes(O: int, out: int, hidden: Sequence[int]) -> List[Tuple[int, int]]:
    dims = [O, *hidden, out]
    return list(zip(dims[:-1], dims[1:]))


def policy_sizes(O: int, nu: int):
    return layer_sizes(O, 2 * nu, POLICY_HIDDEN)


def value_sizes(O: int):
    return layer_sizes(O, 1, VALUE_HIDDEN)


def num_params(sizes) -> int:
    return sum(i * o + o for i, o in sizes)


def unflatten(flat, sizes):
    """[(W [in, out], b [out])] views of a flat buffer (torch tensor or numpy array)"""
    out, k = [], 0
    for i, o in sizes:
        W = flat[k:k + i * o].reshape(i, o)
        k += i * o
        out.append((W, flat[k:k + o]))
        k += o
    if k != len(flat):
        raise ValueError(f"flat buffer has {len(flat)} floats, the layout {k}")
    return out


def flatten(layers) -> np.ndarray:
    return np.concatenate([np.concatenate([np.asarray(W, np.float32).ravel(), np.asarray(b, np.float32).ravel()]) for W, b in layers])


def init_params(key, sizes) -> np.ndarray:
    """lecun_uniform weights, zero biases; layer l draws from `key, layer_key = split(key)`"""
    layers = []
    for i, o in sizes:
        key, kl = prng.split2(key)
        lim = np.float32(math.sqrt(3.0 / i))
        layers.append((prng.uniform(kl, (i, o), -lim, lim), np.zeros(o, np.float32)))
    return flatten(layers)


def mlp(x: torch.Tensor, layers) -> torch.Tensor:
    for l, (W, b) in enumerate(layers):
        x = torch.addmm(b, x, W)
        if l + 1 < len(layers):
            x = F.silu(x)
    return x


def normalize(obs, mean, std):
    return (obs - mean) / std


def tanh_log_det_jacobian(x):
    return 2.0 * (LOG2 - x - F.softplus(-2.0 * x))


def log_prob(logits: torch.Tensor, raw: torch.Tensor) -> torch.Tensor:
    """NormalTanhDistribution.log_prob(logits, raw) summed over the action axis"""
    loc, s = logits.chunk(2, dim=-1)
    scale = F.softplus(s) + MIN_STD
    lp = -0.5 * torch.square(raw / scale - loc / scale) - (HALF_LOG_2PI + torch.log(scale))
    return (lp - tanh_log_det_jacobian(raw)).sum(-1)


def entropy(logits: torch.Tensor, eps: torch.Tensor) -> torch.Tensor:
    """NormalTanhDistribution.entropy(logits, key) with eps = normal(key, loc.shape): Normal entropy plus the log-det-Jacobian at
    the reparameterised sample eps * scale + loc, summed over the action axis"""
    loc, s = logits.chunk(2, dim=-1)
    scale = F.softplus(s) + MIN_STD
    ent = 0.5 + (HALF_LOG_2PI + torch.log(scale))
    return (ent + tanh_log_det_jacobian(eps * scale + loc)).sum(-1)


# ---- SAC (brax.training.agents.sac.networks **[brax-recalled]**) -------------------------------------------------------------------
# policy: O -> 256 -> 256 -> 2 Nu, ReLU between layers, the layout above (include/mbd_sac.h reads it); Q: two critics, each
# concat(normalize(obs), action) -> 256 -> 256 -> 1 with ReLU.  The Q buffer is layer-major so that both critics run as one batched
# matmul: W_l [2][in][out], then b_l [2][out], layer by layer.  Init: critic c takes key c of split(key_q) and draws as init_params.
SAC_HIDDEN = (256, 256)
N_CRITICS = 2


def sac_policy_sizes(O: int, nu: int):
    return layer_sizes(O, 2 * nu, SAC_HIDDEN)


def sac_q_sizes(O: int, nu: int):
    """the sizes of one critic"""
    return layer_sizes(O + nu, 1, SAC_HIDDEN)


def sac_q_num_params(O: int, nu: int) -> int:
    return N_CRITICS * num_params(sac_q_sizes(O, nu))


def sac_q_unflatten(flat, sizes):
    """[(W [2, in, out], b [2, 1, out])] views of a layer-major Q buffer"""
    out, k = [], 0
    for i, o in sizes:
        W = flat[k:k + N_CRITICS * i * o].reshape(N_CRITICS, i, o)
        k += N_CRITICS * i * o
        out.append((W, flat[k:k + N_CRITICS * o].reshape(N_CRITICS, 1, o)))
        k += N_CRITICS * o
    if k != len(flat):
        raise ValueError(f"flat buffer has {len(flat)} floats, the layout {k}")
    return out


def sac_q_init(key, sizes) -> np.ndarray:
    critics = [unflatten(init_params(k, sizes), sizes) for k in prng.split(key, N_CRITICS)]
    return np.concatenate([np.concatenate([np.stack([np.asarray(c[l][0]) for c in critics]).ravel(),
                                           np.stack([np.asarray(c[l][1]) for c in critics]).ravel()]) for l in range(len(sizes))])


def relu_mlp(x: torch.Tensor, layers) -> torch.Tensor:
    for l, (W, b) in enumerate(layers):
        x = torch.addmm(b, x, W)
        if l + 1 < len(layers):
            x = F.relu(x)
    return x


def sac_q(layers, x: torch.Tensor, action: torch.Tensor) -> torch.Tensor:
    """Q values [2, n] of both critics at (normalised obs x [n, O], action [n, Nu])"""
    h = torch.cat([x, action], -1).unsqueeze(0).expand(N_CRITICS, -1, -1)
    for l, (W, b) in enumerate(layers):
        h = torch.baddbmm(b, h, W)
        if l + 1 < len(layers):
            h = F.relu(h)
    return h.squeeze(-1)
