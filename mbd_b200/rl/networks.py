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
