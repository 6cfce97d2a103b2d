"""One step of a planner ensemble (DESIGN.md §5l) restated on the in-repo CPU oracle — test infrastructure.

Problem b's step draws Y0s exactly as a nominal step (`orc.sample_Y0s`), rolls every sample out under each member's model
`scaled_env(env, f_k, g_k)` (`orc.xpbd_rollout` of that env's blob), scores each sample by the ordered float32 mean of its K
returns and feeds those scores to the unchanged tail (`opl.reverse_once_stats` / `opl.update`, or `opl`'s path-integral rules).
"""
from __future__ import annotations

import numpy as np

from mbd_b200.envs.vec import scaled_env
from oracle import oracle as orc
from oracle import planner as opl

f32 = np.float32


def ordered_mean(r: np.ndarray) -> np.ndarray:
    """r [N, K] member returns -> [N]: s = r[:, 0]; s = fl(s + r[:, k]) for k = 1 .. K-1; fl(s / K) (divided, not multiplied)"""
    r = np.asarray(r, dtype=f32)
    s = r[:, 0].copy()
    for k in range(1, r.shape[1]):
        s = (s + r[:, k]).astype(f32)
    return (s / f32(r.shape[1])).astype(f32)


def member_returns(env, state, Y0s: np.ndarray, H: int, members) -> np.ndarray:
    """[N, K] returns of Y0s [N, H * Nu] from state under every member (friction, gear), each the oracle rollout of its scaled blob"""
    Y = np.ascontiguousarray(Y0s, dtype=f32).reshape(Y0s.shape[0], H, env.action_size)
    return np.stack([orc.xpbd_rollout(scaled_env(env, f, g).blob, state, Y)["rews"] for f, g in members], axis=1)


def reverse_once(env, state, key, Nsample, H, sigma, Ybar_i, temp, alphas, alphas_bar, i, members) -> dict:
    """one diffusion step of a problem planning with `members` [(friction, gear), ...] (opl.reverse_once with the ensemble's
    scores); returns dict(Y0s, ens_rews [N, K], rews, Ybar, weights, rew_mean, Ybar_im1)"""
    Y0s = orc.sample_Y0s(key, Nsample, H * env.action_size, sigma, Ybar_i)
    ens = member_returns(env, state, Y0s, H, members)
    rews = ordered_mean(ens)
    Ybar, rew_mean, w = opl.reverse_once_stats(rews, Y0s, temp)
    return dict(Y0s=Y0s, ens_rews=ens, rews=rews, Ybar=Ybar, weights=w, rew_mean=rew_mean,
                Ybar_im1=opl.update(np.asarray(Ybar_i, f32), Ybar, alphas, alphas_bar, i))
