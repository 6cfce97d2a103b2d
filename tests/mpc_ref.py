"""The receding-horizon controller (DESIGN.md §5i) restated on the CPU oracle: `oracle/planner.py`'s `reverse_once` and `update`
for the diffusion steps, the oracle's own threefry for the keys and the oracle rollouts (n = 1, H = 1) for the plant.

    control step 0:  rng = PRNGKey(seed); rng, rng_reset = split(rng); rng_exp, rng = split(rng);
                     steps i = Ndiffuse - 1 ... 1 from YN = 0 with the keys of the chain r, k = split(r) from rng_exp
    control step c:  rng, rng_c = split(rng); Ybar_Nwarm = shift(P_{c-1}); steps i = Nwarm ... 1 with r, k = split(r) from rng_c
    execute:         a_c = P_c[0]; s_{c+1}, r_c = env.step(s_c, a_c)
"""
from __future__ import annotations

import numpy as np

from oracle import oracle as orc
from oracle import planner as opl

f32 = np.float32


def shift_rows(P: np.ndarray) -> np.ndarray:
    """P [H, Nu]: row h takes row h + 1, the last row is zero"""
    out = np.zeros_like(P)
    out[:-1] = P[1:]
    return out


def car2d_step(params, x, a):
    """(x', r) of one car2d env step through the oracle rollout"""
    out = orc.car2d_rollout(params, np.asarray(x, f32), np.asarray(a, f32).reshape(1, 1, 2), want_rewss=True, want_traj=True)
    return out["traj"][0, 0].astype(f32), f32(out["rewss"][0, 0])


def run_mpc_car2d(car, seed, Nsample, H, Ndiffuse, Nwarm, Nstep, temp, beta0=1e-4, betaT=1e-2):
    """-> dict(plans [Nstep, H, 2], actions [Nstep, 2], rewards [Nstep], states [Nstep + 1, 3], rew_hist [Nstep])"""
    _, alphas, alphas_bar, sigmas = opl.make_schedule(beta0, betaT, Ndiffuse)
    rng = orc.prng_key(seed)
    rng, _rng_reset = orc.split(rng)     # car2d's reset ignores its key
    x = np.asarray(car.x0, f32)
    plans, actions, rewards, states, rew_hist = [], [], [], [x], []
    P = None
    for c in range(Nstep):
        if c == 0:
            rng_exp, rng = orc.split(rng)
            r, i0, Yb = rng_exp, Ndiffuse - 1, np.zeros(H * 2, f32)
        else:
            rng, rng_c = orc.split(rng)
            r, i0, Yb = rng_c, Nwarm, shift_rows(P).reshape(-1)
        env = opl.OracleEnv("car2d", 2, params=car.params, x0=x)
        for i in range(i0, 0, -1):
            r, k = orc.split(r)
            o = opl.reverse_once(env, k, Nsample, H, float(sigmas[i]), Yb, temp, alphas, alphas_bar, i)
            Yb = o["Ybar_im1"]
            rm = o["rew_mean"]
        P = Yb.reshape(H, 2)
        a = P[0].copy()
        x, rew = car2d_step(car.params, x, a)
        plans.append(P), actions.append(a), rewards.append(rew), states.append(x), rew_hist.append(rm)
    return dict(plans=np.stack(plans), actions=np.stack(actions), rewards=np.asarray(rewards, f32), states=np.stack(states),
                rew_hist=np.asarray(rew_hist, f32))
