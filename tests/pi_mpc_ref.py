"""The receding-horizon controller of the path-integral baselines (DESIGN.md §5j) restated on the CPU oracle: `oracle/planner.py`'s
`update_once` for the refinement steps, the oracle's own threefry for the keys and the oracle car2d rollout (n = 1, H = 1) for the
plant.

    control step 0:  rng = PRNGKey(seed); rng, rng_reset = split(rng); rng_exp, rng = split(rng);
                     steps t = Nrefine - 1 ... 1 from mu = 0, sigma = 1 with the keys of the chain r, k = split(r) from rng_exp
    control step c:  rng, rng_c = split(rng); mu_Nwarm = shift(P_{c-1}); sigma = sigma_warm; steps t = Nwarm ... 1 with
                     r, k = split(r) from rng_c
    execute:         a_c = P_c[0]; s_{c+1}, r_c = env.step(s_c, a_c)
    sigma log:       the sigma control step c ended with: CMA-ES's last sigma', else the sigma the step sampled with
"""
from __future__ import annotations

import numpy as np

from oracle import oracle as orc
from oracle import planner as opl
from tests.mpc_ref import car2d_step, shift_rows

f32 = np.float32


def run_pi_mpc_car2d(car, method, seed, Nsample, H, Nrefine, Nwarm, Nstep, temp, sigma_warm=1.0, trace=None):
    """-> dict(plans [Nstep, H, 2], actions [Nstep, 2], rewards [Nstep], states [Nstep + 1, 3], rew_hist [Nstep], sigmas [Nstep]).
    trace: a list that receives (c, t, update_once's dict) of every refinement step"""
    rng = orc.prng_key(seed)
    rng, _rng_reset = orc.split(rng)     # car2d's reset ignores its key
    x = np.asarray(car.x0, f32)
    plans, actions, rewards, states, rew_hist, sigmas = [], [], [], [x], [], []
    P = None
    for c in range(Nstep):
        if c == 0:
            rng_exp, rng = orc.split(rng)
            r, t0, mu, sigma = rng_exp, Nrefine - 1, np.zeros(H * 2, f32), 1.0
        else:
            rng, rng_c = orc.split(rng)
            r, t0, mu, sigma = rng_c, Nwarm, shift_rows(P).reshape(-1), float(f32(sigma_warm))
        env = opl.OracleEnv("car2d", 2, params=car.params, x0=x)
        for t in range(t0, 0, -1):
            r, k = orc.split(r)
            o = opl.update_once(env, k, Nsample, H, sigma, mu, temp, method)
            if trace is not None:
                trace.append((c, t, o))
            mu, sigma, rm = o["mu"], o["sigma"], o["rew_mean"]
        P = mu.reshape(H, 2)
        a = P[0].copy()
        x, rew = car2d_step(car.params, x, a)
        plans.append(P), actions.append(a), rewards.append(rew), states.append(x), rew_hist.append(rm), sigmas.append(sigma)
    return dict(plans=np.stack(plans), actions=np.stack(actions), rewards=np.asarray(rewards, f32), states=np.stack(states),
                rew_hist=np.asarray(rew_hist, f32), sigmas=np.asarray(sigmas, f32))
