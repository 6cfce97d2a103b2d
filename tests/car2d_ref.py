"""Float64 reference of ONE car2d step, its reward and the demo log-density (upstream mbd/envs/car2d.py) with a running
error radius next to every value.

`k_car2d` / `k_car2d_ps` (csrc/mbd_b200.cu) and `orc_car2d_rollout` (oracle/mbd_oracle.c) are two fp32 restatements of one
association order, compared bit for bit; a misreading present in both passes that comparison.  This module evaluates the
step from the upstream equations in float64 on the same fp32 inputs and gives every output a radius that bounds ANY correct
fp32 evaluation of it.  It shares the value-plus-radius class `R` and the error model of tests/xpbd_ref.py: u = 2^-24, one
rounding per `+ - * / sqrt`, gamma_k * sum|terms| for a sum of k terms (so the bound does not depend on the association
order), `sqrt` in the Hoelder form where its argument is within its radius of 0, and COS_ABS_ERR for `mbd_sincosf` on
|x| <= 1200 (tests/test_fp32_spec.py::test_sincos).

Inputs.  Every state and action word is an exact input (radius 0).  Constants enter as the fp32 values a weak-typed JAX
scalar takes, which are the values `Car2d.params` stores: the obstacle centres, the radius 0.3, dt, dt / 2 and dt / 6 are
read from that table, and pi, 0.2, 0.5 and the goal (0.5, 0) are rounded once to fp32.  The factors 2, 3 and 6 are exact.

The step (car2d.py:77-86):
* clip the action to [-1, 1] (exact);
* rates (car2d.py:10-19): x' = u1 sin(theta) 3, y' = u1 cos(theta) 3, theta' = u0 pi / 3 * 2.  sin and cos are 1-Lipschitz,
  so each is charged the propagated angle radius plus COS_ABS_ERR;
* RK4 (car2d.py:22-27): k1 = f(x), k2 = f(x + dt/2 k1), k3 = f(x + dt/2 k2), k4 = f(x + dt k3),
  x_new = x + dt/6 (k1 + 2 k2 + 2 k3 + k4).  An fp32 product with an exactly zero factor is exactly +-0 and x + (+-0) = x,
  so where u1 = 0 (u0 = 0) the new position (angle) is the old one with radius 0: the collision predicate of a car that
  does not move is evaluated on exact inputs;
* collision (car2d.py:30-32): any_k |x_new[:2] - c_k| < r over the 11 obstacles, evaluated on the NEW state;
* select (car2d.py:83): the old state where the car collides, the new state otherwise.

Branch gate.  Obstacle k's margin dist_k - r carries dist_k's radius.  The car surely collides where some margin is below
minus its radius.  Where no obstacle surely collides and some margin is within its radius, the outcome is undecided: the
result is the interval hull of q and q_new, and the sample is marked `undecided` when the two outcomes differ by more than
JUMP radii in some word, the rule of tests/xpbd_ref.py.  An undecided step is held to one of the two outcomes
(`check_rollout_branches`): it equals the frozen q bit for bit (q is an exact input) or lies within K radii of q_new.

`reward` (car2d.py:88-93) and `logpd` (car2d.py:95-102) evaluate the kernel's per-step reward and demo log-density on given
fp32 states.  For a horizon H longer than the reference path (href rows), step t >= href is compared with the last row,
min(t, href - 1): a choice of this repository; upstream requires H = href.  The clamps at 0.2 and 0.5 are Lipschitz and
need no gate (a distance surely beyond the clamp gives it exactly); the division by 0.5 is exact.  `mean_return` is
tests/pusht_ref.py's sum_t r_t / H.
"""
from __future__ import annotations

import numpy as np

from tests.pusht_ref import mean_return
from tests.xpbd_ref import COS_ABS_ERR, JUMP, U, R, exact_scale, fsum, sqrt, where  # noqa: F401  (U for the tests)

NOBS = 11
PI_F = float(np.float32(np.pi))
GOAL = (float(np.float32(0.5)), 0.0)      # car2d.py:64, xg[:2]
REW_CLAMP = float(np.float32(0.2))        # car2d.py:90
DEMO_CLAMP = 0.5                          # car2d.py:99


def table(P):
    """Car2d.params [obs_center (11 x 2), obs_radius, dt, dt / 2, dt / 6] as float64 values of the stored fp32 words"""
    P = np.asarray(P, dtype=np.float32).astype(np.float64)
    return dict(c=P[:2 * NOBS].reshape(NOBS, 2), r=P[2 * NOBS], dt=P[2 * NOBS + 1], hdt=P[2 * NOBS + 2], sdt=P[2 * NOBS + 3])


def _f64(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def _rates(x, u):
    """car2d.py:10-19"""
    rad = x[2].r + COS_ABS_ERR
    s, c = R(np.sin(x[2].v), rad), R(np.cos(x[2].v), rad)
    return (u[1] * s) * 3.0, (u[1] * c) * 3.0, exact_scale((u[0] * PI_F) / 3.0, 2.0)


def rk4(P, states, actions):
    """the unconstrained RK4 end point of states [n, 3] under actions [n, 2] (clipped here): a tuple of three R [n]"""
    T = table(P)
    s, a = _f64(states), np.clip(_f64(actions), -1.0, 1.0)
    q = tuple(R(s[:, i].copy()) for i in range(3))
    u = (R(a[:, 0].copy()), R(a[:, 1].copy()))
    k1 = _rates(q, u)
    k2 = _rates(tuple(q[i] + k1[i] * T["hdt"] for i in range(3)), u)
    k3 = _rates(tuple(q[i] + k2[i] * T["hdt"] for i in range(3)), u)
    k4 = _rates(tuple(q[i] + k3[i] * T["dt"] for i in range(3)), u)
    qn = [q[i] + fsum([k1[i], exact_scale(k2[i], 2.0), exact_scale(k3[i], 2.0), k4[i]]) * T["sdt"] for i in range(3)]
    still = (a[:, 1] == 0, a[:, 1] == 0, a[:, 0] == 0)     # exact zeros stay exact (module docstring)
    return tuple(where(still[i], q[i], qn[i]) for i in range(3))


def step(P, states, actions):
    """one env step of states [n, 3] under actions [n, 2] -> dict(value [n, 3], radius [n, 3], undecided [n], collide [n]
    (surely collides), straddle [n] (some margin within its radius, no sure collision), new_value / new_radius [n, 3]
    (the outcome without collision, q_new))"""
    T = table(P)
    s = _f64(states)
    q = tuple(R(s[:, i].copy()) for i in range(3))
    qn = rk4(P, states, actions)
    mv, mr = [], []
    for k in range(NOBS):
        dx, dy = qn[0] - T["c"][k, 0], qn[1] - T["c"][k, 1]
        d = sqrt(fsum([dx * dx, dy * dy]))
        mv.append(d.v - T["r"])
        mr.append(d.r)
    mv, mr = np.stack(mv), np.stack(mr)
    sure = (mv < -mr).any(0)                              # dist + radius < r: every fp32 evaluation collides
    straddle = ~sure & ((mv >= -mr) & (mv < mr)).any(0)   # some dist within its radius of r, none surely below
    out = [where(sure, q[i], qn[i]) for i in range(3)]
    jump = np.zeros(len(s), dtype=bool)
    for i in range(3):
        gap = np.abs(qn[i].v - q[i].v)
        jump |= gap > JUMP * qn[i].r
        out[i] = R(np.where(straddle, 0.5 * (q[i].v + qn[i].v), out[i].v),
                   np.where(straddle, 0.5 * gap + np.maximum(q[i].r, qn[i].r), out[i].r))
    return dict(value=np.stack([c.v for c in out], -1), radius=np.stack([c.r for c in out], -1),
                undecided=straddle & jump, collide=sure, straddle=straddle,
                new_value=np.stack([c.v for c in qn], -1), new_radius=np.stack([c.r for c in qn], -1))


def clamp_hi(x, hi):
    """min(x, hi) of a nonnegative x: exactly hi (radius 0) where every fp32 evaluation of x is at least hi, Lipschitz
    (the radius carries over) elsewhere"""
    above = x.v - x.r >= hi
    return R(np.minimum(x.v, hi), np.where(above, 0.0, x.r))


def reward(states):
    """car2d.py:88-93 on fp32 states [..., >= 2]: 1 - (clip(|q[:2] - xg[:2]|, 0, 0.2) / 0.2)^2 -> R [...]"""
    s = _f64(states)
    dx, dy = R(s[..., 0]) - GOAL[0], R(s[..., 1]) - GOAL[1]
    c = clamp_hi(sqrt(fsum([dx * dx, dy * dy])), REW_CLAMP) / REW_CLAMP
    return 1.0 - c * c


def logpd(traj, xref):
    """car2d.py:95-102 on fp32 trajectories [n, H, >= 2] against xref [href, 2], row min(t, href - 1) at step t:
    0 - mean_t (clip(|x_t - xref_t|, 0, 0.5) / 0.5)^2 -> R [n]"""
    t = _f64(traj)
    H = t.shape[1]
    xr = _f64(xref)[np.minimum(np.arange(H), len(xref) - 1)]
    ex, ey = R(t[..., 0]) - xr[:, 0], R(t[..., 1]) - xr[:, 1]
    c = exact_scale(clamp_hi(sqrt(fsum([ex * ex, ey * ey])), DEMO_CLAMP), 1.0 / DEMO_CLAMP)
    sq = c * c
    return -(fsum([R(sq.v[:, k], sq.r[:, k]) for k in range(H)]) / float(H))


def ratio(got, value, radius, mask=None):
    """largest |got - value| / radius over the masked entries: 0 where equal, inf where the radius is 0 and they differ or
    where `got` is not finite"""
    d = np.abs(np.asarray(got, dtype=np.float64) - value)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(d == 0, 0.0, d / radius)
    q = np.where(np.isfinite(d), q, np.inf)
    if mask is not None:
        q = q[mask]
    return float(q.max()) if q.size else 0.0


def check_rollout(P, x0, Y, out, xref=None):
    """a rollout's outputs out = dict(traj [n, H, 3], rewss [n, H], rews [n], logpd [n]) from x0 ([3] or per sample [n, 3])
    under Y [n, H, 2], checked teacher-forced: step t from the rollout's own traj[:, t - 1], which is the fp32 state the
    kernel carries.  -> dict(largest ratio per output, undecided steps, steps)"""
    Y = np.asarray(Y, dtype=np.float32)
    n, H, _ = Y.shape
    traj = np.asarray(out["traj"], dtype=np.float32)
    start = np.broadcast_to(np.asarray(x0, dtype=np.float32).reshape(-1, 1, 3), (n, 1, 3))
    prev = np.concatenate([start, traj[:, :-1]], 1).reshape(-1, 3)
    ref = step(P, prev, Y.reshape(-1, 2))
    ok = ~ref["undecided"]
    res = dict(undecided=int(ref["undecided"].sum()), steps=n * H)
    res["traj"] = ratio(traj.reshape(-1, 3), ref["value"], ref["radius"], ok)
    if out.get("rewss") is not None:
        rw = reward(traj)
        res["rewss"] = ratio(out["rewss"], rw.v, rw.r)
        ret = mean_return(out["rewss"])
        res["rews"] = ratio(out["rews"], ret.v, ret.r)
    if xref is not None and out.get("logpd") is not None:
        lp = logpd(traj, xref)
        res["logpd"] = ratio(out["logpd"], lp.v, lp.r)
    return res


def held_steps(prev, got, ref):
    """the undecided steps held to one outcome: the frozen state q (an exact input, so taking the collision branch means
    equal bit for bit) or within K radii of q_new.  prev [m, 3] the state before, got [m, 3] the state after, ref = step(P,
    prev, Y) -> (best [u], second [u]) over the u undecided steps: the ratio to the nearer outcome (0 for q itself) and to
    the other one, both in radii of q_new"""
    und = ref["undecided"]
    old = np.asarray(prev, np.float32)[und]
    g = np.asarray(got, np.float32)[und]
    frozen = np.array([np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(g, old)], dtype=bool)
    to_new = np.zeros(len(g))
    for j in range(len(g)):
        to_new[j] = ratio(g[j], ref["new_value"][und][j], ref["new_radius"][und][j])
    to_old = np.zeros(len(g))
    for j in range(len(g)):
        to_old[j] = ratio(g[j], old[j].astype(np.float64), ref["new_radius"][und][j])
    best = np.where(frozen, 0.0, to_new)
    second = np.where(frozen, to_new, to_old)
    return best, second


def check_rollout_branches(P, x0, Y, out):
    """check_rollout's teacher-forced steps with every undecided step held to one branch outcome (held_steps) -> dict(held,
    undecided, unchecked (always 0: both outcomes are known), ratio (largest held), second [per held step])"""
    Y = np.asarray(Y, dtype=np.float32)
    n, H, _ = Y.shape
    traj = np.asarray(out["traj"], dtype=np.float32)
    start = np.broadcast_to(np.asarray(x0, dtype=np.float32).reshape(-1, 1, 3), (n, 1, 3))
    prev = np.concatenate([start, traj[:, :-1]], 1).reshape(-1, 3)
    ref = step(P, prev, Y.reshape(-1, 2))
    best, second = held_steps(prev, traj.reshape(-1, 3), ref)
    return dict(held=len(best), undecided=int(ref["undecided"].sum()), unchecked=0, ratio=float(best.max(initial=0.0)),
                second=second, best=best)
