"""Constructed car2d inputs for the float64 check of one env step (tests/car2d_ref.py), shared by the CPU and GPU tests.

A one-step family is (states [m, 3] float32, actions [m, 2] float32): every sample has its own start state.  The `demo`
family is a list of rollouts (x0 [3], Y [n, H, 2]) against the shipped 50-row reference path.  The RK4 displacement of a
step depends on theta and the action only, so a start state whose end point lands on a chosen target is the target minus
the float64 displacement, rounded to fp32 (`aim`); the rounding moves the end point by at most half an ulp of the state.
  nominal         states around the planner's region (|x|, |y| <= 1.5, |theta| <= 2 pi), |u| <= 1
  clip            actions exactly +-1, one ulp inside and outside +-1, +-10 and uniform in [-10, 10]
  still           u1 = +0 and -0 (x and y do not move, so the collision predicate sees exact inputs), some with u0 = 0 too
  boundary        end points within 0 .. 32 ulp of an obstacle circle, inside and outside, on the outer rim of the obstacles
  near_boundary   the same at offsets +-1e-6 .. +-1e-2
  lens            end points at and around the crossings of two overlapping circles (centres 0.3 apart, r = 0.3) and inside
                  the lens between them
  inside          starts inside an obstacle with steps that stay inside and steps that leave
  goal            post-step distance to the goal 0 exactly, in (0, 0.2) and straddling 0.2 (still and moving cars)
  far             |x|, |y| from 1e2 to 1e4
  theta           |theta| from 10 to 1e3 (tests/test_fp32_spec.py::test_sincos proves the sine bound up to 1200)
  demo            H = 40, 50 and 60 rollouts from x0, from starts 0.5 from it and near the goal, distances to the
                  reference rows straddling 0.5
"""
from __future__ import annotations

import numpy as np

import mbd_b200
from tests import car2d_ref as X

FAMILIES = ["nominal", "clip", "still", "boundary", "near_boundary", "lens", "inside", "goal", "far", "theta", "demo"]
# largest fraction of undecided samples (steps) per family: the end point straddles a circle and the car moves
UNDECIDED_CAP = {f: 0.0 for f in FAMILIES}
UNDECIDED_CAP["boundary"] = 0.85
UNDECIDED_CAP["lens"] = 0.4
# largest radius of any state word (m, rad) per family: the check must not pass on any plausible value
RADIUS_CAP = {"nominal": 1e-6, "clip": 1e-6, "still": 1e-6, "boundary": 1e-6, "near_boundary": 1e-6, "lens": 1e-6,
              "inside": 1e-6, "goal": 1e-6, "far": 2e-3, "theta": 2e-4, "demo": 1e-6}
# largest radius of a reward (the reward's slope is at most 2 / 0.2 per m)
REWARD_RADIUS_CAP = 2e-6
# on the nominal family 99 % of the radii are below REL_NOMINAL * u * (|q| + |q_new - q|)
REL_NOMINAL = 16.0
SEED = 20
F32 = np.float32


def car():
    return mbd_b200.envs.get_env("car2d")


def aim(P, targets, theta, actions):
    """start states [m, 3] whose float64 RK4 end point under `actions` is `targets` [m, 2], starting at angles `theta`"""
    th = np.asarray(theta, dtype=F32)
    zero = np.zeros((len(th), 3), F32)
    zero[:, 2] = th
    qn = X.rk4(P, zero, actions)
    st = np.stack([targets[:, 0] - qn[0].v, targets[:, 1] - qn[1].v, th.astype(np.float64)], 1)
    return st.astype(F32)


def _moving(rng, m):
    """actions with |u1| >= 0.3 so the car moves 0.09 .. 0.3 m"""
    u = rng.uniform(-1, 1, (m, 2))
    u[:, 1] = np.sign(u[:, 1] + 1e-9) * rng.uniform(0.3, 1.0, m)
    return u.astype(F32)


def _rim(rng, c, r, per):
    """per points on each obstacle circle that are outside every other obstacle by 1e-2 at least, with their obstacle"""
    pts, owner = [], []
    for k in range(len(c)):
        got = 0
        while got < per:
            phi = rng.uniform(0, 2 * np.pi)
            p = c[k] + r * np.array([np.cos(phi), np.sin(phi)])
            if (np.linalg.norm(c - p, axis=1)[np.arange(len(c)) != k] > r + 1e-2).all():
                pts.append(p)
                owner.append(k)
                got += 1
    return np.array(pts), np.array(owner)


def _circle_targets(P, rng, offsets, per):
    T = X.table(P)
    pts, owner = _rim(rng, T["c"], T["r"], per)
    out = []
    for p, k in zip(pts, owner):
        d = (p - T["c"][k]) / np.linalg.norm(p - T["c"][k])
        for off in offsets:
            out.append(T["c"][k] + (T["r"] + off) * d)
    return np.array(out)


def _nominal_states(rng, m):
    return np.stack([rng.uniform(-1.5, 1.5, m), rng.uniform(-1.5, 1.5, m), rng.uniform(-2 * np.pi, 2 * np.pi, m)], 1).astype(F32)


def one_step(family, P=None, seed=SEED):
    """(states [m, 3], actions [m, 2]) of a one-step family; m is never a multiple of 64"""
    P = car().params if P is None else P
    T = X.table(P)
    rng = np.random.default_rng(seed + FAMILIES.index(family))
    ulp = 2.0 ** -25          # one ulp of a distance in [0.25, 0.5)
    if family == "nominal":
        m = 2001
        return _nominal_states(rng, m), rng.uniform(-1, 1, (m, 2)).astype(F32)
    if family == "clip":
        one = F32(1.0)
        vals = np.array([one, np.nextafter(one, F32(0)), np.nextafter(one, F32(2)), F32(10.0)], F32)
        vals = np.concatenate([vals, -vals, np.zeros(1, F32)])
        grid = np.array([(a, b) for a in vals for b in vals], F32)
        u = np.concatenate([grid, grid, rng.uniform(-10, 10, (300, 2)).astype(F32)])
        return _nominal_states(rng, len(u)), u
    if family == "still":
        m = 401
        st = _nominal_states(rng, m)
        u = rng.uniform(-1, 1, (m, 2)).astype(F32)
        u[:, 1] = np.where(np.arange(m) % 2 == 0, F32(0.0), F32(-0.0))
        u[::3, 0] = F32(0.0)
        k = rng.integers(0, X.NOBS, 100)
        rad = rng.uniform(0, T["r"], 100)
        phi = rng.uniform(0, 2 * np.pi, 100)
        st[:100, 0] = T["c"][k, 0] + rad * np.cos(phi)      # some cars parked inside an obstacle
        st[:100, 1] = T["c"][k, 1] + rad * np.sin(phi)
        return st, u
    if family in ("boundary", "near_boundary"):
        if family == "boundary":
            offs = [s * j * ulp for s in (-1, 1) for j in (0, 1, 2, 4, 8, 16, 32)]
        else:
            offs = [s * e for s in (-1, 1) for e in (1e-6, 1e-5, 1e-4, 1e-3, 1e-2)]
        tg = _circle_targets(P, rng, offs, 5)
        u = _moving(rng, len(tg))
        th = rng.uniform(-np.pi, np.pi, len(tg))
        st = aim(P, tg, th, u)
        if len(st) % 64 == 0:
            st, u = st[:-1], u[:-1]
        return st, u
    if family == "lens":
        c, r = T["c"], T["r"]
        tg = []
        for a in range(X.NOBS):
            for b in range(a + 1, X.NOBS):
                dd = np.linalg.norm(c[a] - c[b])
                if dd > 2 * r - 1e-6:
                    continue
                mid, e = 0.5 * (c[a] + c[b]), (c[b] - c[a]) / dd
                nrm = np.array([-e[1], e[0]])
                h = np.sqrt(r * r - 0.25 * dd * dd)
                for sgn in (-1, 1):
                    x = mid + sgn * h * nrm              # a crossing of the two circles
                    for off in (0.0, ulp, 4 * ulp, 1e-6, 1e-4, 1e-2):
                        for _ in range(3):
                            phi = rng.uniform(0, 2 * np.pi)
                            tg.append(x + off * np.array([np.cos(phi), np.sin(phi)]))
                    for t in (0.1, 0.5, 0.9, 0.99):       # inside the lens, on its axis
                        tg.append(mid + sgn * t * h * nrm)
        tg = np.array(tg)
        u = _moving(rng, len(tg))
        return aim(P, tg, rng.uniform(-np.pi, np.pi, len(tg)), u), u
    if family == "inside":
        m = 501
        k = rng.integers(0, X.NOBS, m)
        rad = rng.uniform(0, 0.28, m)
        phi = rng.uniform(0, 2 * np.pi, m)
        st = np.stack([T["c"][k, 0] + rad * np.cos(phi), T["c"][k, 1] + rad * np.sin(phi), rng.uniform(-np.pi, np.pi, m)], 1)
        return st.astype(F32), _moving(rng, m)
    if family == "goal":
        g = np.array(X.GOAL)
        ds = [0.0, 1e-7, 1e-3, 0.05, 0.1, 0.15, 0.199, 0.2 - 1e-6, 0.2, 0.2 + 1e-6, 0.201, 0.21, 0.25]
        tg = np.array([g + d * np.array([np.cos(p), np.sin(p)]) for d in ds for p in rng.uniform(-1.5, 1.5, 12)])
        tiny = F32(2.0 ** -26)
        exact = np.array([[0.5, 0.0], [np.nextafter(F32(0.5), F32(1)), 0.0], [np.nextafter(F32(0.5), F32(0)), 0.0],
                          [0.5, tiny], [0.5, -tiny], [0.5, 0.2], [0.3125, 0.0], [0.7, 0.0], [0.5, np.nextafter(F32(0.2), F32(1))]])
        still = np.concatenate([exact, tg]).astype(F32)
        su = rng.uniform(-1, 1, (len(still), 2)).astype(F32)
        su[:, 1] = 0.0
        sst = np.concatenate([still, rng.uniform(-np.pi, np.pi, (len(still), 1))], 1).astype(F32)
        mu = _moving(rng, len(tg))
        mst = aim(P, tg, rng.uniform(-np.pi, np.pi, len(tg)), mu)
        return np.concatenate([sst, mst]), np.concatenate([su, mu])
    if family == "far":
        m = 601
        mag = 10.0 ** rng.uniform(2, 4, (m, 2)) * rng.choice([-1, 1], (m, 2))
        st = np.concatenate([mag, rng.uniform(-np.pi, np.pi, (m, 1))], 1).astype(F32)
        return st, rng.uniform(-1.5, 1.5, (m, 2)).astype(F32)
    if family == "theta":
        m = 601
        st = _nominal_states(rng, m)
        st[:, 2] = (10.0 ** rng.uniform(1, 3, m) * rng.choice([-1, 1], m)).astype(F32)
        return st, rng.uniform(-1.5, 1.5, (m, 2)).astype(F32)
    raise ValueError(family)


def rollouts(P=None, xref=None, n=33, seed=SEED):
    """the demo family: [(x0 [3], Y [n, H, 2])] for H = 40, 50, 60, from x0 = xref[0], from starts 0.5 away from it and
    from starts near the goal, with slow and with saturated (|u| > 1) actions"""
    env = car()
    xref = env.xref if xref is None else xref
    rng = np.random.default_rng(seed + FAMILIES.index("demo"))
    starts = [env.x0] + [np.array([xref[0, 0] + 0.5 * np.cos(p), xref[0, 1] + 0.5 * np.sin(p), p], F32)
                         for p in (2.9, 3.1, 3.4)]     # the free side of the start: the others are in the obstacles
    starts += [np.array([0.45, 0.05, 1.0], F32), np.array([0.5, -0.1, -2.0], F32)]     # near the goal: nonzero rewards
    scale = (1.3, 0.4, 1.3, 0.4, 0.4, 0.2)
    out = []
    for H in (40, 50, 60):
        for i, x0 in enumerate(starts):
            Y = rng.normal(size=(n, H, 2)) * scale[i]
            out.append((np.asarray(x0, F32), Y.astype(F32)))
    return out
