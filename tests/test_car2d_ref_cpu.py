"""The CPU oracle's car2d step, reward, return and demo log-density against the float64 reference with a radius per value
(tests/car2d_ref.py), on the constructed families of tests/car2d_families.py.  No GPU needed.

Bit equality between `k_car2d` and the oracle shows that they agree; this file shows that the oracle computes the upstream
step (DESIGN.md §2, "Accuracy contract of the car2d step"): every value within K radii, the bound tight enough to matter,
and a numpy fp32 mirror of the step that meets the bound unmutated and leaves it under each deliberate mistake."""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import car2d_families as F
from tests import car2d_ref as X

K = 2.0
f32 = np.float32


@pytest.fixture(scope="module")
def cases():
    """{family: [(x0 [3] or per sample [m, 3], Y [m, H, 2], xref or None)]}"""
    env = F.car()
    out = {}
    for fam in F.FAMILIES[:-1]:
        st, u = F.one_step(fam, env.params)
        out[fam] = [(st, u[:, None], None)]
    out["demo"] = [(x0, Y, env.xref) for x0, Y in F.rollouts(env.params, env.xref)]
    return out


def oracle_run(P, x0, Y, xref=None):
    """orc.car2d_rollout, one call per distinct start state where every sample has its own"""
    if np.ndim(x0) == 1:
        return orc.car2d_rollout(P, x0, Y, xref=xref, want_rewss=True, want_traj=True)
    n, H, _ = Y.shape
    out = dict(traj=np.zeros((n, H, 3), f32), rewss=np.zeros((n, H), f32), rews=np.zeros(n, f32), logpd=None)
    uniq, inv = np.unique(x0, axis=0, return_inverse=True)
    for j, s in enumerate(uniq):
        idx = np.flatnonzero(inv.reshape(-1) == j)
        o = orc.car2d_rollout(P, s, Y[idx], want_rewss=True, want_traj=True)
        for k in ("traj", "rewss", "rews"):
            out[k][idx] = o[k]
    return out


def evaluate(cases, run, P=None):
    """{family: (largest ratio per output, undecided steps, steps)} of the outputs `run(P, x0, Y, xref)`"""
    P = F.car().params if P is None else P
    rep = {}
    for fam, launches in cases.items():
        worst, und, tot = {}, 0, 0
        for x0, Y, xref in launches:
            res = X.check_rollout(P, x0, Y, run(P, x0, Y, xref), xref)
            und, tot = und + res.pop("undecided"), tot + res.pop("steps")
            for k, v in res.items():
                worst[k] = max(worst.get(k, 0.0), v)
        rep[fam] = (worst, und, tot)
    return rep


def test_oracle_within_the_bound(cases):
    rep = evaluate(cases, oracle_run)
    for fam, (worst, und, tot) in rep.items():
        print(f"{fam:14s} largest |oracle - f64| / radius {({k: round(v, 3) for k, v in worst.items()})}  undecided "
              f"{und}/{tot} = {und / tot:.3f}")
        assert und <= F.UNDECIDED_CAP[fam] * tot, f"{fam}: {und} of {tot} steps undecided"
        for k, v in worst.items():
            assert v <= K, f"{fam} {k}: |oracle - value| = {v:.3g} radii"
    assert max(max(w.values()) for w, _, _ in rep.values()) > 0.5      # the radius is not simply huge


def test_the_bound_is_not_vacuous(cases):
    """every radius is finite and below its family's cap, every reward radius below REWARD_RADIUS_CAP; on the nominal
    family 99 % of the radii are within REL_NOMINAL u of |q| + |q_new - q|; the boundary and lens families have undecided
    samples and decided ones on both sides of the predicate, the near-boundary, inside and lens families both outcomes; the
    demo rows straddle 0.5"""
    P = F.car().params
    for fam, launches in cases.items():
        for x0, Y, xref in launches:
            o = oracle_run(P, x0, Y, xref)
            start = np.broadcast_to(np.reshape(x0, (-1, 1, 3)), (Y.shape[0], 1, 3))
            prev = np.concatenate([start, o["traj"][:, :-1]], 1).reshape(-1, 3)
            ref = X.step(P, prev, Y.reshape(-1, 2))
            ok = ~ref["undecided"]
            r = ref["radius"][ok]
            assert np.isfinite(r).all() and r.max() <= F.RADIUS_CAP[fam], f"{fam}: radius {r.max():.3g}"
            rw = X.reward(o["traj"])
            assert np.isfinite(rw.r).all() and rw.r.max() <= F.REWARD_RADIUS_CAP, (fam, rw.r.max())
            if fam == "nominal":
                q = prev.astype(np.float64)
                rel = ref["radius"] / (X.U * (np.abs(q) + np.abs(ref["value"] - q)))
                assert np.percentile(rel[ok], 99) < F.REL_NOMINAL, np.percentile(rel[ok], 99)
            if fam in ("boundary", "lens"):
                assert ref["undecided"].any(), fam
                assert (ref["collide"] & ok).any() and (~ref["collide"] & ~ref["straddle"]).any(), fam
            if fam in ("near_boundary", "inside", "lens"):
                assert 0.2 < ref["collide"].mean() < 0.95, (fam, ref["collide"].mean())
            if fam == "demo":
                rows = xref[np.minimum(np.arange(Y.shape[1]), len(xref) - 1)]
                d = np.linalg.norm(o["traj"][..., :2] - rows, axis=-1)
                assert (d < 0.5).any() and (d > 0.5).any()


# ---------------------------------------------------------------------------------------------------------------------
# a numpy fp32 mirror of the rollout with deliberate mistakes: the bound must catch each on the family named with it
# ---------------------------------------------------------------------------------------------------------------------
MUTATIONS = {
    "rk4_weights_1111": "nominal",       # k1 + k2 + k3 + k4 instead of k1 + 2 k2 + 2 k3 + k4
    "k4_at_half_step": "nominal",        # k4 = f(x + dt/2 k3)
    "sin_cos_swapped": "nominal",
    "turn_rate_pi_3": "nominal",         # u0 pi / 3 instead of u0 pi / 3 * 2
    "speed_factor_dropped": "nominal",
    "clip_dropped": "clip",
    "collide_on_old_state": "near_boundary",
    "select_inverted": "nominal",
    "last_obstacle_dropped": "near_boundary",
    "radius_0.29": "near_boundary",
    "reward_goal_sign": "goal",          # goal (-0.5, 0)
    "reward_clamp_0.25": "goal",
    "logpd_row_t_plus_1": "demo",
    "logpd_clamp_0.2": "demo",
    "return_over_H_minus_1": "demo",
}


def mirror(mut=None):
    def run(P, x0, Y, xref=None):
        P = np.asarray(P, f32)
        c, r, dt, hdt, sdt = P[:22].reshape(11, 2), P[22], P[23], P[24], P[25]
        if mut == "last_obstacle_dropped":
            c = c[:-1]
        if mut == "radius_0.29":
            r = f32(0.29)
        n, H, _ = Y.shape
        q = np.broadcast_to(np.asarray(x0, f32).reshape(-1, 3), (n, 3)).copy()

        def rates(x, u):
            s, co = (np.sin(x[:, 2].astype(np.float64)).astype(f32), np.cos(x[:, 2].astype(np.float64)).astype(f32))
            if mut == "sin_cos_swapped":
                s, co = co, s
            v = f32(1.0) if mut == "speed_factor_dropped" else f32(3.0)
            w = u[:, 0] * f32(np.pi) / f32(3.0)
            if mut != "turn_rate_pi_3":
                w = w * f32(2.0)
            return np.stack([u[:, 1] * s * v, u[:, 1] * co * v, w], 1)

        traj, rewss = np.zeros((n, H, 3), f32), np.zeros((n, H), f32)
        acc = np.zeros(n, f32)
        for t in range(H):
            u = Y[:, t] if mut == "clip_dropped" else np.clip(Y[:, t], f32(-1), f32(1))
            k1 = rates(q, u)
            k2 = rates(q + hdt * k1, u)
            k3 = rates(q + hdt * k2, u)
            k4 = rates(q + (hdt if mut == "k4_at_half_step" else dt) * k3, u)
            two = f32(1.0) if mut == "rk4_weights_1111" else f32(2.0)
            qn = q + sdt * (((k1 + two * k2) + two * k3) + k4)
            at = q if mut == "collide_on_old_state" else qn
            dd = at[:, None, :2] - c[None]
            col = (np.sqrt(dd[..., 0] * dd[..., 0] + dd[..., 1] * dd[..., 1]) < r).any(1)
            if mut == "select_inverted":
                col = ~col
            q = np.where(col[:, None], q, qn)
            gx = f32(-0.5) if mut == "reward_goal_sign" else f32(0.5)
            e0, e1 = q[:, 0] - gx, q[:, 1] - f32(0.0)
            cc = np.clip(np.sqrt(e0 * e0 + e1 * e1), f32(0), f32(0.25) if mut == "reward_clamp_0.25" else f32(0.2)) / f32(0.2)
            rewss[:, t] = f32(1.0) - cc * cc
            traj[:, t] = q
            if xref is not None:
                row = min(t + 1 if mut == "logpd_row_t_plus_1" else t, len(xref) - 1)
                x0_, x1_ = q[:, 0] - xref[row, 0], q[:, 1] - xref[row, 1]
                c2 = np.clip(np.sqrt(x0_ * x0_ + x1_ * x1_), f32(0), f32(0.2) if mut == "logpd_clamp_0.2" else f32(0.5)) / f32(0.5)
                acc = acc + c2 * c2
        with np.errstate(divide="ignore", invalid="ignore"):
            rews = rewss.sum(1, dtype=f32) / f32(H - 1 if mut == "return_over_H_minus_1" else H)
        logpd = (f32(0.0) - acc / f32(H)) if xref is not None else None
        return dict(traj=traj, rewss=rewss, rews=rews, logpd=logpd)
    return run


def test_unmutated_mirror_meets_the_bound(cases):
    for fam, (worst, und, tot) in evaluate(cases, mirror()).items():
        assert und <= F.UNDECIDED_CAP[fam] * tot, fam
        assert max(worst.values()) <= K, (fam, worst)


@pytest.mark.parametrize("mut", list(MUTATIONS))
def test_every_mistake_leaves_the_bound(cases, mut):
    with np.errstate(over="ignore", invalid="ignore"):
        rep = evaluate(cases, mirror(mut))
    caught = {fam: round(max(w.values()), 1) for fam, (w, _, _) in rep.items() if max(w.values()) > K}
    print(mut, "caught on", caught)
    assert MUTATIONS[mut] in caught, f"{mut}: not caught on {MUTATIONS[mut]} (caught on {sorted(caught)})"
