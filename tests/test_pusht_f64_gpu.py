"""`k_pusht` against the float64 reference of one pushT physics step (tests/pusht_ref.py), without the oracle: one launch per
constructed state (tests/pusht_families.py), NSUB = 1, H = 1, a ragged batch of controls, at mu = 1 and mu = 0 in both
solver modes; the solver's stop in both modes; which solver paths ran; and the rewards of the kernel's own trajectory."""
import numpy as np
import pytest
import torch

import mbd_b200
from mbd_b200 import ops
from mbd_b200.envs.pusht import PT
from tests import pusht_families as F
from tests import pusht_ref as X

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
K = 2.0
MUS = (1.0, 0.0)


def T(a):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device=DEV)


def n_of(fam):
    return 129 if F.FAMILIES.index(fam) % 2 else 77


@pytest.fixture(scope="module")
def cases():
    out = {}
    for mu in MUS:
        P = mbd_b200.envs.get_env("pushT").params.copy()
        P[PT["MU"]] = mu
        for fam in F.FAMILIES:
            out[(mu, fam)] = [(P, st, u, X.step(P, st, u)) for st, u in F.build(fam, n_of(fam))]
    return out


def kernel(P, st, u, mode, iters=None, **kw):
    o = ops.pusht_rollout(T(X.solver_params(P, mode, iters=iters)), T(st), T(u[:, None]), want_final=True)
    return o["final"].cpu().numpy()


@pytest.mark.parametrize("mode", ["fixed", "prod"])
def test_kernel_within_the_float64_bound(cases, mode):
    worst = {}
    for (mu, fam), launches in cases.items():
        und = tot = 0
        for i, (P, st, u, ref) in enumerate(launches):
            got = kernel(P, st, u, mode).astype(np.float64)
            ok = ~ref["undecided"]
            d = np.abs(got - ref["value"])[ok]
            with np.errstate(divide="ignore", invalid="ignore"):
                q = np.where(d == 0, 0.0, d / X.radius(ref, mode)[ok])
            q = float(q.max()) if q.size else 0.0
            worst[(mu, fam)] = max(worst.get((mu, fam), 0.0), q)
            assert q <= K, f"{mode} mu={mu} {fam}[{i}]: {q:.3g} radii"
            und, tot = und + int(ref["undecided"].sum()), tot + len(u)
        assert und <= F.UNDECIDED_CAP[fam] * tot, f"mu={mu} {fam}: {und} of {tot} undecided"
    print(mode, "largest |kernel - f64| / radius:", {k: round(v, 3) for k, v in worst.items()})


def test_fixed_point_and_sweep_cap(cases):
    """TOL = 0: ITERS 4000 and 8000 give the same words unless the sweeps never reach a fixed point; production: a sample
    whose ITERS 100 and 200 words differ hit the 100-sweep cap.  Both fractions are bounded per family and printed."""
    rep, worst_nf = {}, 0.0
    for (mu, fam), launches in cases.items():
        nf = cap = tot = 0
        for P, st, u, ref in launches:
            a = kernel(P, st, u, "fixed")
            moved = (a != kernel(P, st, u, "fixed", iters=8000)).any(1) & ~ref["undecided"]
            nf += int(moved.sum())
            if moved.any():      # the fixed-point radius is not proven for these samples: report how far they are
                d = np.abs(a.astype(np.float64) - ref["value"])[moved]
                with np.errstate(divide="ignore", invalid="ignore"):
                    worst_nf = max(worst_nf, float(np.where(d == 0, 0.0, d / ref["radius"][moved]).max()))
            cap += int((kernel(P, st, u, "prod") != kernel(P, st, u, "prod", iters=200)).any(1).sum())
            tot += len(u)
        rep[(mu, fam)] = (nf, cap, tot)
        assert nf <= F.NOT_FIXED_CAP[fam] * tot, f"mu={mu} {fam}: {nf} of {tot} samples not at a fixed point after 4000 sweeps"
        assert cap <= F.SWEEP_CAP[fam] * tot, f"mu={mu} {fam}: {cap} of {tot} samples hit the 100-sweep cap"
    print("(not at a fixed point after 4000, at the 100-sweep cap, samples):", rep)
    print("largest |kernel - f64| / radius on the samples not at a fixed point:", round(worst_nf, 3))
    assert worst_nf <= K


def test_every_solver_path_runs_on_the_device(cases):
    """the launches above ran the register fast path for both boxes, pt_solve<4>, <8> and <12> through the general branch,
    and the centre-inside branch of both boxes (the reference's diagnostics of the launched states)"""
    paths, inside = {}, set()
    for (mu, fam), launches in cases.items():
        for (_, _, u, ref) in launches:
            paths[ref["path"]] = paths.get(ref["path"], 0) + len(u)
            inside |= set(ref["inside"])
    print("samples per kernel path:", paths, "inside-box branch on boxes", sorted(inside))
    assert set(paths) == set(X.PATHS) and inside == {0, 1}


def test_reward_and_return():
    """at the shipped NSUB = 5 and H = 6: every per-step reward against the float64 reward of the kernel's own state after
    that step, and the return against sum(rewss) / H"""
    env = mbd_b200.envs.get_env("pushT")
    for fam in ("box0", "both", "limits_both", "theta"):
        for st, u in F.build(fam, 77)[:3]:
            Y = np.repeat(u[:, None], 6, 1) * np.float32(0.3) + F.controls(6, 5)[None]
            o = ops.pusht_rollout(env.device_params(), T(st), T(Y), want_traj=True, want_rewss=True)
            traj, rewss, rews = (o[k].cpu().numpy() for k in ("traj", "rewss", "rews"))
            ref = X.reward(traj)
            assert np.all(np.abs(rewss - ref.v) <= K * ref.r), f"{fam}: {np.max(np.abs(rewss - ref.v) / ref.r):.3g} radii"
            ret = X.mean_return(rewss)
            assert np.all(np.abs(rews - ret.v) <= K * ret.r), fam
