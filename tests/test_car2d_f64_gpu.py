"""The car2d kernels against the float64 reference of one env step, its reward, the return and the demo log-density
(tests/car2d_ref.py), without the oracle:
* `k_car2d` (`ops.car2d_rollout`) at n = 1, 77 and 4096 (a ragged last CTA) and H = 1, 40, 50 and 60 against the 50-row
  reference path, from x0 and from family states, every step checked teacher-forced from the kernel's own trajectory;
* `k_car2d` with in-kernel sampling (n_begin > 0, nonzero Ybar and sigma), the actions read back from the Y0s it wrote;
* `k_car2d_ps` through `VecEnv("car2d", B)`: every constructed one-step family (tests/car2d_families.py) as one ragged
  batch of per-sample states."""
import numpy as np
import pytest
import torch

from mbd_b200 import ops
from mbd_b200.envs.vec import VecEnv
from tests import car2d_families as F
from tests import car2d_ref as X

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
K = 2.0
UNDECIDED_ROLLOUT = 1e-4     # random rollouts end a step within the predicate's radius of a circle about once per 1e6 steps


def T(a):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device=DEV)


def _starts(car):
    """x0, and one state of the inside, far, theta and near-goal kinds"""
    return [car.x0, F.one_step("inside", car.params)[0][0], F.one_step("far", car.params)[0][0],
            F.one_step("theta", car.params)[0][3], np.float32([0.45, 0.05, 1.0])]


def _assert_within(res, what):
    und, steps = res.pop("undecided"), res.pop("steps")
    assert und <= UNDECIDED_ROLLOUT * steps, f"{what}: {und} of {steps} steps undecided"
    for k, v in res.items():
        assert v <= K, f"{what} {k}: |kernel - f64| = {v:.3g} radii"
    return max(res.values())


def _host(o):
    return {k: (None if v is None else v.cpu().numpy()) for k, v in o.items()}


@pytest.mark.parametrize("n", [1, 77, 4096])
def test_k_car2d_within_the_float64_bound(n):
    car = F.car()
    params, xref = car.device_params()
    rng = np.random.default_rng(n)
    worst = 0.0
    for H in (1, 40, 50, 60):
        for i, x0 in enumerate(_starts(car)):
            Y = (rng.normal(size=(n, H, 2)) * 1.3).astype(np.float32)       # |u| > 1 on a fifth of the words
            o = _host(ops.car2d_rollout(params, T(x0), T(Y), xref=xref, want_rewss=True, want_traj=True))
            worst = max(worst, _assert_within(X.check_rollout(car.params, x0, Y, o, car.xref), f"n={n} H={H} start {i}"))
    print(f"k_car2d n={n}: largest |kernel - f64| / radius {worst:.3f}")


@pytest.mark.parametrize("n", [77, 4096])
def test_k_car2d_fused_sampling_within_the_float64_bound(n):
    car = F.car()
    params, xref = car.device_params()
    worst = 0.0
    for H in (40, 60):
        for i, x0 in enumerate(_starts(car)[:3]):
            Ybar = (0.6 * np.sin(np.arange(2 * H) * 0.37)).astype(np.float32)
            Y0s = torch.empty((n, H, 2), device=DEV)
            o = _host(ops.car2d_rollout(params, T(x0), Y0s, xref=xref, want_rewss=True, want_traj=True, key=np.uint32([7, i]),
                                        n_total=n + 64 + 5, n_begin=64, sigma=0.8, Ybar=T(Ybar)))
            Y = Y0s.cpu().numpy()
            # the sampler clips to [-1, 1]; the draws reach the clip and follow Ybar
            assert (np.abs(Y) <= 1).all() and (np.abs(Y) == 1).any()
            assert np.corrcoef(Y.mean(0).ravel(), Ybar)[0, 1] > 0.8
            worst = max(worst, _assert_within(X.check_rollout(car.params, x0, Y, o, car.xref), f"fused n={n} H={H} start {i}"))
    print(f"k_car2d fused n={n}: largest |kernel - f64| / radius {worst:.3f}")


def test_vecenv_step_within_the_float64_bound():
    """k_car2d_ps: every family as one batch of per-sample states; raw state against `step`, the reward against `reward`"""
    car = F.car()
    rep = {}
    for fam in F.FAMILIES[:-1]:
        st, u = F.one_step(fam, car.params)
        B = len(st)
        assert B % 64, fam
        venv = VecEnv(car, B)
        venv.set_state(st)
        s = venv.step(T(u))
        raw, rew = s.raw.cpu().numpy().copy(), s.reward.cpu().numpy().copy()
        res = X.check_rollout(car.params, st, u[:, None], dict(traj=raw[:, None], rewss=rew[:, None], rews=rew))
        und, steps = res.pop("undecided"), res.pop("steps")
        rep[fam] = ({k: round(v, 3) for k, v in res.items()}, und, steps)
        assert und <= F.UNDECIDED_CAP[fam] * steps, f"{fam}: {und} of {steps} undecided"
        for k, v in res.items():
            assert v <= K, f"{fam} {k}: |kernel - f64| = {v:.3g} radii"
    for fam, (w, und, steps) in rep.items():
        print(f"k_car2d_ps {fam:14s} largest |kernel - f64| / radius {w}  undecided {und}/{steps}")
