"""Every rollout kernel's undecided samples held to one of their branch outcomes (tests/test_branches_ref_cpu.py), without
the oracle:
* the XPBD kernels through the (model, variant) cases of tests/test_xpbd_f64_gpu.py at n = 1, 77, 129 and 16 x SMs + 37:
  the substep chain on every family state, each undecided substep held to K radii of one consistent assignment of its
  gated predicates (tests/xpbd_ref.py `branch_outcomes`, memoised with the float64 step in horizon_ref.StepMemo);
* the same kernels along the horizon: the relaunched substeps of a few env steps of the env-step chain;
* `k_car2d` from x0 and family starts and from undecided rim states, and `k_car2d_ps` on every constructed one-step family: an undecided step equals the
  frozen state bit for bit or lies within K radii of q_new;
* `k_pusht` on every pushT family at mu = 1 and 0 in both solver modes: within K radii of one enumerated configuration.
The per-env-state kernels `k_rollout<PerEnv>`, `k_rollout_wpl<PerEnv>` and `k_pusht_ps` step a whole env step; they equal the broadcast
kernels above bit for bit from the same state (tests/test_horizon_f64_gpu.py), so these checks hold them too."""
import numpy as np
import pytest
import torch

import mbd_b200
from mbd_b200 import ops
from mbd_b200.envs.pusht import PT
from mbd_b200.envs.vec import VecEnv
from mbd_b200.model import blob as B
from tests import car2d_families as CF
from tests import car2d_ref as CX
from tests import horizon_ref as HR
from tests import pusht_families as PF
from tests import pusht_ref as PX
from tests import xpbd_families as F
from tests.test_horizon_f64_gpu import RELAUNCH_STEPS, _cases_with_n, _rows, big_n, kernel_run, sms
from tests.test_horizon_ref_cpu import HORIZON_MODELS, horizon_actions, horizon_starts
from tests.test_xpbd_f64_gpu import launched_kernel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
K = 2.0
UNCHECKED_CAP = 0.0      # measured 0 on every case (tests/test_branches_ref_cpu.py)
HELD = {}                # (kernel, family) -> (undecided, largest held ratio), printed at the end


def T(a):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device=DEV)


def _note(kernel, fam, und, q):
    a = HELD.get((kernel, fam), (0, 0.0))
    HELD[(kernel, fam)] = (a[0] + und, max(a[1], q))


@pytest.fixture(scope="module")
def memo():
    return HR.StepMemo()


@pytest.mark.parametrize("name,variant,n", _cases_with_n())
def test_xpbd_kernel_undecided_held(tmp_path, memo, name, variant, n):
    env = F.make_env(name, tmp_path)
    n = big_n() if n == "big" else n
    m = env.device_model(torch.device(DEV))
    kern = launched_kernel(env.blob, variant, n, sms())
    run = kernel_run(m, 0)
    nsub = int(env.blob.view(np.int32)[3])
    ops.set_kernel_variant(variant)
    try:
        for fam in (F.FAMILIES if n <= 129 else ["F1", "F5"]):
            und = unc = 0
            for i, (st, u) in enumerate(F.build(env, fam, max(n, 8))):
                u = u[:n]
                ch = HR.substep_chain(run, st, u, nsub)
                rows = _rows(n) if n > 129 else np.arange(n)
                prev = np.concatenate([c[rows] for c in ch[:-1]])
                got = np.concatenate([c[rows] for c in ch[1:]])
                _, q, c, info = HR.step_ratios(memo, env.blob, prev, np.tile(u[rows], (nsub, 1)), got)
                assert q <= K, f"{name} v{variant} n={n} {fam}[{i}]: best assignment {q:.3g} radii"
                und, unc = und + info["undecided"], unc + c
                _note(kern, fam, info["undecided"], q)
            assert unc <= UNCHECKED_CAP * und, f"{name} v{variant} n={n} {fam}: {unc} of {und} undecided substeps unchecked"
    finally:
        ops.set_kernel_variant(0)


@pytest.mark.parametrize("name,variant,n", [c for c in _cases_with_n(HORIZON_MODELS) if c[2] != "big"])
def test_xpbd_kernel_relaunched_horizon_undecided_held(tmp_path, memo, name, variant, n):
    """along the horizon, where most undecided substeps are (the humanoids and gen0 on the floor): from the first two starts
    of tests/test_horizon_f64_gpu.py, the last sample's env steps RELAUNCH_STEPS relaunched one substep at a time from the
    loop's own state, each substep held to its branch outcomes"""
    env = F.make_env(name, tmp_path)
    m = env.device_model(torch.device(DEV))
    kern = launched_kernel(env.blob, variant, n, sms())
    blob = env.blob
    run = kernel_run(m, int(blob.view(np.int32)[B.H_NTRACK]))
    nsub = int(blob.view(np.int32)[3])
    xref = env.xref if name == "humanoidtrack" else None
    ops.set_kernel_variant(variant)
    try:
        und = unc = 0
        for si, (label, st, xr) in enumerate(horizon_starts(env, name, run, xref)[:2]):
            Y = horizon_actions(env.action_size, n, 50, 1000 + si)
            _, traj = HR.env_step_chain(run, st, Y, xr)
            ok = HR.finite_samples(traj)
            if not ok.any():
                continue
            b = int(np.flatnonzero(ok)[-1])
            prev = HR.previous_states(st, traj)
            for t in RELAUNCH_STEPS:
                ch = HR.relaunch_chain(run, prev[b, t], Y[b, t], nsub)
                assert HR.same_bits(ch[-1], traj[b, t]), f"{name} v{variant} n={n} {label}: substeps of env step {t}"
                _, q, c, info = HR.step_ratios(memo, blob, np.stack(ch[:-1]), np.tile(Y[b, t], (nsub, 1)), np.stack(ch[1:]))
                assert q <= K, f"{name} v{variant} n={n} {label} step {t}: best assignment {q:.3g} radii"
                und, unc = und + info["undecided"], unc + c
                _note(kern, "horizon relaunch", info["undecided"], q)
        assert unc <= UNCHECKED_CAP * und, f"{name} v{variant} n={n}: {unc} of {und} undecided substeps unchecked"
    finally:
        ops.set_kernel_variant(0)


def _car_starts(car):
    return [car.x0, CF.one_step("inside", car.params)[0][0], CF.one_step("boundary", car.params)[0][0],
            CF.one_step("lens", car.params)[0][0], np.float32([0.45, 0.05, 1.0])]


@pytest.mark.parametrize("n", [1, 77, 4096])
def test_k_car2d_undecided_held(n):
    """random rollouts from five starts, and a launch from each of the first undecided rim-family states with its own
    action in every sample (random actions seldom end a step on a circle, so that launch keeps the test from passing
    vacuously)"""
    car = CF.car()
    params, xref = car.device_params()
    rng = np.random.default_rng(n)
    st, u = CF.one_step("boundary", car.params)
    seen = 0
    for i in np.flatnonzero(CX.step(car.params, st, u)["undecided"])[:4]:
        Y = np.broadcast_to(u[i], (n, 1, 2)).copy()
        o = ops.car2d_rollout(params, T(st[i]), T(Y), xref=xref, want_rewss=True, want_traj=True)
        res = CX.check_rollout_branches(car.params, st[i], Y, dict(traj=o["traj"].cpu().numpy()))
        _note("k_car2d", "rim", res["undecided"], res["ratio"])
        seen += res["undecided"]
        assert res["ratio"] <= K, f"n={n} rim state {i}: {res['ratio']:.3g} radii from both outcomes"
    assert seen >= n
    for H in (1, 50):
        for i, x0 in enumerate(_car_starts(car)):
            Y = (rng.normal(size=(n, H, 2)) * 1.3).astype(np.float32)
            o = ops.car2d_rollout(params, T(x0), T(Y), xref=xref, want_rewss=True, want_traj=True)
            res = CX.check_rollout_branches(car.params, x0, Y, dict(traj=o["traj"].cpu().numpy()))
            _note("k_car2d", f"start {i}", res["undecided"], res["ratio"])
            assert res["ratio"] <= K, f"n={n} H={H} start {i}: {res['ratio']:.3g} radii from both outcomes"


def test_k_car2d_ps_undecided_held():
    car = CF.car()
    seen = 0
    for fam in CF.FAMILIES[:-1]:
        st, u = CF.one_step(fam, car.params)
        venv = VecEnv(car, len(st))
        venv.set_state(st)
        raw = venv.step(T(u)).raw.cpu().numpy().copy()
        res = CX.check_rollout_branches(car.params, st, u[:, None], dict(traj=raw[:, None]))
        _note("k_car2d_ps", fam, res["undecided"], res["ratio"])
        seen += res["undecided"]
        assert res["ratio"] <= K, f"{fam}: {res['ratio']:.3g} radii from both outcomes"
    assert seen > 0


@pytest.mark.parametrize("mode", ["fixed", "prod"])
def test_k_pusht_undecided_held(mode):
    seen = 0
    for mu in (1.0, 0.0):
        P = mbd_b200.envs.get_env("pushT").params.copy()
        P[PT["MU"]] = mu
        for fam in PF.FAMILIES:
            n = 129 if PF.FAMILIES.index(fam) % 2 else 77
            for i, (st, u) in enumerate(PF.build(fam, n)):
                ref = PX.step(P, st, u)
                if not ref["undecided"].any():
                    continue
                o = ops.pusht_rollout(T(PX.solver_params(P, mode)), T(st), T(u[:, None]), want_final=True)
                b, _ = PX.held_ratios(o["final"].cpu().numpy(), ref, mode)
                seen += len(b)
                _note(f"k_pusht {mode}", f"mu={mu} {fam}", len(b), float(b.max()))
                assert b.max() <= K, f"{mode} mu={mu} {fam}[{i}]: {b.max():.3g} radii from every configuration"
    assert seen > 0


def test_report():
    print("(kernel, family): (undecided, largest held ratio)")
    for k, v in sorted(HELD.items(), key=str):
        if v[0]:
            print(f"  {k}: {v[0]}, {v[1]:.3f}")
