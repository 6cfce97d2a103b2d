"""Batched solves without a device: mbd_batch_step_launch refuses bad arguments before any CUDA call (with a message),
run_diffusion_batch checks its Args before touching the device, and the run_mbd sweep driver parses the reference's flags."""
import ctypes

import pytest

from mbd_b200 import _lib
from mbd_b200.planners.mbd_planner import Args, run_diffusion_batch

FAKE = 0x1000   # never dereferenced: every case below fails validation, which runs before the first CUDA call


def _plan(**kw):
    """a car2d plan that passes every check except the one a test breaks"""
    p = _lib.StepPlan()
    for f in ("car_params_dev", "state_init_dev", "params_dev", "ctl_dev", "Ybars_dev", "Y0s_dev", "rews_dev", "rews_all_dev",
              "logp_dev", "weights_dev", "runs_dev", "partial_dev", "scalars_dev"):
        setattr(p, f, FAKE)
    p.n_total, p.n_begin, p.n_local, p.H, p.nu, p.P, p.rank, p.temp = 64, 0, 64, 40, 2, 1, 0, 0.1
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _reject(p, B=4, Nd=10):
    L = _lib.lib()
    rc = L.mbd_batch_step_launch(ctypes.byref(p), B, Nd, None, None)
    return rc, L.mbd_last_error().decode()


@pytest.mark.parametrize("kw,B,Nd,msg", [
    ({}, 0, 10, "B must be at least 1"),
    ({}, -3, 10, "B must be at least 1"),
    ({}, 4, 1, "Ndiffuse must be at least 2"),
    ({"P": 2, "peer_base_ptrs": ctypes.cast(FAKE, ctypes.POINTER(ctypes.c_uint64))}, 4, 10, "P must be 1"),
    ({"n_local": 32}, 4, 10, "n_local == n_total"),
    ({"n_begin": 32, "n_local": 32}, 4, 10, "n_local == n_total"),
    ({"H": 4000, "nu": 2}, 4, 10, "H * Nu exceeds 27 * 256 columns"),
    ({"state_init_dev": None}, 4, 10, "state_init must be set"),
    ({"ctl_dev": None}, 4, 10, "params / ctl / Ybars must be set"),
    ({"weights_dev": None}, 4, 10, "a work buffer is NULL"),
    ({"nu": 3}, 4, 10, "nu == 2"),
    ({"car_params_dev": None}, 4, 10, "needs car_params"),
    ({"env_kind": _lib.ENV_PUSHT, "xref_dev": FAKE, "href": 5, "logpd_dev": FAKE, "logpd_all_dev": FAKE}, 4, 10,
     "pushT has no demonstration"),
    ({"n_total": 1 << 20, "n_local": 1 << 20, "H": 100, "nu": 2}, 16, 10, "below 2^31"),
], ids=["B0", "Bneg", "Nd1", "P2", "nlocal", "nbegin", "columns", "state", "ctl", "weights", "nu", "carparams", "pusht-demo",
        "index-range"])
def test_batch_launch_rejects_with_message(kw, B, Nd, msg):
    rc, err = _reject(_plan(**kw), B, Nd)
    assert rc == -1, (rc, err)
    assert err.startswith("mbd_batch_step_launch: ") and msg in err, err


def test_null_plan_rejected():
    L = _lib.lib()
    assert L.mbd_batch_step_launch(None, 2, 10, None, None) == -1
    assert "plan is NULL" in L.mbd_last_error().decode()


def _args(**kw):
    base = dict(env_name="car2d", Nsample=64, Hsample=40, Ndiffuse=10, not_render=True, disable_recommended_params=True)
    base.update(kw)
    return Args(**base)


@pytest.mark.parametrize("field,value", [("env_name", "pushT"), ("Nsample", 128), ("Hsample", 30), ("Ndiffuse", 20),
                                         ("enable_demo", True)])
def test_batch_fields_must_agree(field, value):
    args = [_args(seed=0), _args(seed=1), _args(seed=2, **{field: value})]
    with pytest.raises(ValueError, match=f"same {field}"):
        run_diffusion_batch(args)


def test_batch_requires_not_render():
    with pytest.raises(ValueError, match="not_render"):
        run_diffusion_batch([_args(seed=0), _args(seed=1, not_render=False)])


def test_batch_refuses_multiple_ranks(monkeypatch):
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(ValueError, match="WORLD_SIZE"):
        run_diffusion_batch([_args(seed=0), _args(seed=1)])


def test_batch_recommended_params_applied_before_the_check():
    """apply_recommended_params runs per Args first: humanoidrun's Nsample override makes 16 and 8192 agree"""
    a = [Args(env_name="humanoidrun", Nsample=16, not_render=True), Args(env_name="humanoidrun", seed=1, not_render=False)]
    with pytest.raises(ValueError, match="not_render"):
        run_diffusion_batch(a)
    assert a[0].Nsample == a[1].Nsample == 8192


def test_batch_varying_fields_are_allowed_by_the_check():
    from mbd_b200.planners.mbd_planner import check_batch_args
    check_batch_args([_args(seed=0, temp_sample=0.1, beta0=1e-4, betaT=1e-2), _args(seed=5, temp_sample=0.4, beta0=2e-4, betaT=2e-2)])


def test_run_mbd_args_tyro():
    import tyro
    from mbd_b200.scripts import run_mbd
    a = tyro.cli(run_mbd.Args, args=["--algo", "path_integral", "--update_method", "cma-es", "--mode", "temp", "--env_name", "hopper"])
    assert (a.algo, a.update_method, a.mode, a.env_name) == ("path_integral", "cma-es", "temp", "hopper")
    d = tyro.cli(run_mbd.Args, args=[])
    assert (d.algo, d.update_method, d.mode, d.env_name) == ("mbd", "mppi", "seed", "ant")


def test_run_mbd_sweeps_match_the_reference():
    from mbd_b200.scripts import run_mbd
    s = run_mbd.seed_args(run_mbd.Args(env_name="hopper"))
    assert [a.seed for a in s] == list(range(8)) and all(a.not_render and a.env_name == "hopper" for a in s)
    t = run_mbd.temp_args(run_mbd.Args(env_name="hopper"))
    assert [a.temp_sample for a in t] == [0.01, 0.03, 0.06, 0.1, 0.2, 0.4, 0.6, 0.8]
    assert all(a.seed == 0 and a.disable_recommended_params and a.not_render for a in t)
    with pytest.raises(ValueError, match="mode"):
        run_mbd.main(["--mode", "neither"])
