"""Batched path-integral solves without a device: mbd_pi_batch_step_launch refuses bad arguments before any CUDA call (with a
message), run_path_integral_batch checks its Args before touching the device, mbd_pi_bufs is 24 bytes, a CEM index row holds the
picks and their count, and run_mbd's --pi_batch builds the same sweeps as the sequential path."""
import ctypes

import numpy as np
import pytest

from mbd_b200 import _lib
from mbd_b200.planners.path_integral import Args, check_pi_batch_args, run_path_integral_batch

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


def _bufs(**kw):
    b = _lib.PiBufs(FAKE, FAKE, FAKE)
    for k, v in kw.items():
        setattr(b, k, v)
    return b


def _reject(p, B=4, Nr=10, method=1, bufs=None, tail_only=0):
    L = _lib.lib()
    rc = L.mbd_pi_batch_step_launch(ctypes.byref(p) if p is not None else None, B, Nr, method, None,
                                    ctypes.byref(bufs if bufs is not None else _bufs()), tail_only, None)
    return rc, L.mbd_last_error().decode()


@pytest.mark.parametrize("kw,B,Nr,method,bufs,msg", [
    ({}, 4, 10, 0, None, "unknown method"),
    ({}, 4, 10, 4, None, "unknown method"),
    ({"P": 2, "peer_base_ptrs": ctypes.cast(FAKE, ctypes.POINTER(ctypes.c_uint64))}, 4, 10, 1, None, "P must be 1"),
    ({}, 4, 1, 2, None, "Nrefine must be at least 2"),
    ({}, 0, 10, 1, None, "B must be at least 1"),
    ({}, 4, 10, 2, {"sigma_hist_dev": None}, "CMA-ES needs sigma_hist and cma_scratch"),
    ({}, 4, 10, 2, {"cma_scratch_dev": None}, "CMA-ES needs sigma_hist and cma_scratch"),
    ({}, 4, 10, 3, {"cem_idx_dev": None}, "CEM needs cem_idx"),
    ({"xref_dev": FAKE, "href": 5, "logpd_dev": FAKE, "logpd_all_dev": FAKE}, 4, 10, 1, None, "no demonstration"),
    ({"n_local": 32}, 4, 10, 1, None, "n_local == n_total"),
    ({"H": 4000, "nu": 2}, 4, 10, 1, None, "H * Nu exceeds 27 * 256 columns"),
    ({"state_init_dev": None}, 4, 10, 1, None, "state_init must be set"),
    ({"weights_dev": None}, 4, 10, 3, None, "a work buffer is NULL"),
    ({"n_total": 1 << 20, "n_local": 1 << 20, "H": 100, "nu": 2}, 16, 10, 1, None, "below 2^31"),
], ids=["method0", "method4", "P2", "Nr1", "B0", "cma-hist", "cma-scratch", "cem-idx", "demo", "nlocal", "columns", "state",
        "weights", "index-range"])
def test_pi_launch_rejects_with_message(kw, B, Nr, method, bufs, msg):
    rc, err = _reject(_plan(**kw), B, Nr, method, _bufs(**(bufs or {})))
    assert rc == -1, (rc, err)
    assert err.startswith("mbd_pi_batch_step_launch: ") and msg in err, err


def test_pi_launch_null_plan_and_bufs_rejected():
    L = _lib.lib()
    assert L.mbd_pi_batch_step_launch(None, 2, 10, 1, None, ctypes.byref(_bufs()), 0, None) == -1
    assert "plan is NULL" in L.mbd_last_error().decode()
    assert L.mbd_pi_batch_step_launch(ctypes.byref(_plan()), 2, 10, 1, None, None, 0, None) == -1
    assert "bufs is NULL" in L.mbd_last_error().decode()


def test_pi_tail_only_skips_the_env_checks_only():
    """tail_only does not need an initial state; the other checks stay"""
    rc, err = _reject(_plan(state_init_dev=None, Y0s_dev=None), tail_only=1)
    assert rc == -1 and "a work buffer is NULL" in err, err


def test_pi_bufs_size_and_cem_slots():
    assert ctypes.sizeof(_lib.PiBufs) == 24 and _lib.PI_IDX_STRIDE > _lib.PI_TOPK


def _args(**kw):
    base = dict(env_name="car2d", Nsample=64, Hsample=40, Nrefine=10, disable_recommended_params=True)
    base.update(kw)
    return Args(**base)


@pytest.mark.parametrize("field,value", [("env_name", "pushT"), ("Nsample", 128), ("Hsample", 30), ("Nrefine", 20),
                                         ("update_method", "cem")])
def test_pi_batch_fields_must_agree(field, value):
    args = [_args(seed=0), _args(seed=1), _args(seed=2, **{field: value})]
    with pytest.raises(ValueError, match=f"same {field}"):
        run_path_integral_batch(args)


def test_pi_batch_unknown_method_is_a_key_error():
    with pytest.raises(KeyError):
        run_path_integral_batch([_args(update_method="nope"), _args(seed=1, update_method="nope")])


def test_pi_batch_needs_two_refinement_steps():
    with pytest.raises(ValueError, match="Nrefine must be at least 2"):
        run_path_integral_batch([_args(Nrefine=1)])


def test_pi_batch_refuses_multiple_ranks(monkeypatch):
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(ValueError, match="WORLD_SIZE"):
        run_path_integral_batch([_args(seed=0), _args(seed=1)])


def test_pi_batch_varying_fields_are_allowed_by_the_check():
    check_pi_batch_args([_args(seed=0, temp_sample=0.1), _args(seed=5, temp_sample=0.4)])


def test_pi_batch_recommended_params_applied_per_problem(monkeypatch):
    """apply_recommended_params runs per Args before the check: pushT's Hsample / Nrefine overrides make the problems agree,
    and the recommended temperature replaces each swept one (path_integral.py:86-91)"""
    monkeypatch.setenv("WORLD_SIZE", "2")   # stop right after the checks, before the device
    a = [Args(env_name="pushT", Hsample=10, temp_sample=0.05), Args(env_name="pushT", seed=1, Nrefine=7, temp_sample=0.6)]
    with pytest.raises(ValueError, match="WORLD_SIZE"):
        run_path_integral_batch(a)
    assert all(x.Hsample == 40 and x.Nrefine == 200 and x.temp_sample == 0.2 and x.Nsample == 2048 for x in a)
    b = [Args(env_name="car2d", temp_sample=0.05, disable_recommended_params=True), Args(env_name="car2d", temp_sample=0.6,
                                                                                      disable_recommended_params=True)]
    with pytest.raises(ValueError, match="WORLD_SIZE"):
        run_path_integral_batch(b)
    assert [x.temp_sample for x in b] == [0.05, 0.6]


def test_run_mbd_pi_batch_flag_parses():
    import tyro
    from mbd_b200.scripts import run_mbd
    a = tyro.cli(run_mbd.Args, args=["--algo", "path_integral", "--pi_batch", "--mode", "temp", "--env_name", "hopper"])
    assert a.pi_batch and a.algo == "path_integral"
    assert not tyro.cli(run_mbd.Args, args=[]).pi_batch


def test_run_mbd_pi_sweeps_match_the_sequential_path():
    """--pi_batch hands run_path_integral_batch the very Args list the sequential loop runs one by one, including the
    reference's temperature-sweep quirk (no disable_recommended_params, no update_method)"""
    from mbd_b200.scripts import run_mbd
    s = run_mbd.pi_seed_args(run_mbd.Args(env_name="hopper", update_method="cem"))
    assert s == [Args(seed=k, env_name="hopper", update_method="cem") for k in range(8)]
    t = run_mbd.pi_temp_args(run_mbd.Args(env_name="hopper", update_method="cem"))
    assert t == [Args(seed=0, env_name="hopper", temp_sample=float(x)) for x in run_mbd.TEMPS]
    assert all(a.update_method == "mppi" and not a.disable_recommended_params for a in t)


def test_run_mbd_pi_batch_dispatch(monkeypatch):
    """--pi_batch calls run_path_integral_batch once with the sweep; without it run_path_integral runs once per problem"""
    from mbd_b200.planners import path_integral
    from mbd_b200.scripts import run_mbd
    calls = []
    monkeypatch.setattr(path_integral, "run_path_integral_batch", lambda al: calls.append(("batch", list(al))) or np.zeros(len(al)))
    monkeypatch.setattr(path_integral, "run_path_integral", lambda a: calls.append(("one", a)) or 0.0)
    import torch
    monkeypatch.setattr(torch.cuda, "synchronize", lambda: None)
    run_mbd.main(["--algo", "path_integral", "--pi_batch", "--mode", "temp", "--env_name", "car2d"])
    assert len(calls) == 1 and calls[0][0] == "batch" and calls[0][1] == run_mbd.pi_temp_args(run_mbd.Args(env_name="car2d"))
    calls.clear()
    run_mbd.main(["--algo", "path_integral", "--mode", "seed", "--env_name", "car2d"])
    assert [c[0] for c in calls] == ["one"] * 8
