"""Planner ensembles without a GPU (DESIGN.md §5l): the ctypes mirror of the new mbd_step_plan fields, the C refusals (all before any
CUDA call), the refusals of the engine and of the controllers' check_args, the member-major table, the run_mpc driver, and the
oracle restatement of one ensemble step against the oracle's nominal step."""
import ctypes

import numpy as np
import pytest

from mbd_b200 import _lib, prng
from mbd_b200.envs import get_env
from mbd_b200.planners import engine as eng
from mbd_b200.planners import mbd_mpc, pi_mpc
from oracle import planner as opl
from tests import ens_ref

FAKE = 0x1000   # never dereferenced: every case below fails validation, which runs before the first CUDA call


def test_abi_sizes_match_the_ctypes_mirror():
    out = (ctypes.c_int32 * 8)()
    n = _lib.lib().mbd_ens_abi_sizes(out, 8)
    P = _lib.StepPlan
    assert list(out[:n]) == [ctypes.sizeof(P), P.ens_factors_dev.offset, P.ens_rews_dev.offset, P.ens_k.offset, _lib.ENS_MAXK]
    assert P.ens_factors_dev.offset == P.timeout_cycles.offset + 8     # appended: every other offset stays
    assert ctypes.sizeof(P) == P.ens_k.offset + 8


def _plan(**kw):
    """a car2d batch plan that passes every check but the ensemble's"""
    p = _lib.StepPlan()
    for f in ("car_params_dev", "state_init_dev", "params_dev", "ctl_dev", "Ybars_dev", "Y0s_dev", "rews_dev", "rews_all_dev",
              "logp_dev", "weights_dev", "runs_dev", "partial_dev", "scalars_dev"):
        setattr(p, f, FAKE)
    p.n_total, p.n_begin, p.n_local, p.H, p.nu, p.P, p.rank, p.temp = 64, 0, 64, 40, 2, 1, 0, 0.1
    for k, v in kw.items():
        setattr(p, k, v)
    return p


TABLE = dict(ens_factors_dev=FAKE, ens_rews_dev=FAKE, ens_k=3)
DEMO = dict(xref_dev=FAKE, href=5, logpd_dev=FAKE, logpd_all_dev=FAKE)
CASES = [
    (dict(ens_factors_dev=FAKE, ens_k=3), 4, "both ens_factors and ens_rews"),
    (dict(ens_rews_dev=FAKE, ens_k=3), 4, "both ens_factors and ens_rews"),
    (dict(ens_rews_dev=FAKE), 4, "both ens_factors and ens_rews"),
    (dict(TABLE, ens_k=0), 4, "ens_k must be in 1 .. MBD_ENS_MAXK"),
    (dict(TABLE, ens_k=17), 4, "ens_k must be in 1 .. MBD_ENS_MAXK"),
    (dict(TABLE, ens_k=-1), 4, "ens_k must be in 1 .. MBD_ENS_MAXK"),
    (dict(ens_k=2), 4, "ens_k must be 0 without an ensemble table"),
    (TABLE, 4, "xpbd"),
    (dict(TABLE, env_kind=_lib.ENV_PUSHT), 4, "xpbd"),
    (dict(TABLE, ens_k=1), 1, "xpbd"),
    (dict(TABLE, **DEMO), 4, "demonstration"),
    (dict(TABLE, ens_k=16, n_total=1 << 14, n_local=1 << 14, H=1), 1 << 13, "B * N * ens_k must stay below 2^31"),
]
IDS = ["table-only", "rews-only", "rews-only-k0", "k0", "k17", "kneg", "k-no-table", "car2d", "pusht", "car2d-B1", "demo", "range"]


@pytest.mark.parametrize("kw,B,msg", CASES, ids=IDS)
def test_batch_step_refuses(kw, B, msg):
    L = _lib.lib()
    rc = L.mbd_batch_step_launch(ctypes.byref(_plan(**kw)), B, 10, None, None)
    err = L.mbd_last_error().decode()
    assert rc == -1 and err.startswith("mbd_batch_step_launch: ") and msg in err, (rc, err)


@pytest.mark.parametrize("kw,B,msg", CASES, ids=IDS)
def test_pi_batch_step_refuses(kw, B, msg):
    L = _lib.lib()
    bufs = _lib.PiBufs(FAKE, FAKE, FAKE)
    rc = L.mbd_pi_batch_step_launch(ctypes.byref(_plan(**kw)), B, 10, _lib.PI_METHODS["mppi"], None, ctypes.byref(bufs), 0, None)
    err = L.mbd_last_error().decode()
    assert rc == -1 and err.startswith("mbd_pi_batch_step_launch: ") and msg in err, (rc, err)


@pytest.mark.parametrize("entry", ["mbd_step_launch", "mbd_step_launch_ev", "mbd_step_tail_launch"])
@pytest.mark.parametrize("kw", [TABLE, dict(ens_factors_dev=FAKE), dict(ens_rews_dev=FAKE), dict(ens_k=1)],
                         ids=["table", "factors", "rews", "k"])
def test_single_solve_entries_refuse_an_ensemble(entry, kw):
    L = _lib.lib()
    p = _plan(**kw)
    if entry == "mbd_step_launch_ev":
        rc = L.mbd_step_launch_ev(ctypes.byref(p), None, None, None, None, None)
    else:
        rc = getattr(L, entry)(ctypes.byref(p), None)
    err = L.mbd_last_error().decode()
    assert rc == -1 and err.startswith(entry + ": ") and "no planner ensemble" in err, (rc, err)


# ---- the engine's table ------------------------------------------------------------------------------------------------------
BAD = [float("nan"), float("inf"), -float("inf"), -1.0, -1e-30, 1e39]   # 1e39 is finite in float64 but not in float32


def test_table_is_member_major_within_each_problem():
    al = [mbd_mpc.Args(seed=b, env_name="hopper", plan_friction=(1.0, 0.5 + b, 2.0), plan_gear=(0.7, 1.0, 1.3 + b)) for b in range(2)]
    t = mbd_mpc.plan_ensemble(al)
    tab = eng.ensemble_table(t, 2, get_env("hopper"), False)
    assert tab.dtype == np.float32 and tab.shape == (2, 3, 2) and tab.flags.c_contiguous
    flat = tab.reshape(-1)
    for b in range(2):
        for k in range(3):
            row = b * 3 + k      # the kernels' factor row of member k of problem b
            assert flat[2 * row] == np.float32(al[b].plan_friction[k]) and flat[2 * row + 1] == np.float32(al[b].plan_gear[k])
    assert mbd_mpc.plan_ensemble([mbd_mpc.Args()]) is None


@pytest.mark.parametrize("bad", BAD)
def test_table_refuses_bad_values(bad):
    t = np.ones((2, 3, 2))
    t[1, 2, 1] = bad
    with pytest.raises(ValueError, match="finite and >= 0"):
        eng.ensemble_table(t, 2, get_env("hopper"), False)


@pytest.mark.parametrize("shape", [(2, 3), (1, 3, 2), (2, 0, 2), (2, 17, 2), (2, 3, 3), (2, 3, 2, 1)])
def test_table_refuses_bad_shapes(shape):
    with pytest.raises(ValueError, match="shape"):
        eng.ensemble_table(np.ones(shape), 2, get_env("hopper"), False)


def test_engine_refuses_before_touching_the_device():
    """the engine checks its ensemble first: these raise ValueError on a machine without a GPU"""
    for env_name in ("car2d", "pushT"):
        with pytest.raises(ValueError, match="xpbd"):
            eng.BatchedDiffusionEngine(get_env(env_name), 16, 8, [0.1], False, [None], 10, ensemble=np.ones((1, 2, 2)))
    with pytest.raises(ValueError, match="demonstration"):
        eng.BatchedDiffusionEngine(get_env("humanoidtrack"), 16, 8, [0.1], True, [None], 10, ensemble=np.ones((1, 2, 2)))
    with pytest.raises(ValueError, match="finite"):
        eng.BatchedDiffusionEngine(get_env("hopper"), 16, 8, [0.1, 0.1], False, [None, None], 10,
                                   ensemble=np.full((2, 2, 2), -1.0))
    from mbd_b200.planners.path_integral import BatchedPathIntegralEngine
    with pytest.raises(ValueError, match="shape"):
        BatchedPathIntegralEngine(get_env("hopper"), 16, 8, [0.1], [None], 10, "mppi", ensemble=np.ones((2, 2, 2)))


# ---- the controllers' Args ----------------------------------------------------------------------------------------------------
def _margs(**kw):
    return mbd_mpc.Args(env_name=kw.pop("env_name", "hopper"), Ndiffuse=10, Nwarm=3, Nstep=2, not_render=True,
                        disable_recommended_params=True, **kw)


def _pargs(**kw):
    return pi_mpc.Args(env_name=kw.pop("env_name", "hopper"), Nrefine=10, Nwarm=3, Nstep=2, not_render=True,
                       disable_recommended_params=True, **kw)


@pytest.mark.parametrize("make,check", [(_margs, mbd_mpc.check_args), (_pargs, pi_mpc.check_args)], ids=["mbd", "pi"])
def test_check_args_refuses_bad_ensembles(make, check):
    check([make(), make(seed=1)], True)
    check([make(plan_friction=(1.0, 0.5), plan_gear=(0.7, 1.3)), make(seed=1, plan_friction=(0.0, 2.0), plan_gear=(1.0, 1.0))], True)
    check([make(plan_friction=(1.0,) * 16, plan_gear=(1.0,) * 16)], True)
    with pytest.raises(ValueError, match="same length"):
        check([make(plan_friction=(1.0, 0.5), plan_gear=(1.0,))], True)
    with pytest.raises(ValueError, match="at most 16"):
        check([make(plan_friction=(1.0,) * 17, plan_gear=(1.0,) * 17)], True)
    with pytest.raises(ValueError, match="same number of ensemble members"):
        check([make(plan_friction=(1.0, 0.5), plan_gear=(1.0, 1.0)), make(seed=1, plan_friction=(1.0,), plan_gear=(1.0,))], True)
    with pytest.raises(ValueError, match="same number of ensemble members"):
        check([make(), make(seed=1, plan_friction=(1.0,), plan_gear=(1.0,))], True)
    for bad in BAD:
        for f, g in (((bad,), (1.0,)), ((1.0,), (bad,))):
            with pytest.raises(ValueError, match="finite and >= 0"):
                check([make(plan_friction=f, plan_gear=g)], True)
    for env_name in ("car2d", "pushT"):
        check([make(env_name=env_name)], False)
        with pytest.raises(ValueError, match="xpbd"):
            check([make(env_name=env_name, plan_friction=(1.0,), plan_gear=(1.0,))], False)


def test_run_mpc_script_passes_the_ensemble_to_every_algorithm():
    from mbd_b200.scripts import run_mpc
    a = run_mpc.Args(env_name="hopper", Nsample=64, Hsample=8, Nsolve=10, Nwarm=3, Nstep=2, plan_friction=(1.0, 1.0, 1.0),
                     plan_gear=(0.7, 1.0, 1.3))
    for al in [run_mpc.mbd_args(a)] + [run_mpc.pi_args(a, m) for m in run_mpc.BASELINES]:
        assert all(x.plan_friction == (1.0, 1.0, 1.0) and x.plan_gear == (0.7, 1.0, 1.3) for x in al)
        assert mbd_mpc.plan_ensemble(al).shape == (len(al), 3, 2)
    nominal = run_mpc.Args()
    assert all(x.plan_friction == () and x.plan_gear == () for x in run_mpc.mbd_args(nominal) + run_mpc.pi_args(nominal, "cem"))


def test_run_mpc_script_parses_the_ensemble_flags():
    import tyro
    from mbd_b200.scripts import run_mpc
    a = tyro.cli(run_mpc.Args, args=["--plan_friction", "1", "1", "1", "--plan_gear", "0.7", "1", "1.3"])
    assert tuple(a.plan_friction) == (1.0, 1.0, 1.0) and tuple(a.plan_gear) == (0.7, 1.0, 1.3)


# ---- the oracle restatement ---------------------------------------------------------------------------------------------------
def _oracle_inputs(env_name="hopper", N=24, H=6):
    env = get_env(env_name)
    rng, rng_reset = prng.split(prng.PRNGKey(4))
    state = env.reset(rng_reset).pipeline_state.raw
    _, alphas, alphas_bar, sigmas = opl.make_schedule(1e-4, 1e-2, 10)
    Ybar = np.random.default_rng(5).uniform(-0.5, 0.5, H * env.action_size).astype(np.float32)
    return env, state, prng.split(rng)[1], N, H, float(sigmas[7]), Ybar, alphas, alphas_bar


def test_oracle_unit_ensemble_is_the_nominal_step():
    env, state, key, N, H, sigma, Ybar, alphas, alphas_bar = _oracle_inputs()
    got = ens_ref.reverse_once(env, state, key, N, H, sigma, Ybar, 0.1, alphas, alphas_bar, 7, [(1.0, 1.0)])
    want = opl.reverse_once(opl.OracleEnv("xpbd", env.action_size, blob=env.blob, state=state), key, N, H, sigma, Ybar, 0.1, alphas,
                            alphas_bar, 7)
    for f in ("Y0s", "rews", "Ybar", "weights", "Ybar_im1"):
        assert np.array_equal(np.asarray(got[f]).view(np.uint32), np.asarray(want[f]).view(np.uint32)), f
    assert got["ens_rews"].shape == (N, 1) and np.array_equal(got["ens_rews"][:, 0], want["rews"])


def test_oracle_ordered_mean():
    r = np.float32([[1e8, 1.0, -1e8], [0.1, 0.2, 0.3]])
    m = ens_ref.ordered_mean(r)
    assert m[0] == np.float32(0.0)      # fl(fl(1e8 + 1) - 1e8) = 0: the member order is part of the definition
    assert m[1] == np.float32(np.float32(np.float32(0.1) + np.float32(0.2)) + np.float32(0.3)) / np.float32(3)
    assert np.array_equal(ens_ref.ordered_mean(r[:, :1]), r[:, 0])


def test_oracle_members_differ():
    """members that scale gear and friction change the returns: the ensemble's score is not the nominal one"""
    env, state, key, N, H, sigma, Ybar, alphas, alphas_bar = _oracle_inputs()
    got = ens_ref.reverse_once(env, state, key, N, H, sigma, Ybar, 0.1, alphas, alphas_bar, 7, [(1.0, 0.7), (1.0, 1.0), (0.5, 1.3)])
    e = got["ens_rews"]
    assert e.shape == (N, 3) and not np.array_equal(e[:, 0], e[:, 1]) and not np.array_equal(e[:, 2], e[:, 1])
    assert np.array_equal(got["rews"], ens_ref.ordered_mean(e))
