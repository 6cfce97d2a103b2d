"""The receding-horizon controller of the path-integral baselines without a GPU: its key table, the argument checks, the refusals
of mbd_mpc_pi_advance and the CPU restatement of the controller on the oracle (tests/pi_mpc_ref.py)."""
import ctypes

import numpy as np
import pytest

import mbd_b200
from mbd_b200 import _lib, prng
from mbd_b200.planners import engine as eng
from mbd_b200.planners import mbd_mpc, pi_mpc
from mbd_b200.planners.pi_mpc import Args
from tests import pi_mpc_ref

METHODS = ("mppi", "cma-es", "cem")


def test_key_table_restates_prng():
    """the controller's keys are mpc_keys with Nrefine in the place of Ndiffuse: cold = run_path_integral's chain, warm[c] = rows
    1 .. Nwarm of key_chain(rng_c, Nwarm + 1)"""
    seed, Nr, Nwarm, Nstep = 5, 9, 3, 4
    rng_reset, cold, warm = mbd_mpc.mpc_keys(seed, Nr, Nwarm, Nstep)
    rng = prng.PRNGKey(seed)
    rng, rr = prng.split(rng)              # run_path_integral: rng, rng_reset = split(rng)
    rng_exp, rng = prng.split(rng)         #                    rng_exp, rng = split(rng)
    assert (rng_reset == rr).all() and (cold == eng.key_chain(rng_exp, Nr)).all()
    r = rng_exp
    for t in range(Nr - 1, 0, -1):         #                    r, k = split(r) per step
        r, k = prng.split(r)
        assert (cold[t] == k).all()
    for c in range(1, Nstep):
        rng, rng_c = prng.split(rng)
        assert (warm[c] == eng.key_chain(rng_c, Nwarm + 1)[1:]).all()
    assert pi_mpc.Controller.steps_field == "Nrefine" and mbd_mpc.Controller.steps_field == "Ndiffuse"


def test_key_table_matches_the_oracle_threefry(orc):
    seed, Nr, Nwarm, Nstep = 11, 8, 2, 4
    _, cold, warm = mbd_mpc.mpc_keys(seed, Nr, Nwarm, Nstep)
    rng = orc.prng_key(seed)
    rng, _ = orc.split(rng)
    rng_exp, rng = orc.split(rng)
    r = rng_exp
    for t in range(Nr - 1, 0, -1):
        r, k = orc.split(r)
        assert (cold[t] == k).all()
    for c in range(1, Nstep):
        rng, r = orc.split(rng)
        for j in range(Nwarm, 0, -1):
            r, k = orc.split(r)
            assert (warm[c, j - 1] == k).all()


def _args(**kw):
    base = dict(env_name="car2d", Nsample=64, Hsample=8, Nrefine=10, Nwarm=3, Nstep=5, not_render=True,
                disable_recommended_params=True)
    base.update(kw)
    return Args(**base)


@pytest.mark.parametrize("kw, msg", [
    (dict(Nwarm=0), "Nwarm"),
    (dict(Nwarm=10), "Nwarm"),
    (dict(Nstep=0), "Nstep"),
    (dict(sigma_warm=0.0), "sigma_warm"),
    (dict(sigma_warm=-1.0), "sigma_warm"),
    (dict(sigma_warm=float("nan")), "sigma_warm"),
    (dict(sigma_warm=float("inf")), "sigma_warm"),
])
def test_argument_checks(kw, msg, monkeypatch):
    """every refusal is a ValueError raised before the controller touches the device"""
    monkeypatch.setattr(pi_mpc, "Controller", None)     # reaching the device would be a TypeError here
    with pytest.raises(ValueError, match=msg):
        pi_mpc.run_pi_mpc(_args(**kw))
    with pytest.raises(ValueError, match=msg):
        pi_mpc.run_pi_mpc_batch([_args(), _args(seed=1, **kw)])


def test_unknown_method_is_a_key_error(monkeypatch):
    monkeypatch.setattr(pi_mpc, "Controller", None)
    with pytest.raises(KeyError):
        pi_mpc.run_pi_mpc(_args(update_method="nope"))
    with pytest.raises(KeyError):
        pi_mpc.run_pi_mpc_batch([_args(update_method="nope"), _args(seed=1, update_method="nope")])


def test_batch_checks(monkeypatch):
    monkeypatch.setattr(pi_mpc, "Controller", None)
    for kw in (dict(Nsample=32), dict(Hsample=6), dict(Nwarm=2), dict(Nstep=4), dict(Nrefine=11), dict(env_name="pushT"),
               dict(update_method="cem"), dict(sigma_warm=0.5)):
        with pytest.raises(ValueError, match="same " + next(iter(kw))):
            pi_mpc.run_pi_mpc_batch([_args(), _args(seed=1, **kw)])
    with pytest.raises(ValueError, match="not_render"):
        pi_mpc.run_pi_mpc_batch([_args(not_render=False)])
    with pytest.raises(ValueError, match="at least one"):
        pi_mpc.run_pi_mpc_batch([])
    pi_mpc.check_args([_args(seed=0, temp_sample=0.1), _args(seed=5, temp_sample=0.4)], batch=True)   # these may differ
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(ValueError, match="WORLD_SIZE"):
        pi_mpc.run_pi_mpc(_args())
    with pytest.raises(ValueError, match="WORLD_SIZE"):
        pi_mpc.run_pi_mpc_batch([_args(), _args(seed=1)])


def test_recommended_params_are_applied_first(monkeypatch):
    """pushT's recommended Nrefine (200) makes Nwarm = 150 valid, as path_integral's override would"""
    seen = []
    monkeypatch.setattr(pi_mpc, "Controller", lambda env, args_list: seen.append(args_list) or (_ for _ in ()).throw(KeyError))
    with pytest.raises(KeyError):
        pi_mpc.run_pi_mpc(Args(env_name="pushT", Nwarm=150, Nstep=2, not_render=True))
    a = seen[0][0]
    assert (a.Nrefine, a.Hsample, a.temp_sample) == (200, 40, 0.2)


def test_comparison_driver_gives_every_algorithm_the_same_problem():
    """scripts/run_mpc.py: mbd and the baselines get the same seeds, Nsample, Hsample, solve length, Nwarm and Nstep"""
    from mbd_b200.scripts import run_mpc
    a = run_mpc.Args(env_name="hopper", Nsample=256, Hsample=20, Nsolve=30, Nwarm=4, Nstep=7, sigma_warm=0.3)
    m = run_mpc.mbd_args(a)
    assert [x.seed for x in m] == list(range(8))
    for method in run_mpc.BASELINES:
        p = run_mpc.pi_args(a, method)
        for x, y in zip(m, p):
            assert (x.seed, x.env_name, x.Nsample, x.Hsample, x.Ndiffuse, x.Nwarm, x.Nstep, x.temp_sample) == \
                   (y.seed, y.env_name, y.Nsample, y.Hsample, y.Nrefine, y.Nwarm, y.Nstep, y.temp_sample)
            assert y.update_method == method and y.sigma_warm == 0.3 and y.not_render and x.not_render
        pi_mpc.check_args(p, batch=True)
    mbd_mpc.check_args(m, batch=True)


# ---- the C ABI --------------------------------------------------------------------------------------------------------------
def test_mpc_pi_plan_extends_mpc_plan():
    P = _lib.MpcPiPlan
    assert P.base.offset == 0 and P.sigma_warm.offset == ctypes.sizeof(_lib.MpcPlan)


BUFS = ("params_dev", "ctl_dev", "Ybars_dev", "rew_hist_dev", "keys_dev", "mpc_ctl_dev", "env_actions_dev", "env_state_dev",
        "env_reward_dev", "actions_dev", "rewards_dev", "states_dev", "rew_hist_log_dev")
ACT_BUFS = set(BUFS) - {"env_reward_dev", "rewards_dev"}
RECORD_BUFS = {"mpc_ctl_dev", "env_state_dev", "states_dev", "env_reward_dev", "rewards_dev"}


def _plan(sigma_warm=1.0, sigma_log_dev=0xF000, **kw):
    p = _lib.MpcPiPlan()
    b = p.base
    b.B, b.H, b.nu, b.Ndiffuse, b.Nwarm, b.Nstep, b.state_words = 2, 8, 2, 10, 3, 5, 3
    for i, name in enumerate(BUFS):
        setattr(b, name, 0x1000 * (i + 1))      # never dereferenced: every call below is refused before any CUDA call
    for k, v in kw.items():
        setattr(b, k, v)
    p.sigma_warm, p.sigma_log_dev = sigma_warm, sigma_log_dev
    return p


def _refused(p, mode, what):
    L = _lib.lib()
    assert L.mbd_mpc_pi_advance(ctypes.byref(p) if p is not None else None, mode, None) == -1
    err = L.mbd_last_error().decode()
    assert err.startswith("mbd_mpc_pi_advance: ") and what in err, err


def test_mpc_pi_advance_refuses_missing_buffers():
    _refused(None, _lib.MPC_ACT, "plan is NULL")
    for mode, need in ((_lib.MPC_ACT, ACT_BUFS), (_lib.MPC_RECORD, RECORD_BUFS)):
        for b in sorted(need):
            _refused(_plan(**{b: None}), mode, "a buffer is missing")
    _refused(_plan(sigma_log_dev=None), _lib.MPC_ACT, "a buffer is missing")


@pytest.mark.parametrize("kw, what", [
    (dict(B=0), "B must be"), (dict(B=_lib.VEC_MAX_B + 1), "B must be"), (dict(H=0), "H and nu"), (dict(nu=0), "H and nu"),
    (dict(H=28 * 256, nu=1), "27 * 256"), (dict(Ndiffuse=1, Nwarm=1), "Ndiffuse"), (dict(Nwarm=0), "Nwarm"),
    (dict(Nwarm=10), "Nwarm"), (dict(Nstep=0), "Nstep"), (dict(state_words=0), "state_words"),
])
def test_mpc_pi_advance_refuses_bad_shapes(kw, what):
    for mode in (_lib.MPC_ACT, _lib.MPC_RECORD):
        _refused(_plan(**kw), mode, what)


def test_mpc_pi_advance_refuses_unknown_modes():
    for mode in (-1, 2, 7):
        _refused(_plan(), mode, "unknown mode")


@pytest.mark.parametrize("sigma", [0.0, -0.5, float("nan"), float("inf"), float("-inf")])
def test_mpc_pi_advance_refuses_bad_sigma_warm(sigma):
    for mode in (_lib.MPC_ACT, _lib.MPC_RECORD):
        _refused(_plan(sigma_warm=sigma), mode, "sigma_warm")


# ---- the oracle restatement -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS)
def test_pi_mpc_ref_control_step_0_is_the_oracle_refinement(orc, method):
    """control step 0 of the CPU controller is an open-loop oracle refinement (update_once from mu = 0, sigma = 1 along the
    chain from rng_exp); every warm control step starts from sigma_warm; the plant is the oracle car2d step"""
    from oracle import oracle as o
    from oracle import planner as opl
    car = mbd_b200.envs.get_env("car2d")
    Nn, H, Nr, Nwarm, Nstep, temp, sw = 64, 8, 10, 3, 4, 0.1, 0.5
    trace = []
    ref = pi_mpc_ref.run_pi_mpc_car2d(car, method, 0, Nn, H, Nr, Nwarm, Nstep, temp, sigma_warm=sw, trace=trace)
    rng = o.prng_key(0)
    rng, _ = o.split(rng)
    r, _ = o.split(rng)
    env = opl.OracleEnv("car2d", 2, params=car.params, x0=car.x0)
    mu, sigma = np.zeros(H * 2, np.float32), 1.0
    for _t in range(Nr - 1, 0, -1):
        r, k = o.split(r)
        out = opl.update_once(env, k, Nn, H, sigma, mu, temp, method)
        mu, sigma = out["mu"], out["sigma"]
    assert (ref["plans"][0].reshape(-1).view(np.uint32) == mu.view(np.uint32)).all()
    assert ref["rew_hist"][0] == out["rew_mean"] and ref["sigmas"][0] == np.float32(sigma)
    assert (ref["actions"] == ref["plans"][:, 0]).all()
    assert ref["states"].shape == (Nstep + 1, 3) and np.isfinite(ref["states"]).all() and np.isfinite(ref["plans"]).all()
    for c in range(Nstep):
        x, rew = pi_mpc_ref.car2d_step(car.params, ref["states"][c], ref["actions"][c])
        assert (x == ref["states"][c + 1]).all() and rew == ref["rewards"][c]
    assert [(c, t) for c, t, _ in trace] == [(0, t) for t in range(Nr - 1, 0, -1)] + \
        [(c, t) for c in range(1, Nstep) for t in range(Nwarm, 0, -1)]
    if method == "cma-es":
        assert len(set(ref["sigmas"].tolist())) > 1 and (ref["sigmas"] >= np.float32(1e-3)).all()
    else:
        assert ref["sigmas"].tolist() == [1.0] + [sw] * (Nstep - 1)
