"""The receding-horizon controller without a GPU: its key table, the shift, the argument checks, the refusals of mbd_mpc_advance and the
CPU restatement of the controller on the oracle (tests/mpc_ref.py)."""
import ctypes

import numpy as np
import pytest

import mbd_b200
from mbd_b200 import _lib, prng
from mbd_b200.planners import engine as eng
from mbd_b200.planners import mbd_mpc
from mbd_b200.planners.mbd_mpc import Args
from tests import mpc_ref


def test_key_table_restates_prng():
    """cold = run_diffusion's key chain; warm[c] = rows 1 .. Nwarm of key_chain(rng_c, Nwarm + 1), rng, rng_c = split(rng)"""
    seed, Nd, Nwarm, Nstep = 7, 12, 4, 6
    rng_reset, cold, warm = mbd_mpc.mpc_keys(seed, Nd, Nwarm, Nstep)
    rng = prng.PRNGKey(seed)
    rng, rr = prng.split(rng)
    rng_exp, rng = prng.split(rng)
    assert (rng_reset == rr).all()
    assert cold.dtype == np.uint32 and (cold == eng.key_chain(rng_exp, Nd)).all()
    # the chain of run_diffusion (mbd_planner.py:103) written out: steps Nd - 1 ... 1
    r = rng_exp
    for i in range(Nd - 1, 0, -1):
        r, k = prng.split(r)
        assert (cold[i] == k).all()
    assert warm.shape == (Nstep, Nwarm, 2) and warm.dtype == np.uint32 and not warm[0].any()
    for c in range(1, Nstep):
        rng, r = prng.split(rng)
        for j in range(Nwarm, 0, -1):
            r, k = prng.split(r)
            assert (warm[c, j - 1] == k).all(), (c, j)
    assert len({tuple(k) for k in warm[1:].reshape(-1, 2)}) == (Nstep - 1) * Nwarm


def test_key_table_matches_the_oracle_threefry(orc):
    seed, Nd, Nwarm, Nstep = 3, 10, 3, 5
    _, cold, warm = mbd_mpc.mpc_keys(seed, Nd, Nwarm, Nstep)
    rng = orc.prng_key(seed)
    rng, _ = orc.split(rng)
    rng_exp, rng = orc.split(rng)
    r = rng_exp
    for i in range(Nd - 1, 0, -1):
        r, k = orc.split(r)
        assert (cold[i] == k).all()
    for c in range(1, Nstep):
        rng, r = orc.split(rng)
        for j in range(Nwarm, 0, -1):
            r, k = orc.split(r)
            assert (warm[c, j - 1] == k).all()


def test_shift():
    P = np.arange(24, dtype=np.float32).reshape(2, 4, 3)
    S = mbd_mpc.shift(P)
    assert (S[:, :3] == P[:, 1:]).all() and (S[:, 3] == 0).all()
    assert (mpc_ref.shift_rows(P[0]) == S[0]).all()
    import torch
    assert (mbd_mpc.shift(torch.as_tensor(P)).numpy() == S).all()


def _args(**kw):
    base = dict(env_name="car2d", Nsample=64, Hsample=8, Ndiffuse=10, Nwarm=3, Nstep=5, not_render=True,
                disable_recommended_params=True)
    base.update(kw)
    return Args(**base)


@pytest.mark.parametrize("kw, msg", [
    (dict(Nwarm=0), "Nwarm"),
    (dict(Nwarm=10), "Nwarm"),
    (dict(Nstep=0), "Nstep"),
    (dict(enable_demo=True), "enable_demo"),
])
def test_argument_checks(kw, msg, monkeypatch):
    """every refusal is a ValueError raised before the controller touches the device"""
    monkeypatch.setattr(mbd_mpc, "Controller", None)     # reaching the device would be a TypeError here
    with pytest.raises(ValueError, match=msg):
        mbd_mpc.run_mpc(_args(**kw))
    with pytest.raises(ValueError, match=msg):
        mbd_mpc.run_mpc_batch([_args(), _args(seed=1, **kw)])


def test_batch_checks(monkeypatch):
    monkeypatch.setattr(mbd_mpc, "Controller", None)
    for kw in (dict(Nsample=32), dict(Hsample=6), dict(Nwarm=2), dict(Nstep=4), dict(Ndiffuse=11), dict(env_name="pushT")):
        with pytest.raises(ValueError, match="same " + next(iter(kw))):
            mbd_mpc.run_mpc_batch([_args(), _args(seed=1, **kw)])
    with pytest.raises(ValueError, match="not_render"):
        mbd_mpc.run_mpc_batch([_args(not_render=False)])
    with pytest.raises(ValueError, match="at least one"):
        mbd_mpc.run_mpc_batch([])
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(ValueError, match="WORLD_SIZE"):
        mbd_mpc.run_mpc(_args())
    with pytest.raises(ValueError, match="WORLD_SIZE"):
        mbd_mpc.run_mpc_batch([_args(), _args(seed=1)])


def test_recommended_params_are_applied_first(monkeypatch):
    """pushT's recommended Ndiffuse (200) makes Nwarm = 150 valid, as the planner's override would"""
    seen = []
    monkeypatch.setattr(mbd_mpc, "Controller", lambda env, args_list: seen.append(args_list) or (_ for _ in ()).throw(KeyError))
    with pytest.raises(KeyError):
        mbd_mpc.run_mpc(Args(env_name="pushT", Nwarm=150, Nstep=2, not_render=True))
    a = seen[0][0]
    assert (a.Ndiffuse, a.Hsample, a.temp_sample) == (200, 40, 0.2)


# ---- the C ABI --------------------------------------------------------------------------------------------------------------
BUFS = ("params_dev", "ctl_dev", "Ybars_dev", "rew_hist_dev", "keys_dev", "mpc_ctl_dev", "env_actions_dev", "env_state_dev",
        "env_reward_dev", "actions_dev", "rewards_dev", "states_dev", "rew_hist_log_dev")
ACT_BUFS = set(BUFS) - {"env_reward_dev", "rewards_dev"}
RECORD_BUFS = {"mpc_ctl_dev", "env_state_dev", "states_dev", "env_reward_dev", "rewards_dev"}


def _plan(**kw):
    p = _lib.MpcPlan()
    p.B, p.H, p.nu, p.Ndiffuse, p.Nwarm, p.Nstep, p.state_words = 2, 8, 2, 10, 3, 5, 3
    for i, b in enumerate(BUFS):
        setattr(p, b, 0x1000 * (i + 1))      # never dereferenced: every call below is refused before any CUDA call
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _refused(p, mode, what):
    L = _lib.lib()
    assert L.mbd_mpc_advance(ctypes.byref(p) if p is not None else None, mode, None) == -1
    assert what in L.mbd_last_error().decode(), L.mbd_last_error().decode()


def test_mpc_advance_refuses_missing_buffers():
    _refused(None, _lib.MPC_ACT, "plan is NULL")
    for mode, need in ((_lib.MPC_ACT, ACT_BUFS), (_lib.MPC_RECORD, RECORD_BUFS)):
        for b in sorted(need):
            _refused(_plan(**{b: None}), mode, "a buffer is missing")


@pytest.mark.parametrize("kw, what", [
    (dict(B=0), "B must be"), (dict(B=_lib.VEC_MAX_B + 1), "B must be"), (dict(H=0), "H and nu"), (dict(nu=0), "H and nu"),
    (dict(H=28 * 256, nu=1), "27 * 256"), (dict(Ndiffuse=1, Nwarm=1), "Ndiffuse"), (dict(Nwarm=0), "Nwarm"),
    (dict(Nwarm=10), "Nwarm"), (dict(Nstep=0), "Nstep"), (dict(state_words=0), "state_words"),
])
def test_mpc_advance_refuses_bad_shapes(kw, what):
    for mode in (_lib.MPC_ACT, _lib.MPC_RECORD):
        _refused(_plan(**kw), mode, what)


def test_mpc_advance_refuses_unknown_modes():
    for mode in (-1, 2, 7):
        _refused(_plan(), mode, "unknown mode")


# ---- the oracle restatement -------------------------------------------------------------------------------------------------
def test_mpc_ref_control_step_0_is_the_oracle_solve(orc):
    """control step 0 of the CPU controller is the oracle run_diffusion's Yi[-1]; later control steps stay finite, inside [-1, 1]
    (a weighted mean of clipped samples through the update is not clipped, so only loosely) and move the car"""
    from oracle import planner as opl
    car = mbd_b200.envs.get_env("car2d")
    ref = mpc_ref.run_mpc_car2d(car, seed=0, Nsample=64, H=8, Ndiffuse=10, Nwarm=3, Nstep=5, temp=0.1)
    _, Yi, rews = opl.run_diffusion(opl.OracleEnv("car2d", 2, params=car.params, x0=car.x0), 0, 64, 8, 10, 0.1)
    assert (ref["plans"][0].reshape(-1).view(np.uint32) == Yi[-1].view(np.uint32)).all()
    assert ref["rew_hist"][0] == rews[-1]
    assert (ref["actions"] == ref["plans"][:, 0]).all()
    assert ref["states"].shape == (6, 3) and np.isfinite(ref["states"]).all()
    assert (ref["states"][0] == car.x0).all() and not (ref["states"][1] == ref["states"][0]).all()
    # the plant: s_{c+1} = env.step(s_c, a_c) through the oracle rollout, one step at a time
    for c in range(5):
        x, r = mpc_ref.car2d_step(car.params, ref["states"][c], ref["actions"][c])
        assert (x == ref["states"][c + 1]).all() and r == ref["rewards"][c]
