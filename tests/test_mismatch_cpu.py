"""Model factors of the vector env without a GPU (DESIGN.md §5k): the refusals of VecEnv.set_model_factors, of the controllers'
check_args and of the C ABI, the blob of scaled_env (the specification of env b) against the nominal blob word by word, and
mbd_vec_plan.factors_dev appended after every other field."""
import ctypes

import numpy as np
import pytest
import torch

from mbd_b200 import _lib
from mbd_b200.envs import get_env
from mbd_b200.envs import vec as vec_mod
from mbd_b200.model import blob as B
from mbd_b200.planners import mbd_mpc, pi_mpc
from tests.test_vecenv_cpu import _plan

XPBD = ["hopper", "ant", "humanoidrun", "halfcheetah", "walker2d", "cartpole"]
BAD = [float("nan"), float("inf"), -float("inf"), -1.0, -1e-30, 1e39]   # 1e39 is finite in float64 but not in float32


def _venv(env_name, num_envs=3):
    """a VecEnv shell: what set_model_factors reads before it allocates.  Its device is cuda, so any device call raises (no GPU
    here, or a tensor the test would see) — the refusals must come first."""
    v = vec_mod.VecEnv.__new__(vec_mod.VecEnv)
    v.env, v.num_envs, v.spec = get_env(env_name), num_envs, vec_mod.env_spec(get_env(env_name))
    v.device, v.plan, v.factors = torch.device("cuda", 0), _lib.VecPlan(), None
    return v


@pytest.mark.parametrize("bad", BAD)
@pytest.mark.parametrize("which", ["friction", "gear"])
def test_set_model_factors_refuses_bad_values(which, bad):
    v = _venv("hopper")
    for val in (bad, [1.0, bad, 1.0]):
        with pytest.raises(ValueError, match="finite and >= 0"):
            v.set_model_factors(**{which: val})
    assert v.factors is None and not v.plan.factors_dev


@pytest.mark.parametrize("shape", [(2,), (4,), (3, 1), (1, 3), (3, 2)])
def test_set_model_factors_refuses_wrong_shapes(shape):
    v = _venv("hopper")
    for which in ("friction", "gear"):
        with pytest.raises(ValueError, match="shape"):
            v.set_model_factors(**{which: np.ones(shape)})
    assert v.factors is None and not v.plan.factors_dev


@pytest.mark.parametrize("env_name", ["car2d", "pushT"])
def test_set_model_factors_refuses_flat_envs(env_name):
    v = _venv(env_name)
    for kw in (dict(friction=0.5), dict(gear=1.0), {}):
        with pytest.raises(ValueError, match="xpbd"):
            v.set_model_factors(**kw)
    assert v.factors is None and not v.plan.factors_dev
    with pytest.raises(ValueError, match="xpbd"):
        vec_mod.scaled_env(get_env(env_name), 0.5, 1.0)


def test_factor_column():
    assert vec_mod.factor_column(0.5, 3, "f").tolist() == [0.5] * 3
    c = vec_mod.factor_column(torch.tensor([0.0, 0.3, 1.7]), 3, "f")
    assert c.dtype == np.float32 and (c == np.float32([0.0, 0.3, 1.7])).all()


def _margs(**kw):
    return mbd_mpc.Args(env_name=kw.pop("env_name", "hopper"), Ndiffuse=10, Nwarm=3, Nstep=2, not_render=True,
                        disable_recommended_params=True, **kw)


def _pargs(**kw):
    return pi_mpc.Args(env_name=kw.pop("env_name", "hopper"), Nrefine=10, Nwarm=3, Nstep=2, not_render=True,
                       disable_recommended_params=True, **kw)


@pytest.mark.parametrize("make,check", [(_margs, mbd_mpc.check_args), (_pargs, pi_mpc.check_args)], ids=["mbd", "pi"])
def test_check_args_refuses_bad_plants(make, check):
    check([make(), make(seed=1, plant_friction=0.0, plant_gear=2.5)], True)     # per problem, not shared
    for f in ("plant_friction", "plant_gear"):
        for bad in BAD[:5]:
            with pytest.raises(ValueError, match="finite and >= 0"):
                check([make(), make(seed=1, **{f: bad})], True)
        for env_name in ("car2d", "pushT"):
            check([make(env_name=env_name, **{f: 1.0})], False)
            with pytest.raises(ValueError, match="xpbd"):
                check([make(env_name=env_name, **{f: 0.9})], False)


def test_run_mpc_script_passes_the_plant_to_every_algorithm():
    from mbd_b200.scripts import run_mpc
    a = run_mpc.Args(env_name="hopper", Nsample=64, Hsample=8, Nsolve=10, Nwarm=3, Nstep=2, plant_friction=0.5, plant_gear=1.3)
    for al in [run_mpc.mbd_args(a)] + [run_mpc.pi_args(a, m) for m in run_mpc.BASELINES]:
        assert all(x.plant_friction == 0.5 and x.plant_gear == 1.3 for x in al)


@pytest.mark.parametrize("entry", ["mbd_vec_step", "mbd_vec_set_state", "mbd_vec_reset", "mbd_vec_world_poses"])
@pytest.mark.parametrize("kind", ["pusht", "car2d"])
def test_abi_refuses_factors_for_flat_envs(entry, kind):
    L = _lib.lib()
    fields = dict(factors_dev=0x5000)
    if kind == "car2d":
        fields.update(kind=_lib.VEC_CAR2D, nq=3, done_rule=0)
    P = _plan(**fields)
    if entry == "mbd_vec_reset":
        rc = L.mbd_vec_reset(ctypes.byref(P), ctypes.c_void_p(0x4000), None)
    elif entry == "mbd_vec_world_poses":
        rc = L.mbd_vec_world_poses(ctypes.byref(P), ctypes.c_void_p(0x4000), ctypes.c_void_p(0x4000), None)
    else:
        rc = getattr(L, entry)(ctypes.byref(P), None)
    assert rc == -1
    err = L.mbd_last_error().decode()
    assert err.startswith(entry) and "xpbd envs only" in err, err


def test_factors_dev_is_appended():
    V = _lib.VecPlan
    assert V.factors_dev.offset == V.steps_dev.offset + 8 == ctypes.sizeof(V) - 8   # appended: every other offset stays


def _word_masks():
    """(friction words, gear words) of the blob: field 4 of every contact slot and D_GEAR of every dof slot, every link"""
    fr, gr = np.zeros(B.BLOB_WORDS, bool), np.zeros(B.BLOB_WORDS, bool)
    for l in range(B.MAXL):
        for ci in range(B.MAXCON):
            fr[B.HDR_WORDS + (B.F_CON0 + ci * B.CON_STRIDE + 4) * B.MAXL + l] = True
        for k in range(B.MAXDOF):
            gr[B.HDR_WORDS + (B.F_DOF0 + k * B.DOF_STRIDE + B.D_GEAR) * B.MAXL + l] = True
    return fr, gr


@pytest.mark.parametrize("env_name", XPBD)
@pytest.mark.parametrize("friction,gear", [(0.3, 1.4), (1.7, 0.5), (0.0, 1.0), (1.0, 0.7), (1.0, 1.0)])
def test_scaled_env_blob_differs_in_exactly_the_factored_words(env_name, friction, gear):
    env = get_env(env_name)
    sc = vec_mod.scaled_env(env, friction, gear)
    assert type(sc) is type(env) and sc.sys is not env.sys and sc.blob is not env.blob
    nom, got = env.blob.view(np.float32), sc.blob.view(np.float32)
    fr, gr = _word_masks()
    rest = ~(fr | gr)
    assert (env.blob[rest] == sc.blob[rest]).all()
    for mask, f in ((fr, friction), (gr, gear)):
        want = (nom[mask] * np.float32(f)).astype(np.float32)
        assert (want.view(np.uint32) == got[mask].view(np.uint32)).all()
    # the factors reach words that matter: every env here has actuators, and all but cartpole have contacts
    assert (nom[gr] != 0).any() and (nom[fr] != 0).any() == (env_name != "cartpole")
    moved = (gear != 1.0) or (friction != 1.0 and env_name != "cartpole")
    assert (env.blob != sc.blob).any() == moved
    # the env it came from is untouched
    assert (env.blob == get_env(env_name).blob).all()
