"""Domain randomisation without a GPU (DESIGN.md §5n): the host specification dr_factors against a direct numpy restatement in both
threefry layouts, the key roots of the trainers and of run_mpc's policy row against the controllers' chains, every refusal (the C ABI's
before any CUDA call, VecEnv.set_domain_randomization's before any device call, the trainers' and the CLIs'), the new CLI flags, and
the layout of mbd_vec_dr beside an unchanged mbd_vec_plan."""
import ctypes

import numpy as np
import pytest
import torch

from mbd_b200 import _lib, prng
from mbd_b200.envs import get_env
from mbd_b200.envs import vec as vec_mod
from mbd_b200.planners import mbd_mpc
from mbd_b200.rl import ppo, sac
from tests.test_vecenv_cpu import _plan

f32 = np.float32
FAKE = 0x5000   # never dereferenced: every case below fails validation, which runs before the first CUDA call
RANGES = [((0.5, 1.5), (0.7, 1.3)), ((0.0, 2.0), (1.0, 1.0)), ((1.0, 1.0), (1.0, 1.0)), ((0.3, 0.3), (0.0, 4.0))]


@pytest.fixture(params=[False, True], ids=["legacy", "partitionable"])
def layout(request):
    prng.set_layout(request.param)
    try:
        yield request.param
    finally:
        prng.set_layout(False)


# ---- the host specification ---------------------------------------------------------------------------------------------------
def _restated(key, e, fr, gr, part):
    """dr_factors written out with threefry2x32 blocks: fold_in, split(., 2) and uniform(., (1,)) of prng's two layouts"""
    tf = prng.threefry2x32
    a, b = tf(key, np.uint32([0]), np.uint32([e]))
    k = np.uint32([a[0], b[0]])
    if part:
        kf, kg = [np.uint32([x[0] for x in tf(k, np.uint32([0]), np.uint32([i]))]) for i in (0, 1)]
        bits = [np.bitwise_xor(*tf(kk, np.uint32([0]), np.uint32([0])))[0] for kk in (kf, kg)]
    else:
        o0, o1 = tf(k, np.uint32([0, 1]), np.uint32([2, 3]))   # random_bits(k, 4) = o0 | o1, rows of two
        kf, kg = np.uint32([o0[0], o0[1]]), np.uint32([o1[0], o1[1]])
        bits = [tf(kk, np.uint32([0]), np.uint32([0]))[0][0] for kk in (kf, kg)]   # random_bits(., 1): counters (0, 0), word 0
    out = []
    for bb, (lo, hi) in zip(bits, (fr, gr)):
        u = (np.uint32([bb]) >> np.uint32(9) | np.uint32(0x3F800000)).view(f32)[0] - f32(1)
        out.append(max(f32(lo), f32(u * (f32(hi) - f32(lo)) + f32(lo))))
    return out


@pytest.mark.parametrize("fr,gr", RANGES)
def test_dr_factors_against_the_restatement(layout, fr, gr):
    for seed in range(3):
        for b, key in enumerate(prng.split(prng.PRNGKey((2 << 32) | seed), 5)):
            for e in (0, 1, 2, 7, 1000, 2 ** 31 - 1):
                f, g = vec_mod.dr_factors(key, e, fr, gr)
                rf, rg = _restated(key, e, fr, gr, layout)
                assert f.dtype == f32 and g.dtype == f32
                assert f.view(np.uint32) == rf.view(np.uint32) and g.view(np.uint32) == rg.view(np.uint32), (seed, b, e)


def test_equal_bounds_give_the_bound(layout):
    for key in prng.split(prng.PRNGKey(9), 16):
        for e in range(6):
            for v in (0.0, 0.3, 1.0, 2.5):
                f, g = vec_mod.dr_factors(key, e, (v, v), (v, v))
                assert f == f32(v) and g == f32(v)


def test_draws_stay_in_range_and_differ(layout):
    fr, gr = (0.5, 1.5), (0.7, 1.3)
    draws = np.array([[vec_mod.dr_factors(k, e, fr, gr) for e in range(20)] for k in prng.split(prng.PRNGKey(3), 20)])
    assert (draws[..., 0] >= f32(0.5)).all() and (draws[..., 0] <= f32(1.5)).all()
    assert (draws[..., 1] >= f32(0.7)).all() and (draws[..., 1] <= f32(1.3)).all()
    flat = draws.reshape(-1, 2)
    assert len({tuple(x) for x in flat.tolist()}) == len(flat)      # every (env, episode) its own plant
    assert len(set(flat[:, 0].tolist())) == len(flat) and len(set(flat[:, 1].tolist())) == len(flat)


# ---- key roots ------------------------------------------------------------------------------------------------------------------
def _rows(a):
    return {tuple(int(x) for x in r) for r in np.asarray(a, np.uint32).reshape(-1, 2)}


def test_key_roots_share_no_key_with_the_controllers():
    from mbd_b200.scripts import run_mpc
    seeds, Nstep = range(8), 50
    ctl = set()
    for s in seeds:
        rng_reset, cold, warm = mbd_mpc.mpc_keys(s, 100, 10, Nstep)
        ctl |= _rows(rng_reset) | _rows(cold) | _rows(warm[1:]) | _rows(mbd_mpc.member_keys(s, Nstep))
        ctl |= _rows(prng.PRNGKey(s)) | _rows(prng.PRNGKey((1 << 32) | s))
    new = set()
    for s in seeds:
        new |= _rows(ppo.dr_keys(s, 2048)) | _rows(run_mpc.policy_keys(s, Nstep))
        new |= _rows(prng.PRNGKey((2 << 32) | s)) | _rows(prng.PRNGKey((3 << 32) | s))
    assert len(new) == 8 * (2048 + Nstep + 2)
    assert not new & ctl
    assert np.array_equal(ppo.dr_keys(5, 128), prng.split(np.uint32([2, 5]), 128))
    assert np.array_equal(run_mpc.policy_keys(5, 50), prng.split(np.uint32([3, 5]), 50))
    assert sac.dr_keys is ppo.dr_keys
    with pytest.raises(ValueError, match="seed"):
        ppo.dr_keys(-1, 4)
    with pytest.raises(ValueError, match="seed"):
        run_mpc.policy_keys(1 << 32, 4)


def test_fold_in_moved_to_prng():
    assert ppo.fold_in is prng.fold_in and sac.fold_in is prng.fold_in
    k = np.uint32([7, 11])
    o0, o1 = prng.threefry2x32(k, np.uint32([0]), np.uint32([5]))
    assert np.array_equal(prng.fold_in(k, 5), np.uint32([o0[0], o1[0]]))


# ---- the C ABI ------------------------------------------------------------------------------------------------------------------
def test_dr_struct_leaves_the_plan_as_it_was():
    V, D = _lib.VecPlan, _lib.VecDr
    assert V.factors_dev.offset == V.steps_dev.offset + 8 == ctypes.sizeof(V) - 8   # mbd_vec_plan keeps its layout
    assert D.keys_dev.offset == 0 and D.episodes_dev.offset == 8 and D.range.offset == 16 and ctypes.sizeof(D) == 32


def _xpbd(**kw):
    """an xpbd plan whose model and kinematics pointers are never dereferenced: the DR checks come first"""
    base = dict(kind=_lib.VEC_XPBD, params_dev=None, model=0x2000, kin_dev=0x3000, obs_layout=0, nq=7, nqd=6, nu=3, factors_dev=FAKE)
    base.update(kw)
    return _plan(**base)


def _dr(rng=(0.5, 1.5, 0.7, 1.3), keys=FAKE, episodes=FAKE):
    D = _lib.VecDr()
    D.keys_dev, D.episodes_dev = keys, episodes
    D.range[:] = list(rng)
    return D


NAN, INF = float("nan"), float("inf")
ABI_CASES = [
    (lambda: (_plan(), _dr()), "xpbd envs only"),
    (lambda: (_plan(kind=_lib.VEC_CAR2D, nq=3, done_rule=0), _dr()), "xpbd envs only"),
    (lambda: (_xpbd(), None), "dr is NULL"),
    (lambda: (_xpbd(factors_dev=None), _dr()), "needs the plan's factors_dev"),
    (lambda: (_xpbd(), _dr(keys=None)), "needs keys_dev and episodes_dev"),
    (lambda: (_xpbd(), _dr(episodes=None)), "needs keys_dev and episodes_dev"),
    (lambda: (_xpbd(), _dr(rng=(NAN, 1, 1, 1))), "finite and >= 0"),
    (lambda: (_xpbd(), _dr(rng=(1, INF, 1, 1))), "finite and >= 0"),
    (lambda: (_xpbd(), _dr(rng=(1, 1, -INF, 1))), "finite and >= 0"),
    (lambda: (_xpbd(), _dr(rng=(-0.1, 1, 1, 1))), "finite and >= 0"),
    (lambda: (_xpbd(), _dr(rng=(1, 1, 1, -1e-30))), "finite and >= 0"),
    (lambda: (_xpbd(), _dr(rng=(1.5, 0.5, 1, 1))), "lo <= hi"),
    (lambda: (_xpbd(), _dr(rng=(1, 1, 1.3, 0.7))), "lo <= hi"),
]


@pytest.mark.parametrize("case", range(len(ABI_CASES)))
@pytest.mark.parametrize("entry", ["mbd_vec_step_dr", "mbd_vec_reset_dr"])
def test_abi_refuses_bad_randomization(entry, case):
    make, msg = ABI_CASES[case]
    P, D = make()
    d = ctypes.byref(D) if D is not None else None
    L = _lib.lib()
    if entry == "mbd_vec_reset_dr":
        rc = L.mbd_vec_reset_dr(ctypes.byref(P), d, ctypes.c_void_p(0x4000), None)
    else:
        rc = L.mbd_vec_step_dr(ctypes.byref(P), d, None)
    assert rc == -1   # MBD_EINVAL
    err = L.mbd_last_error().decode()
    assert err.startswith(entry) and msg in err, err


def test_abi_dr_entries_keep_the_plan_checks():
    """a good DR struct on a bad plan: the plan's own refusals still apply"""
    L = _lib.lib()
    P = _xpbd(model=None)
    assert L.mbd_vec_step_dr(ctypes.byref(P), ctypes.byref(_dr()), None) == -1
    assert "needs a model" in L.mbd_last_error().decode()
    P = _xpbd(model=None)
    assert L.mbd_vec_reset_dr(ctypes.byref(P), ctypes.byref(_dr()), None, None) == -1


# ---- VecEnv.set_domain_randomization --------------------------------------------------------------------------------------------
def _venv(env_name, num_envs=3):
    """a VecEnv shell whose device is cuda: any device call raises here, so every refusal must come first"""
    v = vec_mod.VecEnv.__new__(vec_mod.VecEnv)
    v.env, v.num_envs, v.spec = get_env(env_name), num_envs, vec_mod.env_spec(get_env(env_name))
    v.device, v.plan, v.factors, v.dr, v.dr_keys, v.dr_episodes = torch.device("cuda", 0), _lib.VecPlan(), None, None, None, None
    return v


BAD_RANGES = [((NAN, 1.0), (1.0, 1.0)), ((1.0, 1.0), (0.5, INF)), ((-0.5, 1.0), (1.0, 1.0)), ((1.0, 1.0), (-1.0, -0.5)),
              ((1.5, 0.5), (1.0, 1.0)), ((1.0, 1.0), (1.3, 0.7)), ((1e39, 1e39), (1.0, 1.0)),
              ((1.0,), (1.0, 1.0)), ((1.0, 1.0, 1.0), (1.0, 1.0)), (1.0, (1.0, 1.0)), (("a", "b"), (1.0, 1.0)), (None, (1.0, 1.0))]


@pytest.mark.parametrize("fr,gr", BAD_RANGES)
def test_set_domain_randomization_refuses_bad_ranges(fr, gr):
    v = _venv("hopper")
    with pytest.raises(ValueError, match="range"):
        v.set_domain_randomization(fr, gr, np.zeros((3, 2), np.uint32))
    assert v.factors is None and v.dr_episodes is None and v.dr is None and not v.plan.factors_dev


@pytest.mark.parametrize("keys", [np.zeros((2, 2), np.uint32), np.zeros((3,), np.uint32), np.zeros((3, 3), np.uint32),
                                  np.zeros((1, 3, 2), np.uint32), torch.zeros((3, 2), dtype=torch.float32),
                                  torch.zeros((3, 1), dtype=torch.int32)], ids=["B-1", "flat", "3x3", "3d", "float", "3x1"])
def test_set_domain_randomization_refuses_wrong_keys(keys):
    v = _venv("hopper")
    with pytest.raises(ValueError, match="keys must be uint32"):
        v.set_domain_randomization((0.5, 1.5), (0.7, 1.3), keys)
    assert v.factors is None and v.dr_episodes is None and v.dr is None


@pytest.mark.parametrize("env_name", ["car2d", "pushT"])
def test_set_domain_randomization_refuses_flat_envs(env_name):
    v = _venv(env_name)
    with pytest.raises(ValueError, match="xpbd"):
        v.set_domain_randomization((0.5, 1.5), (0.7, 1.3), np.zeros((3, 2), np.uint32))
    assert v.factors is None and v.dr is None


def test_dr_range_accepts_good_ranges():
    assert np.array_equal(vec_mod.dr_range((0.5, 1.5), [0, 0]), f32([0.5, 1.5, 0, 0]))
    assert np.array_equal(vec_mod.dr_range(np.array([1, 1]), torch.tensor([0.7, 1.3])), f32([1, 1, 0.7, 1.3]))


# ---- the trainers and the CLIs --------------------------------------------------------------------------------------------------
def test_check_randomization():
    hop = get_env("hopper")
    assert ppo.check_randomization(None, hop) is None
    fr, gr = ppo.check_randomization(dict(friction_range=(0.5, 1.5)), hop)
    assert fr == (f32(0.5), f32(1.5)) and gr == (1.0, 1.0)
    for bad in (dict(friction=(0.5, 1.5)), dict(friction_range=(0.5, 1.5), mass_range=(1, 1)), ((0.5, 1.5), (1, 1)),
                dict(friction_range=(1.5, 0.5)), dict(gear_range=(-1, 1)), dict(gear_range=(1, NAN))):
        with pytest.raises(ValueError):
            ppo.check_randomization(bad, hop)
    for name in ("car2d", "pushT"):
        with pytest.raises(ValueError, match="xpbd"):
            ppo.check_randomization(dict(friction_range=(1, 1)), get_env(name))


@pytest.mark.parametrize("env_name", ["car2d", "pushT"])
def test_trainers_refuse_flat_envs_before_the_device(env_name):
    """the refusal comes before the trainers ask for a GPU"""
    dr = dict(friction_range=(0.5, 1.5), gear_range=(1.0, 1.0))
    with pytest.raises(ValueError, match="xpbd"):
        ppo.train(env_name, num_timesteps=1000, episode_length=10, num_envs=4, batch_size=4, num_minibatches=1, randomization=dr)
    with pytest.raises(ValueError, match="xpbd"):
        sac.train(env_name, num_timesteps=1000, episode_length=10, num_envs=4, randomization=dr)


def test_train_cli_flags_parse():
    from mbd_b200.rl import train_brax, train_sac
    a = train_brax.parse_args(["--env_name", "halfcheetah", "--dr_friction", "0.5", "1.5", "--dr_gear", "0.7", "1.3"])
    assert train_brax.randomization(a) == dict(friction_range=(0.5, 1.5), gear_range=(0.7, 1.3))
    a = train_brax.parse_args(["--dr_gear", "0.7", "1.3"])
    assert train_brax.randomization(a) == dict(friction_range=(1.0, 1.0), gear_range=(0.7, 1.3))
    assert train_brax.randomization(train_brax.parse_args([])) is None
    b = train_sac.parse_args(["--learner", "fused", "--dr_friction", "0.5", "1.5", "--num_timesteps", "100"])
    assert b.learner == "fused" and b.num_timesteps == 100
    assert train_brax.randomization(b) == dict(friction_range=(0.5, 1.5), gear_range=(1.0, 1.0))
    for argv in (["--dr_friction", "0.5"], ["--dr_gear", "a", "b"]):
        with pytest.raises(SystemExit):
            train_sac.parse_args(argv)


def test_train_cli_refuses_dr_on_pusht():
    from mbd_b200.rl import train_brax
    with pytest.raises(ValueError, match="xpbd"):
        train_brax.main(["--env_name", "pushT", "--dr_friction", "0.5", "1.5", "--num_timesteps", "10"])


def test_run_mpc_policy_flags():
    import tyro

    from mbd_b200.scripts import run_mpc
    a = tyro.cli(run_mpc.Args, args=["--policy", "results/hopper/params_dr.npz", "--policy_algo", "sac", "--plant_gear", "0.7"])
    assert a.policy == "results/hopper/params_dr.npz" and a.policy_algo == "sac" and a.plant_gear == 0.7
    run_mpc.check_policy_args(a)
    run_mpc.check_policy_args(run_mpc.Args())
    for kw, msg in ((dict(policy="p.npz"), "--policy_algo"), (dict(policy="p.npz", policy_algo="td3"), "--policy_algo"),
                    (dict(policy_algo="ppo"), "--policy")):
        with pytest.raises(ValueError, match=msg):
            run_mpc.check_policy_args(run_mpc.Args(**kw))
    with pytest.raises(ValueError, match="--policy_algo"):     # before any controller runs
        run_mpc.main(["--policy", "p.npz"])
