"""Worst-m scores and drawn members of the planner ensemble without a GPU (DESIGN.md §5m): ens_worst in the former pad word and the
size of the draw plan, every C refusal (all before any CUDA call), the refusals of the engines and of the controllers' check_args, the member
key chain, the numpy worst-m specification on constructed families, and the run_mpc driver."""
import ctypes
import itertools

import numpy as np
import pytest

from mbd_b200 import _lib, prng
from mbd_b200.envs import get_env
from mbd_b200.planners import engine as eng
from mbd_b200.planners import mbd_mpc, pi_mpc
from tests import ens_ref, ens_risk_ref

FAKE = 0x1000   # never dereferenced: every case below fails validation, which runs before the first CUDA call
f32 = np.float32


def test_ens_worst_takes_the_pad_word():
    P = _lib.StepPlan
    assert P.ens_worst.offset == P.ens_k.offset + 4 and ctypes.sizeof(P) == P.ens_k.offset + 8   # the former pad word
    assert ctypes.sizeof(_lib.EnsDrawPlan) == 48


# ---- the C refusals -----------------------------------------------------------------------------------------------------------
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
CASES = [
    (dict(ens_worst=1), "ens_worst must be 0 without an ensemble table"),
    (dict(ens_worst=-1), "ens_worst must be 0 without an ensemble table"),
    (dict(TABLE, ens_worst=4), "ens_worst must be in 0 .. ens_k"),
    (dict(TABLE, ens_worst=-1), "ens_worst must be in 0 .. ens_k"),
    (dict(TABLE, ens_k=1, ens_worst=2), "ens_worst must be in 0 .. ens_k"),
]
IDS = ["no-table", "no-table-neg", "above-k", "neg", "above-k1"]


@pytest.mark.parametrize("kw,msg", CASES, ids=IDS)
def test_batch_steps_refuse(kw, msg):
    L = _lib.lib()
    rc = L.mbd_batch_step_launch(ctypes.byref(_plan(**kw)), 4, 10, None, None)
    err = L.mbd_last_error().decode()
    assert rc == -1 and err.startswith("mbd_batch_step_launch: ") and msg in err, (rc, err)
    bufs = _lib.PiBufs(FAKE, FAKE, FAKE)
    rc = L.mbd_pi_batch_step_launch(ctypes.byref(_plan(**kw)), 4, 10, _lib.PI_METHODS["cem"], None, ctypes.byref(bufs), 0, None)
    err = L.mbd_last_error().decode()
    assert rc == -1 and err.startswith("mbd_pi_batch_step_launch: ") and msg in err, (rc, err)


def test_worst_within_k_passes_the_ensemble_checks():
    """ens_worst in 0 .. ens_k gets past the ensemble checks to the next refusal (a car2d table has no positional model)"""
    L = _lib.lib()
    for w in range(4):
        rc = L.mbd_batch_step_launch(ctypes.byref(_plan(**TABLE, ens_worst=w)), 4, 10, None, None)
        err = L.mbd_last_error().decode()
        assert rc == -1 and "xpbd" in err, (w, err)


@pytest.mark.parametrize("entry", ["mbd_step_launch", "mbd_step_launch_ev", "mbd_step_tail_launch"])
def test_single_solve_entries_refuse_ens_worst(entry):
    L = _lib.lib()
    p = _plan(ens_worst=1)
    if entry == "mbd_step_launch_ev":
        rc = L.mbd_step_launch_ev(ctypes.byref(p), None, None, None, None, None)
    else:
        rc = getattr(L, entry)(ctypes.byref(p), None)
    err = L.mbd_last_error().decode()
    assert rc == -1 and err.startswith(entry + ": ") and "no planner ensemble" in err, (rc, err)


@pytest.mark.parametrize("args,msg", [
    ((None, FAKE, 8, 3, 1), "a buffer is NULL"),
    ((FAKE, None, 8, 3, 1), "a buffer is NULL"),
    ((FAKE, FAKE, 0, 3, 1), "count must be at least 1"),
    ((FAKE, FAKE, 8, 0, 0), "K must be in 1 .. MBD_ENS_MAXK"),
    ((FAKE, FAKE, 8, 17, 1), "K must be in 1 .. MBD_ENS_MAXK"),
    ((FAKE, FAKE, 8, 3, 4), "worst must be in 0 .. K"),
    ((FAKE, FAKE, 8, 3, -1), "worst must be in 0 .. K"),
], ids=["rews-in", "rews-out", "count", "k0", "k17", "above-k", "neg"])
def test_ens_score_refuses(args, msg):
    L = _lib.lib()
    rc = L.mbd_ens_score(*args, None)
    err = L.mbd_last_error().decode()
    assert rc == -1 and err.startswith("mbd_ens_score: ") and msg in err, (rc, err)


def _draw_plan(**kw):
    p = _lib.EnsDrawPlan()
    p.B, p.K, p.Nstep = 4, 3, 10
    p.keys_dev = p.ranges_dev = p.mpc_ctl_dev = p.ens_factors_dev = FAKE
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@pytest.mark.parametrize("kw,msg", [
    (dict(keys_dev=None), "a buffer is NULL"),
    (dict(ranges_dev=None), "a buffer is NULL"),
    (dict(mpc_ctl_dev=None), "a buffer is NULL"),
    (dict(ens_factors_dev=None), "a buffer is NULL"),
    (dict(B=0), "B must be in 1..65536"),
    (dict(B=65537), "B must be in 1..65536"),
    (dict(K=0), "K must be in 1 .. MBD_ENS_MAXK"),
    (dict(K=17), "K must be in 1 .. MBD_ENS_MAXK"),
    (dict(Nstep=0), "Nstep must be at least 1"),
], ids=["keys", "ranges", "ctl", "factors", "B0", "Bbig", "K0", "K17", "Nstep"])
def test_ens_draw_refuses(kw, msg):
    L = _lib.lib()
    rc = L.mbd_ens_draw(ctypes.byref(_draw_plan(**kw)), None)
    err = L.mbd_last_error().decode()
    assert rc == -1 and err.startswith("mbd_ens_draw: ") and msg in err, (rc, err)
    rc = L.mbd_ens_draw(None, None)
    assert rc == -1 and "plan is NULL" in L.mbd_last_error().decode()


# ---- the engines --------------------------------------------------------------------------------------------------------------
def test_engines_refuse_ens_worst_before_touching_the_device():
    """these raise ValueError on a machine without a GPU: the check runs before the engine asks for a device"""
    from mbd_b200.planners.path_integral import BatchedPathIntegralEngine
    env = get_env("hopper")
    mk = [lambda **kw: eng.BatchedDiffusionEngine(env, 16, 8, [0.1], False, [None], 10, **kw),
          lambda **kw: BatchedPathIntegralEngine(env, 16, 8, [0.1], [None], 10, "mppi", **kw)]
    for make in mk:
        with pytest.raises(ValueError, match="needs a planner ensemble"):
            make(ens_worst=1)
        with pytest.raises(ValueError, match=r"0 \.\. K = 2"):
            make(ensemble=np.ones((1, 2, 2)), ens_worst=3)
        with pytest.raises(ValueError, match=r"0 \.\. K = 2"):
            make(ensemble=np.ones((1, 2, 2)), ens_worst=-1)
        for bad in (True, 1.0, "1"):
            with pytest.raises(ValueError, match="must be an int"):
                make(ensemble=np.ones((1, 2, 2)), ens_worst=bad)
    assert eng.check_ens_worst(0, None) == 0 and eng.check_ens_worst(np.int64(2), 2) == 2


# ---- the controllers' Args ----------------------------------------------------------------------------------------------------
def _margs(**kw):
    return mbd_mpc.Args(env_name=kw.pop("env_name", "hopper"), Ndiffuse=10, Nwarm=3, Nstep=2, not_render=True,
                        disable_recommended_params=True, **kw)


def _pargs(**kw):
    return pi_mpc.Args(env_name=kw.pop("env_name", "hopper"), Nrefine=10, Nwarm=3, Nstep=2, not_render=True,
                       disable_recommended_params=True, **kw)


DRAW = dict(plan_members=4, plan_friction_range=(0.5, 1.5), plan_gear_range=(0.7, 1.3))
FIXED = dict(plan_friction=(1.0, 1.0, 1.0), plan_gear=(0.7, 1.0, 1.3))


@pytest.mark.parametrize("make,check", [(_margs, mbd_mpc.check_args), (_pargs, pi_mpc.check_args)], ids=["mbd", "pi"])
def test_check_args_accepts(make, check):
    check([make(**DRAW), make(seed=1, **DRAW)], True)
    check([make(**DRAW, plan_worst=2), make(seed=2 ** 32 - 1, **DRAW, plan_worst=2)], True)
    check([make(**FIXED, plan_worst=1), make(seed=1, **FIXED, plan_worst=1)], True)
    check([make(**FIXED, plan_worst=3)], True)
    check([make(plan_members=16, plan_friction_range=(1.0, 1.0), plan_gear_range=(0.0, 0.0), plan_worst=16)], True)
    check([make(**DRAW), make(seed=1, plan_members=4, plan_friction_range=(0.0, 2.0), plan_gear_range=(1.0, 1.0))], True)


@pytest.mark.parametrize("make,check", [(_margs, mbd_mpc.check_args), (_pargs, pi_mpc.check_args)], ids=["mbd", "pi"])
def test_check_args_refuses(make, check):
    def refuses(al, match):
        with pytest.raises(ValueError, match=match):
            check(al, True)
    refuses([make(**DRAW, **FIXED)], "excludes plan_friction")
    refuses([make(plan_members=4, plan_gear_range=(0.7, 1.3))], r"plan_friction_range must be \(lo, hi\)")
    refuses([make(plan_members=4, plan_friction_range=(0.5, 1.5))], r"plan_gear_range must be \(lo, hi\)")
    for bad in [(1.0,), (0.5, 1.0, 1.5), (1.5, 0.5), (-0.1, 1.0), (0.5, float("inf")), (float("nan"), 1.0), (0.5, 1e39)]:
        refuses([make(**{**DRAW, "plan_gear_range": bad})], "plan_gear_range must be")
        refuses([make(**{**DRAW, "plan_friction_range": bad})], "plan_friction_range must be")
    refuses([make(plan_friction_range=(0.5, 1.5))], "needs plan_members")
    refuses([make(**FIXED, plan_gear_range=(0.5, 1.5))], "needs plan_members")
    for M in (-1, 17, 1.5, True):
        refuses([make(**{**DRAW, "plan_members": M})], "plan_members must be an int")
    refuses([make(**DRAW, plan_worst=5)], r"plan_worst must be in 0 \.\. K = 4")
    refuses([make(**FIXED, plan_worst=4)], r"plan_worst must be in 0 \.\. K = 3")
    refuses([make(**DRAW, plan_worst=-1)], r"plan_worst must be in 0 \.\. K = 4")
    refuses([make(plan_worst=1)], "needs a planner ensemble")
    refuses([make(**DRAW, plan_worst=1.0)], "plan_worst must be an int")
    refuses([make(**DRAW), make(seed=1, **{**DRAW, "plan_members": 3})], "same number of ensemble members")
    refuses([make(**DRAW), make(seed=1, plan_friction=(1.0,) * 4, plan_gear=(1.0,) * 4)], "draw its members")
    refuses([make(**DRAW), make(seed=1, plan_friction=(1.0,) * 3, plan_gear=(1.0,) * 3)], "same number of ensemble members")
    refuses([make(**DRAW, plan_worst=1), make(seed=1, **DRAW, plan_worst=2)], "same plan_worst")
    refuses([make(**FIXED, plan_worst=1), make(seed=1, **FIXED)], "same plan_worst")
    refuses([make(seed=-1, **DRAW)], "seed in 0 .. 2")
    refuses([make(seed=2 ** 32, **DRAW)], "seed in 0 .. 2")
    for env_name in ("car2d", "pushT"):
        with pytest.raises(ValueError, match="xpbd"):
            check([make(env_name=env_name, **DRAW)], False)
        with pytest.raises(ValueError, match="needs a planner ensemble"):
            check([make(env_name=env_name, plan_worst=1)], False)


def test_drawn_ensemble_starts_as_unit_members():
    al = [_margs(seed=b, **DRAW) for b in range(3)]
    t = mbd_mpc.plan_ensemble(al)
    assert t.dtype == np.float32 and t.shape == (3, 4, 2) and (t == 1).all()


# ---- the member key chain and the draw ------------------------------------------------------------------------------------------
def test_member_keys_restated():
    for s in (0, 1, 7, 2 ** 32 - 1):
        want = prng.split(np.array([1, s], np.uint32), 50)
        assert np.array_equal(mbd_mpc.member_keys(s, 50), want)


def test_member_keys_never_collide_with_the_controller_keys():
    """seeds 0 .. 7 at the closed-loop settings: no member key (nor its two sub-keys) equals any key of mpc_keys (rng_reset, the
    cold chain, every warm row) of any of the seeds"""
    Nd, Nw, Ns = 100, 10, 50
    ctl = set()
    for s in range(8):
        rr, cold, warm = mbd_mpc.mpc_keys(s, Nd, Nw, Ns)
        ctl.add(tuple(int(x) for x in rr))
        ctl.update(tuple(int(x) for x in k) for k in cold)
        ctl.update(tuple(int(x) for x in k) for k in warm[1:].reshape(-1, 2))
    mem = set()
    for s in range(8):
        for k in mbd_mpc.member_keys(s, Ns):
            mem.add(tuple(int(x) for x in k))
            mem.update(tuple(int(x) for x in sub) for sub in prng.split(k))
    assert len(mem) == 8 * Ns * 3          # distinct among themselves too
    assert not (mem & ctl)


def test_draw_members_specification():
    key = mbd_mpc.member_keys(3, 5)[2]
    m = mbd_mpc.draw_members(key, 7, (0.5, 1.5), (0.7, 1.3))
    kf, kg = prng.split(key)
    assert m.dtype == np.float32 and m.shape == (7, 2)
    assert np.array_equal(m[:, 0], prng.uniform(kf, (7,), 0.5, 1.5)) and np.array_equal(m[:, 1], prng.uniform(kg, (7,), 0.7, 1.3))
    assert (m[:, 0] >= f32(0.5)).all() and (m[:, 0] < f32(1.5)).all() and (m[:, 1] >= f32(0.7)).all() and (m[:, 1] < f32(1.3)).all()
    same = mbd_mpc.draw_members(key, 16, (1.0, 1.0), (0.0, 0.0))
    assert (same[:, 0] == f32(1.0)).all() and (same[:, 1] == f32(0.0)).all() and not np.signbit(same).any()
    assert len(set(m[:, 0].tolist())) == 7


# ---- the worst-m specification ------------------------------------------------------------------------------------------------
def _brute(row, m):
    """one row, the definition read literally: Python's sort on (value, member index)"""
    if any(np.isnan(row)):
        return ens_risk_ref.NAN
    order = sorted(range(len(row)), key=lambda k: (float(row[k]), k))
    s = f32(row[order[0]])
    with np.errstate(over="ignore", invalid="ignore"):
        for j in range(1, m):
            s = f32(s + row[order[j]])
        s = f32(s / f32(m))
    return ens_risk_ref.NAN if np.isnan(s) else s


def families(K: int, seed: int = 0) -> np.ndarray:
    """[rows, K] constructed member returns: random, ties, ±0 in both orders, ±inf, NaN, and huge values whose sums cancel"""
    g = np.random.default_rng(1000 * K + seed)
    rows = [g.standard_normal(K), g.integers(-2, 3, K).astype(np.float64), np.zeros(K), -np.zeros(K),
            np.where(np.arange(K) % 2, 0.0, -0.0), np.where(np.arange(K) % 2, -0.0, 0.0),
            np.full(K, 1e38), np.full(K, -1e38), g.standard_normal(K) * 1e30]
    for special in (np.inf, -np.inf, np.nan):
        for pos in {0, K // 2, K - 1}:
            r = g.standard_normal(K)
            r[pos] = special
            rows.append(r)
    r = g.standard_normal(K)
    r[0], r[-1] = np.inf, -np.inf
    rows.append(r)
    r = g.standard_normal(K)
    r[:] = r[0]
    rows.append(r)
    return np.asarray(rows, dtype=f32)


@pytest.mark.parametrize("K", range(1, 17))
def test_worst_m_specification(K):
    r = families(K)
    for m in range(K + 1):
        got = ens_risk_ref.worst_m(r, m)
        if m == 0:
            assert np.array_equal(got.view(np.uint32), ens_ref.ordered_mean(r).view(np.uint32))
            continue
        want = np.array([_brute(row, m) for row in r], dtype=f32)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (K, m)
    # m = 1 is the minimum exactly, signed zeros by member order
    fin = r[~np.isnan(r).any(axis=1)]
    w1 = ens_risk_ref.worst_m(fin, 1)
    assert np.array_equal(w1, fin.min(axis=1))
    z = np.where(np.arange(K) % 2, 0.0, -0.0).astype(f32)[None]
    assert np.signbit(ens_risk_ref.worst_m(z, 1)[0]) and not np.signbit(ens_risk_ref.worst_m(-z, 1)[0])


def test_worst_m_is_order_free_up_to_signed_zeros():
    g = np.random.default_rng(3)
    r = g.standard_normal((64, 9)).astype(f32)
    for perm in itertools.islice(itertools.permutations(range(9)), 0, 2000, 97):
        for m in range(1, 10):
            assert np.array_equal(ens_risk_ref.worst_m(r[:, list(perm)], m), ens_risk_ref.worst_m(r, m))


def test_worst_m_refuses_m_outside_k():
    with pytest.raises(ValueError):
        ens_risk_ref.worst_m(np.zeros((2, 3), f32), 4)


# ---- the run_mpc driver -------------------------------------------------------------------------------------------------------
def test_run_mpc_script_passes_the_new_flags_to_every_algorithm():
    from mbd_b200.scripts import run_mpc
    a = run_mpc.Args(env_name="hopper", Nsample=64, Hsample=8, Nsolve=10, Nwarm=3, Nstep=2, plan_members=4,
                     plan_friction_range=(0.5, 1.5), plan_gear_range=(0.7, 1.3), plan_worst=2)
    for al in [run_mpc.mbd_args(a)] + [run_mpc.pi_args(a, m) for m in run_mpc.BASELINES]:
        assert all(x.plan_members == 4 and x.plan_friction_range == (0.5, 1.5) and x.plan_gear_range == (0.7, 1.3)
                   and x.plan_worst == 2 for x in al)
        (mbd_mpc if isinstance(al[0], mbd_mpc.Args) else pi_mpc).check_args(al, True)
    nominal = run_mpc.Args()
    assert all(x.plan_members == 0 and x.plan_worst == 0 and x.plan_friction_range == () and x.plan_gear_range == ()
               for x in run_mpc.mbd_args(nominal) + run_mpc.pi_args(nominal, "cem"))


def test_run_mpc_script_parses_the_new_flags():
    import tyro
    from mbd_b200.scripts import run_mpc
    a = tyro.cli(run_mpc.Args, args=["--plan_members", "4", "--plan_friction_range", "0.5", "1.5", "--plan_gear_range", "0.7", "1.3",
                                     "--plan_worst", "2"])
    assert a.plan_members == 4 and a.plan_worst == 2
    assert tuple(a.plan_friction_range) == (0.5, 1.5) and tuple(a.plan_gear_range) == (0.7, 1.3)
    b = tyro.cli(run_mpc.Args, args=["--plan_friction", "1", "1", "1", "--plan_gear", "0.7", "1", "1.3", "--plan_worst", "1"])
    assert b.plan_worst == 1 and tuple(b.plan_gear) == (0.7, 1.0, 1.3)
