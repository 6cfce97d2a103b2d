"""Worst-m scores and drawn members of the planner ensemble on the device (DESIGN.md §5m): the sample returns of a real ensemble step
and of constructed member returns equal the numpy worst-m specification bit for bit; identical members with ens_worst = 1 are today's
nominal step; permuting the members leaves the scores unchanged; k_ens_draw equals the host draw; and the receding-horizon
controllers with worst-m scores and drawn members replay on the device as they run with the host in the loop."""
import numpy as np
import pytest
import torch

from mbd_b200 import _lib, ops, prng
from mbd_b200.envs import get_env
from mbd_b200.planners import mbd_mpc, pi_mpc
from mbd_b200.planners.engine import BatchedDiffusionEngine, key_chain, make_schedule
from mbd_b200.planners.path_integral import BatchedPathIntegralEngine
from tests import ens_risk_ref
from tests.conftest import assert_bit_exact
from tests.test_ens_risk_cpu import families

pytestmark = pytest.mark.gpu

METHODS = ["mbd", "mppi", "cma-es", "cem"]
ND = 6
_cache = {}


def _env(name):
    if name not in _cache:
        _cache[name] = get_env(name)
    return _cache[name]


def _host(t):
    return t.detach().cpu().numpy()


def _members(B, K, seed=0):
    t = np.random.default_rng(seed).uniform(0.4, 1.6, (B, K, 2)).astype(np.float32)
    t[0, 0] = 1.0
    return t


def _engine(env_name, method, B, N, H, ensemble=None, ens_worst=0, seeds=None):
    """a batched engine of B problems (problem b: reset and key chain of seed seeds[b]) armed at its first step"""
    env = _env(env_name)
    seeds = list(range(B)) if seeds is None else seeds
    states, keys = [], []
    for s in seeds:
        rng, rng_reset = prng.split(prng.PRNGKey(s))
        states.append(env.reset(rng_reset))
        keys.append(key_chain(prng.split(rng)[0], ND))
    temps = [0.1 + 0.05 * b for b in range(B)]
    if method == "mbd":
        e = BatchedDiffusionEngine(env, N, H, temps, False, states, ND, ensemble=ensemble, ens_worst=ens_worst)
        _, al, ab, sg = make_schedule(1e-4, 1e-2, ND)
        e.load_schedule(keys, [sg] * B, [al] * B, [ab] * B)
    else:
        e = BatchedPathIntegralEngine(env, N, H, temps, states, ND, method, ensemble=ensemble, ens_worst=ens_worst)
        e.load_schedule(keys)
    e.set_step(ND - 1)
    return e


def _same_state(a, b, what):
    for f in ("Ybars", "rew_hist", "rews", "Y0s"):
        assert_bit_exact(_host(getattr(a, f)), _host(getattr(b, f)), f"{what}: {f}")
    if getattr(a, "update_method", None) == "cma-es":
        assert_bit_exact(_host(a.sigma_hist), _host(b.sigma_hist), f"{what}: sigma_hist")


# ---- 1. the score is the specification --------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("K", [1, 3, 9, 16])
@pytest.mark.parametrize("env_name", ["hopper", "humanoidrun"])
def test_step_scores_are_the_specification(env_name, K, method):
    """one step of 2 problems at every m: the member returns are those of the mean's step, the sample returns worst_m of them, and
    the next iterate the tail of those returns (m = 0 is the ordered mean)"""
    B, N, H = 2, 64, 8
    table = _members(B, K, seed=K)
    ref = None
    for m in range(K + 1):
        e = _engine(env_name, method, B, N, H, ensemble=table, ens_worst=m)
        e.step()
        ens, rews = _host(e.ens_rews), _host(e.rews)
        assert_bit_exact(rews, ens_risk_ref.worst_m(ens, m), f"m = {m}: rews = worst_m(ens_rews)")
        if ref is None:
            ref = ens
        assert_bit_exact(ens, ref, f"m = {m}: ens_rews = the mean's")
        assert np.isfinite(_host(e.Ybars)).all()


@pytest.mark.parametrize("K", range(1, 17))
def test_constructed_scores_are_the_specification(K):
    """mbd_ens_score on constructed member returns (ties, ±0 in both orders, ±inf, NaN, cancelling sums) at every m.  The mean
    (m = 0, §5l's k_ens_mean) defines no NaN bit pattern: there a NaN only has to meet a NaN"""
    r = np.concatenate([families(K, seed) for seed in range(4)] + [np.random.default_rng(K).standard_normal((300, K))]).astype(np.float32)
    dev = torch.as_tensor(r, device="cuda")
    for m in range(K + 1):
        got, want = _host(ops.ens_score(dev, m)), ens_risk_ref.worst_m(r, m)
        if m == 0:
            nan = np.isnan(want)
            assert np.array_equal(np.isnan(got), nan), f"K = {K}, m = 0: NaN positions"
            got, want = got[~nan], want[~nan]
        assert_bit_exact(got, want, f"K = {K}, m = {m}")


# ---- 2. identical members reproduce the nominal step --------------------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("K", [1, 4, 16])
def test_identical_unit_members_are_the_nominal_step(K, method):
    B, N, H = 2, 128, 12
    nom = _engine("hopper", method, B, N, H)
    e = _engine("hopper", method, B, N, H, ensemble=np.ones((B, K, 2), np.float32), ens_worst=1)
    for _ in range(3):
        nom.step()
        e.step()
    _same_state(e, nom, f"K = {K}")


# ---- 3. member order does not matter ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", ["mbd", "cem"])
def test_member_order_does_not_matter(method):
    B, N, H, K = 2, 128, 12, 5
    table = _members(B, K, seed=21)
    perm = [3, 0, 4, 2, 1]
    for m in range(1, K + 1):
        a = _engine("hopper", method, B, N, H, ensemble=table, ens_worst=m)
        b = _engine("hopper", method, B, N, H, ensemble=table[:, perm], ens_worst=m)
        for _ in range(2):
            a.step()
            b.step()
        _same_state(a, b, f"m = {m}")
        assert_bit_exact(_host(b.ens_rews), _host(a.ens_rews)[:, :, perm], f"m = {m}: permuted member returns")


# ---- 4. the draw is the host specification ------------------------------------------------------------------------------------
RANGES = [((0.5, 1.5), (0.7, 1.3)), ((1.0, 1.0), (0.7, 1.3)), ((0.0, 2.0), (0.0, 0.0)), ((0.0, 0.0), (1.0, 1.0)), ((3.0, 7.5), (0.25, 0.5))]


@pytest.mark.parametrize("K", [1, 3, 16])
def test_draw_is_the_host_specification(K):
    B, Nstep = 5, 9
    seeds = [0, 1, 7, 12345, 2 ** 32 - 1]
    keys = np.stack([mbd_mpc.member_keys(s, Nstep) for s in seeds])
    ranges = np.array([fr + gr for fr, gr in RANGES], np.float32)
    d = torch.device("cuda")
    keys_t = torch.as_tensor(keys.view(np.int32), device=d).contiguous()
    ranges_t = torch.as_tensor(ranges, device=d)
    ctl = torch.zeros(B, device=d, dtype=torch.int32)
    out = torch.zeros((B, K, 2), device=d)
    p = _lib.EnsDrawPlan()
    p.B, p.K, p.Nstep = B, K, Nstep
    p.keys_dev, p.ranges_dev, p.mpc_ctl_dev, p.ens_factors_dev = keys_t.data_ptr(), ranges_t.data_ptr(), ctl.data_ptr(), out.data_ptr()
    sentinel = np.float32(-7.0)
    for cs in ([0] * B, [1, 2, 3, 4, 8], [8, 0, 5, 9, 12], [Nstep] * B, [-1, 3, Nstep + 100, 6, 2]):
        out.fill_(float(sentinel))
        ctl.copy_(torch.tensor(cs, dtype=torch.int32))
        ops.ens_draw(p)
        got = _host(out)
        for b, c in enumerate(cs):
            if 0 <= c < Nstep:
                want = mbd_mpc.draw_members(keys[b, c], K, ranges[b, :2], ranges[b, 2:])
                assert_bit_exact(got[b], want, f"problem {b}, control step {c}")
            else:
                assert (got[b] == sentinel).all(), f"problem {b}: control step {c} is outside the loop, nothing is written"
        assert_bit_exact(_host(ctl), np.array(cs, np.int32), "the draw leaves the counters")
    # lo == hi is exactly lo
    ctl.zero_()
    ops.ens_draw(p)
    got = _host(out)
    assert (got[1, :, 0] == np.float32(1.0)).all() and (got[2, :, 1] == 0).all() and (got[3, :, 0] == 0).all()


# ---- 5. the closed loop -------------------------------------------------------------------------------------------------------
SETTINGS = {"fixed-worst1": dict(plan_friction=(1.0, 1.0, 1.0), plan_gear=(0.7, 1.0, 1.3), plan_worst=1),
            "drawn-mean": dict(plan_members=3, plan_friction_range=(0.5, 1.5), plan_gear_range=(0.7, 1.3)),
            "drawn-worst2": dict(plan_members=3, plan_friction_range=(0.5, 1.5), plan_gear_range=(0.7, 1.3), plan_worst=2)}


def mpc_args(env_name, B=2, Nstep=20, seed0=0, **kw):
    return [mbd_mpc.Args(seed=seed0 + 3 * b, env_name=env_name, Nsample=64, Hsample=8, Ndiffuse=6, Nwarm=2, Nstep=Nstep,
                         temp_sample=(0.1, 0.2, 0.05)[b % 3], plant_gear=(0.7, 1.3, 1.0)[b % 3], not_render=True,
                         disable_recommended_params=True, **kw) for b in range(B)]


def pi_args(env_name, B=2, Nstep=20, seed0=0, **kw):
    return [pi_mpc.Args(seed=seed0 + 3 * b, env_name=env_name, update_method="mppi", Nsample=64, Hsample=8, Nrefine=6, Nwarm=2,
                        Nstep=Nstep, sigma_warm=0.7, temp_sample=(0.1, 0.2, 0.05)[b % 3], plant_gear=(0.7, 1.3, 1.0)[b % 3],
                        not_render=True, disable_recommended_params=True, **kw) for b in range(B)]


def _assert_result(r, q, what, rows=slice(None)):
    for f in ("actions", "rewards", "states", "rew_hist"):
        assert_bit_exact(getattr(r, f)[rows], getattr(q, f), f"{what}: {f}")


@pytest.mark.parametrize("setting", list(SETTINGS))
@pytest.mark.parametrize("mod,make", [(mbd_mpc, mpc_args), (pi_mpc, pi_args)], ids=["mbd", "mppi"])
@pytest.mark.parametrize("env_name", ["hopper", "ant", "humanoidrun"])
def test_graph_replay_equals_the_host_driven_loop(env_name, mod, make, setting):
    """20 control steps of 2 seeds: actions, rewards, states and rew_hist bit for bit; with drawn members the device's last draw is
    the host's draw of the last control step"""
    kw = SETTINGS[setting]
    al = make(env_name, **kw)
    env = mod._prepare(al, batch=True)
    dev = mod.Controller(env, al)
    r = dev.run()
    host = mod.Controller(env, al, host=True)
    _assert_result(r, host.run_host_driven(), f"{env_name} {setting}")
    assert np.isfinite(r.states).all() and (_host(dev.mpc_ctl) == 20).all()
    if "plan_members" in kw:
        assert_bit_exact(_host(dev.engine.ens_factors), host.draws[:, -1], "the last control step's members")
        assert not np.array_equal(host.draws[:, 0], host.draws[:, 1]), "the members are drawn afresh"


@pytest.mark.parametrize("mod,make", [(mbd_mpc, mpc_args), (pi_mpc, pi_args)], ids=["mbd", "mppi"])
def test_problem_of_a_batch_is_its_solo_run(mod, make):
    kw = SETTINGS["drawn-worst2"]
    al = make("hopper", B=3, Nstep=8, **kw)
    _, res = (mbd_mpc.run_mpc_batch if mod is mbd_mpc else pi_mpc.run_pi_mpc_batch)(al, return_result=True)
    for b in range(3):
        solo = mod.Controller(mod._prepare([al[b]], batch=True), [al[b]]).run()
        _assert_result(res, solo, f"problem {b}", rows=slice(b, b + 1))


@pytest.mark.parametrize("mod,make", [(mbd_mpc, mpc_args), (pi_mpc, pi_args)], ids=["mbd", "mppi"])
def test_degenerate_draw_is_the_nominal_controller(mod, make):
    al = make("hopper", Nstep=10, plan_members=4, plan_friction_range=(1.0, 1.0), plan_gear_range=(1.0, 1.0), plan_worst=1)
    env = mod._prepare(al, batch=True)
    r = mod.Controller(env, al).run()
    nominal = make("hopper", Nstep=10)
    _assert_result(r, mod.Controller(env, nominal).run(), "nominal")
