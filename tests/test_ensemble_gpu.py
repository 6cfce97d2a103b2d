"""Planner ensembles on the device (DESIGN.md §5l): a unit ensemble is today's batched step bit for bit; with K members every member
return is the rollout of its scaled model, the sample return is the ordered fp32 mean, the tail is today's tail on those returns and
the step agrees with the CPU oracle; both kernel mappings and every batch size give the same bits; captured steps follow in-place
rewrites of the table; and the receding-horizon controllers plan with an ensemble on the device as on the host."""
import numpy as np
import pytest

from mbd_b200 import _lib, ops, prng
from mbd_b200.envs import get_env
from mbd_b200.envs.vec import scaled_env
from mbd_b200.planners import mbd_mpc, pi_mpc
from mbd_b200.planners.engine import BatchedDiffusionEngine, key_chain, make_schedule
from mbd_b200.planners.path_integral import BatchedPathIntegralEngine
from tests import ens_ref
from tests.conftest import assert_bit_exact

pytestmark = pytest.mark.gpu

METHODS = ["mbd", "mppi", "cma-es", "cem"]
ND = 6
_cache = {}


def _env(name):
    if name not in _cache:
        _cache[name] = get_env(name)
    return _cache[name]


def _members(B, K, seed=0):
    """[B, K, 2] members that differ per problem (member 0 of problem 0 is the nominal model)"""
    t = np.random.default_rng(seed).uniform(0.4, 1.6, (B, K, 2)).astype(np.float32)
    t[0, 0] = 1.0
    return t


def _engine(env_name, method, B, N, H, ensemble=None, seeds=None):
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
        e = BatchedDiffusionEngine(env, N, H, temps, False, states, ND, ensemble=ensemble)
        _, al, ab, sg = make_schedule(1e-4, 1e-2, ND)
        e.load_schedule(keys, [sg] * B, [al] * B, [ab] * B)
    else:
        e = BatchedPathIntegralEngine(env, N, H, temps, states, ND, method, ensemble=ensemble)
        e.load_schedule(keys)
    e.set_step(ND - 1)
    return e


def _host(t):
    return t.detach().cpu().numpy()


def _same_state(a, b, what, rows=slice(None)):
    for f in ("Ybars", "rew_hist", "rews", "Y0s"):
        assert_bit_exact(_host(getattr(a, f))[rows], _host(getattr(b, f)), f"{what}: {f}")
    if getattr(a, "update_method", None) == "cma-es":
        assert_bit_exact(_host(a.sigma_hist)[rows], _host(b.sigma_hist), f"{what}: sigma_hist")


# ---- a unit ensemble is today's step ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("env_name,N", [("hopper", 256), ("ant", 256), ("humanoidrun", 4096)])
def test_unit_ensemble_is_todays_step(env_name, N, method):
    """one member (1, 1): every Ybars row, rew_hist and rews of 3 steps equal the nominal batched step's, bit for bit.  Humanoidrun's
    nominal step at 2 x 4096 samples runs the packed kernel, the ensemble the warp-per-link one"""
    B, H = 2, 16
    nom = _engine(env_name, method, B, N, H)
    ens = _engine(env_name, method, B, N, H, ensemble=np.ones((B, 1, 2), np.float32))
    for _ in range(3):
        nom.step()
        ens.step()
    _same_state(ens, nom, f"{env_name} {method}")
    assert_bit_exact(_host(ens.ens_rews)[:, :, 0], _host(ens.rews), "ens_rews")


# ---- K members ----------------------------------------------------------------------------------------------------------------
def _tail_again(e, i):
    """the tail alone (launches 2 and 3 of today's step) on the buffers the ensemble step left, re-armed at step i: MBD problem by
    problem with mbd_step_tail_launch on a single-problem view of the plan, a baseline with its tail-only batched launch"""
    e.ctl[:, 0].fill_(i)
    if isinstance(e, BatchedPathIntegralEngine):
        e.tail_step()
        return
    src, B, N, HNu, Nd = e._plan_c, e.B, e.N, e.HNu, e.Nd
    nruns = (N + ops.RUN - 1) // ops.RUN
    temps = _host(e.temps)
    for b in range(B):
        p = _lib.StepPlan.from_buffer_copy(src)
        off = lambda base, words: base + 4 * words   # noqa: E731
        p.params_dev, p.ctl_dev = off(src.params_dev, b * Nd * _lib.STEP_PARAMS_WORDS), off(src.ctl_dev, b * _lib.STEP_CTL_WORDS)
        p.Ybars_dev, p.rew_hist_dev = off(src.Ybars_dev, b * Nd * HNu), off(src.rew_hist_dev, b * Nd)
        p.Y0s_dev = off(src.Y0s_dev, b * N * HNu)
        p.rews_dev = p.rews_all_dev = off(src.rews_dev, b * N)
        p.logp_dev, p.weights_dev = off(src.logp_dev, b * N), off(src.weights_dev, b * N)
        p.runs_dev, p.scalars_dev = off(src.runs_dev, b * nruns * HNu), off(src.scalars_dev, b * 4)
        p.temp = float(temps[b])
        p.ens_factors_dev, p.ens_rews_dev, p.ens_k = None, None, 0
        ops.step_tail_launch(p)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("env_name,K", [("hopper", 3), ("hopper", 9), ("humanoidrun", 3)])
def test_members(env_name, K, method):
    B, N, H = 3, 128, 12
    env = _env(env_name)
    table = _members(B, K, seed=K)
    nom = _engine(env_name, method, B, N, H)
    e = _engine(env_name, method, B, N, H, ensemble=table)
    nom.step()
    e.step()
    Y0s, ens, rews = _host(e.Y0s), _host(e.ens_rews), _host(e.rews)
    assert_bit_exact(Y0s, _host(nom.Y0s), "Y0s = the nominal step's")
    st = _host(e.state_init)
    for b in range(B):
        Yb = e.Y0s[b].view(N, H, env.action_size)
        want = ens_ref.member_returns(env, st[b], Y0s[b], H, table[b])
        for k in range(K):
            spec = scaled_env(env, *table[b, k]).device_model()
            got = ops.rollout(spec, e.state_init[b], Yb)["rews"]
            assert_bit_exact(ens[b, :, k], _host(got), f"problem {b}, member {k}: ops.rollout of its scaled model")
        assert_bit_exact(ens[b], want, f"problem {b}: the oracle's member returns")
        assert_bit_exact(rews[b], ens_ref.ordered_mean(ens[b]), f"problem {b}: ordered mean")
    assert not np.array_equal(rews, _host(nom.rews))
    # the tail is today's tail on these returns
    step = _host(e.Ybars)[:, ND - 2].copy()
    _tail_again(e, ND - 1)
    assert_bit_exact(_host(e.Ybars)[:, ND - 2], step, "next Ybars row = the tail alone")
    # the diffusion update against the oracle (the tolerance of test_planner_gpu.py)
    if method == "mbd":
        _, al, ab, sg = make_schedule(1e-4, 1e-2, ND)
        params = _host(e.params).view(np.uint32)
        for b in range(B):
            o = ens_ref.reverse_once(env, st[b], params[b, ND - 1, 0:2], N, H, float(sg[ND - 1]), np.zeros(H * env.action_size, np.float32),
                                     float(_host(e.temps)[b]), al, ab, ND - 1, table[b])
            assert_bit_exact(o["Y0s"], Y0s[b], f"problem {b}: oracle Y0s")
            assert_bit_exact(o["rews"], rews[b], f"problem {b}: oracle sample returns")
            err = np.abs(step[b] - o["Ybar_im1"]).max() / max(np.abs(o["Ybar_im1"]).max(), 1e-6)
            assert err < 1e-4, f"problem {b}: Ybar differs from the oracle by {err}"


@pytest.mark.parametrize("method", ["mbd", "cem"])
def test_mappings_and_batches(method):
    """humanoidrun, 512 samples x 3 members: one problem runs the lane-per-link kernel (1536 rollouts), four the warp-per-link one
    (6144); problem b of the batch of four equals its batch of one under either mapping, over three steps"""
    B, N, H, K = 4, 512, 12, 3
    table = _members(B, K, seed=7)
    big = _engine("humanoidrun", method, B, N, H, ensemble=table)
    for _ in range(3):
        big.step()
    for b in range(B):
        one = _engine("humanoidrun", method, 1, N, H, ensemble=table[b:b + 1], seeds=[b])
        one.temps.copy_(big.temps[b:b + 1])
        for _ in range(3):
            one.step()
        _same_state(big, one, f"problem {b}", rows=slice(b, b + 1))
        assert_bit_exact(_host(big.ens_rews)[b:b + 1], _host(one.ens_rews), f"problem {b}: ens_rews")


@pytest.mark.parametrize("method", ["mbd", "cma-es"])
def test_graph_replay_follows_set_ensemble(method):
    B, N, H, K = 3, 256, 12, 3
    T0, T1 = _members(B, K, seed=11), _members(B, K, seed=12)
    eager, kept, g = (_engine("hopper", method, B, N, H, ensemble=T0) for _ in range(3))
    ptr = g.ens_factors.data_ptr()
    g.capture()
    for s in range(4):
        if s == 2:
            eager.set_ensemble(T1)
            g.set_ensemble(T1)
            assert g.ens_factors.data_ptr() == ptr
        eager.step()
        kept.step()
        g.step()
        _same_state(g, eager, f"replay {s}")
        assert_bit_exact(_host(g.ens_rews), _host(eager.ens_rews), f"replay {s}: ens_rews")
    assert not np.array_equal(_host(g.ens_rews), _host(kept.ens_rews)), "the rewrite changed nothing"
    with pytest.raises(ValueError, match="shape"):
        g.set_ensemble(np.ones((B, K + 1, 2)))


# ---- the controllers ----------------------------------------------------------------------------------------------------------
GEAR = dict(plan_friction=(1.0, 1.0, 1.0), plan_gear=(0.7, 1.0, 1.3))


def mpc_args(Nstep=10, **kw):
    return [mbd_mpc.Args(seed=3 * b, env_name="hopper", Nsample=256, Hsample=16, Ndiffuse=10, Nwarm=3, Nstep=Nstep, temp_sample=0.1,
                         plant_gear=(1.0, 0.7, 1.3)[b], not_render=True, disable_recommended_params=True, **kw) for b in range(3)]


def pi_args(Nstep=10, **kw):
    return [pi_mpc.Args(seed=3 * b, env_name="hopper", update_method="mppi", Nsample=256, Hsample=16, Nrefine=10, Nwarm=3, Nstep=Nstep,
                        sigma_warm=0.7, temp_sample=0.1, plant_gear=(1.0, 0.7, 1.3)[b], not_render=True,
                        disable_recommended_params=True, **kw) for b in range(3)]


def _assert_result(r, q, what, rows=slice(None)):
    for f in ("actions", "rewards", "states", "rew_hist"):
        assert_bit_exact(getattr(r, f)[rows], getattr(q, f), f"{what}: {f}")


@pytest.mark.parametrize("mod,make", [(mbd_mpc, mpc_args), (pi_mpc, pi_args)], ids=["mbd", "mppi"])
def test_graph_replay_equals_the_host_driven_loop(mod, make):
    al = make(**GEAR)
    env = mod._prepare(al, batch=True)
    dev = mod.Controller(env, al)
    assert dev.engine.ens_factors is not None and dev.engine.ens_factors.shape == (3, 3, 2)
    r = dev.run()
    _assert_result(r, mod.Controller(env, al, host=True).run_host_driven(), "host-driven")
    nominal = mod.Controller(env, make()).run()
    assert not np.array_equal(r.actions, nominal.actions), "the ensemble changed no action"


def test_unit_ensemble_is_todays_run_mpc():
    al = mpc_args(plan_friction=(1.0,), plan_gear=(1.0,))
    _, res = mbd_mpc.run_mpc_batch(al, return_result=True)
    _, q = mbd_mpc.run_mpc(mpc_args()[0], return_result=True)
    _assert_result(res, q, "problem 0", rows=slice(0, 1))
