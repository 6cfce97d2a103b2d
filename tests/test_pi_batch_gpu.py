"""The path-integral baselines as device steps (BatchedPathIntegralEngine / mbd_pi_batch_step_launch): one step against the CPU
oracle, the tail on constructed returns against the float64 radii of tests/pi_tail_ref.py, batches against B = 1 bit for bit,
graph replay against eager launches, and the device path against the host-driven run_path_integral step by step."""
import math

import numpy as np
import pytest
import torch

import mbd_b200
from mbd_b200 import _lib, ops, prng
from mbd_b200.planners import engine as eng
from mbd_b200.planners.mbd_planner import final_reward
from mbd_b200.planners.path_integral import Args, BatchedPathIntegralEngine, PathIntegralEngine, run_path_integral_batch
from oracle import planner as opl
from tests import pi_tail_ref as pr
from tests import tail_ref as tr
from tests.conftest import assert_bit_exact

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RTOL = 1e-4          # test_path_integral_update_once_vs_oracle
METHODS = ("mppi", "cma-es", "cem")
f32 = np.float32


def N(t):
    return t.detach().cpu().numpy()


def _close(a, b, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    err = np.abs(a - b).max() / max(np.abs(b).max(), 1e-6)
    assert err <= RTOL, f"{what}: max rel-to-scale error {err:.3e} > {RTOL}"


def _reset(env, seed):
    rng = prng.PRNGKey(seed=seed)
    rng, rng_reset = prng.split(rng)
    return env.reset(rng_reset), prng.split(rng)[0]


def _oracle_env(env, st):
    if env.kind == "xpbd":
        return opl.OracleEnv("xpbd", env.action_size, blob=env.blob, state=st.pipeline_state.raw)
    if env.kind == "pusht":
        return opl.OracleEnv("pusht", 2, params=env.params, x0=st.pipeline_state.raw)
    return opl.OracleEnv("car2d", 2, params=env.params, x0=env.x0)


def _stage(e, b, key, mu, sigma, t=1):
    """host-side inputs of step t of problem b: key, sigma_t (params row t) and mu_t (Ybars row t)"""
    row = np.zeros(_lib.STEP_PARAMS_WORDS, np.uint32)
    row[0:2] = np.asarray(key, np.uint32)
    row[2] = f32(sigma).view(np.uint32)
    e.params[b, t].copy_(torch.from_numpy(row.view(np.int32)))
    e.Ybars[b, t].copy_(torch.as_tensor(np.asarray(mu, f32), device=DEV))


def _sigma(e, b, t):
    return float(e.params[b, t, 2:3].cpu().numpy().view(f32)[0])


# ---- 1. one step against the CPU oracle ------------------------------------------------------------------------------------

ONE_STEP = [("humanoidrun", 256, 50), ("humanoidrun", 77, 50), ("hopper", 128, 50), ("car2d", 64, 40), ("pushT", 128, 40)]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("env_name,Nn,H", ONE_STEP, ids=[f"{e}-{n}" for e, n, _ in ONE_STEP])
def test_one_step_vs_oracle(orc, env_name, Nn, H, method):
    env = mbd_b200.envs.get_env(env_name)
    st, _ = _reset(env, 0)
    HNu = H * env.action_size
    key = np.uint32([21, 12])
    mu0 = (np.random.default_rng(5).normal(size=HNu) * 0.2).astype(f32)
    ref = opl.update_once(_oracle_env(env, st), key, Nn, H, 0.8, mu0, 0.1, method)
    e = BatchedPathIntegralEngine(env, Nn, H, [0.1], [st], 2, method)
    _stage(e, 0, key, mu0, 0.8)
    e.set_step(1)
    e.step()
    e.check_exchange()
    assert_bit_exact(N(e.Y0s[0]), ref["Y0s"], "Y0s")
    assert_bit_exact(N(e.rews[0]), ref["rews"], "returns")
    _close(N(e.Ybars[0, 0]), ref["mu"], f"{method} mean")
    _close(e.rew_hist[0, 1].item(), ref["rew_mean"], "rews.mean()")
    if method == "cma-es":
        assert abs(_sigma(e, 0, 0) - ref["sigma"]) <= 1e-5 * max(1.0, ref["sigma"])
        assert float(e.sigma_hist[0, 0].item()) == _sigma(e, 0, 0)
    if method == "cem":
        assert np.array_equal(e.cem_indices(0), ref["idx"])


# ---- 2. tail-only launches on constructed returns --------------------------------------------------------------------------

def _tail(method, fams, Nn, HNu, temp, sigma=0.6, Y=None, mu=None):
    """one problem per family, launches 2 and 3 of step 1 only, on an engine without an env (Nu = 1, so that H * Nu can be any
    column count); returns (engine, inputs)"""
    B = len(fams)
    e = BatchedPathIntegralEngine(None, Nn, HNu, [temp] * B, [None] * B, 2, method, inputs=eng.LaunchInputs.none(), nu=1)
    e.load_schedule([np.zeros((2, 2), np.uint32)] * B)   # sigma 1 in every row; row 1 is staged below
    ins = []
    for b, fam in enumerate(fams):
        f = tr.make_family(fam, Nn, seed=b)
        Yb, mub = tr.make_samples(Nn, HNu, seed=b) if Y is None else (Y, mu)
        e.rews[b].copy_(torch.from_numpy(f["rews"]))
        e.Y0s[b].copy_(torch.from_numpy(np.ascontiguousarray(Yb)))
        _stage(e, b, np.zeros(2, np.uint32), mub, sigma)
        ins.append((f, Yb, mub))
    e.set_step(1)
    e.tail_step()
    torch.cuda.synchronize()
    e.check_exchange()
    assert (N(e.ctl[:, 0]) == 0).all()
    return e, ins


CEM_FAMS = ("normal", "constant", "tie", "dominant", "guard_below", "offset")


@pytest.mark.parametrize("Nn", [1, 7, 10, 11, 8193])
@pytest.mark.parametrize("temp", [0.01, 0.1, 1.0])
def test_cem_tail_indices_and_mean(Nn, temp):
    """the index set is argsort(w_dev, stable)[::-1][:10] of the device's own weights — ties (mass ties at temp 0.01, where most
    weights are exactly 0; the constant family; two-way ties) included — and the mean lies within its float64 radius"""
    HNu = 37
    e, ins = _tail("cem", CEM_FAMS, Nn, HNu, temp)
    for b, (f, Y, _) in enumerate(ins):
        w = N(e.weights[b])
        want = pr.cem_indices(w)
        got = e.cem_indices(b)
        assert np.array_equal(got, want), f"{CEM_FAMS[b]} N={Nn} T={temp}: {got} vs {want} (nonzero weights {(w > 0).sum()})"
        tr.check_columns(N(e.Ybars[b, 0]), pr.cem_mean_reference(Y, got), pr.cem_mean_radius(Y, got), f"{CEM_FAMS[b]} mean")
    if temp == 0.01 and Nn > 10:
        assert (N(e.weights[0]) == 0).any(), "at T = 0.01 some weights of the normal family should underflow to exactly 0"
        assert (N(e.weights[3]) > 0).sum() < 10, "the dominant family at T = 0.01 should leave fewer than 10 nonzero weights"


CMA_FAMS = ("normal", "offset", "guard_above", "constant", "dominant")


@pytest.mark.parametrize("Nn,HNu", [(1, 1), (63, 257), (1025, 850), (8193, 256)])
@pytest.mark.parametrize("method", ["mppi", "cma-es"])
def test_mppi_cma_tail_within_f64_radii(method, Nn, HNu):
    temp, sigma = 0.1, 0.6
    e, ins = _tail(method, CMA_FAMS, Nn, HNu, temp, sigma)
    nruns = math.ceil(Nn / 64)
    for b, (f, Y, mu) in enumerate(ins):
        what = f"{method} {CMA_FAMS[b]} N={Nn} HNu={HNu}"
        ref = tr.reference(f["rews"], temp, Y0s=Y, mu=mu)
        sc = N(e.scalars[b])
        tr.check_stats(ref, f["rews"], sc[0], sc[1], tr.cluster_depth(Nn), what)
        wb = tr.weight_bounds(ref, tr.cluster_depth(Nn), sc[0], sc[1])
        tr.check_weights(ref, N(e.weights[b]), wb, what + ": weights")
        tr.check_columns(N(e.Ybars[b, 0]), ref["Ybar"], tr.ybar_bound(ref, Y, wb["rho"], tr.wsum_depth(nruns)), what + ": mean")
        if method == "cma-es":
            want, _ = pr.cma_sigma_reference(ref, sigma)
            rad = pr.cma_sigma_radius(ref, Y, mu, wb["rho"], tr.wsum_depth(nruns), sigma, pr.cma_mean_depth(HNu))
            pr.check_scalar(_sigma(e, b, 0), want, rad, what + ": sigma'")
            assert float(e.sigma_hist[b, 0].item()) == _sigma(e, b, 0)
        else:
            assert _sigma(e, b, 0) == 1.0 and float(e.sigma_hist[b, 0].item()) == 1.0, "MPPI leaves sigma alone"


def test_cma_floor_when_samples_equal_the_mean():
    Nn, HNu = 300, 120
    mu = (np.random.default_rng(2).normal(size=HNu) * 0.3).astype(f32)
    Y = np.repeat(mu[None], Nn, axis=0)
    e, _ = _tail("cma-es", ("normal", "constant"), Nn, HNu, 0.1, 0.9, Y=Y, mu=mu)
    for b in range(2):
        assert _sigma(e, b, 0) == float(f32(1e-3)) and float(e.sigma_hist[b, 0].item()) == float(f32(1e-3))


# ---- 3. batches against B = 1, bit for bit ---------------------------------------------------------------------------------

def _pargs(env_name, B, Nn, H, method, Nr=12):
    temps = [0.1, 0.05, 0.3, 0.2, 0.15, 0.5, 0.08, 1.0]
    return [Args(seed=3 * b + 1, env_name=env_name, Nsample=Nn, Hsample=H, Nrefine=Nr, update_method=method, temp_sample=temps[b % 8],
                 disable_recommended_params=True) for b in range(B)]


def _solve(env, args_list, graph=False):
    """(engine, Ybars, rew_hist, sigma_hist, rew_final) of one batched solve of args_list"""
    ins = [_reset(env, a.seed) for a in args_list]
    a0 = args_list[0]
    e = BatchedPathIntegralEngine(env, a0.Nsample, a0.Hsample, [a.temp_sample for a in args_list], [i[0] for i in ins], a0.Nrefine,
                                  a0.update_method)
    e.load_schedule([eng.key_chain(i[1], a0.Nrefine) for i in ins])
    e.set_step(a0.Nrefine - 1)
    if graph:
        e.capture()
    for _ in range(a0.Nrefine - 1):
        e.step()
    e.check_exchange()
    fin = [final_reward(env, e.problem(b), e.Ybars[b, 0]) for b in range(e.B)]
    return e, N(e.Ybars), N(e.rew_hist), N(e.sigma_hist), fin


def _assert_matches_solo(env, args_list, out, what):
    _, Yb, rh, sh, fin = out
    for b, a in enumerate(args_list):
        _, Ys, rs, ss, fs = _solve(env, [a])
        assert_bit_exact(Yb[b], Ys[0], f"{what} problem {b}: mu trajectory")
        assert_bit_exact(rh[b], rs[0], f"{what} problem {b}: rew_hist")
        assert_bit_exact(sh[b], ss[0], f"{what} problem {b}: sigma history")
        assert fin[b] == fs[0], f"{what} problem {b}: rew_final"


BATCH_ENVS = [("car2d", 64, 40), ("hopper", 128, 50), ("humanoidrun", 256, 50), ("pushT", 128, 40)]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("env_name,Nn,H", BATCH_ENVS, ids=[e for e, _, _ in BATCH_ENVS])
def test_batch_matches_single_problems(env_name, Nn, H, method):
    env = mbd_b200.envs.get_env(env_name)
    al = _pargs(env_name, 2, Nn, H, method)
    _assert_matches_solo(env, al, _solve(env, al), f"{env_name} {method} B=2")
    perm = [al[1], al[0]]
    _assert_matches_solo(env, perm, _solve(env, perm), f"{env_name} {method} permuted")
    if method == "cma-es":
        sh = _solve(env, al)[3]
        assert len(np.unique(sh[0])) > 1, "CMA-ES should move sigma"


@pytest.mark.parametrize("method", METHODS)
def test_batch_of_17(method):
    env = mbd_b200.envs.get_env("car2d")
    al = _pargs("car2d", 17, 63, 40, method, Nr=6)
    _assert_matches_solo(env, al, _solve(env, al), f"car2d {method} B=17")


@pytest.mark.parametrize("variant", [0, 1, 2, 8])
@pytest.mark.parametrize("method", METHODS)
def test_humanoid_variants(variant, method):
    env = mbd_b200.envs.get_env("humanoidrun")
    al = _pargs("humanoidrun", 2, 77, 50, method, Nr=6)
    ops.set_kernel_variant(variant)
    try:
        _assert_matches_solo(env, al, _solve(env, al), f"variant {variant} {method}")
    finally:
        ops.set_kernel_variant(0)


@pytest.mark.parametrize("method", METHODS)
def test_run_path_integral_batch_surface(method, capsys):
    al = _pargs("car2d", 3, 64, 40, method, Nr=6)
    rf, mus = run_path_integral_batch(al, return_trajectory=True)
    assert rf.shape == (3,) and len(mus) == 3 and mus[0].shape == (5, 40, 2) and np.isfinite(rf).all()
    env = mbd_b200.envs.get_env("car2d")
    _, Yb, _, _, fin = _solve(env, _pargs("car2d", 3, 64, 40, method, Nr=6))
    for b in range(3):
        assert_bit_exact(N(mus[b]).reshape(5, -1), Yb[b, 4::-1], f"problem {b}: trajectory layout")
        assert rf[b] == fin[b]


# ---- 4. graph replay against eager; a replay past the last step writes nothing ----------------------------------------------

@pytest.mark.parametrize("method", METHODS)
def test_graph_replay_matches_eager_and_stops_at_the_end(method):
    env = mbd_b200.envs.get_env("hopper")
    al = _pargs("hopper", 3, 128, 50, method, Nr=8)
    eager = _solve(env, al)
    e, Yb, rh, sh, fin = _solve(env, al, graph=True)
    for x, y, what in ((Yb, eager[1], "mu"), (rh, eager[2], "rew_hist"), (sh, eager[3], "sigma history")):
        assert_bit_exact(x, y, f"graph vs eager: {what}")
    assert fin == eager[4]
    canary = 1234.5
    e.Ybars[:, -1].fill_(canary)
    e.sigma_hist[:, -1].fill_(canary)
    e.params[:, -1, 2].fill_(int(f32(canary).view(np.int32)))
    before = [t.clone() for t in (e.Ybars, e.sigma_hist, e.params, e.rew_hist)]
    e.step()                     # one replay too many: every problem's counter is at 0
    torch.cuda.synchronize()
    for t0, t1 in zip(before, (e.Ybars, e.sigma_hist, e.params, e.rew_hist)):
        assert torch.equal(t0, t1), "a step past the end wrote into the tables"
    assert (N(e.ctl[:, 2]) == 2).all()
    with pytest.raises(ops.MbdError, match=r"problems \[0, 1, 2\]"):
        e.check_exchange()


# ---- 5. the device path against the host-driven run_path_integral, one step at a time -------------------------------------

@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("env_name,Nn,H", [("car2d", 64, 40), ("hopper", 256, 50)])
def test_device_step_vs_host_step(env_name, Nn, H, method):
    """At every step of the host chain, the host's mu_t and sigma_t are staged into the device engine, so chaos cannot amplify
    a difference.  The two paths compute the softmax in different reduction orders (k_softmax_weights, one CTA, against the
    8-CTA cluster of k_step_weights), so the weights differ in the last bits and nothing downstream is bit-exact: MPPI's mean
    is held to the statistics tolerance of test_step_matches_round1_kernels, CMA-ES's sigma to 1e-5 relative, and CEM's index
    set must agree wherever the host's 10th and 11th weights differ.  car2d's collision freeze gives many samples the same
    return, and at temp 0.1 many weights are exactly 0, so its 10th and 11th weights were equal at every step of this chain and
    the CEM comparison is vacuous there; hopper must compare at least one step."""
    env = mbd_b200.envs.get_env(env_name)
    st, rng_exp = _reset(env, 1)
    Nr, temp = 8, 0.1
    keys = eng.key_chain(rng_exp, Nr)
    host = PathIntegralEngine(env, Nn, H, temp, st, method)
    dev = BatchedPathIntegralEngine(env, Nn, H, [temp], [st], 2, method)
    mu = torch.zeros(H * env.action_size, device=DEV)
    out = torch.empty_like(mu)
    sigma = 1.0
    checked = 0
    for t in range(Nr - 1, 0, -1):
        _stage(dev, 0, keys[t], N(mu), sigma)
        dev.set_step(1)
        dev.step()
        dev.check_exchange()
        _, sigma_new, _ = host.update_once(keys[t], mu, sigma, out)
        assert_bit_exact(N(dev.rews[0]), N(host.rews_local), f"step {t}: returns")
        wh, wd = N(host.weights), N(dev.weights[0])
        assert np.allclose(wd, wh, rtol=2e-6, atol=1e-12), f"step {t}: weights"
        if method == "cem":
            srt = np.sort(wh)[::-1]
            if Nn <= 10 or srt[9] != srt[10]:
                assert set(dev.cem_indices(0).tolist()) == set(torch.sort(host.weights, stable=True).indices.flip(0)[:10].tolist())
                checked += 1
        else:
            Ymax = float(np.abs(N(host.Y0s)).max())
            assert np.abs(N(dev.Ybars[0, 0]) - N(out)).max() <= 4e-6 * max(Ymax, 1e-6), f"step {t}: mean"
            if method == "cma-es":
                assert abs(_sigma(dev, 0, 0) - sigma_new) <= 1e-5 * sigma_new, f"step {t}: sigma {_sigma(dev, 0, 0)} vs {sigma_new}"
        mu, sigma = out.clone(), sigma_new
    assert method != "cem" or env_name == "car2d" or checked > 0
