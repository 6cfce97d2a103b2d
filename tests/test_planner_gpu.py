"""reverse_once / run_diffusion on the GPU against the numpy planner oracle (rtol 1e-4, the
tolerance north_star states for fp32), shard-count invariance (bit-exact) and the env surface."""
import os

import numpy as np
import pytest
import torch

import mbd_b200
from mbd_b200 import ops, prng
from mbd_b200.planners import engine as eng
from mbd_b200.planners.mbd_planner import Args, run_diffusion
from mbd_b200.planners.sharding import tree_sum_rows
from oracle import planner as opl
from tests.conftest import assert_bit_exact

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RTOL = 1e-4  # north_star: "within 1e-4 relative fp32"


def N(t):
    return t.detach().cpu().numpy()


def _close(a, b, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(np.abs(b).max(), 1e-6)
    err = np.abs(a - b).max() / scale
    assert err <= RTOL, f"{what}: max rel-to-scale error {err:.3e} > {RTOL}"


@pytest.mark.parametrize("demo", [False, True])
def test_reverse_once_car2d_vs_oracle(orc, demo):
    car = mbd_b200.envs.get_env("car2d")
    Nn, H, temp, i = 512, 50, 0.1, 60
    _, alphas, alphas_bar, sigmas = opl.make_schedule(1e-4, 1e-2, 100)
    key = np.uint32([9, 8])
    Ybar_i = (np.random.default_rng(0).normal(size=100) * 0.3).astype(np.float32)
    oenv = opl.OracleEnv("car2d", 2, params=car.params, x0=car.x0)
    ref = opl.reverse_once(oenv, key, Nn, H, float(sigmas[i]), Ybar_i, temp, alphas, alphas_bar, i,
                           xref=car.xref if demo else None, rew_xref=car.rew_xref)
    e = eng.DiffusionEngine(car, Nn, H, temp, demo, car.reset(None))
    out, rew = e.reverse_once(key, float(sigmas[i]), torch.as_tensor(Ybar_i, device=DEV), eng.update_coef(alphas, alphas_bar, i))
    assert_bit_exact(N(e.Y0s), ref["Y0s"]); assert_bit_exact(N(e.rews_local), ref["rews"])
    if demo:
        assert_bit_exact(N(e.logpd_local), ref["logpd"])
    _close(N(e.weights), ref["weights"], "softmax weights")
    _close(N(out), ref["Ybar_im1"], "Ybar_im1")
    _close(rew.item(), ref["rew_mean"], "rews.mean()")
    assert abs(N(e.weights).sum() - 1) < 1e-5


def test_reverse_once_humanoidrun_vs_oracle(orc, humanoidrun_setup):
    env, blob, st = humanoidrun_setup
    Nn, H, temp, i = 256, 50, 0.1, 299
    _, alphas, alphas_bar, sigmas = opl.make_schedule(1e-4, 1e-2, 300)
    key = prng.split(prng.split(prng.split(prng.PRNGKey(0))[0])[0])[1]
    Ybar_i = np.zeros(850, np.float32)
    oenv = opl.OracleEnv("xpbd", 17, blob=blob, state=st)
    ref = opl.reverse_once(oenv, key, Nn, H, float(sigmas[i]), Ybar_i, temp, alphas, alphas_bar, i)
    e = eng.DiffusionEngine(env, Nn, H, temp, False, st)
    out, rew = e.reverse_once(key, float(sigmas[i]), torch.zeros(850, device=DEV), eng.update_coef(alphas, alphas_bar, i))
    assert_bit_exact(N(e.rews_local), ref["rews"], "per-sample returns")
    _close(N(out), ref["Ybar_im1"], "Ybar_im1"); _close(rew.item(), ref["rew_mean"], "rews.mean()")
    # index work is bit-exact: the best sample is the same one
    assert int(N(e.weights).argmax()) == int(ref["weights"].argmax())


def test_reverse_once_humanoidtrack_demo_vs_oracle(orc):
    env = mbd_b200.envs.get_env("humanoidtrack")
    st = env.reset(None).pipeline_state.raw
    Nn, H, temp, i = 128, 50, 0.1, 80
    _, alphas, alphas_bar, sigmas = opl.make_schedule(1e-4, 1e-2, 100)
    key = np.uint32([77, 1])
    oenv = opl.OracleEnv("xpbd", 17, blob=env.blob, state=st)
    ref = opl.reverse_once(oenv, key, Nn, H, float(sigmas[i]), np.zeros(850, np.float32), temp, alphas, alphas_bar, i,
                           xref=env.xref, rew_xref=env.rew_xref)
    e = eng.DiffusionEngine(env, Nn, H, temp, True, st)
    out, rew = e.reverse_once(key, float(sigmas[i]), torch.zeros(850, device=DEV), eng.update_coef(alphas, alphas_bar, i))
    assert_bit_exact(N(e.rews_local), ref["rews"]); assert_bit_exact(N(e.logpd_local), ref["logpd"])
    _close(N(e.weights), ref["weights"], "weights (demo blend)"); _close(N(out), ref["Ybar_im1"], "Ybar_im1")


def test_std_guard_uniform_weights():
    """rews.std() < 1e-4 -> 1 (mbd_planner.py:112): constant rewards give uniform weights."""
    n = 256
    rews = torch.full((n,), 0.25, device=DEV)
    w = torch.empty(n, device=DEV); sc = torch.zeros(4, device=DEV); scratch = torch.empty(n, device=DEV)
    ops.softmax_weights(rews, None, 0, n, 0.1, 0.0, w, sc, scratch)
    assert np.allclose(N(w), 1 / n, rtol=1e-6) and N(sc)[1] == 1.0 and np.isclose(N(sc)[0], 0.25)


@pytest.mark.parametrize("demo", [False, True], ids=["humanoidrun", "humanoidtrack-demo"])
@pytest.mark.parametrize("P", [2, 4, 8])
def test_shard_count_invariance_bit_exact(humanoidrun_setup, P, demo):
    """P ranks EMULATED on one GPU (one engine + stream per rank, plain device buffers as the peers' symmetric memory): the
    very kernels of a sharded run — cross-GPU flag rendezvous, peer loads of the returns inside the statistics kernel,
    peer loads of the rank partials inside the update kernel — give the single-rank result bit for bit, over two
    consecutive steps (flag epochs, ticket reset, step counter)."""
    if demo:
        env = mbd_b200.envs.get_env("humanoidtrack"); st = env.reset(None).pipeline_state.raw
    else:
        env, blob, st = humanoidrun_setup
    Nn, H, temp, Nd = 1024, 50, 0.1, 100
    _, alphas, alphas_bar, sigmas = opl.make_schedule(1e-4, 1e-2, Nd)
    keys = eng.key_chain(np.uint32([4, 4]), Nd)
    e1 = eng.DiffusionEngine(env, Nn, H, temp, demo, st, Ndiffuse=Nd)
    e1.load_schedule(keys, sigmas, alphas, alphas_bar); e1.set_step(Nd - 1)
    e1.step(); e1.step()
    ranks = eng.DiffusionEngine.make_emulated_ranks(env, Nn, H, temp, demo, st, P, Ndiffuse=Nd)
    for e in ranks:
        e.load_schedule(keys, sigmas, alphas, alphas_bar); e.set_step(Nd - 1)
    eng.DiffusionEngine.step_emulated_ranks(ranks)
    eng.DiffusionEngine.step_emulated_ranks(ranks)
    torch.cuda.synchronize()
    for e in ranks:
        e.check_exchange()
        assert int(e.ctl[0].item()) == Nd - 3 and int(e.ctl[1].item()) == 2
        assert_bit_exact(N(e.Ybars[Nd - 3:Nd - 1]), N(e1.Ybars[Nd - 3:Nd - 1]), f"rank {e.rank} of {P}: iterates")
        assert_bit_exact(N(e.rew_hist), N(e1.rew_hist), "rews.mean() history")
        assert_bit_exact(N(e.rews_all), N(e1.rews_all), "gathered returns")
    assert_bit_exact(np.concatenate([N(e.weights) for e in ranks]), N(e1.weights), "softmax weights")
    assert_bit_exact(np.concatenate([N(e.Y0s) for e in ranks]), N(e1.Y0s), "sampled actions")


def test_exchange_timeout_poisons_the_output(humanoidrun_setup, monkeypatch):
    """a peer that never shows up: the rendezvous times out, ctl.err is set and the step's outputs are NaN — a stale
    or missing exchange can never be mistaken for a result (ADVICE r1: the former peer-gather kernel used stale data after a timeout)"""
    monkeypatch.setenv("MBD_XCHG_TIMEOUT_S", "0.005")
    env, blob, st = humanoidrun_setup
    _, alphas, alphas_bar, sigmas = opl.make_schedule(1e-4, 1e-2, 10)
    ranks = eng.DiffusionEngine.make_emulated_ranks(env, 256, 50, 0.1, False, st, 2, Ndiffuse=10)
    for e in ranks:
        e.load_schedule(eng.key_chain(np.uint32([1, 1]), 10), sigmas, alphas, alphas_bar); e.set_step(9)
    eng.DiffusionEngine.step_emulated_ranks(ranks, ranks=[0])     # rank 1 never launches
    torch.cuda.synchronize()
    assert int(ranks[0].ctl[2].item()) == 1 and np.isnan(N(ranks[0].Ybars[8])).all() and np.isnan(N(ranks[0].weights)).all()
    with pytest.raises(ops.MbdError, match="rendezvous timed out"):
        ranks[0].check_exchange()


def test_step_graph_replay_equals_direct_launches(humanoidrun_setup):
    """a captured step replayed k times == k direct launches, bit for bit (parameters come from device memory)"""
    env, blob, st = humanoidrun_setup
    Nd = 8
    _, alphas, alphas_bar, sigmas = opl.make_schedule(1e-4, 1e-2, Nd)
    keys = eng.key_chain(np.uint32([2, 5]), Nd)
    outs = []
    for graph in (False, True):
        e = eng.DiffusionEngine(env, 512, 50, 0.1, False, st, Ndiffuse=Nd)
        e.load_schedule(keys, sigmas, alphas, alphas_bar); e.set_step(Nd - 1)
        if graph:
            e.capture()
        for _ in range(Nd - 1):
            e.step()
        torch.cuda.synchronize()
        assert int(e.ctl[0].item()) == 0
        outs.append((N(e.Ybars).copy(), N(e.rew_hist).copy()))
    assert_bit_exact(outs[0][0], outs[1][0], "iterates"); assert_bit_exact(outs[0][1], outs[1][1], "reward history")


def test_step_matches_round1_kernels(humanoidrun_setup):
    """the fused tail (cluster statistics + last-CTA tree/update) against the separate round-1 kernels, which stay in the
    ABI for path_integral: same weighted-mean order (bit-exact given equal weights), statistics within 1e-6"""
    env, blob, st = humanoidrun_setup
    Nn, H = 2048, 50
    _, alphas, alphas_bar, sigmas = opl.make_schedule(1e-4, 1e-2, 100)
    coef = eng.update_coef(alphas, alphas_bar, 70)
    key = np.uint32([4, 4]); Ybar_i = torch.as_tensor((np.random.default_rng(0).normal(size=850) * 0.1).astype(np.float32), device=DEV)
    e = eng.DiffusionEngine(env, Nn, H, 0.1, False, st)
    out, rew = e.reverse_once(key, float(sigmas[70]), Ybar_i, coef)
    w = torch.empty(Nn, device=DEV); sc = torch.zeros(4, device=DEV); scratch = torch.empty(Nn, device=DEV)
    ops.softmax_weights(e.rews_local, None, 0, Nn, 0.1, 0.0, w, sc, scratch)
    assert np.allclose(N(w), N(e.weights), rtol=2e-6, atol=1e-12) and np.allclose(N(sc)[:2], N(e.scalars)[:2], rtol=1e-6)
    runs = torch.empty(((Nn + 63) // 64) * 850, device=DEV); ref = torch.empty(850, device=DEV)
    nr = ops.weighted_sum_runs(e.weights, e.Y0s, 850, runs)
    ops.update(runs, nr, 850, Ybar_i, coef, ref)
    assert_bit_exact(N(out), N(ref), "tree + update")


def test_run_diffusion_car2d_matches_oracle_solve(orc, capsys):
    """BASELINE config 1 (car2d, Nsample=64, Hsample=40, full solve) + a demo solve, end to end
    through the reference-facing API."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "car2d_oracle.npz"))
    rf, Yi = run_diffusion(Args(env_name="car2d", Nsample=64, Hsample=40, not_render=True), return_trajectory=True)
    out = capsys.readouterr().out
    assert "override temp_sample to 0.1" in out and "init sigma = 6.30e-01" in out
    assert Yi.shape == (99, 40, 2)
    _close(N(Yi[-1]).reshape(-1), g["Yi_last"], "final iterate"); _close(rf, float(g["rew_final"]), "rew_final")
    # demo branch, short chain (Ndiffuse=9): every iterate within 1e-3 of the oracle chain.  Long chains
    # amplify last-ulp differences of the statistics through car2d's collision freeze, so the full demo
    # solve is only checked for its outcome: the planner reaches the goal region like the oracle run does.
    _, Yis = run_diffusion(Args(env_name="car2d", Nsample=512, Hsample=50, Ndiffuse=9, enable_demo=True, not_render=True),
                           return_trajectory=True)
    assert np.abs(N(Yis).reshape(8, -1) - g["Yi_short_demo"]).max() < 1e-3
    rfd, Yid = run_diffusion(Args(env_name="car2d", Nsample=512, Hsample=50, enable_demo=True, not_render=True), return_trajectory=True)
    assert rfd > 0.1 and float(g["rew_final_demo"]) > 0.1


def test_run_diffusion_humanoidrun_short(humanoidrun_setup, tmp_path, monkeypatch):
    """a short humanoidrun solve through Args/run_diffusion: artefact shape + improving reward"""
    a = Args(env_name="humanoidrun", Nsample=512, Ndiffuse=12, disable_recommended_params=True, not_render=True)
    rf, Yi = run_diffusion(a, return_trajectory=True)
    assert Yi.shape == (11, 50, 17) and np.isfinite(N(Yi)).all() and np.isfinite(rf)
    assert float(N(Yi).max()) <= 1.0 and float(N(Yi).min()) >= -1.0


def test_env_surface_step_equals_rollout(orc, humanoidrun_setup):
    """env.reset/step (reference surface) steps the same kernel: H single steps == one rollout."""
    env, blob, st = humanoidrun_setup
    rng, rng_reset = prng.split(prng.PRNGKey(0))
    state = env.reset(rng_reset)
    us = np.clip(np.random.default_rng(3).normal(size=(6, 17)), -1, 1).astype(np.float32)
    rews = []
    for t in range(6):
        state = env.step(state, us[t]); rews.append(state.reward)
    ref = orc.xpbd_rollout(blob, st, us[None], want_rewss=True, want_final=True)
    assert_bit_exact(np.float32(rews), ref["rewss"][0]); assert_bit_exact(state.pipeline_state.raw, ref["final"][0])
    assert state.obs.shape == (47,)
    assert np.isclose(state.reward, env._get_reward(state.pipeline_state), atol=1e-5)
    r2 = mbd_b200.utils.eval_us(env.step, env.reset(rng_reset), us)
    assert_bit_exact(r2, ref["rewss"][0])
    car = mbd_b200.envs.get_env("car2d")
    s = car.reset(None)
    s = car.step(s, np.float32([0.3, 1.0]))
    assert s.pipeline_state.shape == (3,) and s.pipeline_state[0] < -0.5
    rr, xs = mbd_b200.utils.rollout_us(car.step, car.reset(None), np.float32([[0.3, 1.0]] * 3))
    assert len(xs) == 3 and np.allclose(xs[0], s.pipeline_state)


@pytest.mark.parametrize("method", ["mppi", "cma-es", "cem"])
def test_path_integral_update_once_vs_oracle(orc, humanoidrun_setup, method):
    """SURVEY 8f.1: MPPI / CMA-ES / CEM updates on the same kernels; CEM's top-10 index set is bit-exact."""
    from mbd_b200.planners.path_integral import PathIntegralEngine
    env, blob, st = humanoidrun_setup
    Nn, H = 256, 50
    key = np.uint32([21, 12])
    mu0 = (np.random.default_rng(5).normal(size=850) * 0.2).astype(np.float32)
    oenv = opl.OracleEnv("xpbd", 17, blob=blob, state=st)
    ref = opl.update_once(oenv, key, Nn, H, 0.8, mu0, 0.1, method)
    e = PathIntegralEngine(env, Nn, H, 0.1, st, method)
    out = torch.empty(850, device=DEV)
    mu, sigma, rew = e.update_once(key, torch.as_tensor(mu0, device=DEV), 0.8, out)
    assert_bit_exact(N(e.rews_local), ref["rews"])
    _close(N(mu), ref["mu"], f"{method} mean"); _close(rew.item(), ref["rew_mean"], "rews.mean()")
    assert abs(sigma - ref["sigma"]) <= 1e-5 * max(1.0, ref["sigma"])
    if method == "cem":
        idx = torch.sort(e.weights, stable=True).indices.flip(0)[:10].cpu().numpy()
        assert np.array_equal(idx, ref["idx"])


def test_run_path_integral_cli_surface(capsys):
    from mbd_b200.planners.path_integral import Args as PArgs, run_path_integral
    rf, mus = run_path_integral(PArgs(env_name="car2d", Nsample=128, Nrefine=6, update_method="cma-es"), return_trajectory=True)
    assert mus.shape == (5, 50, 2) and np.isfinite(rf) and "override temp_sample" in capsys.readouterr().out
    with pytest.raises(KeyError):
        run_path_integral(PArgs(env_name="car2d", Nsample=64, Nrefine=3, update_method="nope"))
