"""Batched solves (BatchedDiffusionEngine / mbd_batch_step_launch / run_diffusion_batch) against B stand-alone solves of the
same Args: full Ybars tables, rew_hist and rew_final, bit for bit.  Every batch mixes seeds, temperatures and betas."""
import numpy as np
import pytest
import torch

import mbd_b200
from mbd_b200 import ops, prng
from mbd_b200.planners import engine as eng
from mbd_b200.planners.mbd_planner import Args, final_reward, run_diffusion, run_diffusion_batch
from tests.conftest import assert_bit_exact

pytestmark = pytest.mark.gpu


def N(t):
    return t.detach().cpu().numpy()


def mixed_args(env_name, B, Nsample, Hsample, Ndiffuse, demo=False):
    """B Args of one env and shape; seed, temp_sample, beta0 and betaT vary from problem to problem"""
    temps = [0.1, 0.05, 0.3, 0.2, 0.15, 0.5, 0.08, 1.0]
    return [Args(seed=3 * b + 1, env_name=env_name, Nsample=Nsample, Hsample=Hsample, Ndiffuse=Ndiffuse, enable_demo=demo,
                 temp_sample=temps[b % 8], beta0=1e-4 * (1 + b % 3), betaT=1e-2 * (1 + 0.5 * (b % 2)), not_render=True,
                 disable_recommended_params=True) for b in range(B)]


def problem_inputs(env, a):
    """reset state, key chain and schedule of one problem, derived from its seed exactly as run_diffusion does"""
    rng = prng.PRNGKey(seed=a.seed)
    rng, rng_reset = prng.split(rng)
    st = env.reset(rng_reset)
    _, alphas, alphas_bar, sigmas = eng.make_schedule(a.beta0, a.betaT, a.Ndiffuse)
    rng_exp, rng = prng.split(rng)
    return st, eng.key_chain(rng_exp, a.Ndiffuse), (sigmas, alphas, alphas_bar)


def solo(env, a):
    """one stand-alone DiffusionEngine solve: (Ybars, rew_hist, rew_final)"""
    st, keys, (sig, al, ab) = problem_inputs(env, a)
    e = eng.DiffusionEngine(env, a.Nsample, a.Hsample, a.temp_sample, a.enable_demo, st, Ndiffuse=a.Ndiffuse)
    e.load_schedule(keys, sig, al, ab)
    e.set_step(a.Ndiffuse - 1)
    for _ in range(a.Ndiffuse - 1):
        e.step()
    e.check_exchange()
    return N(e.Ybars), N(e.rew_hist), final_reward(env, e, e.Ybars[0])


def make_batch(env, args_list):
    ins = [problem_inputs(env, a) for a in args_list]
    a0 = args_list[0]
    be = eng.BatchedDiffusionEngine(env, a0.Nsample, a0.Hsample, [a.temp_sample for a in args_list], a0.enable_demo,
                                    [i[0] for i in ins], a0.Ndiffuse)
    be.load_schedule([i[1] for i in ins], [i[2][0] for i in ins], [i[2][1] for i in ins], [i[2][2] for i in ins])
    be.set_step(a0.Ndiffuse - 1)
    return be


def run_batch(env, args_list, graph=False):
    """(engine, Ybars [B,Nd,HNu], rew_hist [B,Nd], rew_final [B]) of one batched solve"""
    be = make_batch(env, args_list)
    if graph:
        be.capture()
    for _ in range(args_list[0].Ndiffuse - 1):
        be.step()
    be.check_exchange()
    finals = [final_reward(env, be.problem(b), be.Ybars[b, 0]) for b in range(be.B)]
    return be, N(be.Ybars), N(be.rew_hist), finals


def assert_matches_solo(env, args_list, Yb, rh, finals, what=""):
    for b, a in enumerate(args_list):
        Ys, rs, fs = solo(env, a)
        assert_bit_exact(Yb[b], Ys, f"{what} problem {b}: Ybars")
        assert_bit_exact(rh[b], rs, f"{what} problem {b}: rew_hist")
        assert finals[b] == fs, f"{what} problem {b}: rew_final {finals[b]!r} vs {fs!r}"


# ---- 1. one test per env kind --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("demo", [False, True], ids=["car2d", "car2d-demo"])
def test_car2d_full_solve_matches_run_diffusion(demo):
    """car2d 64 x 40, B = 8, the full 100 steps, through the planner entry points (graph capture on both sides)"""
    env = mbd_b200.envs.get_env("car2d")
    args = mixed_args("car2d", 8, 64, 40, 100, demo)
    rew_b, Yis = run_diffusion_batch(mixed_args("car2d", 8, 64, 40, 100, demo), return_trajectory=True)
    assert rew_b.shape == (8,)
    for b, a in enumerate(args):
        rew_s, Yi = run_diffusion(a, return_trajectory=True)
        assert rew_b[b] == rew_s, f"problem {b}: rew_final {rew_b[b]!r} vs {rew_s!r}"
        assert_bit_exact(N(Yis[b]), N(Yi), f"problem {b}: Yi")
    _, Yb, rh, finals = run_batch(env, args)
    assert_matches_solo(env, args, Yb, rh, finals, "car2d")
    assert not np.array_equal(Yb[0], Yb[1])   # the problems really differ


@pytest.mark.parametrize("env_name,B,Ns,H,Nd,demo", [
    ("pushT", 4, 256, 40, 5, False),
    ("hopper", 8, 1024, 50, 5, False),
    ("humanoidtrack", 3, 256, 50, 5, True),
    ("humanoidrun", 8, 1024, 50, 4, False),   # 8192 samples in all: the packed kernel; each stand-alone solve runs variant 1
])
def test_env_kind_matches_solo(env_name, B, Ns, H, Nd, demo):
    env = mbd_b200.envs.get_env(env_name)
    args = mixed_args(env_name, B, Ns, H, Nd, demo)
    _, Yb, rh, finals = run_batch(env, args)
    assert_matches_solo(env, args, Yb, rh, finals, env_name)
    assert np.isfinite(Yb).all()


# ---- 2. every explicit kernel variant --------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", [1, 2, 3, 8])
def test_kernel_variants_ragged(variant):
    """B = 3 at a ragged N = 100 on humanoidrun: every variant's batched launch equals the stand-alone solves"""
    env = mbd_b200.envs.get_env("humanoidrun")
    args = mixed_args("humanoidrun", 3, 100, 50, 3)
    ref = [solo(env, a) for a in args]
    ops.set_kernel_variant(variant)
    try:
        _, Yb, rh, finals = run_batch(env, args)
    finally:
        ops.set_kernel_variant(0)
    for b in range(3):
        assert_bit_exact(Yb[b], ref[b][0], f"variant {variant} problem {b}: Ybars")
        assert_bit_exact(rh[b], ref[b][1], f"variant {variant} problem {b}: rew_hist")
        assert finals[b] == ref[b][2]


# ---- 3. order independence -------------------------------------------------------------------------------------------------
def test_permuting_problems_permutes_results():
    env = mbd_b200.envs.get_env("car2d")
    args = mixed_args("car2d", 6, 64, 40, 12)
    _, Yb, rh, fin = run_batch(env, args)
    perm = [4, 0, 5, 2, 1, 3]
    _, Yp, rp, fp = run_batch(env, [args[k] for k in perm])
    for i, k in enumerate(perm):
        assert_bit_exact(Yp[i], Yb[k], f"position {i} (problem {k}): Ybars")
        assert_bit_exact(rp[i], rh[k], f"position {i} (problem {k}): rew_hist")
        assert fp[i] == fin[k]


# ---- 4. edge shapes on car2d -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Ns", [1, 63, 8193])
def test_car2d_edge_sample_counts(Ns):
    """8193 is one more than the 8192-thread stride of the statistics cluster"""
    env = mbd_b200.envs.get_env("car2d")
    args = mixed_args("car2d", 3, Ns, 40, 4)
    _, Yb, rh, finals = run_batch(env, args)
    assert_matches_solo(env, args, Yb, rh, finals, f"N={Ns}")


@pytest.mark.parametrize("B", [1, 2, 17])
def test_car2d_edge_batch_sizes(B):
    """B = 17: 136 statistics CTAs, more than the GPU has SMs"""
    env = mbd_b200.envs.get_env("car2d")
    args = mixed_args("car2d", B, 64, 40, 4)
    _, Yb, rh, finals = run_batch(env, args)
    assert_matches_solo(env, args, Yb, rh, finals, f"B={B}")


@pytest.mark.parametrize("env_name,Ns,demo", [("car2d", 64, True), ("humanoidrun", 256, False)])
def test_batch_of_one_equals_step_launch(env_name, Ns, demo):
    """B = 1 through mbd_batch_step_launch equals mbd_step_launch, step by step, including the scalars and weights"""
    env = mbd_b200.envs.get_env(env_name)
    a = mixed_args(env_name, 1, Ns, 40, 5, demo)[0]
    st, keys, (sig, al, ab) = problem_inputs(env, a)
    e = eng.DiffusionEngine(env, a.Nsample, a.Hsample, a.temp_sample, a.enable_demo, st, Ndiffuse=a.Ndiffuse)
    e.load_schedule(keys, sig, al, ab); e.set_step(a.Ndiffuse - 1)
    be = make_batch(env, [a])
    for _ in range(a.Ndiffuse - 1):
        e.step(); be.step()
        torch.cuda.synchronize()
        assert_bit_exact(N(be.Y0s[0]), N(e.Y0s), "Y0s"); assert_bit_exact(N(be.rews[0]), N(e.rews_local), "returns")
        assert_bit_exact(N(be.weights[0]), N(e.weights), "weights"); assert_bit_exact(N(be.scalars[0]), N(e.scalars), "scalars")
    assert_bit_exact(N(be.Ybars[0]), N(e.Ybars), "Ybars"); assert_bit_exact(N(be.rew_hist[0]), N(e.rew_hist), "rew_hist")
    assert N(be.ctl[0]).tolist() == N(e.ctl).tolist()


# ---- 5. graph capture and the past-the-end guard -------------------------------------------------------------------------
def test_graph_replay_equals_direct_and_stops_past_the_end():
    env = mbd_b200.envs.get_env("car2d")
    args = mixed_args("car2d", 5, 64, 40, 8, demo=True)
    _, Yd, rd, fd = run_batch(env, args)
    be, Yg, rg, fg = run_batch(env, args, graph=True)
    assert_bit_exact(Yg, Yd, "graph vs direct: Ybars"); assert_bit_exact(rg, rd, "graph vs direct: rew_hist")
    assert fg == fd
    assert N(be.ctl[:, 0]).tolist() == [0] * 5 and N(be.ctl[:, 2]).tolist() == [0] * 5
    # canaries in every problem's last row (YN, read only by the first step): a step past the end would write row -1 of
    # problem b, which is problem b - 1's last row
    Nd = args[0].Ndiffuse
    be.Ybars[:, Nd - 1].fill_(12345.0)
    before = (N(be.Ybars).copy(), N(be.rew_hist).copy(), N(be.scalars).copy(), N(be.weights).copy())
    be.step()   # one replay past the last step
    torch.cuda.synchronize()
    assert N(be.ctl[:, 2]).tolist() == [2] * 5, "every problem's control block reports the past-the-end step"
    assert N(be.ctl[:, 0]).tolist() == [0] * 5
    assert_bit_exact(N(be.Ybars), before[0], "past-the-end replay: Ybars (canaries included)")
    assert_bit_exact(N(be.rew_hist), before[1], "past-the-end replay: rew_hist")
    assert_bit_exact(N(be.scalars), before[2], "past-the-end replay: scalars")
    assert_bit_exact(N(be.weights), before[3], "past-the-end replay: weights")
    with pytest.raises(ops.MbdError, match=r"problems \[0, 1, 2, 3, 4\]"):
        be.check_exchange()


def test_check_exchange_names_the_problem():
    env = mbd_b200.envs.get_env("car2d")
    be = make_batch(env, mixed_args("car2d", 4, 64, 40, 4))
    be.ctl[2, 2] = 2
    with pytest.raises(ops.MbdError, match=r"problems \[2\]"):
        be.check_exchange()
