"""Round-2 envs: slide (prismatic) dofs, hopper / walker2d / ant / halfcheetah / cartpole (BASELINE configs 2 and 3 and the
SURVEY 8f.3 rows).  CPU part: known-answer physics of the oracle's slide-dof code, FK <-> IK round trips, registry and
reward formulas.  GPU part: the CUDA kernels against the oracle, bit for bit, at the BASELINE shapes."""
import os

import numpy as np
import pytest

import mbd_b200
from mbd_b200 import prng
from mbd_b200.envs.generic import GenericPositionalEnv
from mbd_b200.model import blob as B
from mbd_b200.model import mjcf
from oracle import oracle as orc
from oracle import planner as opl
from tests.conftest import assert_bit_exact

FIX = os.path.join(os.path.dirname(__file__), "fixtures")
NEW_ENVS = ["hopper", "walker2d", "ant", "halfcheetah", "cartpole"]
# (Nsample, Hsample) of BASELINE.json configs 2 and 3; the f3 envs at the planner's default 2048 would only cost oracle time
SHAPES = {"hopper": (1024, 50), "ant": (4096, 50), "walker2d": (512, 50), "halfcheetah": (512, 50), "cartpole": (512, 50)}


def _cpu_state(env, seed=0):
    """the env's reset without touching the GPU (ant / halfcheetah draw qd with the sampling kernel in `reset`)"""
    rng, r1, r2 = prng.split(prng.split(prng.PRNGKey(seed))[1], 3)
    q = env.sys.init_q.astype(np.float32)
    name = type(env).__name__
    if name in ("Ant", "HalfCheetah"):
        q = q + prng.uniform(r1, (env.sys.q_size(),), minval=-0.1, maxval=0.1)
        qd = np.float32(0.1) * orc.normal(r2, (env.sys.qd_size(),))
    elif name == "Cartpole":
        q = q + prng.uniform(r1, (env.sys.q_size(),), minval=-0.01, maxval=0.01) + np.array([0.0, np.pi], np.float32)
        qd = prng.uniform(r2, (env.sys.qd_size(),), minval=-0.01, maxval=0.01)
    else:
        q = q + prng.uniform(r1, (env.sys.q_size(),), minval=-5e-3, maxval=5e-3)
        qd = prng.uniform(r2, (env.sys.qd_size(),), minval=-5e-3, maxval=5e-3)
    return env.pipeline_init(q, qd).raw


# ---------------------------------------------------------------------------------------------------------------
# CPU: model compiler, registry, oracle physics
# ---------------------------------------------------------------------------------------------------------------
def test_registry_has_every_positional_env_of_the_reference():
    """upstream mbd/envs/__init__.py:13-33: every name resolves (pushT, the generalized-backend env, included)"""
    for name in NEW_ENVS + ["humanoidrun", "humanoidtrack", "humanoidstandup", "car2d", "pushT"]:
        assert mbd_b200.envs.get_env(name) is not None
    with pytest.raises(ValueError, match="Unknown environment"):
        mbd_b200.envs.get_env("nope")


def test_model_facts():
    hop = mbd_b200.envs.get_env("hopper")
    assert hop.sys.link_types == "3111" and hop.action_size == 3 and hop._n_frames == 20 and np.isclose(hop.dt, 0.04)
    assert list(hop.sys.dof_is_slide[:3]) == [True, True, False] and hop.sys.init_q[1] == 1.25     # rootz ref
    assert hop.blob.view(np.int32)[B.HDR_WORDS + B.F_SLIDE * B.MAXL + 0] == 0b011
    assert hop.blob.view(np.float32)[B.H_RW0] == 1.0
    w2 = mbd_b200.envs.get_env("walker2d")
    assert w2.sys.link_types == "3111111" and w2.action_size == 6 and w2.blob.view(np.float32)[B.H_RW0] == np.float32(1.1)
    ant = mbd_b200.envs.get_env("ant")
    assert ant.sys.link_types == "f11111111" and ant.action_size == 8 and ant._n_frames == 10 and ant.sys.dt == 0.005
    assert np.all(ant.sys.act_gear == 200.0) and len(ant.sys.contacts) == 8                        # 4 foot capsules x 2 caps
    assert [ant.sys.act_names[i] for i in range(2)] == ["hip_4", "ankle_4"]                          # Gym actuator order
    hc = mbd_b200.envs.get_env("halfcheetah")
    assert hc.sys.link_types == "3111111" and hc.action_size == 6 and hc._n_frames == 16 and np.isclose(hc.dt, 0.05)
    assert np.isclose(hc.sys.mass.sum(), 14.0)                                                      # settotalmass
    cp = mbd_b200.envs.get_env("cartpole")
    assert cp.sys.link_types == "11" and cp.action_size == 1 and cp._n_frames == 4 and cp.sys.dt == 0.005
    assert list(cp.sys.dof_is_slide) == [True, False] and list(cp.sys.dof_limit[0]) == [-1.0, 1.0]


@pytest.mark.parametrize("name", NEW_ENVS)
def test_fk_ik_round_trip(name):
    """kinematics.forward then kinematics.inverse returns the joint coordinates (slide dofs included)"""
    env = mbd_b200.envs.get_env(name)
    rng = np.random.default_rng(1)
    q = env.sys.init_q.copy()
    lo = 7 if env.sys.link_types[0] == "f" else 0
    q[lo:] += rng.uniform(-0.2, 0.2, size=q.size - lo)
    qd = rng.uniform(-0.5, 0.5, size=env.sys.qd_size())
    ps = env.pipeline_init(q, qd)
    assert np.allclose(ps.q[lo:], q[lo:], atol=2e-5), (ps.q, q)
    assert np.allclose(ps.qd[(6 if lo else 0):], qd[(6 if lo else 0):], atol=2e-4)


def test_slide_dof_known_answers():
    """a single body on a limited, actuated slide joint along x (tests/fixtures/slider.xml):
    * constant force F = gear * u: semi-implicit Euler gives v_n = n dt F / m exactly (up to fp32), the body stays on the axis
      although gravity pulls it (the XPBD positional constraint removes everything but the free component);
    * at the range limit the free component beyond the limit becomes an error: the body stops at x = hi."""
    env = GenericPositionalEnv(os.path.join(FIX, "slider.xml"), n_frames=1)
    m, dt, F = float(env.sys.mass[0]), 0.002, 10.0 * 0.5
    st = env.pipeline_init(env.sys.init_q, np.zeros(1)).raw
    n = 40
    out = orc.xpbd_rollout(env.blob, st, np.full((1, n, 1), 0.5, np.float32), want_final=True)["final"][0, 0]
    assert np.isclose(out[10], n * dt * F / m, rtol=1e-4)                 # xd_i.vel.x
    assert np.isclose(out[0], dt * dt * F / m * n * (n + 1) / 2, rtol=1e-4)  # semi-implicit Euler position
    assert abs(out[1]) < 1e-6 and abs(out[2] - 0.5) < 1e-4 and abs(out[12]) < 5e-2   # y, z pinned against gravity
    assert np.allclose(out[3:7], [1, 0, 0, 0], atol=1e-6)                 # and no rotation
    far = orc.xpbd_rollout(env.blob, st, np.full((1, 1500, 1), 1.0, np.float32), want_final=True)["final"][0, 0]
    assert 0.3 - 1e-3 < far[0] < 0.3 + 2e-2                               # stopped by the joint limit (XPBD: soft by joint_scale_pos)


def test_planar_roots_stay_in_their_plane():
    for name in ("hopper", "walker2d", "halfcheetah"):
        env = mbd_b200.envs.get_env(name)
        st = _cpu_state(env)
        us = np.clip(np.random.default_rng(3).normal(size=(4, 30, env.action_size)), -1, 1).astype(np.float32)
        fin = orc.xpbd_rollout(env.blob, st, us, want_final=True)["final"]
        assert np.isfinite(fin).all()
        assert np.abs(fin[:, 0, 1]).max() < 1e-4                          # root y
        qw, qy = fin[:, 0, 3], fin[:, 0, 5]
        assert np.abs(fin[:, 0, 4]).max() < 1e-4 and np.abs(fin[:, 0, 6]).max() < 1e-4   # rotation about y only
        assert np.allclose(qw * qw + qy * qy, 1.0, atol=1e-5)


def test_reward_formulas_against_the_reference_expressions():
    """hopper.py:57-65, walker2d.py:56-61, cartpole.py:44 evaluated on the oracle's final state, in float64 with a running
    error bound (tests/xpbd_ref.py), and within the absolute tolerances this test has always used"""
    from tests import xpbd_ref
    for name, z0 in (("hopper", 1.0), ("walker2d", 1.1)):
        env = mbd_b200.envs.get_env(name)
        assert env.blob.view(np.float32)[B.H_RW0] == np.float32(z0)
        st = _cpu_state(env)
        us = np.clip(np.random.default_rng(4).normal(size=(1, 1, env.action_size)), -1, 1).astype(np.float32)
        o = orc.xpbd_rollout(env.blob, st, us, want_rewss=True, want_final=True)
        r = xpbd_ref.reward_post(env.blob, o["final"])
        assert abs(o["rewss"][0, 0] - r.v[0]) <= min(2.0 * r.r[0], 2e-6)
    env = mbd_b200.envs.get_env("cartpole")
    st = _cpu_state(env)
    o = orc.xpbd_rollout(env.blob, st, np.float32([[[0.7]]]), want_rewss=True, want_final=True)
    r = xpbd_ref.reward_post(env.blob, o["final"])
    assert abs(o["rewss"][0, 0] - r.v[0]) <= min(2.0 * r.r[0], 1e-5)
    ps = env._make_pipeline_state(o["final"][0])
    assert np.isclose(r.v[0], np.cos(ps.q[1]) - np.abs(ps.qd[0]), atol=1e-5)     # the same quantity through kinematics.inverse


def test_cartpole_energy_sanity():
    """a motor push moves the cart along +x and swings the (hanging) pole; nothing leaves the rail plane"""
    env = mbd_b200.envs.get_env("cartpole")
    st = _cpu_state(env)
    fin = orc.xpbd_rollout(env.blob, st, np.full((1, 25, 1), 1.0, np.float32), want_final=True)["final"][0]
    assert fin[0, 0] > 0.05 and abs(fin[0, 1]) < 1e-5 and abs(fin[0, 2]) < 2e-3 and abs(fin[1, 1]) < 1e-4   # the pole's weight sags the single-iteration XPBD joint by < 2 mm


# ---------------------------------------------------------------------------------------------------------------
# GPU: kernels vs oracle, bit for bit
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("name", NEW_ENVS)
def test_rollout_kernels_match_oracle_bit_exact(name, variant):
    import torch
    from mbd_b200 import ops
    env = mbd_b200.envs.get_env(name)
    st = _cpu_state(env)
    n, H = (96, 50) if name in ("ant",) else (130, 50)
    us = np.clip(np.random.default_rng(5).normal(size=(n, H, env.action_size)) * 0.7, -1, 1).astype(np.float32)
    ref = orc.xpbd_rollout(env.blob, st, us, want_rewss=True, want_final=True)
    ops.set_kernel_variant(variant)
    try:
        m = env.device_model(torch.device("cuda:0"))
        out = ops.rollout(m, torch.as_tensor(st, device="cuda:0"), torch.as_tensor(us, device="cuda:0"), want_rewss=True, want_final=True)
    finally:
        ops.set_kernel_variant(0)
    assert_bit_exact(out["final"].cpu().numpy(), ref["final"], f"{name} final states")
    assert_bit_exact(out["rewss"].cpu().numpy(), ref["rewss"], f"{name} per-step rewards")
    assert_bit_exact(out["rews"].cpu().numpy(), ref["rews"], f"{name} returns")


@pytest.mark.gpu
@pytest.mark.parametrize("name", NEW_ENVS)
def test_reverse_once_at_baseline_shapes_vs_oracle(name):
    """BASELINE.json configs 2 (hopper 1024 x 50) and 3 (ant 4096 x 50), and the f3 envs: one diffusion step through the
    engine (auto kernel selection) — sampled noise and per-sample returns bit-exact, Ybar and rews.mean() within 1e-4"""
    import torch
    from mbd_b200.planners import engine as eng
    env = mbd_b200.envs.get_env(name)
    st = _cpu_state(env)
    Nn, H = SHAPES[name]
    Nu, temp, i = env.action_size, 0.1, 99
    _, alphas, alphas_bar, sigmas = opl.make_schedule(1e-4, 1e-2, 100)
    key = prng.split(prng.PRNGKey(11))[1]
    Ybar_i = (np.random.default_rng(2).normal(size=H * Nu) * 0.2).astype(np.float32)
    oenv = opl.OracleEnv("xpbd", Nu, blob=env.blob, state=st)
    ref = opl.reverse_once(oenv, key, Nn, H, float(sigmas[i]), Ybar_i, temp, alphas, alphas_bar, i)
    e = eng.DiffusionEngine(env, Nn, H, temp, False, st)
    out, rew = e.reverse_once(key, float(sigmas[i]), torch.as_tensor(Ybar_i, device="cuda:0"), eng.update_coef(alphas, alphas_bar, i))
    assert_bit_exact(e.Y0s.cpu().numpy(), ref["Y0s"], "sampled actions")
    assert_bit_exact(e.rews_local.cpu().numpy(), ref["rews"], "per-sample returns")
    scale = max(np.abs(ref["Ybar_im1"]).max(), 1e-6)
    assert np.abs(out.cpu().numpy() - ref["Ybar_im1"]).max() / scale < 1e-4
    assert abs(rew.item() - ref["rew_mean"]) <= 1e-4 * max(abs(ref["rew_mean"]), 1e-6) + 1e-6
    assert int(e.weights.argmax().item()) == int(ref["weights"].argmax())


@pytest.mark.gpu
@pytest.mark.parametrize("name", NEW_ENVS)
def test_env_surface_step_equals_planner_rollout(name):
    """env.reset / env.step (the reference's env surface) runs the same kernel as the planner: stepping H times equals
    one rollout of the same actions, bit for bit"""
    import torch
    from mbd_b200 import ops
    env = mbd_b200.envs.get_env(name)
    state = env.reset(prng.split(prng.PRNGKey(0))[1])
    H = 4
    us = np.clip(np.random.default_rng(9).normal(size=(H, env.action_size)), -1, 1).astype(np.float32)
    m = env.device_model(torch.device("cuda:0"))
    ro = ops.rollout(m, torch.as_tensor(state.pipeline_state.raw, device="cuda:0"), torch.as_tensor(us[None], device="cuda:0"),
                     want_rewss=True, want_final=True)
    s, rs = state, []
    for t in range(H):
        s = env.step(s, us[t])
        rs.append(s.reward)
    assert_bit_exact(s.pipeline_state.raw, ro["final"][0].cpu().numpy())
    assert_bit_exact(np.float32(rs), ro["rewss"][0].cpu().numpy())
    assert s.obs.shape == state.obs.shape and np.isfinite(s.obs).all()
