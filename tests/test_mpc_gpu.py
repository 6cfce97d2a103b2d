"""The receding-horizon controller on the device (mbd_mpc_advance, mbd_b200/planners/mbd_mpc.py): control step 0 against
run_diffusion, the graph-replayed loop against the host-driven loop and against eager launches, batch invariance, the CPU
restatement on car2d, and a control check on hopper."""
import numpy as np
import pytest
import torch

import mbd_b200
from mbd_b200 import ops
from mbd_b200.planners import mbd_mpc
from mbd_b200.planners.mbd_mpc import Args, Controller
from mbd_b200.planners.mbd_planner import Args as PlannerArgs
from mbd_b200.planners.mbd_planner import run_diffusion
from tests import mpc_ref
from tests.conftest import assert_bit_exact

pytestmark = pytest.mark.gpu
RTOL = 1e-4   # tests/test_planner_gpu.py: a solve against the oracle


def N(t):
    return t.detach().cpu().numpy()


def margs(env_name, B, Nsample=256, Hsample=16, Ndiffuse=10, Nwarm=3, Nstep=20, seed0=0):
    """B Args of one env and shape; seed, temp_sample, beta0 and betaT vary from problem to problem"""
    temps = [0.1, 0.05, 0.3, 0.2, 0.15, 0.5, 0.08, 1.0]
    return [Args(seed=seed0 + 3 * b, env_name=env_name, Nsample=Nsample, Hsample=Hsample, Ndiffuse=Ndiffuse, Nwarm=Nwarm,
                 Nstep=Nstep, temp_sample=temps[b % 8], beta0=1e-4 * (1 + b % 3), betaT=1e-2 * (1 + 0.5 * (b % 2)),
                 not_render=True, disable_recommended_params=True) for b in range(B)]


def controller(args_list, host=False):
    env = mbd_mpc._prepare(args_list, batch=True)
    return env, Controller(env, args_list, host=host)


def assert_same(r, q, what):
    for f in ("actions", "rewards", "states", "rew_hist"):
        assert_bit_exact(getattr(r, f), getattr(q, f), f"{what}: {f}")


@pytest.mark.parametrize("env_name", ["car2d", "hopper", "pushT"])
def test_control_step_0_is_run_diffusion(env_name):
    """P_0 = run_diffusion's Yi[-1] bit for bit; a_0 = P_0[0]; s_1 and r_0 = host env.step(s_0, a_0)"""
    args_list = margs(env_name, 2, Nstep=1)
    env, ctl = controller(args_list)
    res = ctl.run()
    for b, a in enumerate(args_list):
        pa = PlannerArgs(**{k: getattr(a, k) for k in PlannerArgs.__dataclass_fields__})
        _, Yi = run_diffusion(pa, return_trajectory=True)
        assert_bit_exact(N(ctl.engine.Ybars[b, 0]), N(Yi[-1]).reshape(-1), "P_0")
        assert_bit_exact(res.actions[b, 0], N(Yi[-1][0]), "a_0")
        s1 = env.step(ctl.host_states[b], N(Yi[-1][0]))
        assert_bit_exact(res.states[b, 0], mbd_mpc.host_raw(env, ctl.host_states[b]), "s_0")
        assert_bit_exact(res.states[b, 1], mbd_mpc.host_raw(env, s1), "s_1")
        assert_bit_exact(res.rewards[b, 0], np.float32(s1.reward), "r_0")
        assert_bit_exact(res.rew_hist[b, 0], N(ctl.engine.rew_hist[b, 1]), "rew_hist")


@pytest.mark.parametrize("env_name", ["hopper", "ant", "pushT", "car2d", "humanoidrun"])
def test_graph_replay_equals_the_host_driven_loop(env_name):
    """20 control steps of 2 seeds: actions, rewards, states and rew_hist bit for bit against eager steps with the host in the
    loop (plan to the host, host env.step, warm start / keys / step counter written with torch)"""
    args_list = margs(env_name, 2)
    _, dev = controller(args_list)
    r = dev.run()
    _, host = controller(args_list, host=True)
    q = host.run_host_driven()
    assert_same(r, q, env_name)
    assert np.isfinite(r.states).all() and np.isfinite(r.rewards).all()
    ctl = N(dev.engine.ctl)
    assert (ctl[:, 0] == 0).all() and (ctl[:, 2] == 0).all()
    assert (N(dev.mpc_ctl) == 20).all()


def test_graph_replay_equals_eager_launches():
    args_list = margs("hopper", 3, Nstep=8)
    _, g = controller(args_list)
    r = g.run(graph=True)
    assert g.graph is not None
    _, e = controller(args_list)
    q = e.run(graph=False)
    assert e.graph is None
    assert_same(r, q, "graph vs eager")
    for c in (g, e):
        ctl = N(c.engine.ctl)
        assert (ctl[:, 0] == 0).all() and (ctl[:, 2] == 0).all()


def test_batch_invariance():
    """problem b of run_mpc_batch (8 seeds, mixed temperatures and betas) is run_mpc of that seed bit for bit"""
    args_list = margs("hopper", 8, Nsample=128, Ndiffuse=8, Nwarm=3, Nstep=6)
    rew, res = mbd_mpc.run_mpc_batch(args_list, return_result=True)
    assert rew.shape == (8,)
    for b, a in enumerate(margs("hopper", 8, Nsample=128, Ndiffuse=8, Nwarm=3, Nstep=6)):
        r1, q = mbd_mpc.run_mpc(a, return_result=True)
        assert r1 == rew[b]
        for f in ("actions", "rewards", "states", "rew_hist"):
            assert_bit_exact(getattr(res, f)[b], getattr(q, f)[0], f"problem {b}: {f}")


def test_past_the_last_control_step_nothing_changes():
    """an ACT or RECORD launch after the last control step writes nothing: the logs, plan rows and counters stay"""
    _, c = controller(margs("car2d", 2, Nstep=3))
    c.run()
    before = [N(t).copy() for t in (c.actions, c.rewards, c.states, c.rew_hist, c.engine.Ybars, c.engine.params, c.engine.ctl,
                                    c.mpc_ctl)]
    from mbd_b200 import _lib
    ops.mpc_advance(c.plan, _lib.MPC_ACT)
    ops.mpc_advance(c.plan, _lib.MPC_ACT)
    after = [N(t) for t in (c.actions, c.rewards, c.states, c.rew_hist, c.engine.Ybars, c.engine.params, c.engine.ctl, c.mpc_ctl)]
    for x, y in zip(before, after):
        assert (x.view(np.uint32) == y.view(np.uint32)).all()


def test_against_the_cpu_restatement_car2d(orc):
    """control steps 0 and 1 within the tolerance of a solve against the oracle (tests/test_planner_gpu.py)"""
    car = mbd_b200.envs.get_env("car2d")
    ref = mpc_ref.run_mpc_car2d(car, seed=0, Nsample=64, H=8, Ndiffuse=10, Nwarm=3, Nstep=2, temp=0.1)
    for Nstep in (1, 2):
        a = margs("car2d", 1, Nsample=64, Hsample=8, Ndiffuse=10, Nwarm=3, Nstep=Nstep)[0]
        _, c = controller([a])
        res = c.run()
        P = N(c.engine.Ybars[0, 0]).reshape(8, 2)
        want = ref["plans"][Nstep - 1]
        err = np.abs(P.astype(np.float64) - want).max() / max(np.abs(want).max(), 1e-6)
        assert err <= RTOL, f"P_{Nstep - 1}: {err:.3e}"
        err_s = np.abs(res.states[0, Nstep] - ref["states"][Nstep]).max() / np.abs(ref["states"][Nstep]).max()
        assert err_s <= RTOL, f"s_{Nstep}: {err_s:.3e}"


# Measured on an H100 80GB HBM3 (700 W): closed loop 3.737 / 3.990 / 4.104 / 3.862 / 4.140 against zero action -0.090 / -0.109 /
# -0.082 / -0.105 / -0.087 over seeds 0 ... 4, gains 3.83 to 4.23, mean 4.06.  The threshold is half the smallest gain.
CONTROL_MARGIN = 1.9


def test_closed_loop_beats_zero_action_on_hopper():
    """hopper, 5 seeds: the closed-loop mean reward over Nstep control steps exceeds that of the zero-action rollout from the
    same reset state, on average over the seeds by more than CONTROL_MARGIN"""
    Nstep = 50
    args_list = [Args(seed=s, env_name="hopper", Nsample=1024, Hsample=50, Ndiffuse=100, Nwarm=10, Nstep=Nstep, not_render=True)
                 for s in range(5)]
    rew, res = mbd_mpc.run_mpc_batch(args_list, return_result=True)
    env = mbd_b200.envs.get_env("hopper")
    m = env.device_model()
    zero = []
    for b in range(5):
        s0 = torch.as_tensor(res.states[b, 0], device=m.device)
        zero.append(float(ops.rollout(m, s0, torch.zeros((1, Nstep, env.action_size), device=m.device))["rews"][0].item()))
    gain = rew - np.asarray(zero)
    print(f"closed loop {rew}, zero action {zero}, gain {gain}, mean gain {gain.mean():.4f}")
    assert gain.mean() > CONTROL_MARGIN
