"""The vector env on the device against the host env of one state (each env class is the specification): reset, 30 steps, batch
invariance across the kernel variants the step selects, set_state against the planner's rollout, graph capture, the episode wrapper /
auto-reset and the world poses.  Raw states and rewards are held bit for bit, observations and kinematic outputs to one float32 ulp."""
import numpy as np
import pytest
import torch

from mbd_b200 import ops, prng
from mbd_b200.envs import get_env
from mbd_b200.envs.vec import VecEnv
from tests.vecenv_ref import wrapper_step

pytestmark = pytest.mark.gpu

ENVS = ["humanoidrun", "humanoidstandup", "humanoidtrack", "hopper", "walker2d", "cartpole", "ant", "halfcheetah", "pushT", "car2d"]
B = 33
_cache = {}


def _env(name):
    if name not in _cache:
        _cache[name] = get_env(name)
    return _cache[name]


def _ulp(dev, host, what):
    dev, host = np.asarray(dev, np.float32).ravel(), np.asarray(host, np.float32).ravel()
    err = np.abs(dev.astype(np.float64) - host.astype(np.float64))
    ok = (err <= np.spacing(np.abs(host)).astype(np.float64)) | (err <= 1e-12)
    assert ok.all(), f"{what}: {np.count_nonzero(~ok)} of {ok.size} beyond 1 ulp, worst {err.max():.3g}"


def _bits(a, b, what):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{what} differs"


def _raw(s):
    ps = s.pipeline_state
    return np.asarray(ps if isinstance(ps, np.ndarray) else ps.raw, np.float32)


def _actions(env, T, n, seed):
    return np.random.default_rng(seed).uniform(-1, 1, (T, n, env.action_size)).astype(np.float32)


@pytest.mark.parametrize("name", ENVS)
def test_reset_matches_host(name):
    env = _env(name)
    keys = prng.split(prng.PRNGKey(7), B)
    venv = VecEnv(env, B)
    st = venv.reset(keys)
    host = [env.reset(keys[b]) for b in range(B)]
    raw = st.raw.cpu().numpy().reshape(B, -1)
    hraw = np.stack([_raw(h).ravel() for h in host])
    if name in ("pushT", "car2d"):
        _bits(raw, hraw, "reset state (the noise itself)")
    else:
        _ulp(raw, hraw, "reset raw state")
    _ulp(st.obs.cpu().numpy(), np.stack([np.asarray(h.obs, np.float32) for h in host]), "reset obs")
    assert np.array_equal(st.reward.cpu().numpy(), np.float32([h.reward for h in host]))
    assert np.array_equal(st.done.cpu().numpy(), np.float32([h.done for h in host]))
    assert not st.steps.any() and not st.truncation.any()


@pytest.mark.parametrize("name", ENVS)
def test_steps_match_host_loop(name):
    env = _env(name)
    keys = prng.split(prng.PRNGKey(11), B)
    host = [env.reset(keys[b]) for b in range(B)]
    venv = VecEnv(env, B)
    venv.set_state(np.stack([_raw(h) for h in host]))
    acts = _actions(env, 30, B, seed=1)
    for t in range(30):
        st = venv.step(torch.as_tensor(acts[t], device="cuda"))
        host = [env.step(host[b], acts[t, b]) for b in range(B)]
        _bits(st.raw.cpu().numpy().reshape(B, -1), np.stack([_raw(h).ravel() for h in host]), f"raw state, step {t}")
        _bits(st.reward.cpu().numpy(), np.float32([h.reward for h in host]), f"reward, step {t}")
        _ulp(st.obs.cpu().numpy(), np.stack([np.asarray(h.obs, np.float32) for h in host]), f"obs, step {t}")
        assert np.array_equal(st.done.cpu().numpy(), np.float32([h.done for h in host])), f"done, step {t}"


@pytest.mark.parametrize("name", ["humanoidrun", "humanoidstandup", "hopper", "ant", "pushT", "car2d"])
@pytest.mark.parametrize("n", [1, 4096])
def test_batch_invariance_across_sizes_and_permutations(name, n):
    """B = 33 is the reference; its envs are embedded (permuted) in a batch of n, which for the 11-link models at 4096 runs the
    warp-per-link kernel instead of the lane-per-link one, and for n = 1 a single env"""
    env = _env(name)
    keys = prng.split(prng.PRNGKey(3), max(n, B))
    acts = _actions(env, 5, max(n, B), seed=4)
    ref = VecEnv(env, B)
    ref.reset(keys[:B])
    outs = []
    for t in range(5):
        s = ref.step(torch.as_tensor(acts[t, :B], device="cuda"))
        outs.append((s.raw.clone(), s.obs.clone(), s.reward.clone()))
    rng = np.random.default_rng(n)
    perm = rng.permutation(max(n, B))
    pos = np.argsort(perm)[:B] if n >= B else None   # where env b of the reference sits in the permuted batch
    big = VecEnv(env, n)
    sel = perm[:n] if n >= B else np.array([5])
    big.reset(keys[sel])
    for t in range(5):
        s = big.step(torch.as_tensor(acts[t, sel], device="cuda"))
        idx = torch.as_tensor(pos if n >= B else [0], device="cuda")
        src = torch.as_tensor(np.arange(B) if n >= B else [5], device="cuda")
        for a, r in zip((s.raw, s.obs, s.reward), outs[t]):
            _bits(a[idx].cpu().numpy(), r[src].cpu().numpy(), f"batch of {n}, step {t}")


@pytest.mark.parametrize("name", ["humanoidrun", "hopper", "pushT", "car2d"])
def test_set_state_then_step_equals_rollout(name):
    env = _env(name)
    acts = torch.as_tensor(_actions(env, 1, B, seed=9)[0], device="cuda")
    venv = VecEnv(env, B)
    if name == "pushT":
        x0 = torch.as_tensor(env.reset(prng.PRNGKey(0)).pipeline_state.raw, device="cuda")
        ref = ops.pusht_rollout(env.device_params(), x0, acts[:, None, :].contiguous(), want_final=True)
        venv.set_state(x0.expand(B, -1))
        st = venv.step(acts)
        _bits(st.raw.cpu().numpy(), ref["final"].cpu().numpy(), "state")
    elif name == "car2d":
        x0 = torch.as_tensor(env.x0, device="cuda")
        ref = ops.car2d_rollout(env.device_params()[0], x0, acts[:, None, :].contiguous(), want_traj=True)
        venv.set_state(x0.expand(B, -1))
        st = venv.step(acts)
        _bits(st.raw.cpu().numpy(), ref["traj"][:, 0].cpu().numpy(), "state")
    else:
        state_init = torch.as_tensor(env.reset(prng.PRNGKey(0)).pipeline_state.raw, device="cuda")
        ref = ops.rollout(env.device_model(), state_init, acts[:, None, :].contiguous(), want_final=True)
        venv.set_state(state_init.expand(B, -1, -1))
        st = venv.step(acts)
        _bits(st.raw.cpu().numpy(), ref["final"].cpu().numpy(), "state")
    _bits(st.reward.cpu().numpy(), ref["rews"].cpu().numpy(), "reward")


@pytest.mark.parametrize("name", ["humanoidrun", "hopper", "pushT"])
def test_graph_replay_equals_eager(name):
    env = _env(name)
    keys = prng.split(prng.PRNGKey(5), 256)
    acts = torch.as_tensor(_actions(env, 20, 256, seed=6), device="cuda")
    eager = VecEnv(env, 256, episode_length=7)
    eager.reset(keys)
    ref = []
    for t in range(20):
        s = eager.step(acts[t])
        ref.append(torch.cat([s.raw.reshape(256, -1), s.obs, s.reward[:, None], s.done[:, None], s.truncation[:, None], s.steps[:, None]], 1).clone())
    venv = VecEnv(env, 256, episode_length=7)
    venv.reset(keys)
    venv.step(acts[0])   # warm-up outside the capture (first-use setup), then start over
    venv.reset(keys)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            venv.step()
    torch.cuda.current_stream().wait_stream(s)
    for t in range(20):
        venv.actions.copy_(acts[t])
        g.replay()
        st = venv._view()
        got = torch.cat([st.raw.reshape(256, -1), st.obs, st.reward[:, None], st.done[:, None], st.truncation[:, None], st.steps[:, None]], 1)
        _bits(got.cpu().numpy(), ref[t].cpu().numpy(), f"replay {t}")


@pytest.mark.parametrize("name", ["hopper", "pushT"])
def test_auto_reset_against_host_restatement(name):
    env = _env(name)
    ep, n = 5, 64
    keys = prng.split(prng.PRNGKey(21), n)
    acts = _actions(env, 17, n, seed=8)
    wrapped = VecEnv(env, n, episode_length=ep)
    plain = VecEnv(env, n)
    s0 = wrapped.reset(keys)
    first_raw, first_obs = s0.raw.clone(), s0.obs.clone()
    plain.reset(keys)
    done, steps = np.zeros(n, np.float32), np.zeros(n, np.float32)
    for t in range(17):
        pre = wrapped.state.clone()
        plain.set_state(pre)             # the same physics step from the same states, without the wrapper
        p = plain.step(torch.as_tensor(acts[t], device="cuda"))
        w = wrapped.step(torch.as_tensor(acts[t], device="cuda"))
        env_done = p.done.cpu().numpy()
        done, trunc, steps, reset = wrapper_step(done, steps, env_done, ep)
        _bits(w.done.cpu().numpy(), done, f"done {t}")
        _bits(w.truncation.cpu().numpy(), trunc, f"truncation {t}")
        _bits(w.steps.cpu().numpy(), steps, f"steps {t}")
        _bits(w.reward.cpu().numpy(), p.reward.cpu().numpy(), f"reward {t}")
        m = torch.as_tensor(reset, device="cuda")
        exp_raw = torch.where(m.view(-1, *[1] * (p.raw.dim() - 1)), first_raw, p.raw)
        exp_obs = torch.where(m[:, None], first_obs, p.obs)
        _bits(w.raw.cpu().numpy(), exp_raw.cpu().numpy(), f"state {t}")
        _bits(w.obs.cpu().numpy(), exp_obs.cpu().numpy(), f"obs {t}")
    assert (steps <= ep).all()


@pytest.mark.parametrize("name", ["humanoidrun", "humanoidtrack", "hopper", "cartpole", "ant"])
def test_world_poses_match_host(name):
    env = _env(name)
    venv = VecEnv(env, B)
    venv.reset(prng.split(prng.PRNGKey(2), B))
    venv.step(torch.as_tensor(_actions(env, 1, B, seed=2)[0], device="cuda"))
    pos, rot = venv.world_poses()
    hs = [venv.pipeline_state(b) for b in range(B)]
    _ulp(pos.cpu().numpy(), np.stack([h.x.pos for h in hs]), "x.pos")
    _ulp(rot.cpu().numpy(), np.stack([h.x.rot for h in hs]), "x.rot")


def test_humanoidtrack_rejects_episode_length():
    from mbd_b200._lib import MbdError
    venv = VecEnv(_env("humanoidtrack"), 4, episode_length=5)
    with pytest.raises(MbdError, match="time-counter done"):
        venv.step()
