"""The recorded rollout (`ops.rollout(..., want_traj=True)`, k_rollout_wpl<Traj>) and the diffusion-process page on the device:
every recorded state against H successive one-step `ops.rollout` calls, bit for bit, on the shipped humanoids, hopper, ant and a
random model, at one sample, 77 and more than 16 per SM (which crosses every kernel the selector picks for the plain rollout); the
other outputs against the rollout without a record; the world poses of every iterate against host `env.step`; pushT; and the
whole script against the host-stepped path."""
import numpy as np
import pytest
import torch

import mbd_b200
from mbd_b200 import ops, prng
from mbd_b200.envs import get_env
from mbd_b200.scripts import vis_diffusion as vd
from tests import modelgen

pytestmark = pytest.mark.gpu
H = 4


def _bits(a, b, what):
    a = np.ascontiguousarray(a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a, np.float32)
    b = np.ascontiguousarray(b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else b, np.float32)
    assert a.shape == b.shape, f"{what}: shape {a.shape} != {b.shape}"
    bad = np.count_nonzero(a.view(np.uint32) != b.view(np.uint32))
    assert bad == 0, f"{what}: {bad} of {a.size} words differ"


def _big_n():
    return 16 * torch.cuda.get_device_properties(0).multi_processor_count + 37


def _env(name, tmp_path):
    if name == "random":
        xml, facts = modelgen.random_model(7)
        p = tmp_path / "model_7.xml"
        p.write_text(xml)
        env = mbd_b200.envs.GenericPositionalEnv(str(p), n_frames=3)
        return env, env.pipeline_init(env.sys.init_q, np.zeros(env.sys.qd_size())).raw
    env = get_env(name)
    return env, env.reset(prng.split(prng.PRNGKey(1))[1]).pipeline_state.raw


@pytest.mark.parametrize("n", [1, 77, "big"])
@pytest.mark.parametrize("name", ["humanoidrun", "humanoidtrack", "hopper", "ant", "random"])
def test_recorded_states_equal_one_step_rollouts(name, n, tmp_path):
    n = _big_n() if n == "big" else n
    env, raw = _env(name, tmp_path)
    m = env.device_model()
    raw0 = torch.as_tensor(np.asarray(raw, np.float32), device=m.device)
    rng = np.random.default_rng(n)
    us = torch.as_tensor(np.clip(rng.normal(size=(n, H, m.nu)) * 0.7, -1, 1).astype(np.float32), device=m.device)
    rec = ops.rollout(m, raw0, us, want_traj=True, want_final=True, want_rewss=True)
    plain = ops.rollout(m, raw0, us, want_final=True, want_rewss=True)
    assert rec["traj"].shape == (n, H, m.L, 13)
    _bits(rec["final"], plain["final"], "final state")
    _bits(rec["rews"], plain["rews"], "returns")
    _bits(rec["rewss"], plain["rewss"], "per-step rewards")
    _bits(rec["traj"][:, -1], plain["final"], "last recorded state")
    steps = torch.empty_like(rec["traj"])
    for i in range(n):
        st = raw0
        for t in range(H):
            st = ops.rollout(m, st, us[i:i + 1, t:t + 1].contiguous(), want_final=True)["final"][0]
            steps[i, t] = st
    _bits(rec["traj"], steps, f"recorded states of {name}, n = {n}")


@pytest.mark.parametrize("name", ["hopper", "humanoidtrack"])
def test_world_poses_equal_host_steps(name):
    env = get_env(name)
    state = env.reset(prng.split(prng.PRNGKey(0))[1])
    us = np.clip(np.random.default_rng(5).normal(size=(5, 6, env.action_size)) * 0.7, -1, 1).astype(np.float32)
    pos, rot = vd.device_rollouts(env, state, us)
    hpos, hrot = vd.host_rollouts(env, state, us)
    assert pos.shape == (5, 6, env.sys.num_links(), 3)
    _bits(pos, hpos, f"{name} x.pos")
    _bits(rot, hrot, f"{name} x.rot")


def test_world_poses_cross_a_chunk_boundary():
    """more states than one vector env holds: the chunks (the last one padded) give what one pass per state gives"""
    env = get_env("hopper")
    m = env.device_model()
    raw0 = torch.as_tensor(env.reset(prng.PRNGKey(3)).pipeline_state.raw, device=m.device)
    us = torch.rand((1400, 50, env.action_size), device=m.device) * 2 - 1
    before = vd.rollout_states_device(env, raw0, us).reshape(-1, *raw0.shape)
    assert before.shape[0] > mbd_b200._lib.VEC_MAX_B
    pos, rot = vd.world_poses(env, before)
    sel = [0, 1, mbd_b200._lib.VEC_MAX_B - 1, mbd_b200._lib.VEC_MAX_B, before.shape[0] - 1]
    for i in sel:
        ps = env._make_pipeline_state(before[i].cpu().numpy())
        _bits(pos[i], ps.x.pos, f"x.pos of state {i}")
        _bits(rot[i], ps.x.rot, f"x.rot of state {i}")


def test_pusht_poses_equal_host_steps():
    env = get_env("pushT")
    state = env.reset(prng.split(prng.PRNGKey(0))[1])
    us = np.random.default_rng(6).uniform(-1, 1, size=(4, 7, 2)).astype(np.float32)
    pos, rot = vd.device_rollouts(env, state, us)
    hpos, hrot = vd.host_rollouts(env, state, us)
    _bits(pos, hpos, "pushT x.pos")
    _bits(rot, hrot, "pushT x.rot")


def test_script_page_equals_the_host_stepped_page(tmp_path):
    env = get_env("humanoidtrack")
    mu = np.clip(np.random.default_rng(8).normal(size=(19, 50, env.action_size)) * 0.5, -1, 1).astype(np.float32)
    np.save(tmp_path / "mu_0ts.npy", mu)
    out = vd.main(["--env_name", "humanoidtrack", "--path", str(tmp_path)])
    page = open(out).read()
    us = vd.load_iterates(str(tmp_path), env.action_size)
    assert us.shape[0] == 20
    hpos, hrot = vd.rollouts("humanoidtrack", env, us, cache=None, host=True)
    assert page == vd.render_page("humanoidtrack", env, hpos, hrot)
    # a second run reads the cache and writes the same page
    assert open(vd.main(["--env_name", "humanoidtrack", "--path", str(tmp_path)])).read() == page
