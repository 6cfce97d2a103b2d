"""SAC on the device: k_sac_act bit for bit against the host harness of include/mbd_sac.h, the replay ring against rows built from the
vector env step by step, k_sac_sample against its host restatement, the statistics against float64, graph replay against eager
launches, determinism of training, and a short learning run.

The learning run (tests/sac_ref.learn_config: hopper at the reference's configuration, the prefill and 600 training steps, 85 k env
steps) is calibrated by scripts/gpu_sac_timing.py (profiles/h100_sac.json, "learning_check", H100 80GB HBM3 at 400 W, 31 s a run).  Over
seeds 0 .. 4 the evaluation return rose from 2620 / 2436 / 2854 / 13973 / 625 to 36311 / 32324 / 29925 / 34654 / 31142: every seed gained
at least 20681, and the returns of the five seeds spread by 13348 before and 6386 after.  The test asks seed 0 (a gain of 33691) for a
gain of 15000, above both spreads and below every seed's gain."""
import numpy as np
import pytest
import torch

from mbd_b200 import _lib, ops, prng
from mbd_b200.envs import get_env
from mbd_b200.envs.vec import VecEnv
from mbd_b200.rl import sac
from tests import ppo_ref, sac_ref
from tests.test_sac_cpu import host_act, random_policy, sac_harness  # noqa: F401  (sac_harness: the fixture of the host build)

pytestmark = pytest.mark.gpu
LEARN_MARGIN = 15000.0
_envs = {}


def _env(name):
    if name not in _envs:
        _envs[name] = get_env(name)
    return _envs[name]


def _bits(a, b, what):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), \
        f"{what}: {np.count_nonzero(a.view(np.uint32) != b.view(np.uint32))} of {a.size} differ"


def _small_trainer(name, B=8, cap=20, episode_length=5, seed=0, G=4, mb=16, steps=3, min_replay=16):
    c = sac.counts(10 ** 9, B, min_replay, 2)
    num_timesteps = c.prefill_env_steps + steps * B
    return sac.SACTrainer(_env(name), num_timesteps, episode_length, B, 16, 6e-4, 0.997, seed, mb, 2, True, 30.0, 0.005, min_replay,
                          cap, G)


@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("B", [1, 33, 128, 4096])
@pytest.mark.parametrize("name", ["hopper", "cartpole", "halfcheetah", "pushT", "humanoidrun"])
def test_act_matches_host_harness(sac_harness, name, B, part):
    prng.set_layout(bool(part))
    try:
        venv = VecEnv(_env(name), B)
        venv.reset(prng.split(prng.PRNGKey(3), B))
        O, nu = venv.spec.obs_size, venv.spec.nu
        policy, mean, std, _ = random_policy(O, nu, 7)
        d = venv.device
        pol, m, s = (torch.from_numpy(a).to(d) for a in (policy, mean, std))
        key = prng.PRNGKey(B + 5)
        actor = sac.Actor(venv, pol, m, s)
        obs = venv.obs.cpu().numpy()
        actor.act(key)
        got = venv.actions.cpu().numpy()
        eps = sac_ref.normal_host(key, (B, nu))
    finally:
        prng.set_layout(False)
    a_h, _, _ = host_act(sac_harness, policy, mean, std, obs, eps)
    _bits(got, a_h, "actions")
    assert actor.ctl.cpu().tolist() == [1, 1, 0, 0]


def test_ring_matches_the_vector_env_across_auto_reset_and_wrap():
    tr = _small_trainer("cartpole", B=8, cap=20, episode_length=3, steps=10)
    v = tr.venv
    ring = sac_ref.RingRef(tr.cap, tr.R)
    O, nu = tr.O, tr.nu
    dones = []
    for _ in range(7):                       # 56 rows through a ring of 20: wraps twice, and the capacity is not a multiple of B
        obs = v.obs.cpu().numpy().copy()
        ops.sac_act(tr.plan, _lib.SAC_ACT)
        act = v.actions.cpu().numpy().copy()
        ops.vec_step(v.plan)
        ops.sac_record(tr.plan)
        rows = np.zeros((tr.B, tr.R), np.float32)
        rows[:, :O], rows[:, O:O + nu] = obs, act
        rows[:, O + nu], rows[:, O + nu + 1] = v.reward.cpu().numpy(), 1 - v.done.cpu().numpy()
        rows[:, O + nu + 2:2 * O + nu + 2], rows[:, 2 * O + nu + 2] = v.obs.cpu().numpy(), v.truncation.cpu().numpy()
        dones.append(v.done.cpu().numpy())
        ring.insert(rows)
        torch.cuda.synchronize()
        _bits(tr.ring.cpu().numpy(), ring.data, "ring")
        _bits(tr.stage.cpu().numpy(), obs, "staged obs")
        assert tr.ring_ctl.cpu().tolist() == [ring.pos, ring.size, 0, 0]
    assert np.any(np.array(dones) == 1), "no auto-reset happened"
    assert tr.act_ctl.cpu().tolist() == [7, 7, 0, 0]


@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("size", [1, 8192, 5001, 1 << 20])
def test_sample_matches_host(size, part):
    prng.set_layout(bool(part))
    try:
        tr = _small_trainer("hopper", B=128, cap=1 << 20, G=64, mb=512, min_replay=128)
        rng = np.random.default_rng(size)
        pos = int(rng.integers(0, tr.cap))
        data = rng.normal(size=(tr.cap, tr.R)).astype(np.float32)
        tr.ring.copy_(torch.from_numpy(data))
        tr.ring_ctl.copy_(torch.tensor([pos, size, 0, 0], dtype=torch.int32))
        tr.sample_ctl[0] = 1                                  # training step row 1 of the noise keys
        ops.sac_sample(tr.plan)
        torch.cuda.synchronize()
        bk, idx, rows, eps = sac_ref.sample_host(data, pos, size, tr.keys.buffer, tr.keys.noise[1], tr.G, tr.mb, tr.nu)
    finally:
        prng.set_layout(False)
    assert np.array_equal(tr.idx.cpu().numpy(), idx)
    _bits(tr.batch.cpu().numpy(), rows, "gathered rows")
    _bits(tr.eps.cpu().numpy(), eps, "noise")
    ctl = tr.sample_ctl.cpu().numpy()
    assert ctl[0] == 2 and ctl[1] == 0 and np.array_equal(ctl[2:].view(np.uint32), bk)


def test_obs_stats_against_float64():
    tr = _small_trainer("halfcheetah", B=64, cap=256)
    st = (0.0, np.zeros(tr.O), np.zeros(tr.O))
    for _ in range(3):
        obs = tr.venv.obs.cpu().numpy().copy()
        tr.actor_step()
        st, std = ppo_ref.running_update(st, obs)
    torch.cuda.synchronize()
    stat = tr.stat.cpu().numpy()
    assert stat[0] == st[0]
    np.testing.assert_allclose(stat[1:1 + tr.O], st[1], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(tr.mean.cpu().numpy(), st[1], rtol=1.2e-7, atol=1e-12)
    np.testing.assert_allclose(tr.std.cpu().numpy(), std, rtol=1.2e-7)


def _run(tr, steps):
    tr.prefill()
    for _ in range(steps):
        tr.training_step()
    torch.cuda.synchronize()
    return [t.detach().cpu().numpy().copy() for t in (tr.learner.policy, tr.learner.q, tr.learner.target_q, tr.learner.log_alpha,
                                                        tr.std, tr.ring)]


def test_graph_replay_equals_eager():
    a, b = _small_trainer("hopper", seed=4), _small_trainer("hopper", seed=4)
    b.capture()
    ra, rb = _run(a, 3), _run(b, 3)
    for name, x, y in zip(("policy", "q", "target_q", "log_alpha", "obs std", "ring"), ra, rb):
        _bits(x, y, name)
    assert np.isfinite(ra[0]).all() and not np.array_equal(ra[0], sac.nets.init_params(a.keys.policy, sac.nets.sac_policy_sizes(a.O, a.nu)))


def test_training_is_deterministic():
    runs = []
    for _ in range(2):
        tr = _small_trainer("pushT", seed=9)
        tr.capture()
        p = _run(tr, 3)
        runs.append((p, tr.evaluate()))
    for name, x, y in zip(("policy", "q", "target_q", "log_alpha", "obs std", "ring"), runs[0][0], runs[1][0]):
        _bits(x, y, name)
    assert runs[0][1] == runs[1][1]


def test_short_run_learns():
    curve = []
    cfg = sac_ref.learn_config(0)
    sac.train(environment=sac_ref.LEARN_ENV, progress_fn=lambda n, m: curve.append((n, m["eval/episode_reward"])), **cfg)
    assert [n for n, _ in curve] == [0, cfg["num_timesteps"]]
    assert curve[1][1] > curve[0][1] + LEARN_MARGIN, curve


def test_actor_without_key_table_needs_a_key():
    venv = VecEnv(_env("hopper"), 2)
    venv.reset(prng.split(prng.PRNGKey(0), 2))
    policy, mean, std, _ = random_policy(venv.spec.obs_size, venv.spec.nu, 1)
    actor = sac.Actor(venv, *(torch.from_numpy(a).cuda() for a in (policy, mean, std)))
    actor.act(prng.PRNGKey(1))
    with pytest.raises(ValueError, match="key"):
        actor.act()
