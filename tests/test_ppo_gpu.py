"""PPO on the device: k_ppo_act bit for bit against the host harness of include/mbd_ppo.h, the rollout records against the vector
env step by step, GAE against its float32 restatement, the statistics against float64, graph replay against eager launches,
determinism of training, and a short learning run.

The learning run (tests/ppo_ref.learn_config: halfcheetah at the reference's configuration, three training steps) is calibrated by
scripts/gpu_ppo_timing.py (profiles/h100_ppo.json, "learning_check", H100 80GB HBM3 at 400 W, 1.5-1.6 s a run).  Over seeds 0 .. 4 the
evaluation return rose from -188.5 / -216.0 / -236.5 / -161.3 / -166.0 to 222.4 / 189.4 / 192.3 / 383.7 / 393.4: every seed gained at
least 405, and the returns of the five seeds spread by 75 before and 204 after.  The test asks seed 0 (a gain of 411) for a gain of 250,
above both spreads and well below every seed's gain."""
import numpy as np
import pytest
import torch

from mbd_b200 import _lib, ops, prng
from mbd_b200.blackbox.mbd_mnist import normal_host
from mbd_b200.envs import get_env
from mbd_b200.envs.vec import VecEnv
from mbd_b200.rl import ppo
from tests import ppo_ref
from tests.test_ppo_cpu import harness, host_act, random_policy  # noqa: F401  (harness: the fixture of the host build)

pytestmark = pytest.mark.gpu
LEARN_MARGIN = 250.0
_envs = {}


def _env(name):
    if name not in _envs:
        _envs[name] = get_env(name)
    return _envs[name]


def _bits(a, b, what):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), \
        f"{what}: {np.count_nonzero(a.view(np.uint32) != b.view(np.uint32))} of {a.size} differ"


def _small_trainer(name, B=8, T=4, batch=4, nmb=4, E=2, episode_length=7, seed=0, evals=2):
    c = ppo.counts(10 ** 9, B, batch, nmb, T, evals)
    steps = 2 * batch * nmb * T    # two training steps per epoch
    return ppo.PPOTrainer(_env(name), steps * c.num_evals_after_init, episode_length, B, 16, 3e-4, 1e-3, 0.97, seed, T, batch, nmb, E,
                          evals, True, 1.0, 0.3, 0.95)


@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("B", [1, 33, 4096])
@pytest.mark.parametrize("name", ["cartpole", "pushT", "halfcheetah", "ant", "humanoidrun"])
def test_act_matches_host_harness(harness, name, B, part):
    prng.set_layout(bool(part))
    try:
        venv = VecEnv(_env(name), B)
        venv.reset(prng.split(prng.PRNGKey(3), B))
        O, nu = venv.spec.obs_size, venv.spec.nu
        policy, mean, std, _ = random_policy(O, nu, 7)
        d = venv.device
        pol, m, s = (torch.from_numpy(a).to(d) for a in (policy, mean, std))
        key = prng.PRNGKey(B + 5)
        act = ppo.Actor(venv, pol, m, s)
        obs = venv.obs.cpu().numpy()
        act.act(key)
        got = venv.actions.cpu().numpy()
        eps = normal_host(key, (B, nu))
    finally:
        prng.set_layout(False)
    a_h, raw_h, lp_h = host_act(harness, policy, mean, std, obs, eps)
    _bits(got, a_h, "actions")
    # raw and log_prob through the training mode's records
    tr_raw = torch.zeros((1, B, nu), device=d)
    tr_lp = torch.zeros((1, B), device=d)
    obs_rec = torch.zeros((2, B, O), device=d)
    z = [torch.zeros((1, B), device=d) for _ in range(3)]
    keys = torch.from_numpy(key.reshape(1, 2).view(np.int32)).to(d)
    ctl = torch.zeros(4, device=d, dtype=torch.int32)
    P = act.plan
    P.act_keys_dev, P.act_ctl_dev, P.act_key_rows = keys.data_ptr(), ctl.data_ptr(), 1
    P.obs_dev, P.raw_dev, P.logp_dev = obs_rec.data_ptr(), tr_raw.data_ptr(), tr_lp.data_ptr()
    P.reward_dev, P.disc_dev, P.trunc_dev = (t.data_ptr() for t in z)
    prng.set_layout(bool(part))
    try:
        ops.ppo_act(P, _lib.PPO_ACT)
        torch.cuda.synchronize()
    finally:
        prng.set_layout(False)
    _bits(tr_raw[0].cpu().numpy(), raw_h, "raw")
    _bits(tr_lp[0].cpu().numpy(), lp_h, "log_prob")
    _bits(obs_rec[0].cpu().numpy(), obs, "recorded obs")
    assert ctl.cpu().tolist() == [1, 1, 0, 0]


def test_records_match_the_vector_env_across_auto_reset():
    tr = _small_trainer("cartpole", episode_length=3)
    S = tr.U * tr.T
    v = tr.venv
    obs, rew, done, trunc = [], [], [], []
    for _ in range(S):
        obs.append(v.obs.cpu().numpy().copy())
        ops.ppo_act(tr.plan, _lib.PPO_ACT)
        ops.vec_step(v.plan)
        rew.append(v.reward.cpu().numpy().copy())
        done.append(v.done.cpu().numpy().copy())
        trunc.append(v.truncation.cpu().numpy().copy())
    obs.append(v.obs.cpu().numpy().copy())
    ops.ppo_act(tr.plan, _lib.PPO_RECORD)
    torch.cuda.synchronize()
    assert np.any(np.array(done) == 1) and np.any(np.array(trunc) == 1), "no auto-reset happened"
    _bits(tr.obs.cpu().numpy(), np.array(obs), "obs")
    _bits(tr.reward.cpu().numpy(), np.array(rew), "reward")
    _bits(tr.disc.cpu().numpy(), 1 - np.array(done), "discount")
    _bits(tr.trunc.cpu().numpy(), np.array(trunc), "truncation")
    assert tr.act_ctl.cpu().tolist() == [0, S, 0, 0]


def test_gae_matches_restatement():
    tr = _small_trainer("halfcheetah", B=20, T=5, batch=300, nmb=2, E=1)   # mb 300: one thread per trajectory, idle threads
    rng = np.random.default_rng(0)
    S, B, T, mb = tr.U * tr.T, tr.B, tr.T, tr.mb
    reward = rng.normal(size=(S, B)).astype(np.float32)
    disc = (rng.uniform(size=(S, B)) > 0.1).astype(np.float32)
    trunc = ((disc == 0) & (rng.uniform(size=(S, B)) > 0.5)).astype(np.float32)
    values = rng.normal(size=(T + 1, mb)).astype(np.float32)
    traj = rng.permutation(tr.U * B)[:mb].astype(np.int32)
    for t, a in ((tr.reward, reward), (tr.disc, disc), (tr.trunc, trunc)):
        t.copy_(torch.from_numpy(a))
    tr.sel.copy_(torch.from_numpy(traj[None]))
    vals = torch.from_numpy(values).cuda()
    tr.mb_ctl[1] = 3
    tr.plan.values_dev = vals.data_ptr()
    ops.ppo_gae(tr.plan)
    torch.cuda.synchronize()
    vs, adv = ppo_ref.gae_kernel_f32(reward, disc, trunc, values, traj, B, T, 1.0, 0.97, 0.95)
    _bits(tr.vs.cpu().numpy(), vs, "vs")
    _bits(tr.adv.cpu().numpy(), adv, "advantages")
    key = tr.keys.loss.reshape(-1, 2)[3]
    _bits(tr.ent_eps.cpu().numpy(), normal_host(key, (T, mb, tr.nu)), "entropy noise")


def test_gae_many_trajectories_per_thread():
    tr = _small_trainer("cartpole", B=1024, T=3, batch=2048, nmb=1, E=1)
    rng = np.random.default_rng(1)
    S, B, T, mb = tr.U * tr.T, tr.B, tr.T, tr.mb
    reward = rng.normal(size=(S, B)).astype(np.float32)
    disc = (rng.uniform(size=(S, B)) > 0.05).astype(np.float32)
    trunc = np.zeros((S, B), np.float32)
    values = rng.normal(size=(T + 1, mb)).astype(np.float32)
    traj = rng.permutation(tr.U * B)[:mb].astype(np.int32)
    for t, a in ((tr.reward, reward), (tr.disc, disc), (tr.trunc, trunc)):
        t.copy_(torch.from_numpy(a))
    tr.sel.copy_(torch.from_numpy(traj[None]))
    vals = torch.from_numpy(values).cuda()
    tr.plan.values_dev = vals.data_ptr()
    ops.ppo_gae(tr.plan)
    torch.cuda.synchronize()
    vs, adv = ppo_ref.gae_kernel_f32(reward, disc, trunc, values, traj, B, T, 1.0, 0.97, 0.95)
    _bits(tr.vs.cpu().numpy(), vs, "vs")
    _bits(tr.adv.cpu().numpy(), adv, "advantages")


def test_obs_stats_against_float64():
    tr = _small_trainer("halfcheetah", B=64, T=5, batch=64, nmb=2)
    rng = np.random.default_rng(2)
    st = (0.0, np.zeros(tr.O), np.zeros(tr.O))
    for k in range(3):
        x = rng.normal(k, 1.0 + k, tr.obs.shape).astype(np.float32)
        tr.obs.copy_(torch.from_numpy(x))
        ops.ppo_obs_stats(tr.plan)
        st, std = ppo_ref.running_update(st, x[:-1])
    torch.cuda.synchronize()
    stat = tr.stat.cpu().numpy()
    assert stat[0] == st[0]
    np.testing.assert_allclose(stat[1:1 + tr.O], st[1], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(tr.mean.cpu().numpy(), st[1], rtol=1.2e-7, atol=1e-12)
    np.testing.assert_allclose(tr.std.cpu().numpy(), std, rtol=1.2e-7)


def test_graph_replay_equals_eager_unroll():
    a, b = _small_trainer("halfcheetah", seed=4), _small_trainer("halfcheetah", seed=4)
    b.capture()
    for _ in range(a.U):
        a.unroll()
        b._unroll_graph.replay()
    torch.cuda.synchronize()
    for name in ("obs", "raw", "logp", "reward", "disc", "trunc"):
        _bits(getattr(a, name).cpu().numpy(), getattr(b, name).cpu().numpy(), name)


def test_training_is_deterministic():
    runs = []
    for _ in range(2):
        tr = _small_trainer("pushT", seed=9)
        tr.capture()
        for _ in range(2):
            tr.training_step()
        ev = tr.evaluate()
        runs.append((tr.theta.detach().cpu().numpy(), tr.std.cpu().numpy(), ev))
    _bits(runs[0][0], runs[1][0], "parameters")
    _bits(runs[0][1], runs[1][1], "obs std")
    assert runs[0][2] == runs[1][2]
    assert np.isfinite(runs[0][0]).all()


def test_short_run_learns():
    curve = []
    cfg = ppo_ref.learn_config(0)
    ppo.train(environment=ppo_ref.LEARN_ENV, progress_fn=lambda n, m: curve.append((n, m["eval/episode_reward"])), **cfg)
    assert [n for n, _ in curve] == [0, cfg["num_timesteps"]]
    assert curve[1][1] > curve[0][1] + LEARN_MARGIN, curve


def test_actor_without_key_table_needs_a_key():
    venv = VecEnv(_env("cartpole"), 2)
    venv.reset(prng.split(prng.PRNGKey(0), 2))
    O, nu = venv.spec.obs_size, venv.spec.nu
    policy, mean, std, _ = random_policy(O, nu, 1)
    actor = ppo.Actor(venv, *(torch.from_numpy(a).cuda() for a in (policy, mean, std)))
    actor.act(prng.PRNGKey(1))
    with pytest.raises(ValueError, match="key"):
        actor.act()
