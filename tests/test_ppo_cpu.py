"""PPO without a GPU: GAE and the running statistics against hand-built cases, NormalTanh against scipy, the acting arithmetic of
include/mbd_ppo.h (built with g++) against float64, the parameter layout, the reference's table and derived counts, the key chain,
the ABI's refusals and the CLI errors.

Acting bound (host harness against float64, the same eps): within 2 radii of the float64 contract (tests/rl_ref.py), and
|act - act64| <= 4e-6, |raw - raw64| <= 2e-6 (1 + |raw64|) and
|logp - logp64| <= 1e-4 (1 + |logp64|).  The fp32 functions are accurate to a few ulp (tests/test_fp32_spec.py); the sums over up to
128 inputs and the cancellation in 1 - 2 / (exp(2|x|) + 1) near 0 set the rest."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
import torch
from scipy import stats

from mbd_b200 import _lib, prng
from mbd_b200.blackbox.mbd_mnist import normal_host
from mbd_b200.rl import networks as nets
from mbd_b200.rl import ppo, train_brax
from tests import ppo_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_f32p = ctypes.POINTER(ctypes.c_float)


def _fp(a):
    return a.ctypes.data_as(_f32p)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("ppo") / "libppo_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "host_ppo", "ppo_harness.cpp"), "-o", so], check=True,
                   env={**os.environ, "CC": "", "CXX": ""})
    return ctypes.CDLL(so)


def host_act(L, policy, mean, std, obs, eps):
    B, O = obs.shape
    nu = eps.shape[1]
    act, raw, logp = np.zeros((B, nu), np.float32), np.zeros((B, nu), np.float32), np.zeros(B, np.float32)
    arrs = [np.ascontiguousarray(a, np.float32) for a in (policy, mean, std, obs, eps)]
    L.ppo_act_host(*[_fp(a) for a in arrs], B, O, nu, _fp(act), _fp(raw), _fp(logp))
    return act, raw, logp


def random_policy(O, nu, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    p = nets.init_params(prng.PRNGKey(seed), nets.policy_sizes(O, nu))
    layers = nets.unflatten(p.copy(), nets.policy_sizes(O, nu))
    for W, b in layers:
        b[:] = rng.normal(0, 0.3, b.shape) * scale
    flat = nets.flatten(layers)
    mean = rng.normal(0, 1, O).astype(np.float32)
    std = rng.uniform(0.2, 3.0, O).astype(np.float32)
    obs = (mean + std * rng.normal(0, 1.5, (64, O))).astype(np.float32)
    return flat, mean, std, obs


# ---- GAE ---------------------------------------------------------------------------------------------------------------------------
def test_gae_all_truncated_is_zero():
    T, n = 6, 5
    rng = np.random.default_rng(0)
    vs, adv = ppo_ref.compute_gae(np.ones((T, n)), np.zeros((T, n)), rng.normal(size=(T, n)), rng.normal(size=(T, n)),
                                  rng.normal(size=n), 0.95, 0.97)
    assert np.all(adv == 0)


def test_gae_lambda_one_is_discounted_return_minus_value():
    T, n, g = 7, 4, 0.9
    rng = np.random.default_rng(1)
    r, v, boot = rng.normal(size=(T, n)), rng.normal(size=(T, n)), rng.normal(size=n)
    vs, adv = ppo_ref.compute_gae(np.zeros((T, n)), np.zeros((T, n)), r, v, boot, 1.0, g)
    ret = np.zeros((T, n))
    acc = boot
    for t in range(T - 1, -1, -1):
        acc = r[t] + g * acc
        ret[t] = acc
    np.testing.assert_allclose(vs - v, ret - v, atol=1e-12)
    np.testing.assert_allclose(vs, ret, atol=1e-12)


def test_gae_termination_cuts_the_recursion():
    T, n = 6, 3
    rng = np.random.default_rng(2)
    r, v, boot = rng.normal(size=(T, n)), rng.normal(size=(T, n)), rng.normal(size=n)
    term = np.zeros((T, n))
    term[2] = 1.0
    vs, adv = ppo_ref.compute_gae(np.zeros((T, n)), term, r, v, boot, 0.95, 0.99)
    r2 = r.copy()
    r2[3:] += 100.0                   # anything after the termination cannot reach steps 0..2
    vs2, adv2 = ppo_ref.compute_gae(np.zeros((T, n)), term, r2, v, boot, 0.95, 0.99)
    np.testing.assert_array_equal(vs[:3], vs2[:3])
    np.testing.assert_allclose(vs[2], r[2], atol=1e-12)   # terminal step: vs = reward


def test_gae_kernel_order_matches_float64():
    B, T, U, mb = 6, 5, 2, 8
    rng = np.random.default_rng(3)
    S = U * T
    reward = rng.normal(size=(S, B)).astype(np.float32)
    disc = (rng.uniform(size=(S, B)) > 0.1).astype(np.float32)
    trunc = ((disc == 0) & (rng.uniform(size=(S, B)) > 0.5)).astype(np.float32)
    values = rng.normal(size=(T + 1, mb)).astype(np.float32)
    traj = rng.permutation(U * B)[:mb]
    vs32, adv32 = ppo_ref.gae_kernel_f32(reward, disc, trunc, values, traj, B, T, 2.0, 0.97, 0.95)
    u, b = traj // B, traj % B
    rows = (u * T)[None, :] + np.arange(T)[:, None]
    tr = trunc[rows, b].astype(np.float64)
    vs, adv = ppo_ref.compute_gae(tr, (1 - disc[rows, b]) * (1 - tr), 2.0 * reward[rows, b].astype(np.float64),
                                  values[:T].astype(np.float64), values[T].astype(np.float64), 0.95, 0.97)
    np.testing.assert_allclose(vs32, vs, atol=1e-5)
    np.testing.assert_allclose(adv32, ppo_ref.normalize_advantage(adv), atol=1e-4)


# ---- statistics, distribution ----------------------------------------------------------------------------------------------------
def test_running_statistics_over_batches_equal_one_shot():
    rng = np.random.default_rng(4)
    batches = [rng.normal(3.0, 2.0, (int(k), 5)) for k in (7, 100, 1, 33)]
    st = (0.0, np.zeros(5), np.zeros(5))
    for x in batches:
        st, std = ppo_ref.running_update(st, x)
    allx = np.concatenate(batches)
    assert st[0] == len(allx)
    np.testing.assert_allclose(st[1], allx.mean(0), rtol=1e-12)
    np.testing.assert_allclose(std, allx.std(0), rtol=1e-12)


def test_normal_tanh_against_scipy():
    rng = np.random.default_rng(5)
    loc, s, raw = rng.normal(size=(50, 3)), rng.normal(size=(50, 3)), rng.normal(size=(50, 3)) * 2
    lp, scale = ppo_ref.normal_tanh(loc, s, raw)
    # density of a = tanh(raw): N(raw) / |d tanh / d raw|
    ref = (stats.norm.logpdf(raw, loc, scale) - np.log1p(-np.tanh(raw) ** 2)).sum(-1)
    np.testing.assert_allclose(lp, ref, rtol=1e-9, atol=1e-9)
    eps = rng.normal(size=(50, 3))
    ent = ppo_ref.entropy(loc, s, eps)
    x = eps * scale + loc
    ref_e = (stats.norm.entropy(loc, scale) + np.log1p(-np.tanh(x) ** 2)).sum(-1)
    np.testing.assert_allclose(ent, ref_e, rtol=1e-9, atol=1e-9)
    t = lambda a: torch.from_numpy(a)   # noqa: E731
    logits = t(np.concatenate([loc, s], -1))
    np.testing.assert_allclose(nets.log_prob(logits, t(raw)).numpy(), lp, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(nets.entropy(logits, t(eps)).numpy(), ent, rtol=1e-12, atol=1e-12)


# ---- the acting arithmetic (host harness of include/mbd_ppo.h) -------------------------------------------------------------------
@pytest.mark.parametrize("O,nu", [(4, 1), (16, 2), (17, 6), (27, 8), (47, 17), (128, 32)])
def test_host_harness_against_float64(harness, O, nu):
    policy, mean, std, obs = random_policy(O, nu, O + nu)
    eps = normal_host(prng.PRNGKey(O), (obs.shape[0], nu))
    act, raw, logp = host_act(harness, policy, mean, std, obs, eps)
    a64, r64, l64 = ppo_ref.policy_act64(policy.astype(np.float64), mean.astype(np.float64), std.astype(np.float64), obs, eps, O, nu)
    assert np.abs(act - a64).max() <= 4e-6
    assert np.all(np.abs(raw - r64) <= 2e-6 * (1 + np.abs(r64)))
    assert np.all(np.abs(logp - l64) <= 1e-4 * (1 + np.abs(l64)))
    # the float64 contract (tests/rl_ref.py, DESIGN.md §2): every word within 2 radii of the reference, whose values are
    # the restatement's
    from tests import rl_ref
    b = rl_ref.act("ppo", policy, mean, std, obs, eps, O, nu)
    for got, want, w64 in ((act, b["act"], a64), (raw, b["raw"], r64), (logp, b["logp"], l64)):
        np.testing.assert_allclose(want.v, w64, rtol=1e-9, atol=1e-9)
        assert rl_ref.ratio(got, want).max() <= 2.0


@pytest.mark.parametrize("part", [0, 1])
def test_host_eps_is_prng_normal(harness, part):
    B, nu = 33, 6
    key = prng.PRNGKey(11)
    out = np.zeros((B, nu), np.float32)
    harness.ppo_eps_host(ctypes.c_uint32(int(key[0])), ctypes.c_uint32(int(key[1])), B, nu, part, _fp(out))
    old = prng._PARTITIONABLE
    prng._PARTITIONABLE = bool(part)
    try:
        ref = normal_host(key, (B, nu))
    finally:
        prng._PARTITIONABLE = old
    assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))


# ---- layout, table, counts, keys -------------------------------------------------------------------------------------------------
def test_parameter_layout_round_trip():
    O, nu = 17, 6
    sizes = nets.policy_sizes(O, nu)
    assert sizes == [(17, 32), (32, 32), (32, 32), (32, 32), (32, 12)]
    flat = np.arange(nets.num_params(sizes), dtype=np.float32)
    layers = nets.unflatten(flat, sizes)
    assert np.array_equal(nets.flatten(layers), flat)
    assert layers[0][0][1, 0] == 32 and layers[0][1][0] == 17 * 32    # W1 is [in][out], its bias follows it
    assert nets.value_sizes(O) == [(17, 256)] + [(256, 256)] * 4 + [(256, 1)]
    p = nets.init_params(prng.PRNGKey(0), sizes)
    for (i, o), (W, b) in zip(sizes, nets.unflatten(p, sizes)):
        assert np.all(b == 0) and np.abs(W).max() <= math.sqrt(3.0 / i) and W.std() > 0.4 * math.sqrt(1.0 / i)
    with pytest.raises(ValueError):
        nets.unflatten(flat[:-1], sizes)


# Brax's step accounting for the reference's table: U, env steps per training step, training steps per epoch
EXPECTED = {"ant": (16, 327680, 34), "walker2d": (8, 327680, 9), "halfcheetah": (8, 327680, 9), "pusher": (4, 245760, 11),
            "pushT": (8, 327680, 34), "humanoidrun": (16, 327680, 34), "humanoidstandup": (16, 491520, 11)}


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_table_and_counts(name):
    cfg = train_brax.ppo_config(name)
    assert cfg["normalize_observations"] and cfg["action_repeat"] == 1
    c = ppo.counts(cfg["num_timesteps"], cfg["num_envs"], cfg["batch_size"], cfg["num_minibatches"], cfg["unroll_length"], cfg["num_evals"])
    assert (c.U, c.env_steps_per_training_step, c.steps_per_epoch) == EXPECTED[name]
    assert c.num_evals_after_init == cfg["num_evals"] - 1
    assert cfg["batch_size"] <= _lib.PPO_MAX_MB


def test_counts_edge_cases():
    assert ppo.counts(1000, 4, 4, 2, 5, 1).num_evals_after_init == 1
    with pytest.raises(ValueError):
        ppo.counts(1000, 3, 4, 2, 5, 1)


def test_key_chain_shapes_and_links():
    c = ppo.counts(2 * 4 * 3 * 2, 4, 4, 2, 3, 3)
    assert (c.U, c.steps_per_epoch, c.num_evals_after_init) == (2, 1, 2)
    K = ppo.key_chain(5, c, 4, 3, 2, 2, 6, 7)
    assert K.env.shape == (4, 2) and K.act.shape == (2, 6, 2) and K.perm.shape == (2, 3, 2, 2) and K.loss.shape == (2, 4, 2)
    assert K.eval_reset.shape == (3, 6, 2) and K.eval_act.shape == (3, 7, 2)
    gk, lk = prng.split(prng.PRNGKey(5))
    lk = ppo.fold_in(lk, 0)
    lk, key_env, eval_key = prng.split(lk, 3)
    assert np.array_equal(K.env, prng.split(key_env, 4))
    assert np.array_equal(K.policy, prng.split(gk)[0]) and np.array_equal(K.value, prng.split(gk)[1])
    epoch_key, _ = prng.split2(lk)
    key = prng.split(epoch_key, 1)[0]
    key_sgd, key_unroll, _ = prng.split(key, 3)
    cur = prng.split2(key_unroll)[0]
    assert np.array_equal(K.act[0, 0], prng.split2(cur)[0])
    _, kperm, kgrad = prng.split(key_sgd, 3)
    assert np.array_equal(K.perm[0, 1, 0], prng.split2(kperm)[1])
    assert np.array_equal(K.loss[0, 0], prng.split2(kgrad)[1])
    uk = prng.split2(eval_key)[1]
    assert np.array_equal(K.eval_reset[0], prng.split(uk, 6)) and np.array_equal(K.eval_act[0, 0], prng.split2(uk)[0])
    assert len({tuple(k) for k in K.act.reshape(-1, 2)}) == K.act.shape[0] * K.act.shape[1]


def test_fold_in_is_one_threefry_block():
    k = prng.PRNGKey(42)
    o0, o1 = prng.threefry2x32(k, np.uint32([0]), np.uint32([7]))
    assert np.array_equal(ppo.fold_in(k, 7), np.array([o0[0], o1[0]], np.uint32))


# ---- ABI ---------------------------------------------------------------------------------------------------------------------------
def _plan(**kw):
    P = _lib.PpoPlan()
    P.B, P.O, P.nu, P.slots, P.unroll, P.mb, P.act_key_rows, P.loss_key_rows = 4, 5, 2, 6, 3, 4, 10, 10
    for name, _ in _lib.PpoPlan._fields_:
        if name.endswith("_dev"):
            setattr(P, name, 0x1000)
    for k, v in kw.items():
        setattr(P, k, v)
    return P


REJECT = [(dict(B=0), "B must be"), (dict(B=_lib.VEC_MAX_B + 1), "B must be"), (dict(O=0), "O must be"), (dict(O=129), "O must be"),
          (dict(nu=0), "nu must be"), (dict(nu=33), "nu must be"), (dict(slots=0), "slots"), (dict(policy_dev=None), "buffer is missing"),
          (dict(act_ctl_dev=None), "buffer is missing")]


@pytest.mark.parametrize("fields,msg", REJECT, ids=[m + "-" + ",".join(f) for f, m in REJECT])
def test_act_rejected_before_cuda(fields, msg):
    L = _lib.lib()
    assert L.mbd_ppo_act(ctypes.byref(_plan(**fields)), _lib.PPO_ACT, None) == -1
    assert msg in L.mbd_last_error().decode()


@pytest.mark.parametrize("fields,msg", [(dict(O=200), "O must be"), (dict(stat_dev=None), "buffer is missing")])
def test_obs_stats_rejected_before_cuda(fields, msg):
    L = _lib.lib()
    assert L.mbd_ppo_obs_stats(ctypes.byref(_plan(**fields)), None) == -1
    assert msg in L.mbd_last_error().decode()


@pytest.mark.parametrize("fields,msg", [(dict(mb=0), "mb must be"), (dict(mb=4097), "mb must be"), (dict(unroll=4), "unroll must divide"),
                                        (dict(values_dev=None), "buffer is missing"), (dict(nu=40), "nu must be")])
def test_gae_rejected_before_cuda(fields, msg):
    L = _lib.lib()
    assert L.mbd_ppo_gae(ctypes.byref(_plan(**fields)), None) == -1
    assert msg in L.mbd_last_error().decode()


def test_act_unknown_mode():
    L = _lib.lib()
    assert L.mbd_ppo_act(ctypes.byref(_plan()), 9, None) == -1
    assert "unknown mode" in L.mbd_last_error().decode()


def test_abi_sizes_match_ctypes():
    out = (ctypes.c_int32 * 16)()
    n = _lib.lib().mbd_ppo_abi_sizes(out, 16)
    P = _lib.PpoPlan
    assert list(out[:n]) == [ctypes.sizeof(P), P.reward_scaling.offset, P.policy_dev.offset, P.env_obs_dev.offset, P.stat_dev.offset,
                             P.ent_eps_dev.offset, _lib.PPO_MAX_OBS, _lib.PPO_MAX_NU, _lib.PPO_MAX_MB, _lib.PPO_STAT_ROWS]


# ---- CLI ---------------------------------------------------------------------------------------------------------------------------
def test_cli_hopper_says_sac_is_not_built():
    with pytest.raises(SystemExit, match="SAC"):
        train_brax.main(["--env_name", "hopper"])


def test_cli_pusher_fails_in_get_env():
    with pytest.raises((NotImplementedError, ValueError)):
        train_brax.main(["--env_name", "pusher"])
