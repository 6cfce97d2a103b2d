"""SAC without a GPU: the acting arithmetic of include/mbd_sac.h (built with g++) against float64, randint's uint32 arithmetic, the
ring against Brax's rolling queue, the hopper row's step accounting, the key chain, the torch fp32 losses and one sgd_step against a
float64 restatement, the ABI's refusals and the CLI errors.

Acting bound (host harness against float64, the same eps): within 2 radii of the float64 contract (tests/rl_ref.py), and
|act - act64| <= 4e-6, |raw - raw64| <= 2e-6 (1 + |raw64|) and
|logp - logp64| <= 1e-4 (1 + |logp64|), the bounds of tests/test_ppo_cpu.py.  The layers are wider here (256 inputs instead of 32)
but ReLU passes errors through without amplification: with weights of lecun scale a unit's accumulated fp32 error stays below
~256 * 2^-24 * sum |x_i w_i|, about 1e-5 relative, and the head's functions are accurate to a few ulp (tests/test_fp32_spec.py).

Loss bound (torch fp32 on CPU against float64 on the same parameters, batch and noise): relative 1e-4 on each loss, and on each
gradient an absolute 1e-4 of the gradient's largest element (sums over 512 rows of fp32 products)."""
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
from mbd_b200.rl import sac, train_brax, train_sac
from tests import sac_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_f32p = ctypes.POINTER(ctypes.c_float)
_u32p = ctypes.POINTER(ctypes.c_uint32)


def _fp(a):
    return a.ctypes.data_as(_f32p)


@pytest.fixture(scope="module")
def sac_harness(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("sac") / "libsac_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "host_sac", "sac_harness.cpp"), "-o", so], check=True,
                   env={**os.environ, "CC": "", "CXX": ""})
    return ctypes.CDLL(so)


def host_act(L, policy, mean, std, obs, eps):
    B, O = obs.shape
    nu = eps.shape[1]
    act, raw, logp = np.zeros((B, nu), np.float32), np.zeros((B, nu), np.float32), np.zeros(B, np.float32)
    arrs = [np.ascontiguousarray(a, np.float32) for a in (policy, mean, std, obs, eps)]
    L.sac_act_host(*[_fp(a) for a in arrs], B, O, nu, _fp(act), _fp(raw), _fp(logp))
    return act, raw, logp


def random_policy(O, nu, seed, n=64):
    rng = np.random.default_rng(seed)
    sizes = nets.sac_policy_sizes(O, nu)
    layers = nets.unflatten(nets.init_params(prng.PRNGKey(seed), sizes).copy(), sizes)
    for W, b in layers:
        b[:] = rng.normal(0, 0.3, b.shape)
    mean = rng.normal(0, 1, O).astype(np.float32)
    std = rng.uniform(0.2, 3.0, O).astype(np.float32)
    obs = (mean + std * rng.normal(0, 1.5, (n, O))).astype(np.float32)
    return nets.flatten(layers), mean, std, obs


# ---- the acting arithmetic -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("O,nu", [(4, 1), (12, 3), (17, 6), (27, 8), (47, 17), (128, 32)])
def test_host_harness_against_float64(sac_harness, O, nu):
    policy, mean, std, obs = random_policy(O, nu, O + nu)
    assert policy.size == nets.num_params(nets.sac_policy_sizes(O, nu))
    eps = normal_host(prng.PRNGKey(O), (obs.shape[0], nu))
    act, raw, logp = host_act(sac_harness, policy, mean, std, obs, eps)
    a64, r64, l64 = sac_ref.policy_act64(policy.astype(np.float64), mean.astype(np.float64), std.astype(np.float64), obs, eps, O, nu)
    assert np.abs(act - a64).max() <= 4e-6
    assert np.all(np.abs(raw - r64) <= 2e-6 * (1 + np.abs(r64)))
    assert np.all(np.abs(logp - l64) <= 1e-4 * (1 + np.abs(l64)))
    # the float64 contract (tests/rl_ref.py, DESIGN.md §2): every word within 2 radii of the reference, whose values are
    # the restatement's
    from tests import rl_ref
    b = rl_ref.act("sac", policy, mean, std, obs, eps, O, nu)
    for got, want, w64 in ((act, b["act"], a64), (raw, b["raw"], r64), (logp, b["logp"], l64)):
        np.testing.assert_allclose(want.v, w64, rtol=1e-9, atol=1e-9)
        assert rl_ref.ratio(got, want).max() <= 2.0


def test_hopper_policy_size():
    assert nets.num_params(nets.sac_policy_sizes(12, 3)) == 70662


@pytest.mark.parametrize("part", [0, 1])
def test_host_split_is_prng_split(sac_harness, part):
    old = prng._PARTITIONABLE
    prng._PARTITIONABLE = bool(part)
    try:
        for seed in (0, 7, 123456):
            key = prng.PRNGKey(seed)
            out = np.zeros(4, np.uint32)
            sac_harness.sac_split2_host(ctypes.c_uint32(int(key[0])), ctypes.c_uint32(int(key[1])), part, out.ctypes.data_as(_u32p))
            assert np.array_equal(out.reshape(2, 2), prng.split(key))
    finally:
        prng._PARTITIONABLE = old


# ---- randint -----------------------------------------------------------------------------------------------------------------------
SPANS = [1, 3, 100_000, 1 << 20, 8192, 1_000_003]


@pytest.mark.parametrize("span", SPANS)
def test_randint_int_equals_uint32(sac_harness, span):
    rng = np.random.default_rng(span)
    hi = rng.integers(0, 1 << 32, 4000, dtype=np.uint64).astype(np.uint32)
    lo = rng.integers(0, 1 << 32, 4000, dtype=np.uint64).astype(np.uint32)
    ref = np.array([sac_ref.randint_int(int(h), int(l), span) for h, l in zip(hi, lo)], np.uint32)
    assert np.array_equal(sac_ref.randint_np(hi, lo, span), ref)
    out = np.zeros(len(hi), np.uint32)
    sac_harness.sac_randint_host(hi.ctypes.data_as(_u32p), lo.ctypes.data_as(_u32p), len(hi), ctypes.c_uint32(span), out.ctypes.data_as(_u32p))
    assert np.array_equal(out, ref)
    assert ref.max() < span


def test_randint_wraps_where_jax_does():
    assert sac_ref.randint_np([0], [0], 1)[0] == 0
    m = 65536 % 100_000
    assert (m * m) % (1 << 32) == 0            # the product wraps to 0: the offset is lo % span
    assert sac_ref.randint_int(12345, 678901, 100_000) == 678901 % 100_000
    assert sac_ref.randint_int(99, 7, 1 << 20) == 7
    assert sac_ref.randint(prng.PRNGKey(0), 10, 5, 5).tolist() == [5] * 10    # maxval <= minval: minval
    assert sac_ref.randint(prng.PRNGKey(0), 10, 5, 3).tolist() == [5] * 10


@pytest.mark.parametrize("span", [3, 8192, 100_000, 1 << 20])
def test_randint_is_uniform(span):
    x = sac_ref.randint(prng.PRNGKey(span), 1 << 18, 0, span)
    assert x.min() >= 0 and x.max() < span
    bins = min(span, 64)
    counts = np.bincount((x * bins) // span, minlength=bins)
    expected = np.array([len(range(-(-(k * span) // bins), -(-((k + 1) * span) // bins))) for k in range(bins)]) * len(x) / span
    assert stats.chisquare(counts, expected).pvalue > 1e-4


# ---- the ring against Brax's queue ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cap,B", [(12, 4), (10, 4), (7, 3), (16, 16), (9, 1)])
def test_ring_equals_rolling_queue(cap, B):
    rng = np.random.default_rng(cap * 100 + B)
    q, r = sac_ref.QueueRef(cap, 3), sac_ref.RingRef(cap, 3)
    n = 0
    for step in range(5 * cap // B + 3):
        upd = np.arange(n, n + B, dtype=np.float32)[:, None] * np.ones(3, np.float32)
        n += B
        q.insert(upd)
        r.insert(upd)
        size = min(n, cap)
        assert q.insert_position - q.sample_position == r.size == size
        assert np.array_equal(q.content(), r.rows(np.arange(size)))
        idx = rng.integers(0, size, 50)
        assert np.array_equal(q.take(idx), r.rows(idx))
        assert np.array_equal(q.content()[:, 0], np.arange(n - size, n, dtype=np.float32))    # the last `size` rows, oldest first


# ---- accounting and keys -----------------------------------------------------------------------------------------------------------
def test_hopper_counts():
    cfg = train_sac.sac_config("hopper")
    c = sac.counts(cfg["num_timesteps"], cfg["num_envs"], cfg["min_replay_size"], cfg["num_evals"])
    assert (c.prefill_steps, c.num_evals_after_init, c.steps_per_epoch) == (64, 19, 2692)
    assert c.num_evals_after_init * c.steps_per_epoch == 51148
    assert c.num_evals_after_init * c.steps_per_epoch * cfg["grad_updates_per_step"] == 3273472
    assert c.prefill_env_steps + c.steps_per_epoch * cfg["num_envs"] == 352768           # the first post-init evaluation
    with pytest.raises(ValueError):
        sac.counts(100, 128, 8192, 20)


@pytest.mark.parametrize("part", [0, 1])
def test_split_many_is_split(part):
    old = prng._PARTITIONABLE
    prng._PARTITIONABLE = bool(part)
    try:
        keys = prng.split(prng.PRNGKey(3), 5)
        for num in (1, 2, 4, 7):
            got = sac.split_many(keys, num)
            for i in range(5):
                assert np.array_equal(got[i], prng.split(keys[i], num))
    finally:
        prng._PARTITIONABLE = old


def _sequential_chain(seed, c, B, G, n_eval_envs, T):
    gk, lk = prng.split(prng.PRNGKey(seed))
    lk = sac.fold_in(lk, 0)
    lk, rb_key, env_key, eval_key = prng.split(lk, 4)
    prefill_key, lk = prng.split(lk)
    k = prng.split(prefill_key, 1)[0]
    act = []
    for _ in range(c.prefill_steps):
        k, nxt = prng.split(k)
        act.append(k)
        k = nxt
    noise = []
    for _ in range(c.num_evals_after_init):
        epoch_key, lk = prng.split(lk)
        k = prng.split(epoch_key, 1)[0]
        for _ in range(c.steps_per_epoch):
            k, nxt = prng.split(k)
            exp_key, key = prng.split(k)
            act.append(exp_key)
            row = []
            for _ in range(G):
                key, ka, kc, kp = prng.split(key, 4)
                row.append([ka, kc, kp])
            noise.append(row)
            k = nxt
    return dict(policy=prng.split(gk)[0], q=prng.split(gk)[1], env=prng.split(env_key, B), buffer=prng.split(rb_key, 1)[0],
                act=np.array(act), noise=np.array(noise))


@pytest.mark.parametrize("part", [0, 1])
def test_key_chain_equals_sequential_loop(part):
    old = prng._PARTITIONABLE
    prng._PARTITIONABLE = bool(part)
    try:
        c = sac.counts(4 * 3 + 4 * 5 * 3, 4, 10, 4)
        assert (c.prefill_steps, c.num_evals_after_init, c.steps_per_epoch) == (3, 3, 5)
        K = sac.key_chain(7, c, 4, 6, 5, 9)
        ref = _sequential_chain(7, c, 4, 6, 5, 9)
        assert K.act.shape == (3 + 15, 2) and K.noise.shape == (15, 6, 3, 2)
        assert K.eval_reset.shape == (4, 5, 2) and K.eval_act.shape == (4, 9, 2)
        for name in ("policy", "q", "env", "buffer", "act", "noise"):
            assert np.array_equal(getattr(K, name), ref[name]), name
        assert len({tuple(k) for k in K.noise.reshape(-1, 2)}) == K.noise.size // 2
    finally:
        prng._PARTITIONABLE = old


# ---- the learner -----------------------------------------------------------------------------------------------------------------
def _learner_case(O=5, nu=2, n=512, seed=0):
    rng = np.random.default_rng(seed)
    policy = nets.init_params(prng.PRNGKey(seed), nets.sac_policy_sizes(O, nu))
    q = nets.sac_q_init(prng.PRNGKey(seed + 1), nets.sac_q_sizes(O, nu))
    target = q + rng.normal(0, 0.02, q.shape).astype(np.float32)
    mean = rng.normal(0, 1, O).astype(np.float32)
    std = rng.uniform(0.5, 2.0, O).astype(np.float32)
    R = 2 * O + nu + 3
    rows = np.zeros((n, R), np.float32)
    rows[:, :O] = mean + std * rng.normal(size=(n, O))
    rows[:, O:O + nu] = np.tanh(rng.normal(size=(n, nu)))
    rows[:, O + nu] = rng.normal(size=n)
    rows[:, O + nu + 1] = (rng.uniform(size=n) > 0.1)
    rows[:, O + nu + 2:2 * O + nu + 2] = mean + std * rng.normal(size=(n, O))
    rows[:, 2 * O + nu + 2] = (rows[:, O + nu + 1] == 0) & (rng.uniform(size=n) > 0.5)
    eps = rng.normal(size=(3, n, nu)).astype(np.float32)
    return policy, q, target, np.float32([0.3]), mean, std, rows, eps


def test_q_layout_round_trip():
    O, nu = 5, 2
    sizes = nets.sac_q_sizes(O, nu)
    assert sizes == [(7, 256), (256, 256), (256, 1)]
    flat = np.arange(nets.sac_q_num_params(O, nu), dtype=np.float32)
    layers = nets.sac_q_unflatten(flat, sizes)
    assert layers[0][0].shape == (2, 7, 256) and layers[0][1].shape == (2, 1, 256)
    assert layers[0][0][1, 0, 0] == 7 * 256 and layers[0][1][0, 0, 0] == 2 * 7 * 256
    q = nets.sac_q_init(prng.PRNGKey(0), sizes)
    c0 = nets.init_params(prng.split(prng.PRNGKey(0), 2)[0], sizes)
    assert np.array_equal(nets.sac_q_unflatten(q, sizes)[1][0][0], nets.unflatten(c0, sizes)[1][0])


def test_losses_and_gradients_against_float64():
    O, nu, rs, gamma = 5, 2, 30.0, 0.997
    policy, q, target, la, mean, std, rows, eps = _learner_case(O, nu)
    t = lambda a, g=False: torch.tensor(a, dtype=torch.float32, requires_grad=g)   # noqa: E731
    pol, qq, lat = t(policy, True), t(q, True), t(la, True)
    ls = sac.losses(pol, qq, t(target), lat, t(mean), t(std), t(rows), t(eps), O, nu, rs, gamma)
    g = [torch.autograd.grad(ls[0], lat, retain_graph=True)[0], torch.autograd.grad(ls[1], qq, retain_graph=True)[0],
         torch.autograd.grad(ls[2], pol, retain_graph=True)[0]]
    ref_l, ga, gq, gp = sac_ref.grads64(policy, q, target, la, mean, std, rows, eps, O, nu, rs, gamma)
    for a, b in zip(ls, ref_l):
        assert abs(float(a.detach()) - b) <= 1e-4 * (1 + abs(b)), (float(a.detach()), b)
    for got, ref in zip(g, (ga, gq, gp)):
        assert np.abs(got.numpy() - ref).max() <= 1e-4 * np.abs(ref).max()
    # each loss reaches only its own parameters
    assert torch.autograd.grad(ls[0], [pol, qq], allow_unused=True) == (None, None)
    assert torch.autograd.grad(ls[2], [qq, lat], allow_unused=True) == (None, None)
    assert torch.autograd.grad(ls[1], [pol, lat], allow_unused=True) == (None, None)


def test_sgd_step_against_float64():
    """one Learner.update: Adam's first step is lr * sign(g) wherever |g| is far above eps, so compare there only; the target is
    (1 - tau) target + tau q_new (lerp in fp32)"""
    O, nu, rs, gamma, lr, tau = 5, 2, 30.0, 0.997, 6e-4, 0.005
    policy, q, target, la, mean, std, rows, eps = _learner_case(O, nu, seed=3)
    L = sac.Learner(policy, q, O, nu, lr, rs, gamma, tau, "cpu")
    L.target_q.copy_(torch.from_numpy(target))
    L.log_alpha.data.copy_(torch.from_numpy(la))
    L.update(torch.from_numpy(rows), torch.from_numpy(eps), torch.from_numpy(mean), torch.from_numpy(std))
    _, ga, gq, gp = sac_ref.grads64(policy, q, target, la, mean, std, rows, eps, O, nu, rs, gamma)
    p64, q64, t64, la64 = sac_ref.first_sgd_step64(policy, q, target, la, ga, gq, gp, lr, sac.ALPHA_LEARNING_RATE, tau)
    for got, ref, g in ((L.policy, p64, gp), (L.q, q64, gq), (L.log_alpha, la64, ga)):
        got = got.detach().numpy()
        sure = np.abs(g) > 1e-3 * np.abs(g).max() + 1e-6
        assert sure.mean() > 0.3
        assert np.abs(got[sure] - ref[sure]).max() <= 1e-6 * (1 + np.abs(ref[sure]).max())
    sure = np.abs(gq) > 1e-3 * np.abs(gq).max() + 1e-6
    assert np.abs(L.target_q.numpy()[sure] - t64[sure]).max() <= 1e-6
    # the target moved towards the new Q, not the old: old-Q Polyak would differ by tau * lr
    old = target * (1 - tau) + q * tau
    assert np.abs(L.target_q.numpy()[sure] - old[sure]).min() > 0.5 * tau * lr


# ---- ABI ---------------------------------------------------------------------------------------------------------------------------
def _plan(**kw):
    P = _lib.SacPlan()
    P.B, P.O, P.nu, P.capacity, P.batch, P.updates, P.act_key_rows, P.noise_key_rows = 4, 5, 2, 16, 8, 2, 10, 10
    for name, _ in _lib.SacPlan._fields_:
        if name.endswith("_dev"):
            setattr(P, name, 0x1000)
    for k, v in kw.items():
        setattr(P, k, v)
    return P


REJECT = [(dict(B=0), "B must be"), (dict(B=_lib.VEC_MAX_B + 1), "B must be"), (dict(O=0), "O must be"), (dict(O=129), "O must be"),
          (dict(nu=0), "nu must be"), (dict(nu=33), "nu must be"), (dict(capacity=3), "capacity"),
          (dict(capacity=_lib.SAC_MAX_CAPACITY + 1), "capacity"), (dict(policy_dev=None), "buffer is missing"),
          (dict(ring_dev=None), "buffer is missing"), (dict(act_ctl_dev=None), "buffer is missing")]


@pytest.mark.parametrize("fields,msg", REJECT, ids=[m + "-" + ",".join(f) for f, m in REJECT])
def test_act_rejected_before_cuda(fields, msg):
    L = _lib.lib()
    assert L.mbd_sac_act(ctypes.byref(_plan(**fields)), _lib.SAC_ACT, None) == -1
    assert msg in L.mbd_last_error().decode()


def test_act_unknown_mode():
    L = _lib.lib()
    assert L.mbd_sac_act(ctypes.byref(_plan()), 7, None) == -1
    assert "unknown mode" in L.mbd_last_error().decode()


@pytest.mark.parametrize("fields,msg", [(dict(ring_ctl_dev=None), "buffer is missing"), (dict(env_trunc_dev=None), "buffer is missing"),
                                        (dict(O=200), "O must be")])
def test_record_rejected_before_cuda(fields, msg):
    L = _lib.lib()
    assert L.mbd_sac_record(ctypes.byref(_plan(**fields)), None) == -1
    assert msg in L.mbd_last_error().decode()


@pytest.mark.parametrize("fields,msg", [(dict(batch=0), "batch and updates"), (dict(updates=0), "batch and updates"),
                                        (dict(noise_keys_dev=None), "buffer is missing"), (dict(noise_key_rows=0), "buffer is missing"),
                                        (dict(batch=1 << 24, updates=64), "below 2^31")])
def test_sample_rejected_before_cuda(fields, msg):
    L = _lib.lib()
    assert L.mbd_sac_sample(ctypes.byref(_plan(**fields)), None) == -1
    assert msg in L.mbd_last_error().decode()


def test_abi_sizes_match_ctypes():
    out = (ctypes.c_int32 * 16)()
    n = _lib.lib().mbd_sac_abi_sizes(out, 16)
    P = _lib.SacPlan
    assert list(out[:n]) == [ctypes.sizeof(P), P.noise_key_rows.offset, P.policy_dev.offset, P.env_obs_dev.offset, P.ring_dev.offset,
                             P.eps_dev.offset, _lib.SAC_MAX_CAPACITY, _lib.SAC_HIDDEN]


# ---- CLI ---------------------------------------------------------------------------------------------------------------------------
def test_cli_ppo_env_points_to_train_brax():
    with pytest.raises(SystemExit, match="train_brax"):
        train_sac.main(["--env_name", "halfcheetah"])


def test_train_brax_hopper_points_to_train_sac():
    with pytest.raises(SystemExit, match="train_sac"):
        train_brax.main(["--env_name", "hopper"])


def test_table_is_the_reference_row():
    cfg = train_sac.sac_config("hopper")
    assert cfg["num_timesteps"] == 6_553_600 and cfg["grad_updates_per_step"] == 64 and cfg["max_replay_size"] == 1 << 20
    assert cfg["reward_scaling"] == 30 and cfg["discounting"] == 0.997 and cfg["learning_rate"] == 6e-4 and cfg["seed"] == 1


def test_train_refuses_what_is_not_built():
    with pytest.raises(NotImplementedError):
        sac.train("hopper", 10000, 10, action_repeat=2)
    with pytest.raises(NotImplementedError):
        sac.train("hopper", 10000, 10, deterministic_eval=True)
