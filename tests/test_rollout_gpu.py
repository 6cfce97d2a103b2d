"""GPU parity tests proper: the CUDA path (through the C ABI) against the CPU oracle and the
committed golden fixtures.  Bit-exact for everything below the planner statistics."""
import os

import numpy as np
import pytest
import torch

import mbd_b200
from mbd_b200 import ops
from tests.conftest import assert_bit_exact

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
DEV = "cuda:0"


def T(a):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device=DEV)


def N(t):
    return None if t is None else t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def hr(humanoidrun_setup):
    env, blob, st = humanoidrun_setup
    return env, blob, st, env.device_model(torch.device(DEV))


def _actions(rng, n, H, nu, scale=0.88):
    return np.clip(rng.normal(size=(n, H, nu)) * scale, -1, 1).astype(np.float32)


@pytest.fixture(params=[1, 2, 3, 8], ids=["v1-lane-per-link", "v2-cta-bar", "v2-named-bar", "pk-group-bar"])
def variant(request):
    ops.set_kernel_variant(request.param)
    yield request.param
    ops.set_kernel_variant(0)


@pytest.mark.parametrize("n,H,nsub", [(1, 1, 1), (8, 1, 1), (5, 2, 3), (8, 1, 7), (37, 5, 0), (64, 50, 0), (129, 7, 0)])
def test_humanoidrun_rollout_bit_exact(orc, hr, variant, n, H, nsub):
    """per physics step (nsub=1), per env step (H=1) and per rollout; ragged n (not a multiple
    of the samples per CTA), n=1 — for every kernel mapping."""
    env, blob, st, m = hr
    Y = _actions(np.random.default_rng(n * 100 + H), n, H, 17)
    ref = orc.xpbd_rollout(blob, st, Y, want_rewss=True, want_final=True, nsub_override=nsub)
    out = ops.rollout(m, T(st), T(Y), want_rewss=True, want_final=True, nsub_override=nsub)
    assert_bit_exact(N(out["final"]), ref["final"], "final state")
    assert_bit_exact(N(out["rewss"]), ref["rewss"], "rewss")
    assert_bit_exact(N(out["rews"]), ref["rews"], "rews")


def test_humanoidrun_saturated_and_zero_actions(orc, hr, variant):
    env, blob, st, m = hr
    Y = np.zeros((24, 50, 17), np.float32)
    Y[8:16] = 1.0; Y[16:] = -1.0
    Y[3, :, 5] = 37.0  # far outside ctrl_range: actuator clip
    ref = orc.xpbd_rollout(blob, st, Y, want_final=True)
    out = ops.rollout(m, T(st), T(Y), want_final=True)
    assert_bit_exact(N(out["final"]), ref["final"])
    assert_bit_exact(N(out["rews"]), ref["rews"])
    assert np.isfinite(ref["final"]).all()


def test_humanoidrun_golden_fixture(hr, variant):
    """the committed oracle fixture (does not need the oracle library at run time)"""
    env, blob, st, m = hr
    g = np.load(os.path.join(G, "humanoidrun_oracle.npz"))
    assert_bit_exact(st, g["state_init"], "reset state")
    out = ops.rollout(m, T(g["state_init"]), T(g["Y0s"]), want_rewss=True, want_final=True)
    assert_bit_exact(N(out["rews"]), g["rews"]); assert_bit_exact(N(out["rewss"]), g["rewss"])
    assert_bit_exact(N(out["final"]), g["final"])
    # and the in-kernel sampling reproduces the fixture's noise from its key
    Y = ops.sample(g["key"], 8192, 0, 32, 850, float(g["sigma"]), torch.zeros(850, device=DEV))
    assert_bit_exact(N(Y).reshape(32, 50, 17), g["Y0s"], "sampled Y0s")


def test_exact_arith(orc):
    """The branch-free device div / rcp / sqrt (hardware fast path written out, include/mbd_fp32.h) are
    correctly rounded on the operand ranges of the path: bit-equal to IEEE (numpy float32) results."""
    import ctypes
    from mbd_b200 import _lib
    rng = np.random.default_rng(0)
    n = 1 << 22

    def run(op, a, b):
        ta, tb = T(a), T(b)
        out = torch.empty(n, device=DEV)
        _lib.check(_lib.lib().mbd_test_arith(op, ctypes.c_void_p(ta.data_ptr()), ctypes.c_void_p(tb.data_ptr()),
                                             ctypes.c_void_p(out.data_ptr()), n, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
                   "mbd_test_arith")
        return N(out)

    mag = lambda lo, hi: (np.float32(10.0) ** rng.uniform(lo, hi, n).astype(np.float32)) * rng.choice(np.float32([-1, 1]), n)
    a, b = mag(-12, 6), np.abs(mag(-9, 9))
    a[:4096] = 0.0; a[4096:8192] = -0.0                      # zero dividends (normalised zero vectors)
    assert_bit_exact(run(0, a, b), a / b, "div")
    assert_bit_exact(run(0, a, -b), a / -b, "div, negative divisor")
    x = np.abs(mag(-12, 12))
    assert_bit_exact(run(1, x, x), np.float32(1.0) / x, "rcp")
    x = np.abs(mag(-28, 20)); x[:4096] = 0.0
    assert_bit_exact(run(2, x, x), np.sqrt(x), "sqrt")
    y, xx = mag(-6, 3), mag(-6, 3)
    y[:1000] = 0.0; xx[500:1500] = 0.0
    assert_bit_exact(run(3, y, xx), orc.fmap("atan2", y, xx), "atan2 (device division inside)")
    # the packed kernel's atan2_ (div_nn_ inside): scalar, and either half of its two-lane instantiation
    for op, what in ((4, "scalar"), (5, "f2 low half"), (6, "f2 high half")):
        assert_bit_exact(run(op, y, xx), orc.fmap("atan2", y, xx), f"packed atan2_, {what}")


def test_sampling_bit_exact(orc):
    key = np.uint32([0xDEADBEEF, 42])
    rng = np.random.default_rng(0)
    Ybar = (rng.normal(size=850) * 0.2).astype(np.float32)
    for (ntot, b, cnt, hnu) in [(512, 128, 64, 850), (7, 0, 7, 3), (8192, 8000, 192, 850), (33, 5, 11, 80)]:
        got = ops.sample(key, ntot, b, cnt, hnu, 0.7, T(Ybar[:hnu]))
        assert_bit_exact(N(got), orc.sample_Y0s(key, ntot, hnu, 0.7, Ybar[:hnu], b, b + cnt), f"sample {ntot},{b},{cnt},{hnu}")
    assert abs(N(got)).max() <= 1.0


def test_fused_sample_rollout_equals_two_step_and_oracle(orc, hr, variant):
    env, blob, st, m = hr
    key = np.uint32([5, 6]); n_total, n_begin, n_local, H = 4096, 1024, 72, 50
    Ybar = (np.random.default_rng(2).normal(size=850) * 0.1).astype(np.float32)
    Y0s = torch.empty((n_local, 850), device=DEV); rews = torch.empty(n_local, device=DEV)
    ops.sample_rollout(m, T(st), key, n_total, n_begin, n_local, H, 0.5, T(Ybar), Y0s, rews)
    refY = orc.sample_Y0s(key, n_total, 850, 0.5, Ybar, n_begin, n_begin + n_local)
    assert_bit_exact(N(Y0s), refY, "fused Y0s")
    assert_bit_exact(N(rews), orc.xpbd_rollout(blob, st, refY.reshape(n_local, H, 17))["rews"], "fused rews")
    two = ops.rollout(m, T(st), ops.sample(key, n_total, n_begin, n_local, 850, 0.5, T(Ybar)).view(n_local, H, 17))
    assert_bit_exact(N(two["rews"]), N(rews))


def test_humanoidtrack_demo_bit_exact(orc, variant):
    env = mbd_b200.envs.get_env("humanoidtrack")
    st = env.reset(None).pipeline_state.raw
    m = env.device_model(torch.device(DEV))
    g = np.load(os.path.join(G, "humanoidtrack_oracle.npz"))
    assert_bit_exact(st, g["state_init"])
    out = ops.rollout(m, T(st), T(g["Y0s"]), xref=T(env.xref), want_track=True, want_rewss=True)
    assert_bit_exact(N(out["rews"]), g["rews"]); assert_bit_exact(N(out["logpd"]), g["logpd"])
    assert_bit_exact(N(out["track"])[:, ::10], g["track"])
    # against the live oracle, ragged n, horizon 60 (clamped reference index: extension, SURVEY F9)
    Y = _actions(np.random.default_rng(9), 21, 60, 17, 0.6)
    ref = orc.xpbd_rollout(env.blob, st, Y, xref=env.xref, want_rewss=True, want_track=True, want_final=True)
    out = ops.rollout(m, T(st), T(Y), xref=T(env.xref), want_rewss=True, want_track=True, want_final=True)
    for k in ("rews", "rewss", "logpd", "track", "final"):
        assert_bit_exact(N(out[k]), ref[k], k)
    # reward is evaluated on the PRE-step state: the first reward does not depend on the action
    assert np.all(ref["rewss"][:, 0] == ref["rewss"][0, 0])


def test_humanoidstandup_bit_exact(orc, variant):
    """contact-heavy env: 15 plane contacts, up to 5 on one link (capsule end caps + spheres)"""
    env = mbd_b200.envs.get_env("humanoidstandup")
    from mbd_b200 import prng
    st = env.reset(prng.split(prng.PRNGKey(0))[1]).pipeline_state.raw
    m = env.device_model(torch.device(DEV))
    Y = _actions(np.random.default_rng(11), 45, 20, 17, 0.8)
    ref = orc.xpbd_rollout(env.blob, st, Y, want_rewss=True, want_final=True)
    out = ops.rollout(m, T(st), T(Y), want_rewss=True, want_final=True)
    assert_bit_exact(N(out["final"]), ref["final"]); assert_bit_exact(N(out["rewss"]), ref["rewss"])
    assert_bit_exact(N(out["rews"]), ref["rews"])


@pytest.mark.parametrize("v", [1, 2])
def test_generic_model_quadruped_bit_exact(orc, v):
    """A model that is NOT one of the reference humanoids (9 links, root with 4 children, capsule feet): the generic
    kernel instantiations (L != 11) of both mappings agree with the oracle bit for bit."""
    from mbd_b200 import prng
    env = mbd_b200.envs.GenericPositionalEnv(os.path.join(os.path.dirname(__file__), "fixtures", "quadruped.xml"), n_frames=5)
    st = env.reset(prng.split(prng.PRNGKey(3))[1]).pipeline_state.raw
    m = env.device_model(torch.device(DEV))
    Y = _actions(np.random.default_rng(21), 70, 30, 8, 0.7)
    ref = orc.xpbd_rollout(env.blob, st, Y, want_rewss=True, want_final=True)
    ops.set_kernel_variant(v)
    try:
        out = ops.rollout(m, T(st), T(Y), want_rewss=True, want_final=True)
    finally:
        ops.set_kernel_variant(0)
    assert_bit_exact(N(out["final"]), ref["final"]); assert_bit_exact(N(out["rews"]), ref["rews"])
    # and the planner runs on it end to end
    from mbd_b200.planners import engine as eng
    _, alphas, alphas_bar, sigmas = eng.make_schedule(1e-4, 1e-2, 50)
    e = eng.DiffusionEngine(env, 256, 30, 0.1, False, st)
    o, rew = e.reverse_once(np.uint32([1, 2]), float(sigmas[40]), torch.zeros(240, device=DEV), eng.update_coef(alphas, alphas_bar, 40))
    assert np.isfinite(N(o)).all() and np.isfinite(rew.item())


def test_car2d_bit_exact(orc):
    car = mbd_b200.envs.get_env("car2d")
    params, xref = car.device_params()
    rng = np.random.default_rng(4)
    for (n, H) in [(64, 40), (1, 1), (77, 50), (130, 60)]:
        Y = _actions(rng, n, H, 2, 1.2) * 1.5  # includes |u| > 1 (env-side clip)
        ref = orc.car2d_rollout(car.params, car.x0, Y, xref=car.xref, want_rewss=True, want_traj=True)
        out = ops.car2d_rollout(params, T(car.x0), T(Y), xref=xref, want_rewss=True, want_traj=True)
        for k in ("rews", "rewss", "logpd", "traj"):
            assert_bit_exact(N(out[k]), ref[k], f"car2d {k} n={n} H={H}")
    # fused in-kernel sampling
    key = np.uint32([3, 4]); n, H = 64, 40
    Ybar = np.zeros(80, np.float32)
    Y0s = torch.empty((n, H, 2), device=DEV)
    out = ops.car2d_rollout(params, T(car.x0), Y0s, key=key, n_total=256, n_begin=64, sigma=0.63, Ybar=T(Ybar))
    refY = orc.sample_Y0s(key, 256, 80, 0.63, Ybar, 64, 128)
    assert_bit_exact(N(Y0s).reshape(n, 80), refY)
    assert_bit_exact(N(out["rews"]), orc.car2d_rollout(car.params, car.x0, refY.reshape(n, H, 2))["rews"])


def test_full_size_properties(orc, hr, variant):
    """BASELINE size (8192 x 50): oracle-checked slice + size-independent properties."""
    env, blob, st, m = hr
    key = np.uint32([1, 2]); n, H = 8192, 50
    Ybar = torch.zeros(850, device=DEV)
    Y0s = torch.empty((n, 850), device=DEV); rews = torch.empty(n, device=DEV)
    ops.sample_rollout(m, T(st), key, n, 0, n, H, 0.8839, Ybar, Y0s, rews)
    r = N(rews)
    assert np.isfinite(r).all() and r.std() > 0.05
    # (a) random slices agree with the oracle bit for bit
    idx = np.r_[0:16, 4000:4016, 8176:8192]
    ref = orc.xpbd_rollout(blob, st, N(Y0s)[idx].reshape(-1, H, 17))
    assert_bit_exact(r[idx], ref["rews"], "full-size slice")
    # (b) shard invariance: a rank that owns [2048, 4096) of 8192 reproduces the same rows
    Y2 = torch.empty((2048, 850), device=DEV); r2 = torch.empty(2048, device=DEV)
    ops.sample_rollout(m, T(st), key, n, 2048, 2048, H, 0.8839, Ybar, Y2, r2)
    assert_bit_exact(N(Y2), N(Y0s)[2048:4096]); assert_bit_exact(N(r2), r[2048:4096])
    # (c) idempotence / determinism: a second launch reproduces every word
    ops.sample_rollout(m, T(st), key, n, 0, n, H, 0.8839, Ybar, Y0s, rews)
    assert_bit_exact(N(rews), r)
    # (d) rewss.mean(-1) == rews (sequential fp32 mean)
    out = ops.rollout(m, T(st), Y0s[:256].view(256, H, 17), want_rewss=True)
    rs = N(out["rewss"])
    acc = np.zeros(256, np.float32)
    for t in range(H):
        acc = acc + rs[:, t]
    assert_bit_exact(acc / np.float32(H), N(out["rews"]))


def test_argument_errors(hr):
    env, blob, st, m = hr
    from mbd_b200._lib import MbdError
    with pytest.raises(MbdError):
        ops.rollout(m, T(st), torch.zeros((4, 5, 3), device=DEV))            # wrong action width
    with pytest.raises(MbdError):
        ops.rollout(m, torch.as_tensor(st), torch.zeros((4, 5, 17)))         # CPU tensors: no fallback
    with pytest.raises(MbdError):
        ops.sample(np.uint32([1, 2]), 10, 8, 5, 4, 1.0, torch.zeros(4, device=DEV))  # slice past the end


def test_partitionable_threefry_layout_on_the_gpu(orc, hr):
    """compatibility switch for JAX >= 0.5 (mbd_set_prng_layout): the in-kernel sampler and the oracle's implement the same
    [jax-recalled] partitionable layout — fused sampling + rollouts agree bit for bit, and differ from the legacy stream"""
    from mbd_b200 import prng
    env, blob, st, m = hr
    key = np.uint32([12, 34]); n, H = 96, 6
    Yb = torch.zeros(H * 17, device=DEV)
    sti = torch.as_tensor(st, device=DEV)
    Y = torch.empty((n, H * 17), device=DEV); r = torch.empty(n, device=DEV)
    ops.sample_rollout(m, sti, key, n, 0, n, H, 0.7, Yb, Y, r)
    legacy = Y.cpu().numpy().copy()
    try:
        prng.set_layout(True); orc.set_prng_layout(True)
        ops.sample_rollout(m, sti, key, n, 0, n, H, 0.7, Yb, Y, r)
        ref = orc.sample_Y0s(key, n, H * 17, 0.7, np.zeros(H * 17, np.float32))
        assert_bit_exact(Y.cpu().numpy(), ref, "partitionable Y0s")
        out = orc.xpbd_rollout(blob, st, ref.reshape(n, H, 17))
        assert_bit_exact(r.cpu().numpy(), out["rews"], "returns")
    finally:
        prng.set_layout(False); orc.set_prng_layout(False)
    assert not np.array_equal(legacy, Y.cpu().numpy())
