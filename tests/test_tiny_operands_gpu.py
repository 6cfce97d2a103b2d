"""The kernels at operands below 2^-101: the tiny-operand families (tests/tiny_families.py) through every rollout kernel
(lane-per-link, the warp-per-link CTA and named-barrier kernels, the packed kernel) at n = 1 and at a ragged n, and through the
vector env's per-env step with and without a factor table; k_ppo_act and k_sac_act on observations within each band of their
mean; and mbd_atan2f / the scalar atan2_ on (y, x) pairs in every band.  Each result equals the host build (the CPU oracle, the
host harnesses, the host atan2) bit for bit, lies within the float64 bound, and is finite wherever the float64 reference is."""
import numpy as np
import pytest
import torch

from mbd_b200 import ops
from mbd_b200.blackbox.mbd_mnist import normal_host
from mbd_b200.envs.vec import VecEnv
from oracle import oracle as O
from tests import tiny_families as T
from tests import xpbd_ref as X
from tests.conftest import assert_bit_exact
from tests.test_fp32_device_gpu import arith
from tests.test_ppo_cpu import harness, host_act  # noqa: F401  (harness: the fixture of the host build)
from tests.test_rl_f64_gpu import ppo_act_dev, sac_act_dev
from tests.test_rl_ref_cpu import check_act
from tests.test_sac_cpu import host_act as sac_host_act
from tests.test_sac_cpu import sac_harness  # noqa: F401
from tests.test_tiny_operands_cpu import K, ratio, site_value
from tests.test_xpbd_f64_gpu import launched_kernel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VARIANTS = (1, 2, 3, 8)     # lane-per-link, warp-per-link (CTA, named barriers), packed: every kernel an 11-link model runs


@pytest.fixture(scope="module")
def env(tmp_path_factory):
    return T.make_env(tmp_path_factory.mktemp("tiny"))


def test_the_variants_launch_different_kernels(env):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert {launched_kernel(env.blob, v, n, sms) for v in VARIANTS for n in (1, 77)} == {"lane-per-link", "wpl-cta", "wpl-named",
                                                                                       "pk-group"}


def _check(env, st, u, got, fam, band, what):
    """got [n, L, 13]: finite, the oracle's bits and within K radii of the float64 step"""
    n = u.shape[0]
    states = np.broadcast_to(st, (n,) + st.shape)
    ref = X.positional_step(env.blob, states, u)
    assert T.in_band(site_value(fam, ref), band).all()
    what = f"{what} {fam} {band}"
    assert np.isfinite(got).all(), f"{what}: {np.count_nonzero(~np.isfinite(got))} words not finite"
    want = O.xpbd_rollout(env.blob, st, u[:, None], want_final=True, nsub_override=1)["final"]
    assert_bit_exact(got, want, f"{what}: device vs oracle")
    q = ratio(got, ref, env.blob, states, u)
    assert q <= K, f"{what}: {q:.3g} radii"


def _cases(env, n):
    return [(fam, band, st, u) for fam in T.FAMILIES for band in T.SITE[fam][1] for st, u in T.build(env, fam, band, n)]


def _t(a):
    return torch.as_tensor(np.ascontiguousarray(a, np.float32), device=DEV)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("n", [1, 77])
def test_rollout_kernels_at_tiny_operands(env, variant, n):
    m = env.device_model(torch.device(DEV))
    ops.set_kernel_variant(variant)
    try:
        for fam, band, st, u in _cases(env, n):
            got = ops.rollout(m, _t(st), _t(u[:, None]), want_final=True, nsub_override=1)["final"].cpu().numpy()
            _check(env, st, u, got, fam, band, f"v{variant} n={n}")
    finally:
        ops.set_kernel_variant(0)


@pytest.mark.parametrize("factors", [False, True])
@pytest.mark.parametrize("n", [1, 77])
def test_vector_env_step_at_tiny_operands(env, n, factors):
    """one step of the vector env (one substep: the fixture's n_frames is 1) from the families' states, through the per-env
    rollout kernel, and through its factor-table form with friction and gear factors of 1 (the nominal step, bit for bit)"""
    venv = VecEnv(env, n)
    if factors:
        venv.set_model_factors(friction=np.ones(n), gear=np.ones(n))
    for fam, band, st, u in _cases(env, n):
        venv.set_state(np.broadcast_to(st, (n,) + st.shape))
        got = venv.step(_t(u)).raw.cpu().numpy().reshape(n, *st.shape)
        _check(env, st, u, got, fam, band, f"vec env n={n}{' factors' if factors else ''}")


@pytest.mark.parametrize("kind,B", [("ppo", 1), ("ppo", 33), ("sac", 1), ("sac", 7)])
def test_act_at_tiny_observations(kind, B, harness, sac_harness):   # noqa: F811
    """k_ppo_act / k_sac_act with every observation within each band of its mean (tests/tiny_families.py): finite, the host
    harness's bits, and within K radii of the float64 acting step"""
    for band, case in T.act_cases(kind, B):
        O, nu, pol, mean, std, obs, key = case
        eps = normal_host(key, (B, nu))
        if kind == "ppo":
            got = ppo_act_dev(*case)
            want = host_act(harness, pol, mean, std, obs, eps)
        else:
            act, _ = sac_act_dev(*case)
            want = sac_host_act(sac_harness, pol, mean, std, obs, eps)
            got = (act, want[1], want[2])
        assert np.isfinite(got[0]).all(), f"{kind} {band}: actions not finite"
        assert_bit_exact(got[0], want[0], f"{kind} B={B} {band}: actions vs the host harness")
        for g, w, name in zip(got[1:], want[1:], ("raw", "logp")):
            assert_bit_exact(g, w, f"{kind} B={B} {band}: {name} vs the host harness")
        check_act(kind, case, got, f"B={B} {band}")


ATAN2_OPS = ("atan2", "pk_atan2")


def _band_values(rng, band, n):
    lo, hi = T.BANDS[band]
    if band == "subnormal":
        bits = rng.integers(1, 1 << 23, n).astype(np.uint32)
        v = bits.view(np.float32)
    else:
        v = np.exp2(rng.uniform(np.log2(lo), np.log2(hi), n)).astype(np.float32) if band != "zero" else np.zeros(n, np.float32)
    return v * rng.choice(np.float32([-1.0, 1.0]), n)


@pytest.mark.parametrize("yb", list(T.BANDS))
@pytest.mark.parametrize("xb", list(T.BANDS))
def test_atan2_at_tiny_operands(orc, yb, xb):
    """(y, x) with |y| in one band and |x| in another (every pair of bands, both in the same band among them): mbd_atan2f and
    the scalar atan2_ equal the host build and lie within ATAN2_ULP ulps of float64"""
    rng = np.random.default_rng([list(T.BANDS).index(yb), list(T.BANDS).index(xb)])
    n = 1 << 16
    y, x = _band_values(rng, yb, n), _band_values(rng, xb, n)
    host = orc.fmap("atan2", y, x)
    ref = np.arctan2(y.astype(np.float64), x.astype(np.float64))
    ar = np.abs(ref.astype(np.float32))
    ulp = (np.nextafter(ar, np.float32(np.inf)) - ar).astype(np.float64)
    off_cut = (y != 0) | (x > 0)     # at y = 0, x < 0 float64 has its branch cut (+-pi by the sign of zero): held to the host only
    for op in ATAN2_OPS:
        got = arith(op, y, x)
        assert np.isfinite(got).all(), f"{op}: {np.count_nonzero(~np.isfinite(got))} of {n} not finite"
        assert_bit_exact(got, host, f"{op} vs the host, |y| {yb}, |x| {xb}")
        e = (np.abs(got - ref) / ulp)[off_cut]
        assert e.size == 0 or e.max() <= X.ATAN2_ULP, f"{op}: {e.max():.3g} ulp"
