"""Accuracy of the shared fp32 math specification (include/mbd_fp32.h) against float64."""
import numpy as np
from scipy.special import erfinv

from tests.test_ppo_cpu import harness  # noqa: F401  (the host build of include/mbd_ppo.h, for its composite functions)


def _ulp_err(got, ref):
    ref32 = ref.astype(np.float32)
    ulp = np.spacing(np.abs(ref32)).astype(np.float64)
    return np.max(np.abs(got.astype(np.float64) - ref) / ulp)


def test_atan2(orc):
    """mbd_atan2f within ATAN2_ULP ulps of float64 atan2 — the bound the float64 reference of the positional step
    (tests/xpbd_ref.py) charges every Euler angle — over the operand ranges the Euler extraction produces"""
    from tests.xpbd_ref import ATAN2_ULP
    rng = np.random.default_rng(0)
    f64 = lambda a: a.astype(np.float64)   # noqa: E731
    y = rng.normal(size=100000).astype(np.float32)
    x = rng.normal(size=100000).astype(np.float32)
    assert _ulp_err(orc.fmap("atan2", y, x), np.arctan2(f64(y), f64(x))) <= ATAN2_ULP
    # |y/x| from 1e-30 to 1e30 in all four quadrants, |x| from 1e-3 to 1e3
    n = 400000
    x = (10.0 ** rng.uniform(-3, 3, n)) * rng.choice([-1.0, 1.0], n)
    y = np.abs(x) * 10.0 ** rng.uniform(-30, 30, n) * rng.choice([-1.0, 1.0], n)
    x, y = x.astype(np.float32), y.astype(np.float32)
    assert _ulp_err(orc.fmap("atan2", y, x), np.arctan2(f64(y), f64(x))) <= ATAN2_ULP
    # y = +-x over the whole normal range
    x = ((10.0 ** rng.uniform(-30, 30, n)) * rng.choice([-1.0, 1.0], n)).astype(np.float32)
    for y in (x, -x):
        assert _ulp_err(orc.fmap("atan2", y, x), np.arctan2(f64(y), f64(x))) <= ATAN2_ULP
    # axes: exact
    yy = np.float32([0, 0, 1, -1, 3e-30, -3e-30])
    xx = np.float32([1, -1, 0, 0, 0, 0])
    got = orc.fmap("atan2", yy, xx)
    assert got.tolist() == [0.0, np.float32(np.pi), np.float32(np.pi / 2), -np.float32(np.pi / 2), np.float32(np.pi / 2), -np.float32(np.pi / 2)]
    # signed zeros: the sign tests are `x < 0` and `y < 0`, so a negative zero counts as positive.  atan2(-0, x > 0) is +0
    # (IEEE: -0), atan2(-0, x < 0) is +pi (IEEE: -pi) and atan2(+-0, +-0) is +0 (IEEE: +-0 or +-pi).  The float64 reference
    # treats an exact zero y with x < 0 as the branch cut (both +-pi).
    yy = np.float32([0.0, -0.0, 0.0, -0.0, 0.0, -0.0, 0.0, -0.0])
    xx = np.float32([1.0, 1.0, -1.0, -1.0, 0.0, 0.0, -0.0, -0.0])
    got = orc.fmap("atan2", yy, xx)
    pi = np.float32(np.pi)
    assert got.tolist() == [0.0, 0.0, pi, pi, 0.0, 0.0, 0.0, 0.0]
    assert not np.signbit(got).any()


def test_sincos(orc):
    """mbd_sincosf within COS_ABS_ERR (absolute) of float64 over |x| <= 1200: the bound tests/xpbd_ref.py and
    tests/pusht_ref.py charge every sine and cosine, the latter for slider angles up to 1e3 rad"""
    from tests.xpbd_ref import COS_ABS_ERR
    rng = np.random.default_rng(1)
    for hi in (40.0, 1200.0):
        a = rng.uniform(-hi, hi, size=200000).astype(np.float32)
        assert np.max(np.abs(orc.fmap("sin", a) - np.sin(a.astype(np.float64)))) < COS_ABS_ERR
        assert np.max(np.abs(orc.fmap("cos", a) - np.cos(a.astype(np.float64)))) < COS_ABS_ERR
    # the fp32 neighbours of multiples of pi / 2 (largest reduced argument error) up to 1200
    k = np.arange(-764, 765)
    a = np.concatenate([np.nextafter(np.float32(k * np.pi / 2), d) for d in (np.float32(-np.inf), np.float32(np.inf))])
    a = np.concatenate([a, np.float32(k * np.pi / 2)])
    assert np.max(np.abs(orc.fmap("sin", a) - np.sin(a.astype(np.float64)))) < COS_ABS_ERR
    assert np.max(np.abs(orc.fmap("cos", a) - np.cos(a.astype(np.float64)))) < COS_ABS_ERR


def test_log_exp(orc):
    rng = np.random.default_rng(2)
    l = np.exp(rng.uniform(-17, 5, size=100000)).astype(np.float32)
    assert _ulp_err(orc.fmap("log", l), np.log(l.astype(np.float64))) <= 3.0 or \
        np.max(np.abs(orc.fmap("log", l) - np.log(l.astype(np.float64)))) < 1e-6
    e = rng.uniform(-86.9, 0, size=100000).astype(np.float32)
    assert _ulp_err(orc.fmap("exp", e), np.exp(e.astype(np.float64))) <= 3.0
    assert orc.fmap("exp", np.float32([-100.0, 0.0]))[0] == 0.0
    assert orc.fmap("exp", np.float32([0.0]))[0] == 1.0


def test_exp_positive(orc):
    """mbd_expf on [0, 88] (mbd_tanhf calls it up to 40, mbd_swishf up to 80) within EXP_REL u relative; above 88 the argument
    is clamped, so the result stays at exp(88)'s word instead of overflowing"""
    from tests.rl_ref import EXP_REL
    rng = np.random.default_rng(4)
    e = np.concatenate([rng.uniform(0, 88, 200000), np.linspace(0, 88, 200001), [20.0, 40.0, 80.0]]).astype(np.float32)
    got, ref = orc.fmap("exp", e).astype(np.float64), np.exp(e.astype(np.float64))
    assert np.max(np.abs(got - ref) / ref) <= EXP_REL * 2.0 ** -24
    top = orc.fmap("exp", np.float32([88.0, 88.5, 88.7, 1e4]))
    assert np.all(top == top[0]) and np.isfinite(top).all()


def test_log_scale_range(orc):
    """mbd_logf within LOG_REL u |log x| over the range log(scale) sees: scale = softplus(s) + 0.001 from its floor up to 2e6
    (tests/rl_ref.py), and over [e^-17, e^5]"""
    from tests.rl_ref import LOG_REL
    rng = np.random.default_rng(5)
    x = np.exp(np.concatenate([rng.uniform(np.log(1e-3), np.log(2e6), 300000), rng.uniform(-17, 5, 100000)])).astype(np.float32)
    x = np.concatenate([x, np.float32([1e-3, 1.0, 1e6, 2e6]), np.nextafter(np.float32(1), np.float32([0, 2]))])
    got, ref = orc.fmap("log", x).astype(np.float64), np.log(x.astype(np.float64))
    assert np.all(np.abs(got - ref) <= LOG_REL * 2.0 ** -24 * np.abs(ref))


def _sweep(lo, hi, n, rng):
    return np.concatenate([rng.uniform(lo, hi, n), np.linspace(lo, hi, n)]).astype(np.float32)


def test_rl_composites(harness):
    """mbd_tanhf, mbd_softplusf and mbd_swishf of include/mbd_ppo.h (through the host harness) against float64 over dense sweeps
    and both sides of every cap, with the constants tests/rl_ref.py charges them (DESIGN.md §2)"""
    import ctypes
    from tests.rl_ref import SOFTPLUS, SWISH_CAP, SWISH_REL, TANH_ABS
    u = 2.0 ** -24
    fp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))   # noqa: E731

    def fm(fn, x):
        x = np.ascontiguousarray(x, np.float32)
        out = np.zeros_like(x)
        harness.ppo_fmap_host(fn, fp(x), x.size, fp(out))
        return out.astype(np.float64)

    rng = np.random.default_rng(6)
    near = lambda c: np.concatenate([np.float32(c) + np.float32(c) * np.float32(2.0 ** -23) * np.arange(-64, 65),   # noqa: E731
                                     np.float32(c) + np.linspace(-0.5, 0.5, 4001)]).astype(np.float32)
    # tanh: the cap at |x| = 20 (2|x| = 40) from both sides, and |x| down to 1e-30 where 1 - 2 / (e + 1) has no relative accuracy
    x = np.concatenate([_sweep(-30, 30, 200000, rng), _sweep(-1e-3, 1e-3, 100000, rng), near(20), near(-20),
                        np.float32(10.0 ** -np.arange(1, 31)), -np.float32(10.0 ** -np.arange(1, 31))])
    t = np.tanh(x.astype(np.float64))
    assert np.all(np.abs(fm(0, x) - t) <= TANH_ABS * u * (1 + np.abs(t)))
    assert np.all(fm(0, np.float32([20.0, 25.0, 1e4])) == 1.0)
    # softplus: |x| up to 1e4 and the regimes of log(1 + e): e kept (x > -8), a few bits of it (-17 .. -8), lost (below -17)
    x = np.concatenate([_sweep(-100, 100, 200000, rng), _sweep(-1e4, 1e4, 100000, rng), _sweep(-20, -8, 100000, rng)])
    sp = np.logaddexp(x.astype(np.float64), 0.0)
    assert np.all(np.abs(fm(1, x) - sp) <= SOFTPLUS * u * (1 + sp))
    # swish: relative above the cap at -80, |x| e^-80 below it, both sides of it; |x| up to 1e5
    x = np.concatenate([_sweep(-100, 100, 200000, rng), _sweep(-1e5, 1e5, 100000, rng), near(-80), _sweep(-1, 1, 50000, rng)])
    xd = x.astype(np.float64)
    with np.errstate(over="ignore"):
        sw = xd / (1.0 + np.exp(-xd))
    tol = np.where(xd >= SWISH_CAP, SWISH_REL * u * np.abs(sw), 1.01 * np.abs(xd) * np.exp(SWISH_CAP)) + 2.0 ** -149
    assert np.all(np.abs(fm(2, x) - sw) <= tol)


def test_erfinv(orc):
    u = np.random.default_rng(3).uniform(-1, 1, size=100000).astype(np.float32)
    got, ref = orc.fmap("erfinv", u), erfinv(u.astype(np.float64))
    assert np.max(np.abs(got - ref) / np.maximum(np.abs(ref), 1e-3)) < 1e-6
    edge = np.float32([-0.99999994, 0.99999994, 0.0])
    assert np.isfinite(orc.fmap("erfinv", edge)).all()
