"""Accuracy of the shared fp32 math specification (include/mbd_fp32.h) against float64."""
import numpy as np
from scipy.special import erfinv


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


def test_erfinv(orc):
    u = np.random.default_rng(3).uniform(-1, 1, size=100000).astype(np.float32)
    got, ref = orc.fmap("erfinv", u), erfinv(u.astype(np.float64))
    assert np.max(np.abs(got - ref) / np.maximum(np.abs(ref), 1e-3)) < 1e-6
    edge = np.float32([-0.99999994, 0.99999994, 0.0])
    assert np.isfinite(orc.fmap("erfinv", edge)).all()
