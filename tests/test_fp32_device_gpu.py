"""The device build of the fp32 math specification (include/mbd_fp32.h, include/mbd_ppo.h, csrc/pk_scalar.cuh) held to float64
on EVERY float32 input its error constants are charged for, and to the host build bit for bit.

The float64 references (tests/xpbd_ref.py, pusht_ref.py, car2d_ref.py, rl_ref.py, mnist_ref.py, bbo_ref.py) charge fixed error
constants to these functions; the kernels run the nvcc build.  A unary fp32 function has at most 2^32 inputs, so the device
evaluates all of those in each charged range beside a float64 reference from CUDA's double libm (mbd_test_sweep) and the
constants become proofs for the build that runs.  atan2 takes two operands: its polynomial and quadrant roundings are swept
exhaustively with a divisor of 1 (the quotient is exact) and the rounding of a general quotient is added analytically.  The
exact division, reciprocal and square root are held bit for bit to the correctly rounded result on their documented domain,
which includes every subnormal and tiny operand the host accepts.
Run with -s to see the measured maxima, their input bits, the planted-mistake margins and the table of what the exact
operations do outside their domain.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
from scipy.special import erfinv

from mbd_b200 import _lib
from tests import bbo_ref, mnist_ref, rl_ref
from tests.conftest import assert_bit_exact
from tests.test_ppo_cpu import harness  # noqa: F401  (the host build of include/mbd_ppo.h)
from tests.xpbd_ref import ATAN2_ULP, COS_ABS_ERR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
f32, f64 = np.float32, np.float64
FLT_MAX = float(np.finfo(f32).max)

# the ops of mbd_test_arith (include/mbd_b200.h)
OP = dict(div=0, rcp=1, sqrt=2, atan2=3, pk_atan2=4, pk_atan2_lo=5, pk_atan2_hi=6, log=7, exp=8, sin=9, cos=10, erfinv=11,
          normal=12, tanh=13, softplus=14, swish=15, pk_rcp=16, pk_div=17, pk_div_nn=18, pk_sqrt=19, pk_rcp_lo=20, pk_rcp_hi=21,
          pk_div_lo=22, pk_div_hi=23, pk_div_nn_lo=24, pk_div_nn_hi=25, pk_sqrt_lo=26, pk_sqrt_hi=27,
          planted_sin=28, planted_exp=29, planted_rcp=30, planted_sqrt=31, planted_div=32, planted_sqrt_noscale=33)
# the metrics of mbd_test_err: ulps of fl(ref), u |ref|, u (1 + |ref|), u, u |x|, exact, atan2 composed with its quotient
ULP, REL, ONEPLUS, ABS, XREL, EXACT, ATANC = range(7)
RCP_OPS = ("rcp", "pk_rcp", "pk_rcp_lo", "pk_rcp_hi")
SQRT_OPS = ("sqrt", "pk_sqrt", "pk_sqrt_lo", "pk_sqrt_hi")
DIV_OPS = ("div", "pk_div", "pk_div_lo", "pk_div_hi")             # any divisor sign
DIV_NN_OPS = ("pk_div_nn", "pk_div_nn_lo", "pk_div_nn_hi")        # divisor >= +0 (atan2_'s |.| / |.|)
# the packed kernel's two-lane rcp_ / div_ / div_nn_ / sqrt_ keep the bare fast path (csrc/pk_scalar.cuh): exact on its domain only
FAST_ONLY = ("pk_rcp_lo", "pk_rcp_hi", "pk_sqrt_lo", "pk_sqrt_hi", "pk_div_lo", "pk_div_hi", "pk_div_nn_lo", "pk_div_nn_hi")

# name: (op, metric, intervals, bound in the metric's unit).  Every float32 of every interval is evaluated.
UNARY = {
    "log": ("log", REL, [(math.exp(-17), 2e6)], rl_ref.LOG_REL),
    "exp": ("exp", REL, [(-87.0, 88.0)], rl_ref.EXP_REL),
    "sin": ("sin", ABS, [(-1200.0, 1200.0)], COS_ABS_ERR / U),
    "cos": ("cos", ABS, [(-1200.0, 1200.0)], COS_ABS_ERR / U),
    "tanh": ("tanh", ONEPLUS, [(-30.0, 30.0)], rl_ref.TANH_ABS),
    "tanh beyond 30": ("tanh", ONEPLUS, [(-FLT_MAX, -30.0), (30.0, FLT_MAX)], rl_ref.TANH_ABS),
    "softplus": ("softplus", ONEPLUS, [(-1e4, 1e4)], rl_ref.SOFTPLUS),
    "swish": ("swish", REL, [(rl_ref.SWISH_CAP, 1e5)], rl_ref.SWISH_REL),
    "swish below the cap": ("swish", XREL, [(-1e5, float(np.nextafter(f32(rl_ref.SWISH_CAP), f32(-np.inf))))],
                            1.01 * math.exp(rl_ref.SWISH_CAP) / U),
}


def b32(x):
    return int(np.asarray(x, f32).view(np.uint32))


def x32(bits):
    return np.asarray(bits, np.uint32).view(f32)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t, off=0):
    return ctypes.c_void_p(t.data_ptr() + off * t.element_size())


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a, f32), device=DEV)


def arith(op, a, b=None):
    """op of mbd_test_arith elementwise; element n-1-i fills the other half of a two-lane op"""
    ta = _dev(a)
    tb = ta if b is None else _dev(b)
    out = torch.empty_like(ta)
    _lib.check(_lib.lib().mbd_test_arith(OP[op], _ptr(ta), _ptr(tb), _ptr(out), ta.numel(), _stream()), "mbd_test_arith")
    return out.cpu().numpy()


def device_err(op, metric, a, b=None):
    ta = _dev(a)
    tb = ta if b is None else _dev(b)
    err = torch.empty(ta.numel(), dtype=torch.float64, device=DEV)
    _lib.check(_lib.lib().mbd_test_err(OP[op], metric, _ptr(ta), _ptr(tb), _ptr(err), ta.numel(), _stream()), "mbd_test_err")
    return err.cpu().numpy()


def span(lo, hi):
    """(first bits, count) of the runs of float32 bit patterns covering [lo, hi]; the two zeros both belong to 0"""
    lo, hi = f32(lo), f32(hi)
    runs = []
    if lo < 0:
        top = hi if hi < 0 else f32(-0.0)
        runs.append((b32(top), b32(lo) - b32(top) + 1))
    if hi >= 0:
        bot = lo if lo > 0 else f32(0.0)
        runs.append((b32(bot), b32(hi) - b32(bot) + 1))
    return runs


def sweep(jobs):
    """jobs: (op, metric, first bits, count, other operand, other first).  Returns per job (largest error, the bits of an input
    reaching it, the number of inputs with a nonzero error, count), all launches queued before one synchronisation"""
    nbs = [min(2048, max(1, -(-c // (256 * 64)))) for _, _, _, c, _, _ in jobs]
    offs = np.concatenate([[0], np.cumsum(nbs)]).astype(np.int64)
    err = torch.empty(int(offs[-1]), dtype=torch.float64, device=DEV)
    bits = torch.empty(int(offs[-1]), dtype=torch.int32, device=DEV)
    cnt = torch.empty(int(offs[-1]), dtype=torch.int32, device=DEV)
    L = _lib.lib()
    for (op, metric, first, count, other, other_first), nb, o in zip(jobs, nbs, offs):
        _lib.check(L.mbd_test_sweep(OP[op], metric, first, count, 1, ctypes.c_float(other), int(other_first), nb,
                                    _ptr(err, int(o)), _ptr(bits, int(o)), _ptr(cnt, int(o)), _stream()), "mbd_test_sweep")
    e, b, c = err.cpu().numpy(), bits.cpu().numpy().view(np.uint32), cnt.cpu().numpy().view(np.uint32).astype(np.int64)
    out = []
    for j, (_, _, _, count, _, _) in enumerate(jobs):
        s = slice(offs[j], offs[j + 1])
        k = int(np.argmax(e[s]))
        out.append((float(e[s][k]), int(b[s][k]), int(c[s].sum()), count))
    return out


def worst(results):
    """the results of several sweeps of one function, merged"""
    e, bits, _, _ = max(results, key=lambda r: r[0])
    return e, bits, sum(r[2] for r in results), sum(r[3] for r in results)


def sweep_unary(op, metric, intervals):
    return worst(sweep([(op, metric, first, count, 0.0, False) for lo, hi in intervals for first, count in span(lo, hi)]))


def _show(title, rows):
    print(f"\n{title}")
    for r in rows:
        print("  " + r)


@pytest.fixture(scope="module")
def unary():
    """every UNARY sweep: name -> (largest error, its input bits, inputs with a nonzero error, inputs)"""
    res = {name: sweep_unary(op, metric, iv) for name, (op, metric, iv, _) in UNARY.items()}
    unit = {ULP: "ulp", REL: "u|ref|", ONEPLUS: "u(1+|ref|)", ABS: "u", XREL: "u|x|"}
    _show("measured maxima of the device build (every float32 of the range)",
          [f"{name:20s} {res[name][0]:10.6g} {unit[UNARY[name][1]]:10s} at x = {float(x32(res[name][1])):>14.9g} (0x{res[name][1]:08x}),"
           f" bound {UNARY[name][3]:.6g}, {res[name][3]} inputs" for name in UNARY])
    return res


def test_unary_exhaustive(unary):
    """log, exp, sin, cos, tanh, softplus and swish within the constants the float64 references charge them, on every float32
    of the charged range"""
    for name, (_, _, _, bound) in UNARY.items():
        e, bits, _, n = unary[name]
        assert n > 0 and e <= bound, f"{name}: {e} > {bound} at 0x{bits:08x}"
    # the same measurements under the other references' constants: bbo's and mnist's relative exp, mnist's log
    assert unary["exp"][0] * U <= bbo_ref.EXP_REL and unary["exp"][0] * U <= mnist_ref.EXP_REL
    assert unary["log"][0] * U <= mnist_ref.LOG_ABS      # |error| <= LOG_ABS max(1, |log x|)


def _atan2_jobs(metric):
    """the 8 octant and sign configurations: (+-t, +-1) and (+-1, +-t) for every float32 t in (0, 1]; the exact zeros are the
    branch cut of the float64 reference and are held to the host build instead (test_atan2_two_d)"""
    jobs, names = [], []
    for swept_first in (True, False):
        for ts in (1, -1):
            for os_ in (1.0, -1.0):
                first = 1 if ts > 0 else 0x80000001
                jobs.append(("atan2", metric, first, b32(1.0), os_, not swept_first))
                t, o = ("t" if ts > 0 else "-t"), ("1" if os_ > 0 else "-1")
                names.append(f"atan2({t}, {o})" if swept_first else f"atan2({o}, {t})")
    return jobs, names


def test_atan2_exhaustive(orc):
    """mbd_atan2f within ATAN2_ULP ulps for every quotient.  With a divisor of 1 the division is exact, so the sweep measures the
    polynomial and the quadrant roundings at every float32 t in (0, 1] in all 8 configurations.  A general (y, x) adds one
    correctly rounded division t = fl(mn / mx), which moves atan by at most u t / (1 + t^2): metric ATANC adds that to the error
    at each t and measures it in ulps of the smallest correctly rounded result the unrounded quotient can have, so the bound
    holds per binade of the result.  (That rounding is correct while the operands lie in the domain of the device division.)"""
    raw_jobs, names = _atan2_jobs(ULP)
    raw = sweep(raw_jobs)
    comp = sweep(_atan2_jobs(ATANC)[0])
    _show("atan2, every t in (0, 1]", [f"{name:16s} {r[0]:.4f} ulp at t = 0x{r[1]:08x}; with the quotient's rounding {c[0]:.4f} ulp"
                                       f" at 0x{c[1]:08x}" for name, r, c in zip(names, raw, comp)])
    for name, c in zip(names, comp):
        assert c[0] <= ATAN2_ULP, f"{name}: {c[0]} ulp at 0x{c[1]:08x}"
    # the device equals the host build at every reported maximum
    for (_, _, _, _, other, of), r, c in zip(raw_jobs, raw, comp):
        t = x32([r[1], c[1]])
        o = np.full(2, other, f32)
        y, x = (o, t) if of else (t, o)
        assert_bit_exact(arith("atan2", y, x), orc.fmap("atan2", y, x), "atan2 at a maximum")


def test_atan2_two_d(orc):
    """2^24 random (y, x) over all four quadrants with |y / x| from 1e-30 to 1e30: within ATAN2_ULP of float64, equal to the
    host build, and the packed kernel's atan2_ (scalar and both halves of its two-lane form) equal to mbd_atan2f"""
    rng = np.random.default_rng(11)
    n = 1 << 24
    x = (10.0 ** rng.uniform(-3, 3, n)) * rng.choice([-1.0, 1.0], n)
    y = np.abs(x) * 10.0 ** rng.uniform(-30, 30, n) * rng.choice([-1.0, 1.0], n)
    x, y = x.astype(f32), y.astype(f32)
    got = arith("atan2", y, x)
    ref = np.arctan2(y.astype(f64), x.astype(f64))
    ar = np.abs(ref.astype(f32))
    ulp = (np.nextafter(ar, f32(np.inf)) - ar).astype(f64)
    e = np.abs(got - ref) / ulp
    print(f"\natan2 2-D: {e.max():.4f} ulp at (y, x) = ({y[e.argmax()]!r}, {x[e.argmax()]!r}) over {n} pairs")
    assert e.max() <= ATAN2_ULP
    assert_bit_exact(got, orc.fmap("atan2", y, x), "atan2, device vs host")
    for op in ("pk_atan2", "pk_atan2_lo", "pk_atan2_hi"):
        assert_bit_exact(arith(op, y, x), got, op)
    # the axes and signed zeros, where the float64 reference has its branch cut
    v = f32([0.0, -0.0, 1.0, -1.0, 3e-30, -3e-30, 2.5, -2.5])
    yy, xx = np.repeat(v, v.size), np.tile(v, v.size)
    assert_bit_exact(arith("atan2", yy, xx), orc.fmap("atan2", yy, xx), "atan2 on the axes")


def test_erfinv_and_normal_exhaustive(orc):
    """mbd_bits_to_normal at every one of the 2^23 uniform values it can draw (bits >> 9), and mbd_erfinvf at the u each one
    passes it: bit for bit the host build.  The spec is XLA's single-precision polynomial, so equality with the host is the
    assertion; the accuracy against scipy's float64 erfinv is printed."""
    bits = np.arange(1 << 23, dtype=np.uint32) << 9
    lo = f32(-0.99999994)
    unit = ((bits >> 9) | 0x3f800000).view(f32) - f32(1.0)       # mbd_bits_to_unit
    u = np.maximum(unit * f32(2.0) + lo, lo)
    host_erfinv = orc.fmap("erfinv", u)
    assert_bit_exact(arith("erfinv", u), host_erfinv, "mbd_erfinvf")
    got = arith("normal", bits.view(f32))
    assert_bit_exact(got, f32(1.41421354) * host_erfinv, "mbd_bits_to_normal")
    ref = math.sqrt(2.0) * erfinv(u.astype(f64))
    d = np.abs(got - ref)
    rel = d / (U * np.abs(ref))
    print(f"\nmbd_bits_to_normal vs scipy: {d.max():.4g} absolute at bits 0x{bits[d.argmax()]:08x} (normal {ref[d.argmax()]:.6g}); "
          f"{rel.max():.4f} u|ref| at bits 0x{bits[rel.argmax()]:08x} (normal {ref[rel.argmax()]:.6g})")


def _exact(results, what):
    for name, (e, bits, cnt, n) in results:
        assert cnt == 0, f"{what} {name}: {cnt} of {n} results not correctly rounded; worst {e:.3g} ulp at 0x{bits:08x}"


def test_rcp_exact():
    """every nonzero float32 with |x| <= 2^126, both signs, subnormals included: the device reciprocal and the packed kernel's
    scalar rcp_ are the correctly rounded 1 / x, which is +-inf below the overflow edge near 2^-128; both halves of rcp_'s
    two-lane form are, for every |x| in [2^-101, 2^126]"""
    jobs, names = [], []
    tiny = float(x32(1))
    for op in RCP_OPS:
        lo = 2.0 ** -101 if op in FAST_ONLY else tiny
        for first, count in span(lo, 2.0 ** 126) + span(-(2.0 ** 126), -lo):
            jobs.append((op, EXACT, first, count, 0.0, False))
            names.append(f"{op} from 0x{first:08x}")
    res = sweep(jobs)
    assert sum(r[3] for r in res) == 4 * b32(2.0 ** 126) + 4 * (b32(2.0 ** 126) - b32(2.0 ** -101) + 1)
    _exact(zip(names, res), "rcp")


def test_sqrt_exact():
    """every float32 in [0, FLT_MAX], subnormals included: the device square root and the packed kernel's scalar sqrt_ are the
    correctly rounded sqrt (arguments below 2^-100 through the exact scaling by 2^126); both halves of sqrt_'s two-lane form
    are, for 0 and every x in [2^-101, FLT_MAX]"""
    jobs, names = [], []
    for op in SQRT_OPS:
        for first, count in [(0, 1)] + span(2.0 ** -101 if op in FAST_ONLY else float(x32(1)), FLT_MAX):
            jobs.append((op, EXACT, first, count, 0.0, False))
            names.append(f"{op} from 0x{first:08x}")
    res = sweep(jobs)
    assert sum(r[3] for r in res) == 2 * 0x7f800000 + 2 * (0x7f800000 - b32(2.0 ** -101) + 1)
    _exact(zip(names, res), "sqrt")


def _dividends(rng, n, emin, emax):
    m = rng.integers(0, 1 << 23, n).astype(np.uint32)
    m[:2] = (0, (1 << 23) - 1)
    e = rng.integers(emin, emax + 1, n).astype(np.uint32) + 127
    s = rng.integers(0, 2, n).astype(np.uint32) << 31
    return (s | (e << 23) | m).view(f32)


def _div_jobs(dividends, eb):
    """every divisor mantissa at exponent eb against each dividend: positive and negative divisors for the division that takes
    any sign, positive ones for div_nn_"""
    pos = ((127 + eb) << 23, 1 << 23)
    jobs = []
    for a in dividends:
        for op in DIV_OPS:
            jobs.append((op, EXACT, pos[0], pos[1], float(a), True))
            jobs.append((op, EXACT, pos[0] | 0x80000000, pos[1], float(a), True))
        for op in DIV_NN_OPS:
            jobs.append((op, EXACT, pos[0], pos[1], float(a), True))
    return jobs


def _midpoint_pairs(rng, n):
    """(a, b) with a / b within 2^-40 relative of the midpoint between two adjacent float32 quotients: for an odd 24-bit B and
    an odd r, Q = -r / B mod 2^25 makes Q B + r a multiple of 2^25, so A = (Q B + r) / 2^25 is an integer below 2^24 and
    A / B = Q / 2^25 + r / (2^25 B), where Q / 2^25 (Q odd, 25 bits) is a midpoint"""
    M = np.uint64((1 << 25) - 1)
    B = (rng.integers(1 << 22, 1 << 23, n).astype(np.uint64) << np.uint64(1)) | np.uint64(1)     # odd, 24 bits
    r = rng.choice(np.array([-7, -5, -3, -1, 1, 3, 5, 7], np.int64), n)
    inv = B.copy()                       # Newton's iteration for 1 / B mod 2^25 (B odd): 5 steps double the bits to 32
    for _ in range(5):
        inv = (inv * ((np.uint64(2) - B * inv) & M)) & M
    Q = ((-r).astype(np.uint64) * inv) & M
    ok = Q >= np.uint64(1 << 24)         # the quotient in [1/2, 1): A < B
    B, r, Q = B[ok], r[ok], Q[ok]
    num = Q * B + r.astype(np.uint64)
    assert np.all(num & M == 0)
    A = num >> np.uint64(25)
    ea = rng.integers(-60, 61, A.size)
    eb = rng.integers(-60, 61, A.size)
    s = rng.choice(np.array([-1.0, 1.0]), A.size)
    a = (s * np.ldexp(A.astype(f64), ea - 23)).astype(f32)
    b = np.ldexp(B.astype(f64), eb - 23).astype(f32)
    mid = np.ldexp(Q.astype(f64), ea - eb - 25)
    assert np.all(np.abs(np.abs(a.astype(f64) / b) / mid - 1.0) < 2.0 ** -40)
    return a, b


def test_div_exact():
    """the device division, the packed kernel's scalar div_ and div_nn_ and both halves of their two-lane forms are the correctly
    rounded quotient: every divisor mantissa against 1024 dividends, zero dividends of both signs, quotients constructed next to
    rounding midpoints, and the edges of the domain (0 < |divisor| <= 2^126, the quotient 0 or normal): divisors and dividends
    below 2^-100, which take the exact scaling by 2^64, down to every subnormal (test_div_tiny_operands)."""
    rng = np.random.default_rng(12)
    res = sweep(_div_jobs(np.concatenate([_dividends(rng, 1024, -20, 20), f32([0.0, -0.0])]), 0))
    assert len(res) == 1026 * 11
    _exact((("mantissas", r) for r in res), "div")
    # the exponent edges: (divisor exponent, dividend exponent) with the divisor at 2^-101 or 2^125, the dividend at 2^-101, or
    # the quotient near 2^126 or 2^-126
    for eb, ea in ((-101, 25), (-101, 0), (-101, -101), (125, 0), (0, -101), (24, -101), (0, 126)):
        _exact(((f"divisor 2^{eb}, dividend 2^{ea}", r) for r in sweep(_div_jobs(_dividends(rng, 16, ea, ea), eb))), "div")
    a = _dividends(rng, 4096, 0, 127)
    for b in (2.0 ** 126, -(2.0 ** 126), 2.0 ** -101, -(2.0 ** -101)):
        bb = np.full(a.size, b, f32)
        aa = a * f32(2.0 ** -101) if abs(b) < 1 else a                 # dividend >= 2^-101, quotient normal and finite
        for op in DIV_OPS + (DIV_NN_OPS if b > 0 else ()):
            assert_bit_exact(arith(op, aa, bb), aa / bb, f"{op}, divisor {b}")
    a, b = _midpoint_pairs(rng, 1 << 21)
    for op in DIV_OPS:
        assert_bit_exact(arith(op, a, b), a / b, f"{op} next to midpoints")
        assert_bit_exact(arith(op, a, -b), a / -b, f"{op} next to midpoints, negative divisor")
    for op in DIV_NN_OPS:
        assert_bit_exact(arith(op, a, b), a / b, f"{op} next to midpoints")
    print(f"\ndivision: {1026 * 11 + 5 * 16 * 11} divisor-mantissa sweeps and {a.size} near-midpoint quotients per op correctly rounded")


def _div_tiny_jobs():
    """(name, job) of every op of the division on sweeps with an operand below 2^-100: (sweep, first bits, count, other operand,
    other first), expanded over the ops (div_nn_ only where the divisor is positive)"""
    t = lambda e, m=1.0: float(f32(m) * f32(2.0 ** e))   # noqa: E731
    specs = [
        ("every subnormal divisor, dividend 1e-30", 1, 0x7fffff, 1e-30, True),
        ("every subnormal divisor, dividend 1.3 2^-140", 1, 0x7fffff, t(-140, 1.3), True),
        ("every subnormal divisor, dividend 0.75 (overflow below ~2^-127)", 1, 0x7fffff, 0.75, True),
        ("divisors in [2^-126, 2^-101), dividend -1.7 2^-110", 0x00800000, b32(2.0 ** -101) - 0x00800000, t(-110, -1.7), True),
        ("divisors in [2^-126, 2^-101), dividend 2^-3", 0x00800000, b32(2.0 ** -101) - 0x00800000, 0.125, True),
        ("every subnormal dividend, divisor 2^-30", 1, 0x7fffff, t(-30), False),
        ("every subnormal dividend, divisor -1.3 2^-27", 1, 0x7fffff, t(-27, -1.3), False),
        ("every subnormal dividend, divisor 2^-140", 1, 0x7fffff, t(-140), False),
        ("every subnormal dividend, divisor 1.1 2^-110", 1, 0x7fffff, t(-110, 1.1), False),
        ("dividends in [2^-126, 2^-101), divisor 1", 0x00800000, b32(2.0 ** -101) - 0x00800000, 1.0, False),
        ("dividends in [2^-126, 2^-101), divisor -0.7", 0x00800000, b32(2.0 ** -101) - 0x00800000, -0.7, False),
        ("dividends in [2^-126, 2^-101), divisor 1.5 2^-120", 0x00800000, b32(2.0 ** -101) - 0x00800000, t(-120, 1.5), False),
        ("divisors in [1, 2), dividend 1.3 2^-125", b32(1.0), 1 << 23, t(-125, 1.3), True),
        ("divisors in [1, 2), dividend 1.3 2^-102", b32(1.0), 1 << 23, t(-102, 1.3), True),
        ("divisors in [2^-20, 2^-19), dividend 3 2^-131", b32(2.0 ** -20), 1 << 23, 3 * 2.0 ** -131, True),
    ]
    out = []
    for name, first, count, other, of in specs:
        for sign in (0, 0x80000000) if of else (0,):
            for op in tuple(o for o in DIV_OPS + (DIV_NN_OPS if (sign == 0 if of else other > 0) else ()) if o not in FAST_ONLY):
                out.append((f"{op}: {name}{', negative divisor' if sign else ''}", (op, EXACT, first | sign, count, other, of)))
    return out


def test_div_tiny_operands():
    """divisors and dividends below 2^-101, subnormals included, wherever the quotient is normal (or overflows for a subnormal
    divisor): the device division and the packed kernel's scalar div_ and div_nn_ are correctly rounded through the exact
    scaling by 2^64"""
    jobs = _div_tiny_jobs()
    res = sweep([j for _, j in jobs])
    _exact(zip([n for n, _ in jobs], res), "div")
    print(f"\ndivision with tiny operands: {sum(r[3] for r in res)} quotients correctly rounded")


def test_exact_ops_outside_their_domain():
    """What the exact operations do outside the documented domain (reciprocals and quotients in the subnormal range under the
    .ftz seed, divisors above 2^126), and the packed kernel's two-lane rcp_ / div_ / sqrt_ / atan2_ below 2^-101: recorded, not
    asserted"""
    rows = [
        ("rcp, |x| in (2^126, FLT_MAX]: 1 / x subnormal", "rcp", b32(2.0 ** 126) + 1, 0x7f7fffff - b32(2.0 ** 126), 0.0, False),
        ("div 1 / b, b in (2^126, FLT_MAX]", "div", b32(2.0 ** 126) + 1, 0x7f7fffff - b32(2.0 ** 126), 1.0, True),
        ("div 2^-120 / b, b in [2^10, 2^11): quotient subnormal", "div", b32(1024.0), 1 << 23, 2.0 ** -120, True),
        ("div a / 2^20, a subnormal: quotient subnormal", "div", 1, 0x7fffff, 2.0 ** 20, False),
    ] + [(f"{op}, x subnormal (bare fast path)", op, 1, 0x7fffff, 0.0, False) for op in FAST_ONLY if "div" not in op] + [
        (f"{op}, x in [2^-126, 2^-101) (bare fast path)", op, 0x00800000, b32(2.0 ** -101) - 0x00800000, 0.0, False)
        for op in FAST_ONLY if "div" not in op] + [
        (f"{op} 1e-30 / b, b subnormal (bare fast path)", op, 1, 0x7fffff, 1e-30, True) for op in FAST_ONLY if "div" in op] + [
        (f"{op} 1.3 2^-110 / b, b in [1, 2) (bare fast path)", op, b32(1.0), 1 << 23, float(f32(1.3) * f32(2.0 ** -110)), True)
        for op in FAST_ONLY if "div" in op]
    res = sweep([(op, EXACT, first, count, other, of) for _, op, first, count, other, of in rows])
    # the two-lane atan2_ divides with the bare div_nn_: against mbd_atan2f on (y, x) with both magnitudes in one band
    rng = np.random.default_rng(16)
    lanes = []
    for band, (lo, hi) in (("subnormal", (1, 0x7fffff)), ("[2^-126, 2^-101)", (0x00800000, b32(2.0 ** -101) - 1))):
        y, x = (rng.integers(lo, hi + 1, 1 << 16).astype(np.uint32).view(f32) * rng.choice(f32([-1, 1]), 1 << 16) for _ in range(2))
        ref = arith("atan2", y, x)
        for op in ("pk_atan2_lo", "pk_atan2_hi"):
            got = arith(op, y, x)
            lanes.append(f"{op}, |y| and |x| {band:17s} {np.count_nonzero(~np.isfinite(got)):>6d} of {y.size} not finite, "
                         f"{np.count_nonzero(got.view(np.uint32) != ref.view(np.uint32)):>6d} differ from mbd_atan2f")
    _show("exact operations outside their domain (not asserted)",
          [f"{name:56s} {cnt:>10d} of {n:>10d} not correctly rounded, worst {e:.4g} ulp at 0x{bits:08x}"
           for (name, *_), (e, bits, cnt, n) in zip(rows, res)] + lanes)
    assert all(r[3] > 0 for r in res)


def _host(orc, harness, op, x):   # noqa: F811
    if op in ("log", "exp", "sin", "cos"):
        return orc.fmap(op, x)
    x = np.ascontiguousarray(x, f32)
    out = np.zeros_like(x)
    fp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))   # noqa: E731
    harness.ppo_fmap_host(("tanh", "softplus", "swish").index(op), fp(x), x.size, fp(out))
    return out


def strata(intervals, rng, n=1 << 24):
    """bit patterns in the intervals: every one whose low k mantissa bits are zero, with the smallest k that leaves at least n;
    the first two and last two of every binade; and 2^20 uniformly random ones"""
    runs = [r for lo, hi in intervals for r in span(lo, hi)]
    total = sum(c for _, c in runs)
    k = max(0, int(math.floor(math.log2(total / n))))
    out = []
    for first, count in runs:
        last = first + count - 1
        out.append(np.arange(-(-first >> k) << k, last + 1, 1 << k, dtype=np.int64))
        e = np.arange((first & 0x7fffffff) >> 23, ((last & 0x7fffffff) >> 23) + 1, dtype=np.int64)
        edges = ((first & 0x80000000) | (e[:, None] << 23) | np.int64([0, 1, 0x7ffffe, 0x7fffff])).ravel()
        out.append(edges[(edges >= first) & (edges <= last)])
        out.append(first + rng.integers(0, count, max(1, (1 << 20) * count // total)))
    return np.concatenate(out).astype(np.uint32)


def test_device_equals_host(unary, orc, harness):   # noqa: F811
    """the device build equals the host build (oracle/, tests/host_ppo) bit for bit at every measured maximum and on a stratified
    set of at least 2^24 inputs per function"""
    rng = np.random.default_rng(13)
    by_fn = {}
    for name, (op, _, iv, _) in UNARY.items():
        by_fn.setdefault(op, ([], []))
        by_fn[op][0].extend(iv)
        by_fn[op][1].append(unary[name][1])
    for op, (iv, maxima) in by_fn.items():
        bits = np.concatenate([strata(iv, rng), np.uint32(maxima)])
        x = bits.view(f32)
        assert x.size >= 1 << 24
        assert_bit_exact(arith(op, x), _host(orc, harness, op, x), f"{op}, device vs host")


NP_REF = {
    "log": np.log, "exp": np.exp, "sin": np.sin, "cos": np.cos, "tanh": np.tanh,
    "softplus": lambda x: np.where(x > 0, x + np.log1p(np.exp(-np.abs(x))), np.log1p(np.exp(np.minimum(x, 0.0)))),
    "swish": lambda x: x / (1.0 + np.exp(-x)),
}


def np_err(metric, a, b, got, ref):
    """mbd_test_err's metrics in numpy float64"""
    got = got.astype(f64)
    d = np.abs(got - ref)
    if metric in (ULP, ATANC):
        p = 0.0
        if metric == ATANC:
            aa, bb = np.abs(a.astype(f64)), np.abs(b.astype(f64))
            t = np.minimum(aa, bb) / np.maximum(aa, bb)
            p = U * t / (1.0 + t * t) * (1.0 + 1e-6)
        ar = np.abs((np.abs(ref) - p).astype(f32))
        return (d + p) / (np.nextafter(ar, f32(np.inf)) - ar).astype(f64)
    d = np.where(np.abs(ref) < 2.0 ** -126, np.maximum(d - 2.0 ** -149, 0.0), d)
    s = {REL: np.abs(ref), ONEPLUS: 1.0 + np.abs(ref), ABS: np.ones_like(ref), XREL: np.abs(a.astype(f64))}[metric]
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(d == 0, 0.0, d / (U * s))


def test_reference_agrees_with_numpy(unary):
    """the device's float64 reference (CUDA's double libm) gives the errors numpy float64 gives, to 1e-6 of the error plus 1e-7
    of the metric's unit, at every measured maximum and at 1e5 random inputs per function"""
    rng = np.random.default_rng(14)
    for name, (op, metric, iv, _) in UNARY.items():
        runs = [r for lo, hi in iv for r in span(lo, hi)]
        bits = np.concatenate([first + rng.integers(0, count, 100000 // len(runs)) for first, count in runs] + [[unary[name][1]]])
        x = bits.astype(np.uint32).view(f32)
        with np.errstate(over="ignore"):
            en = np_err(metric, x, x, arith(op, x), NP_REF[op](x.astype(f64)))
        ed = device_err(op, metric, x)
        assert np.all(np.abs(ed - en) <= 1e-6 * en + 1e-7), f"{name}: {np.abs(ed - en).max()}"
    jobs, names = _atan2_jobs(ATANC)
    for _, _, first, count, other, of in jobs:
        t = (first + rng.integers(0, count, 100000)).astype(np.uint32).view(f32)
        o = np.full(t.size, other, f32)
        y, x = (o, t) if of else (t, o)
        ref = np.arctan2(y.astype(f64), x.astype(f64))
        got = arith("atan2", y, x)
        for metric in (ULP, ATANC):
            en, ed = np_err(metric, y, x, got, ref), device_err("atan2", metric, y, x)
            assert np.all(np.abs(ed - en) <= 1e-6 * en + 1e-7)


def test_planted_mistakes_fail():
    """each planted mistake (a spec function with one step removed, include/mbd_b200.h ops 28-33) fails the check its function
    passes"""
    sin = sweep_unary("planted_sin", ABS, UNARY["sin"][2])
    exp = sweep_unary("planted_exp", REL, UNARY["exp"][2])
    ex = sweep([("planted_rcp", EXACT, b32(1.0), 1 << 23, 0.0, False), ("planted_sqrt", EXACT, b32(1.0), 1 << 24, 0.0, False),
                ("planted_sqrt_noscale", EXACT, 1, 0x7fffff, 0.0, False)]
               + [("planted_div", EXACT, b32(1.0), 1 << 23, float(a), True) for a in _dividends(np.random.default_rng(15), 16, -20, 20)])
    div = worst(ex[3:])
    rows = [f"sin without its 3rd Cody-Waite constant: {sin[0] * U:.4g} absolute at 0x{sin[1]:08x}, {sin[0] * U / COS_ABS_ERR:.4g} x COS_ABS_ERR",
            f"exp without its 2nd Cody-Waite constant: {exp[0]:.4g} u|ref| at 0x{exp[1]:08x}, {exp[0] / rl_ref.EXP_REL:.4g} x EXP_REL"]
    for what, r in (("rcp as the bare rcp.approx seed", ex[0]), ("sqrt without its final FMA", ex[1]),
                    ("sqrt without the scaling, subnormal x", ex[2]), ("div without the remainder", div)):
        rows.append(f"{what}: {r[2]} of {r[3]} not correctly rounded, worst {r[0]:.4g} ulp at 0x{r[1]:08x}")
    _show("planted mistakes", rows)
    assert sin[0] * U > COS_ABS_ERR and exp[0] > rl_ref.EXP_REL
    assert ex[0][2] > 0 and ex[1][2] > 0 and ex[2][2] > 0 and div[2] > 0
