"""Float64 reference of the black-box objectives (upstream mbd/blackbox/mbd_opt.py:34-60) with a derived error bound, a numpy
float32 mirror of k_bbo's documented order (csrc/blackbox.cuh), and a numpy restatement of one whole step.

Error model (that of tests/tail_ref.py): u = 2^-24; every fp32 operation o(a, b) returns o(a, b)(1 + d), |d| <= u.  The bound is a
running error analysis: each intermediate carries its exact-math value v (float64, exact constants pi, 2 pi, e, 0.2, evaluated
at the fp32 inputs Y) and a radius r with |computed - v| <= r:
  add / sub   r = ra + rb + u (|v| + ra + rb)
  mul         r = |a| rb + |b| ra + ra rb + u (|v| + |a| rb + |b| ra + ra rb)
  constant    r = |fp32(c) - c| (fp32(2 pi), fp32(pi), fp32(e), fp32(-0.2); 10, 20, 1, 0.25, 0.5 are exact)
  sin / cos   r = r_arg + SINCOS_ABS (1-Lipschitz, plus the per-call error of mbd_sincosf at an fp32 argument)
  exp         r = e^v (expm1(r_arg) + EXP_REL (1 + expm1(r_arg)))
  sqrt        r = min(ra / sqrt(a), sqrt(ra)) + u (|v| + ...)  (the second, Hoelder, form covers a near 0)
  / n         r = ra / n + u |v|   (n = dim, exact)
  sums        k_bbo's sums have depth k = ceil(dim / 256) - 1 sequential additions per thread plus 8 tree levels: a term passes
              through at most k + 8 roundings, so r_S = sum r_t + gamma_{k+8} sum (|t| + r_t).
The map X = x_min + (x_max - x_min) (Y + 1) / 2 enters through these rules (Y + 1, the product with the span, the exact halving,
the add of x_min).  Arguments reach |2 pi X| <= 10 pi (Rastrigin), |2 pi X| <= 20 pi (Ackley, X in [-5, 10]) and, for Levy
(w in [-0.5, 2]), |pi w + 1| <= 2 pi + 1 and |2 pi w| <= 4 pi; Ackley's exp sees [-2, 0] and [-1, 1].
SINCOS_ABS and EXP_REL are MEASURED, not proven: the largest errors of mbd_sinf / mbd_cosf (absolute, |x| <= 64) and mbd_expf
(relative, [-2.5, 1.5]) over a dense sweep of fp32 arguments through oracle.fmap were 9.2e-8 and 8.2e-8 (1.38 u); the constants
carry a margin over those and tests/test_bbo_ref_cpu.py re-measures them.  SAFETY = 1.01 covers the dropped second-order terms.
"""
from __future__ import annotations

import math

import numpy as np

from tests import tail_ref as tr

f32, f64 = np.float32, np.float64
U = tr.U
SAFETY = tr.SAFETY
SINCOS_ABS = 1.2e-7
EXP_REL = 1.2e-7
THREADS = 256
DOMAINS = {"Ackley": (-5.0, 10.0), "Rastrigin": (-5.0, 5.0), "Levy": (-5.0, 5.0)}
C2PI_F = float(f32(2 * np.pi))
CPI_F = float(f32(np.pi))
E_F = float(f32(np.e))


def sum_depth(dim: int) -> int:
    return max(math.ceil(dim / THREADS) - 1, 0) + int(math.log2(THREADS))


# ---- running error arithmetic --------------------------------------------------------------------------------------------
class R:
    """value v (exact math, float64) and radius r of an fp32 computation of it"""

    def __init__(self, v, r=0.0):
        self.v, self.r = np.asarray(v, f64), np.asarray(r, f64)

    def __add__(self, o):
        o = o if isinstance(o, R) else R(o)
        v = self.v + o.v
        return R(v, self.r + o.r + U * (np.abs(v) + self.r + o.r))

    def __neg__(self):
        return R(-self.v, self.r)

    def __sub__(self, o):
        return self + (-(o if isinstance(o, R) else R(o)))

    def __mul__(self, o):
        o = o if isinstance(o, R) else R(o)
        v = self.v * o.v
        e = np.abs(self.v) * o.r + np.abs(o.v) * self.r + self.r * o.r
        return R(v, e + U * (np.abs(v) + e))

    def half(self):
        return R(self.v * 0.5, self.r * 0.5)


def const(c_exact: float, c_f32: float) -> R:
    return R(c_exact, abs(c_f32 - c_exact))


def r_sin(a: R) -> R:
    return R(np.sin(a.v), a.r + SINCOS_ABS)


def r_cos(a: R) -> R:
    return R(np.cos(a.v), a.r + SINCOS_ABS)


def r_exp(a: R) -> R:
    v = np.exp(a.v)
    m = np.expm1(a.r)
    return R(v, v * (m + EXP_REL * (1 + m)))


def r_sqrt(a: R) -> R:
    v = np.sqrt(np.maximum(a.v, 0.0))
    e = np.minimum(np.where(v > 0, a.r / np.maximum(v, 1e-300), np.inf), np.sqrt(a.r))
    return R(v, e + U * (v + e))


def r_div(a: R, n: float) -> R:
    v = a.v / n
    return R(v, a.r / n + U * np.abs(v))


def r_sum(t: R, depth: int) -> R:
    """sum over the last axis with k_bbo's depth"""
    return R(t.v.sum(-1), t.r.sum(-1) + tr.gamma(depth) * (np.abs(t.v) + t.r).sum(-1))


# ---- the objectives ------------------------------------------------------------------------------------------------------
def _x(Y, x_min, x_max) -> R:
    Y = np.asarray(Y, f32).astype(f64)
    span = R(float(f32(x_max)) - float(f32(x_min)))
    span = R(span.v, U * abs(span.v))
    return R(x_min) + (span * (R(Y) + 1.0)).half()


def reference(fn: str, Y0s, x_min: float, x_max: float):
    """(J64 [N], radius [N]): J = -f(Y) in float64 at the fp32 samples, and the bound on any fp32 evaluation in k_bbo's order"""
    Y = np.asarray(Y0s, f32).reshape(-1, np.shape(Y0s)[-1])
    dim = Y.shape[1]
    depth = sum_depth(dim)
    X = _x(Y, x_min, x_max)
    if fn == "Rastrigin":
        t = X * X - R(10.0) * r_cos(const(2 * np.pi, C2PI_F) * X)
        f = R(10.0 * dim) + r_sum(t, depth)
    elif fn == "Ackley":
        Q = r_sum(X * X, depth)
        C = r_sum(r_cos(const(2 * np.pi, C2PI_F) * X), depth)
        kb = R(-0.2 / math.sqrt(dim), abs(float(f32(-0.2)) - (-0.2)) / math.sqrt(dim) + tr.gamma(2) * 0.2 / math.sqrt(dim))
        part1 = R(-20.0) * r_exp(kb * r_sqrt(Q))
        part2 = -r_exp(r_div(C, float(dim)))
        f = ((part1 + part2) + 20.0) + const(np.e, E_F)
    elif fn == "Levy":
        w = R(1.0) + (X - 1.0) * 0.25
        d = w - 1.0
        p1 = r_sin(const(np.pi, CPI_F) * R(w.v[:, 0], w.r[:, 0]))
        p1 = p1 * p1
        wi, di = R(w.v[:, :-1], w.r[:, :-1]), R(d.v[:, :-1], d.r[:, :-1])
        s = r_sin(const(np.pi, CPI_F) * wi + 1.0)
        t = (di * di) * (R(1.0) + R(10.0) * (s * s))
        wl, dl = R(w.v[:, -1], w.r[:, -1]), R(d.v[:, -1], d.r[:, -1])
        s3 = r_sin(const(2 * np.pi, C2PI_F) * wl)
        p3 = (dl * dl) * (R(1.0) + s3 * s3)
        S = r_sum(t, depth) if dim > 1 else R(np.zeros(Y.shape[0]))
        f = (p1 + S) + p3
    else:
        raise KeyError(fn)
    # the float64 evaluation itself: a few ulps of float64 per term, far below every fp32 radius
    slack = 1e-13 * (np.abs(f.v) + 1.0)
    return -f.v, SAFETY * f.r + slack


# ---- the fp32 mirror of k_bbo's order (numpy; transcendentals through oracle.fmap) ---------------------------------------
def _partials(t, dim):
    """thread tau's running sum over elements tau, tau + 256, ... (onto 0), then the adjacent-pairwise tree over the 256"""
    N = t.shape[0]
    rows = math.ceil(dim / THREADS)
    pad = np.zeros((N, rows * THREADS), f32)
    pad[:, :dim] = t
    acc = np.zeros((N, THREADS), f32)
    for r in range(rows):
        acc = (acc + pad[:, r * THREADS:(r + 1) * THREADS]).astype(f32)
    while acc.shape[1] > 1:
        acc = (acc[:, 0::2] + acc[:, 1::2]).astype(f32)
    return acc[:, 0]


def objective_f32(fn: str, Y0s, x_min: float, x_max: float, fmap, perturb: str = ""):
    """J = -f(Y0s) [N] in k_bbo's fp32 order; fmap = oracle.fmap (mbd_sinf / mbd_cosf / mbd_expf).  `perturb` names a
    deliberate slip the bound must notice: "drop" (the largest term left out), "map" (X mapped onto [x_min, x_max + 1]),
    "cos_x" (cos(X) for cos(2 pi X)), "levy_last" (Levy's last element summed as a middle term)."""
    Y = np.asarray(Y0s, f32).reshape(-1, np.shape(Y0s)[-1])
    N, dim = Y.shape
    span = f32(f32(x_max) - f32(x_min))
    if perturb == "map":
        span = f32(span + f32(1))
    X = (f32(x_min) + (span * (Y + f32(1))).astype(f32) * f32(0.5)).astype(f32)
    c2pi = f32(1) if perturb == "cos_x" else f32(C2PI_F)

    def cos(a):
        return fmap("cos", np.ascontiguousarray(a, f32)).reshape(a.shape)

    def sin(a):
        return fmap("sin", np.ascontiguousarray(a, f32)).reshape(a.shape)

    def exp(a):
        return fmap("exp", np.ascontiguousarray(a, f32)).reshape(a.shape)

    def drop(t):
        if perturb == "drop":
            t = t.copy()
            t[np.arange(N), np.argmax(np.abs(t), axis=1)] = 0
        return t

    if fn == "Rastrigin":
        t = drop((X * X - f32(10) * cos(c2pi * X)).astype(f32))
        f = (f32(10 * dim) + _partials(t, dim)).astype(f32)
    elif fn == "Ackley":
        Q = _partials(drop((X * X).astype(f32)), dim)
        C = _partials(cos(c2pi * X), dim)
        kb = f32(f32(-0.2) / np.sqrt(f32(dim)))
        part1 = (f32(-20) * exp((kb * np.sqrt(Q)).astype(f32))).astype(f32)
        part2 = -exp((C / f32(dim)).astype(f32))
        f = (((part1 + part2).astype(f32) + f32(20)).astype(f32) + f32(E_F)).astype(f32)
    elif fn == "Levy":
        w = (f32(1) + (X - f32(1)) * f32(0.25)).astype(f32)
        d = (w - f32(1)).astype(f32)
        s0 = sin((f32(CPI_F) * w[:, 0]).astype(f32))
        p1 = (s0 * s0).astype(f32)
        s = sin((f32(CPI_F) * w + f32(1)).astype(f32))
        t = ((d * d) * (f32(1) + f32(10) * (s * s))).astype(f32)
        s3 = sin((f32(C2PI_F) * w[:, -1]).astype(f32))
        p3 = ((d[:, -1] * d[:, -1]) * (f32(1) + s3 * s3)).astype(f32)
        if perturb == "levy_last":
            p3 = np.zeros(N, f32)
        else:
            t[:, -1] = 0
        f = ((p1 + _partials(drop(t), dim)).astype(f32) + p3).astype(f32)
    else:
        raise KeyError(fn)
    return (-f).astype(f32)


def check_J(got, J64, rad, what=""):
    got = np.asarray(got, f32).astype(f64)
    err = np.abs(got - J64)
    bad = ~(err <= rad)
    if bad.any():
        n = int(np.argmax(np.where(bad, err / np.maximum(rad, 1e-300), -1.0)))
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.size} values outside their bound; worst n={n}: {got[n]!r} vs "
                             f"{J64[n]!r} (err {err[n]:.3e}, bound {rad[n]:.3e})")


# ---- one whole step, restated on the host ------------------------------------------------------------------------------
def sample(orc, key, sigma: float, mu, init_key, N: int, dim: int):
    """Y0s of one step: clip(normal(key, (N, dim)) * sigma + mean, -1, 1) with the sampler's fp32 arithmetic (product, then sum);
    mean = normal(init_key, (N, dim)) on the first step (mu None), else the row mu"""
    eps = orc.normal(np.asarray(key, np.uint32), (N, dim))
    mean = orc.normal(np.asarray(init_key, np.uint32), (N, dim)) if mu is None else np.asarray(mu, f32)[None]
    return np.clip((eps * f32(sigma)).astype(f32) + mean, f32(-1), f32(1)).astype(f32)


def host_solve(orc, bbo_eval, fn: str, seed: int, N: int, dim: int, Ndiffuse: int, temp: float, sigmas, keys, init_key):
    """the whole solve on the CPU: k_bbo's draws and objective (bit-exact oracles), the MPPI tail in float64
    (tests/tail_ref.py's reference).  Returns ys [Ndiffuse - 1] = Js.max() per step and the final mean."""
    x_min, x_max = DOMAINS[fn]
    mu, ys = None, []
    for t in range(Ndiffuse - 1, 0, -1):
        Y = sample(orc, keys[t], float(sigmas[t]), mu, init_key, N, dim)
        J = bbo_eval(fn, Y, x_min, x_max)
        ys.append(float(J.max()))
        mu = tr.reference(J, temp, Y0s=Y)["Ybar"].astype(f32)
    return np.array(ys), mu
