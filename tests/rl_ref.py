"""Float64 reference of the RL acting step (PPO and SAC policies with the NormalTanh head), GAE with the advantage normalisation,
and the running observation statistics, with a radius per value (DESIGN.md §2, "Accuracy contract of the RL acting step, GAE and
statistics").

The acting kernels, GAE and their host restatements agree bit for bit because they share one fp32 association order; that says
nothing about whether either computes Brax's formulas.  This module evaluates the formulas in float64 on the same fp32 inputs
(policy words, mean, std, obs, eps, rewards, flags, values) and carries next to every value a first-order bound on how far any
correct fp32 evaluation may lie from it (the running-error arithmetic `R` of tests/xpbd_ref.py).  Error model, u = 2^-24:
* `+ - * /` and `sqrt` round once; a dense unit is gamma_{nin+1} * sum |x w| + |b| (order-free) plus the inputs' radii
  through |W|;
* the project's fp32 functions are charged the constants below, each labelled proven or measured (the measuring test named);
  the propagated radius uses the function's Lipschitz constant on the interval the input may take;
* the head's z = r / scale - loc / scale is evaluated as the map it is: with r = fl(eps scale' + loc') the scale' and loc'
  errors cancel, so |z' - eps| <= u (3|eps| + 2|r / scale| + |loc / scale|) whatever the radii of loc and scale;
* GAE is R arithmetic through Brax's recursion; the normalisation is bounded as tests/tail_ref.py bounds a mean and a std;
* the statistics' float64 sums carry gamma64 * (their magnitudes), then the one fp32 rounding of the stored mean and std.
"""
from __future__ import annotations

import math

import numpy as np

from mbd_b200.rl import networks as nets
from tests.xpbd_ref import ETA, R, U, exact_scale, fsum, gamma

f32 = np.float32

# ---- the fp32 functions (include/mbd_fp32.h, include/mbd_ppo.h) -------------------------------------------------------------
EXP_REL = 2.0          # |mbd_expf(x) / exp(x) - 1| <= EXP_REL u on [-87, 88]; measured 1.51 / 1.44, test_fp32_spec.py::test_log_exp,
                       # ::test_exp_positive
LOG_REL = 2.0          # |mbd_logf(x) - log x| <= LOG_REL u |log x| on [e^-17, 2e6]; measured 1.43, ::test_log_scale_range
TANH_ABS = 2.5         # |mbd_tanhf(x) - tanh x| <= TANH_ABS u (1 + |tanh x|); measured 2.00, ::test_rl_composites.  Absolute:
                       # 1 - 2 / (e + 1) has no relative accuracy near 0
SOFTPLUS = 1.5         # |mbd_softplusf(x) - softplus x| <= SOFTPLUS u (1 + softplus x); measured 1.07, ::test_rl_composites.
                       # Absolute below 0: log(1 + e) keeps e to u only, and loses it below x ~ -17
SWISH_REL = 3.5        # |mbd_swishf(x) - swish x| <= SWISH_REL u |swish x| for x >= -80; measured 2.80, ::test_rl_composites
SWISH_CAP = -80.0      # below it exp(-x) is capped at exp(80): |error| <= 1.01 |x| e^-80 (proven: both are below |x| e^-80 (1 + 4u))
SWISH_LIP = 1.0999     # proven: sup |d/dx x sigma(x)| = 1.0998
HALF_LOG_2PI = 0.5 * math.log(2 * math.pi)
LOG2 = math.log(2.0)
MIN_STD = 0.001
NORM_EPS = float(f32(1e-8))   # the advantage normalisation's 1e-8, as the fp32 word both Brax and the kernel add

V64 = 2.0 ** -53


def gamma64(k) -> float:
    return k * V64 / (1.0 - k * V64)


def _f(x, fn_val, lip, err):
    """a function of an R: value fn(x.v), radius lip * x.r + err(|value| + lip * x.r)"""
    v = fn_val(x.v)
    prop = lip * x.r
    return R(v, prop + err(np.abs(v) + prop) + ETA)


def softplus(x: R) -> R:
    with np.errstate(over="ignore"):
        lip = 1.0 / (1.0 + np.exp(-(x.v + x.r)))
    return _f(x, lambda v: np.logaddexp(v, 0.0), lip, lambda a: SOFTPLUS * U * (1.0 + a))


def tanh(x: R) -> R:
    lip = 1.0 / np.cosh(np.minimum(np.maximum(np.abs(x.v) - x.r, 0.0), 350.0)) ** 2
    return _f(x, np.tanh, lip, lambda a: TANH_ABS * U * (1.0 + a))


def _dswish(x):
    with np.errstate(over="ignore"):
        s = 1.0 / (1.0 + np.exp(-x))
    return s * (1.0 + x * (1.0 - s))


def swish(x: R) -> R:
    """the propagated radius uses the largest |swish'| on [v - r, v + r]: swish' rises from its minimum -0.0998 at -2.3994 to its
    maximum 1.0998 at 2.3994 and is monotone on either side of them, so the end points and those two extremes bound it"""
    lo, hi = x.v - x.r, x.v + x.r
    lip = np.maximum(np.abs(_dswish(lo)), np.abs(_dswish(hi)))
    lip = np.where((lo <= 2.3994) & (hi >= 2.3994), SWISH_LIP, lip)
    lip = np.where((lo <= -2.3994) & (hi >= -2.3994), np.maximum(lip, 0.0999), lip)
    with np.errstate(over="ignore"):
        r = _f(x, lambda v: v / (1.0 + np.exp(-v)), lip * 1.0001, lambda a: SWISH_REL * U * a)
    capped = x.v - x.r < SWISH_CAP
    return R(r.v, r.r + np.where(capped, 1.01 * (np.abs(x.v) + x.r) * math.exp(SWISH_CAP), 0.0))


def relu(x: R) -> R:
    """exactly 0 where the input is surely negative, the input's radius elsewhere"""
    return R(np.maximum(x.v, 0.0), np.where(x.v + x.r < 0, 0.0, x.r))


def log(x: R) -> R:
    lo = x.v - x.r
    with np.errstate(divide="ignore", invalid="ignore"):
        prop = np.where(lo > 0, x.r / np.where(lo > 0, lo, 1.0), np.inf)
        v = np.log(x.v)
    return R(v, prop + LOG_REL * U * (np.abs(v) + prop) + ETA)


def dense(x: R, W, b) -> R:
    """x [n, nin] @ W [nin, nout] + b: the inputs' radii through |W| plus gamma_{nin+1} of every term's magnitude"""
    W, b = np.asarray(W, np.float64), np.asarray(b, np.float64)
    aW = np.abs(W)
    prop = x.r @ aW
    mag = (np.abs(x.v) + x.r) @ aW + np.abs(b)
    k = W.shape[0] + 1
    return R(x.v @ W + b, prop + gamma(k) * (mag + prop) + k * ETA)


def normalize(obs, mean, std) -> R:
    """running_statistics.normalize without clipping, (obs - mean) / std, on fp32 words"""
    return (R(np.asarray(obs, f32)) - R(np.asarray(mean, f32))) / R(np.asarray(std, f32))


# ---- the head ---------------------------------------------------------------------------------------------------------------------
def head(loc: R, s: R, eps):
    """NormalTanh: (raw, tanh(raw), the per-component log_prob term, scale, z) of loc, s [n, nu] and eps [n, nu] (fp32 words)"""
    eps = np.asarray(eps, f32).astype(np.float64)
    sp = softplus(s)
    scale = sp + R(np.full_like(sp.v, MIN_STD), np.full_like(sp.v, U * MIN_STD))
    raw = R(eps) * scale + loc
    # z as the map it is (module docstring): the float64 value is eps exactly
    lo = np.maximum(scale.v - scale.r, 1e-300)
    ar = (np.abs(raw.v) + raw.r) / lo
    al = (np.abs(loc.v) + loc.r) / lo
    zr = 1.01 * U * (3 * np.abs(eps) + 2 * ar + al) + 4 * ETA / lo
    z = R(eps, zr)
    c = R(np.full_like(z.v, HALF_LOG_2PI), np.full_like(z.v, U * HALF_LOG_2PI))
    logpdf = -exact_scale(z * z, 0.5) - (c + log(scale))
    l2 = R(np.full_like(z.v, LOG2), np.full_like(z.v, U * LOG2))
    jac = exact_scale(l2 - raw - softplus(exact_scale(raw, -2.0)), 2.0)
    return raw, tanh(raw), logpdf - jac, scale, z


def sum_last(x: R) -> R:
    """the sum over the action components (any order)"""
    return fsum([R(x.v[:, j], x.r[:, j]) for j in range(x.v.shape[1])])


# ---- the two policies -------------------------------------------------------------------------------------------------------------
def act(kind: str, policy, mean, std, obs, eps, O: int, nu: int) -> dict:
    """the acting step of `kind` ("ppo": O -> 32^4 -> 2 Nu with swish; "sac": O -> 256^2 -> 2 Nu with ReLU) in float64 with radii:
    {act, raw, logp: R, pre: the hidden pre-activations' values}"""
    sizes = nets.policy_sizes(O, nu) if kind == "ppo" else nets.sac_policy_sizes(O, nu)
    layers = nets.unflatten(np.asarray(policy, f32).astype(np.float64), sizes)
    x = normalize(obs, mean, std)
    pre = []
    for l, (W, b) in enumerate(layers):
        x = dense(x, W, b)
        if l + 1 < len(layers):
            pre.append(x.v)
            x = swish(x) if kind == "ppo" else relu(x)
    loc, s = R(x.v[:, :nu], x.r[:, :nu]), R(x.v[:, nu:], x.r[:, nu:])
    raw, a, lp, scale, z = head(loc, s, eps)
    return dict(act=a, raw=raw, logp=sum_last(lp), loc=loc, s=s, scale=scale, z=z, pre=pre)


# ---- GAE --------------------------------------------------------------------------------------------------------------------------
def gae_depth(mb: int, T: int) -> int:
    """k_ppo_gae's reduction: P threads (a power of two from 32 to 1024), ceil(mb / P) * T sequential terms each, log2 P levels"""
    P = 32
    while P < mb and P < 1024:
        P *= 2
    return -(-mb // P) * T + int(math.log2(P))


def gae(reward, disc, trunc, values, reward_scaling, discount, lam):
    """compute_gae of Brax (time-major [T, n] fp32 rollout rows of the minibatch, values [T + 1, n] with the bootstrap in row T)
    with the truncation mask; termination = (1 - discount) (1 - truncation): (vs, advantages) as R"""
    rs, g, lm = (float(f32(a)) for a in (reward_scaling, discount, lam))
    T = reward.shape[0]
    rew = R(np.asarray(reward, f32)) * rs
    tr = R(np.asarray(trunc, f32))
    term = (1.0 - R(np.asarray(disc, f32))) * (1.0 - tr)
    tm = 1.0 - tr
    v = R(np.asarray(values, f32))
    row = lambda x, t: R(x.v[t], x.r[t])   # noqa: E731
    boot = row(v, T)
    acc, vnext = R(np.zeros_like(boot.v)), boot
    vs = [None] * T
    for t in range(T - 1, -1, -1):
        c = g * (1.0 - row(term, t))
        delta = (row(rew, t) + c * vnext - row(v, t)) * row(tm, t)
        acc = delta + c * row(tm, t) * lm * acc
        vs[t] = acc + row(v, t)
        vnext = row(v, t)
    adv = []
    for t in range(T):
        vsn = vs[t + 1] if t + 1 < T else boot
        adv.append((row(rew, t) + g * (1.0 - row(term, t)) * vsn - row(v, t)) * row(tm, t))
    st = lambda xs: R(np.stack([x.v for x in xs]), np.stack([x.r for x in xs]))   # noqa: E731
    return st(vs), st(adv)


def normalize_advantages(adv: R, depth: int):
    """(adv - mean) / (std + 1e-8) of the float64 advantages, and the radius of an fp32 implementation that sums with the given
    depth and computes the std about its own fp32 mean m' (population std).

    With rho_i the advantages' radii, a the float64 advantages and N their number:
      |m' - m|              <= dm = gamma_{depth+1} sum (|a| + rho) / N + mean(rho);
      |m' - mean(a')|       <= dm1 = gamma_{depth+1} sum (|a| + rho) / N;
      sd' within (gamma_{depth+3} / 2 + u) of sqrt(var(a') + (m' - mean a')^2), and std(a') within rms(rho) of std(a) (the
      population std is 1-Lipschitz in the RMS norm), so sd' lies in [s_lo, s_hi];
      the output is (a'_i - m') / (sd' + 1e-8) with the numerator within rho_i + dm of a_i - m: its interval over both ranges,
      widened by the two roundings.
    Where std(a) is within its radius of 0 (nearly constant advantages) the denominator may be as small as 1e-8: then only the
    numerator is bounded, and the radius is (rho_i + dm) / 1e-8 — finite, and as large as the formula makes it."""
    a, rho = adv.v.reshape(-1), adv.r.reshape(-1)
    N = a.size
    m = float(a.mean())
    sd = float(a.std())
    mag = float((np.abs(a) + rho).sum()) / N
    dm1 = gamma(depth + 1) * mag
    dm = dm1 + float(rho.mean())
    rms = float(np.sqrt(np.mean(rho * rho)))
    rel = 1.01 * (0.5 * gamma(depth + 3) + U)
    s_lo = max(sd - rms, 0.0) * (1.0 - rel)
    s_hi = math.sqrt((sd + rms) ** 2 + dm1 ** 2) * (1.0 + rel)
    d_lo, d_hi = (s_lo + NORM_EPS) * (1 - U), (s_hi + NORM_EPS) * (1 + U)
    value = (a - m) / (sd + NORM_EPS)
    n_lo, n_hi = (a - m) - (rho + dm), (a - m) + (rho + dm)
    q = np.stack([n_lo / d_lo, n_lo / d_hi, n_hi / d_lo, n_hi / d_hi])
    q_lo, q_hi = q.min(0), q.max(0)
    rad = np.maximum(q_hi - value, value - q_lo) + 2.02 * U * np.maximum(np.abs(q_lo), np.abs(q_hi)) + ETA
    return R(value.reshape(adv.v.shape), rad.reshape(adv.v.shape)), dict(mean=m, std=sd, dm=dm, s_lo=s_lo, s_hi=s_hi)


# ---- running statistics -----------------------------------------------------------------------------------------------------------
def stats_update(state, batch, chunks: int):
    """running_statistics.update (count, mean, summed variance) with one fp32 batch [n, O], in float64, and the radius of an
    implementation whose float64 sums have depth <= 256 + chunks: (new state, {mean, std: R of the stored fp32 words, state
    radii}).  The reference sums about the batch's own mean (two passes), so its value does not depend on the conditioning;
    the radius charges gamma64 of the magnitudes a shifted two-pass or combined form adds (the batch's first row as the shift),
    which is small unless a column's spread is far below its distance from that shift.  std = clip(sqrt(sv / count), 1e-6, 1e6)."""
    count, mean, sv = state
    x = np.asarray(batch, f32).astype(np.float64)
    n = x.shape[0]
    colsum = lambda a: np.ascontiguousarray(a.T).sum(1)   # noqa: E731  (numpy sums a contiguous row pairwise: depth log2 n)
    mean_b = colsum(x) / n
    M2 = colsum((x - mean_b) ** 2)
    new_count = count + n
    delta = mean_b - mean
    new_mean = mean + delta * (n / new_count)
    new_sv = sv + M2 + delta * delta * (count * n / new_count)
    k = 256 + chunks + int(math.ceil(math.log2(n + 1))) + 16
    c = x[0]
    mag_var = ((x - c) ** 2).sum(0) + n * (mean_b - c) ** 2 + sv + delta * delta * (count * n / new_count) + M2
    r_mean = gamma64(k) * (np.abs(x - c).sum(0) / n + np.abs(c) + np.abs(mean) + np.abs(delta) + np.abs(new_mean))
    # delta = (c + S1 / n) - old mean rounds at the magnitude of the means, not of the spread; it enters the variance through
    # delta^2 n_old n / count (twice: the implementation's and the reference's own float64 delta)
    e_d = 2 * (gamma64(k) * np.abs(x - c).sum(0) / n + gamma64(4) * (np.abs(c) + np.abs(mean_b) + np.abs(mean)))
    r_sv = gamma64(k) * mag_var + (2 * np.abs(delta) * e_d + e_d * e_d) * (count * n / new_count)
    raw_std = np.sqrt(new_sv / new_count)
    with np.errstate(divide="ignore", invalid="ignore"):
        r_std = np.where(raw_std > 0, np.minimum(r_sv / new_count / (2 * np.where(raw_std > 0, raw_std, 1.0)),
                                                 np.sqrt(r_sv / new_count)), np.sqrt(r_sv / new_count))
    std = np.clip(raw_std, 1e-6, 1e6)
    out = dict(mean=R(new_mean, r_mean + U * (np.abs(new_mean) + r_mean)),
               std=R(std, r_std + U * (std + r_std)),
               state_mean_r=r_mean, state_sv_r=r_sv)
    return (new_count, new_mean, new_sv), out


# ---- checks -----------------------------------------------------------------------------------------------------------------------
def ratio(got, ref: R) -> np.ndarray:
    """|got - value| / radius per element; a non-finite result or radius counts as infinitely far"""
    g = np.asarray(got, np.float64)
    err = np.abs(g - ref.v)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(err == 0, 0.0, err / ref.r)
    return np.where(np.isfinite(g) & np.isfinite(q), q, np.inf)


def worst(got, ref: R, what: str = "") -> float:
    q = ratio(got, ref)
    return float(q.max()) if q.size else 0.0
