"""Float64 reference of the tail of a diffusion step, with stated error bounds.

The tail is everything of reverse_once after the rollouts (mbd_planner.py:110-133): rews.mean(), population std with the
1e-4 guard, the demo blend with its second normalisation (note the double /temp), the softmax, Ybar = sum_n w_n Y_n and the
update lines 130-133.  The same statistics drive the round-1 planners (path_integral.py: MPPI mean, CMA-ES
sum_n w_n (Y_n - mu)^2).  `reference` evaluates all of it in float64 from the SAME float32 inputs an implementation sees;
the `*_bound` functions say how far an fp32 implementation with a given reduction structure may land from it.  The bounds
are derived below to first order in u = 2^-24 (second-order terms are covered by a 1 % factor) and hold for every
summation order of the given depth, so they do not pin an association: a one-pass variance or an online softmax passes
them exactly when it is as accurate as the current kernels claim to be.

Notation: gamma_k = k u / (1 - k u) bounds the relative error of a sum whose terms each pass through at most k roundings
(Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., Lemma 3.1 / section 4.2).  `depth` is that k for the
implementation's reductions: ceil(N / lanes) sequential additions per lane plus log2(lanes) tree levels; the 8-CTA cluster
kernel has 8192 lanes (13 levels), the round-1 single-CTA kernel 1024 (10 levels), numpy's pairwise sum see `numpy_depth`.

Derivation (weights, non-demo).  An implementation computes L_n = fl(fl(fl(r_n - m')/s')/T) with its own mean m' and
std s'.  Against the float64 logits l_n = (r_n - m)/s/T:
  * m' - m shifts every L_n by the same amount: it cancels in the softmax;
  * s'/s = 1 + eps_s scales L_n - L_max by (1 + eps_s): an error eps_s |Delta_n| in x_n = L_n - L_max, where
    Delta_n = l_n - max l (the float64 log-weight relative to the best sample);
  * three roundings per logit: 3u (|L_n| + |L_max|); the subtraction x_n = L_n - L_max: u |Delta_n|.
So |x_n - Delta_n - shift| <= e_n = (eps_s + u) |Delta_n| + 3u (|L_n| + |L_max|).  mbd_expf is within 4 ulp (8u relative,
tests/test_fp32_spec.py), so each exponential is exp(Delta_n)(1 + eta_n) with eta_n = expm1(e_n) + 8u; a sample whose
x_n may fall below -87 may be flushed to 0 (then eta_n = 1: anything in [0, 2 w_n]).  The sum S carries
sum_m w_m eta_m + gamma_depth, the division one more u:
    |w'_n - w_n| <= rho_n w_n,   rho_n = eta_n + sum_m w_m eta_m + gamma_depth + u          (plus 2^-149 absolute: the
                                                                                              quotient may be subnormal)
which is u (a + b log2 N)(1 + |Delta_n|) with small constants once eps_s is of order u, plus the 3u |L| rounding term of the
logits themselves.  eps_s is NOT always of order u: the variance is computed about the fp32 mean m', so
s'^2 = var + (m' - m)^2 up to rounding.  With a large offset and a tiny spread (mean 1e3, std 1e-2) (m' - m)/s can reach
1e-2 and eps_s 5e-5 — an honest property of the two-pass formula, which the bound states instead of hiding:
    |s' - s_c| <= (gamma_{depth+3}/2 + u) s_c,   s_c = sqrt(var + (m' - m)^2)   (the conditioned reference),
    |m' - m|  <= gamma_{depth+1} sum|r_n| / N.
Demo: l_n = max(l0_n, ld_n) is re-normalised, (l - mean l)/std l/T, which is invariant to the shift and scale that m' and
s' apply to l, so only the per-element roundings of l (E_n below) and the conditioning of the second std enter.

Ybar column j: |Ybar'_j - Ybar_j| <= gamma_k sum_n w_n |Y_nj| (1 + rho_n) + sum_n rho_n w_n |Y_nj|, k = 64 (sequential run)
+ ceil(log2 nruns) + ceil(log2 P) (pairwise trees over runs and ranks).  Update: the error of Ybar and one rounding per
operation are pushed through lines 130-133 term by term (`update_bound`); c1 c2 ~ 1 makes Yi cancel, so the bound is
carried by |c0 Ybar_i| and |c0 Ybar| rather than by the result.
"""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -24
TINY = 2.0 ** -149          # absolute slack of one subnormal ulp: a weight quotient may underflow
FLUSH = -87.0               # mbd_expf returns 0 below this argument
SAFETY = 1.01               # covers the second-order terms the derivation drops

f32, f64 = np.float32, np.float64


def gamma(k) -> float:
    return k * U / (1.0 - k * U)


def cluster_depth(N: int) -> int:
    """k_step_weights: 8192 lanes (8 CTAs x 1024 threads), then 5 + 5 butterfly levels in the CTA and 3 across the cluster"""
    return math.ceil(N / 8192) + 13


def cta_depth(N: int) -> int:
    """k_softmax_weights: 1024 lanes, 5 + 5 butterfly levels"""
    return math.ceil(N / 1024) + 10


def numpy_depth(N: int) -> int:
    """numpy's float32 pairwise sum: blocks of up to 128 elements summed by 8 accumulators (16 terms each) plus 3 levels,
    blocks combined by recursive halving"""
    return math.ceil(min(N, 128) / 8) + 3 + max(0, math.ceil(math.log2(max(N / 128, 1.0))))


def wsum_depth(nruns: int, P: int = 1) -> int:
    """Sum_n w_n Y_n: 64 sequential fmaf per run, an adjacent-pairwise tree over the runs and one over the rank partials"""
    return 64 + math.ceil(math.log2(max(nruns, 1))) + math.ceil(math.log2(max(P, 1)))


# ---- the reference ------------------------------------------------------------------------------------------------------

def _std(x):
    return float(np.sqrt(np.mean((x - np.mean(x)) ** 2)))


def reference(rews, temp, logpd=None, rew_xref=0.0, Y0s=None, Ybar_i=None, coef=None, mu=None) -> dict:
    """mbd_planner.py:110-133 (and path_integral.py:33-52 with `mu`) in float64 from the float32 inputs.  coef: the five fp32
    scalars of engine.update_coef, widened."""
    r = np.asarray(rews, f32).astype(f64)
    N = r.size
    m = float(np.mean(r))
    s = _std(r)
    sg = 1.0 if s < 1e-4 else s
    T = float(f32(temp))
    out = dict(N=N, mean=m, std=s, std_g=sg, guarded=s < 1e-4, T=T, demo=logpd is not None)
    l0 = (r - m) / sg / T
    if logpd is not None:
        pd = np.asarray(logpd, f32).astype(f64)
        mxd = float(pd.max())
        ld = ((pd - mxd) + float(f32(rew_xref)) - m) / sg / T
        l = np.maximum(ld, l0)
        lm, ls = float(np.mean(l)), _std(l)
        out.update(l=l, lmean=lm, lstd=ls, mxd=mxd)
        logp = (l - lm) / ls / T
    else:
        logp = l0
    mx = float(logp.max())
    delta = logp - mx
    e = np.exp(delta)
    S = float(e.sum())
    w = e / S
    out.update(logp=logp, max_logp=mx, delta=delta, S=S, w=w)
    if Y0s is not None:
        Y = np.asarray(Y0s, f32).astype(f64)
        out["Ybar"] = w @ Y
        if mu is not None:
            d = Y - np.asarray(mu, f32).astype(f64)[None]
            out["sqerr"] = w @ (d * d)
        if coef is not None:
            out["Ybar_im1"] = update64(out["Ybar"], Ybar_i, coef)
    return out


def update64(Ybar, Ybar_i, coef):
    c = [float(f32(x)) for x in coef]
    Yi = np.asarray(Ybar_i, f32).astype(f64) * c[0]
    score = c[1] * (-Yi + c[0] * Ybar)
    return c[3] * (Yi + c[2] * score) / c[4]


def update_f32(Ybar, Ybar_i, coef):
    """diffusion_update (csrc/step_tail.cuh) and k_update in their operation order, numpy float32 (no contraction)"""
    c = [f32(x) for x in coef]
    Ybar, Ybar_i = np.asarray(Ybar, f32), np.asarray(Ybar_i, f32)
    Yi = (Ybar_i * c[0]).astype(f32)
    score = (c[1] * ((-Yi) + (c[0] * Ybar).astype(f32)).astype(f32)).astype(f32)
    Yim1 = (c[3] * (Yi + (c[2] * score).astype(f32)).astype(f32)).astype(f32)
    return (Yim1 / c[4]).astype(f32)


# ---- bounds -------------------------------------------------------------------------------------------------------------

def mean_bound(ref, rews, depth: int) -> float:
    """|m' - m| for a float32 sum of the given depth followed by one division"""
    return gamma(depth + 1) * float(np.abs(np.asarray(rews, f32).astype(f64)).sum()) / ref["N"]


def std_conditioned(ref, mean_used: float) -> float:
    """the population std the implementation targets when it centres on its own fp32 mean: sqrt(var + (m' - m)^2)"""
    return math.sqrt(ref["std"] ** 2 + (float(mean_used) - ref["mean"]) ** 2)


def std_rel_bound(depth: int) -> float:
    """|s' - s_c| / s_c: (x - m') rounded (u), squared exactly by fmaf (2u), summed (gamma_depth), divided (u), sqrt (u)"""
    return SAFETY * (0.5 * gamma(depth + 3) + U)


def weight_bounds(ref, depth: int, mean_used: float, std_used: float) -> dict:
    """per-sample relative bound rho_n on the softmax weights, and the bound on S (see the module docstring).

    mean_used / std_used: the (guarded) fp32 mean and std the implementation worked with — checked separately against
    `mean_bound` / `std_rel_bound`, and here only used to size the logit magnitudes and the scale error."""
    N, T = ref["N"], ref["T"]
    delta = ref["delta"]
    ad = np.abs(delta)
    rs = std_rel_bound(depth)
    if ref["guarded"]:
        eps_s = 0.0
    else:
        sc = std_conditioned(ref, mean_used)
        eps_s = abs(sc - ref["std"]) / ref["std"] + rs * sc / ref["std"]
    sg = ref["std_g"]
    if not ref["demo"]:
        Lc = (np.asarray(ref["logp"]) * sg * T + ref["mean"] - float(mean_used)) / float(std_used) / T   # logits as computed
        e = (eps_s / (1.0 - eps_s) + U) * ad + 3 * U * (np.abs(Lc) + abs(float(Lc.max())))
    else:
        # per-element rounding of l = max(l0, ld), in units of the first normalisation (scale s'), see the docstring
        # l0: three roundings (3u |l|); ld: the three sums before the divisions (`_ld_terms`) plus two divisions (<= 3u |l|)
        l = ref["l"]
        alpha = sg / float(std_used)                          # l as computed ~ alpha * l + shift
        shift = (ref["mean"] - float(mean_used)) / float(std_used) / T
        lc = np.abs(alpha * l + shift)
        E = (ref["_ld_terms"] / float(std_used) / T + 3 * U * lc) * SAFETY
        ls_c = alpha * ref["lstd"]                            # std of l as computed, before its own roundings
        # mean of l: summation error plus the element errors; it shifts every logit alike but enters the second std
        dlm = gamma(depth + 1) * float(np.mean(lc)) + float(E.max())
        rmsE = float(np.sqrt(np.mean(E * E)))
        eps_ls = (rmsE + dlm * dlm / (2 * ls_c)) / ls_c + rs
        logp = np.asarray(ref["logp"])
        top = delta > -1.0
        Etop = float(E[top].max())
        e = (eps_ls / (1.0 - eps_ls) + U) * ad + (E + Etop) / ls_c / T + 3 * U * (np.abs(logp) + abs(ref["max_logp"]))
    e = e * SAFETY
    may_flush = delta - e < FLUSH
    eta = np.where(may_flush, 1.0, np.expm1(e) + 8.0 * U * SAFETY)
    w = ref["w"]
    sum_eta = float((w * eta).sum())
    sigma_S = sum_eta + gamma(depth) * (1 + sum_eta)
    rho = SAFETY * (eta + sigma_S + U)
    rho = np.where(may_flush, np.maximum(rho, 1.0), rho)
    return dict(rho=rho, may_flush=may_flush, sigma_S=SAFETY * sigma_S, e=e, eps_s=eps_s)


def prepare_demo_terms(ref, rews, logpd, rew_xref, mean_used):
    """magnitudes of the intermediate sums of ld = ((pd - max pd) + x_ref - m') / s' / T whose roundings enter E_n"""
    pd = np.asarray(logpd, f32).astype(f64)
    a = pd - ref["mxd"]
    b = a + float(f32(rew_xref))
    ref["_ld_terms"] = U * (np.abs(a) + np.abs(b) + np.abs(b - float(mean_used))) * SAFETY


def ybar_bound(ref, Y0s, rho, k: int):
    """per-column bound on Sum_n w_n Y_nj for a float32 accumulation of depth k and weights within rho_n"""
    Y = np.abs(np.asarray(Y0s, f32).astype(f64))
    w = ref["w"]
    return gamma(k) * ((w * (1 + rho)) @ Y) + (w * rho) @ Y + TINY * Y.shape[0]


def sqerr_bound(ref, Y0s, mu, rho, k: int):
    """per-column bound on Sum_n w_n (Y_nj - mu_j)^2: d = Y - mu rounded (u), d*d rounded (u) -> 3u per term, then as Ybar"""
    d = np.asarray(Y0s, f32).astype(f64) - np.asarray(mu, f32).astype(f64)[None]
    d2 = d * d
    w = ref["w"]
    return (gamma(k) + 3 * U) * ((w * (1 + rho)) @ d2) * SAFETY + (w * rho) @ d2 + TINY * d2.shape[0]


def update_bound(Ybar64, Ybar_i, coef, beta):
    """forward error of lines 130-133 given |Ybar' - Ybar| <= beta: every operation adds u times its float64 magnitude and
    scales the error it receives"""
    c = [float(f32(x)) for x in coef]
    Yi = np.asarray(Ybar_i, f32).astype(f64) * c[0]
    t = c[0] * Ybar64
    s1 = -Yi + t
    sc = c[1] * s1
    v = c[2] * sc
    a = Yi + v
    y = c[3] * a
    o = y / c[4]
    eYi = U * np.abs(Yi)
    et = abs(c[0]) * beta + U * np.abs(t)
    es1 = eYi + et + U * np.abs(s1)
    esc = abs(c[1]) * es1 + U * np.abs(sc)
    ev = abs(c[2]) * esc + U * np.abs(v)
    ea = eYi + ev + U * np.abs(a)
    ey = abs(c[3]) * ea + U * np.abs(y)
    eo = ey / abs(c[4]) + U * np.abs(o)
    return SAFETY * eo + TINY


# ---- input families -----------------------------------------------------------------------------------------------------

FAMILIES = ("normal", "offset", "guard_below", "guard_above", "constant", "dominant", "tie",
            "demo_demo", "demo_reward", "demo_mixed")


def _unit(rng, N):
    """N standard-normal draws rescaled to population std exactly 1 (float64), so a family's spread is what it says"""
    z = rng.standard_normal(N)
    if N > 1:
        z = (z - z.mean()) / z.std()
    return z


def make_family(name: str, N: int, seed: int = 0, tie=None) -> dict:
    """float32 per-sample returns (and demo log-densities) of one input family:
      normal       returns -1 + 0.7 z
      offset       1e3 + 1e-2 z: the case a one-pass variance gets catastrophically wrong
      guard_below  std 0.4e-4 (guarded to 1), guard_above std 3e-4 (not guarded): both >= 2x away from the 1e-4 threshold
                   in float64, so fp32 rounding cannot flip the decision
      constant     every return equal: std 0, uniform weights
      dominant     normal plus one sample 8 std above the rest
      tie          normal plus an exact two-way tie 6 std above the rest, at the positions `tie` = (p, q)
      demo_*       the demo blend (mbd_planner.py:116-126) with demonstration log-densities that win for almost every sample
                   (demo_demo), for none (demo_reward) or for about half of them (demo_mixed)"""
    rng = np.random.default_rng(seed * 1000003 + N * 7 + FAMILIES.index(name))
    z = _unit(rng, N)
    out = dict(logpd=None, rew_xref=0.0)
    if name == "offset":
        r = 1e3 + 1e-2 * z
    elif name == "guard_below":
        r = 0.5 + 0.4e-4 * z
    elif name == "guard_above":
        r = 0.5 + 3e-4 * z
    elif name == "constant":
        r = np.full(N, 0.3)
    else:
        r = -1.0 + 0.7 * z
    if name == "dominant":
        r[int(rng.integers(N))] = -1.0 + 0.7 * 8.0
    if name == "tie":
        p, q = (min(t, N - 1) for t in (tie if tie is not None else (0, N - 1)))
        r[p] = r[q] = -1.0 + 0.7 * 6.0
    if name.startswith("demo"):
        pd = -np.abs(rng.standard_normal(N)) * 0.3
        out["logpd"] = pd.astype(f32)
        # ld - l0 = ((pd - max pd) + x_ref - r) / s / T: x_ref far above / below the returns, or in their middle
        out["rew_xref"] = {"demo_demo": 3.0, "demo_reward": -10.0, "demo_mixed": -1.0}[name]
    out["rews"] = np.asarray(r, f32)
    s64 = _std(out["rews"].astype(f64)) if N > 1 else 0.0
    assert s64 == 0.0 or not (0.5e-4 < s64 < 2e-4), f"{name}: float64 std {s64} too close to the 1e-4 guard"
    return out


def make_samples(N: int, HNu: int, seed: int = 0):
    """Y0s in [-1, 1] (what the clip of mbd_planner.py:106 leaves) and an iterate Ybar_i; no exact zeros, so a sentinel's
    row passes through the weighted sum unchanged in sign"""
    rng = np.random.default_rng(seed + 17 * N + HNu)
    Y = np.clip(rng.standard_normal((N, HNu)) * 0.5, -1, 1).astype(f32)
    Y[Y == 0] = f32(0.25)
    Ybar_i = (rng.standard_normal(HNu) * 0.3).astype(f32)
    return Y, Ybar_i


def schedule_coef(i: int = 60, Ndiffuse: int = 100):
    """update coefficients of step i of the default schedule (beta 1e-4 .. 1e-2), as engine.update_coef computes them"""
    betas = np.linspace(1e-4, 1e-2, Ndiffuse).astype(f32)
    alphas = (f32(1) - betas).astype(f32)
    ab = np.cumprod(alphas, dtype=f32)
    one = f32(1)
    return [np.sqrt(ab[i]), one / (one - ab[i]), one - ab[i], one / np.sqrt(alphas[i]), np.sqrt(ab[i - 1])]


# ---- checks (shared by the CPU self-test and the GPU suite) -------------------------------------------------------------

def check_stats(ref, rews, mean_used, std_used, depth, what=""):
    """rews.mean() and the guarded std against their bounds; the guard decision must agree with float64"""
    mb = mean_bound(ref, rews, depth)
    assert abs(float(mean_used) - ref["mean"]) <= mb, f"{what}: mean {float(mean_used)!r} vs {ref['mean']!r} (bound {mb:.3e})"
    if ref["guarded"]:
        assert float(std_used) == 1.0, f"{what}: std {float(std_used)!r} should be guarded to 1 (float64 std {ref['std']:.3e})"
    else:
        sc = std_conditioned(ref, mean_used)
        tol = std_rel_bound(depth) * sc
        assert abs(float(std_used) - sc) <= tol, (f"{what}: std {float(std_used)!r} vs {sc!r} (conditioned on the fp32 mean; "
                                                 f"bound {tol:.3e}, float64 std {ref['std']!r})")


def check_weights(ref, w, wb, what=""):
    w = np.asarray(w, f32).astype(f64)
    assert w.shape == ref["w"].shape, f"{what}: {w.shape} weights vs {ref['w'].shape}"
    err = np.abs(w - ref["w"])
    tol = wb["rho"] * ref["w"] + TINY
    bad = ~(err <= tol)
    if bad.any():
        n = int(np.argmax(np.where(bad, err / np.maximum(tol, 1e-300), -1.0)))
        raise AssertionError(f"{what}: {int(bad.sum())} of {w.size} weights outside their bound; worst at n={n}: "
                             f"{w[n]!r} vs {ref['w'][n]!r} (rel {err[n] / max(ref['w'][n], 1e-300):.3e}, bound "
                             f"{wb['rho'][n]:.3e}, log-weight {ref['delta'][n]:.2f})")


def check_columns(got, want, tol, what=""):
    got = np.asarray(got, f32).astype(f64)
    err = np.abs(got - want)
    bad = ~(err <= tol)
    if bad.any():
        j = int(np.argmax(np.where(bad, err / np.maximum(tol, 1e-300), -1.0)))
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.size} columns outside their bound; worst at j={j}: "
                             f"{got[j]!r} vs {want[j]!r} (err {err[j]:.3e}, bound {tol[j]:.3e})")


def check_step(ref, *, rews, Y0s, Ybar_i, coef, mean_used, std_used, weights, Ybar_im1, depth, nruns, P=1,
               logpd=None, rew_xref=0.0, what=""):
    """everything one tail step produces against the float64 reference"""
    check_stats(ref, rews, mean_used, std_used, depth, what)
    if logpd is not None:
        prepare_demo_terms(ref, rews, logpd, rew_xref, mean_used)
    wb = weight_bounds(ref, depth, mean_used, std_used)
    check_weights(ref, weights, wb, what + ": weights")
    beta = ybar_bound(ref, Y0s, wb["rho"], wsum_depth(nruns, P))
    check_columns(Ybar_im1, ref["Ybar_im1"], update_bound(ref["Ybar"], Ybar_i, coef, beta), what + ": Ybar_im1")
    return wb
