"""Float64 reference of the path-integral update rules (path_integral.py:33-52) with stated error bounds, on top of
tests/tail_ref.py (same u = 2^-24, same gamma_k model, same 1 % SAFETY factor for dropped second-order terms).

CMA-ES scalar  sigma' = max(mean_j sqrt(V_j) * sigma, 1e-3),  V_j = sum_n w_n (Y_nj - mu_j)^2.
  Each V'_j lies within beta_j of V_j (tail_ref.sqerr_bound, with the implementation's weights within rho_n).  The root moves
  by |sqrt(V') - sqrt(V)| <= min(beta / sqrt(V), sqrt(beta)) (the second, Hoelder, form covers V near 0) plus the rounding
  of sqrtf (u sqrt V').  The mean over HNu columns is a sum of depth k_m (the implementation's order, `cma_mean_depth`) and
  one division: gamma_{k_m + 1} times the mean of the (perturbed) roots.  The product with the fp32 sigma adds u, and the
  floor max(., 1e-3) is 1-Lipschitz, so it keeps the radius.
CEM mean  mu_j = (1/c) sum_{k<c} Y_{idx_k, j} for the c = min(N, 10) picked rows (the index SET is checked for equality
  separately): a sum of depth c - 1 and one division, gamma_{c-1} sum_k |Y_kj| / c + u |mu_j|.
"""
from __future__ import annotations

import math

import numpy as np

from tests import tail_ref as tr

f32, f64 = np.float32, np.float64
TOPK = 10


def cma_mean_depth(HNu: int, threads: int = 256) -> int:
    """cma_sigma (csrc/step_tail.cuh): ceil(HNu / 256) sequential additions per thread, 5 warp and 3 cross-warp levels"""
    return math.ceil(HNu / threads) + 5 + int(math.log2(threads // 32))


def cma_sigma_reference(ref, sigma: float):
    """float64 sigma' from tail_ref.reference(..., Y0s, mu=...)['sqerr'] and the fp32 sigma_i; returns (sigma', roots)"""
    roots = np.sqrt(ref["sqerr"])
    return max(float(roots.mean()) * float(f32(sigma)), 1e-3), roots


def cma_sigma_radius(ref, Y0s, mu, rho, k: int, sigma: float, mean_depth: int) -> float:
    """radius of sigma' for an fp32 implementation whose squared-error sums have depth k and whose weights lie within rho"""
    V = ref["sqerr"]
    beta = tr.sqerr_bound(ref, Y0s, mu, rho, k)
    sq = np.sqrt(V)
    dr = np.minimum(np.where(sq > 0, beta / np.maximum(sq, 1e-300), np.inf), np.sqrt(beta)) + tr.U * (sq + np.sqrt(beta))
    HNu = V.size
    m_hi = float((sq + dr).mean())
    rad_mean = float(dr.mean()) + tr.gamma(mean_depth + 1) * m_hi
    s = float(f32(sigma))
    return tr.SAFETY * (rad_mean * s + tr.U * m_hi * s) + tr.TINY * HNu


def cem_indices(w) -> np.ndarray:
    """path_integral.py:50 on the fp32 weights: jnp.argsort is stable, so after [::-1] equal weights come highest index first"""
    return np.argsort(np.asarray(w, f32), kind="stable")[::-1][:TOPK]


def cem_mean_reference(Y0s, idx) -> np.ndarray:
    return np.asarray(Y0s, f32)[np.asarray(idx)].astype(f64).mean(axis=0)


def cem_mean_radius(Y0s, idx) -> np.ndarray:
    Yk = np.abs(np.asarray(Y0s, f32)[np.asarray(idx)].astype(f64))
    c = Yk.shape[0]
    return tr.SAFETY * (tr.gamma(max(c - 1, 0)) * Yk.sum(axis=0) / c + tr.U * np.abs(cem_mean_reference(Y0s, idx))) + tr.TINY


def check_scalar(got: float, want: float, radius: float, what: str = ""):
    assert abs(float(got) - want) <= radius, f"{what}: {float(got)!r} vs {want!r} (err {abs(float(got) - want):.3e}, bound {radius:.3e})"
