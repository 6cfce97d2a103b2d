"""The float64 path-integral reference and its radii (tests/pi_tail_ref.py), checked without a GPU: a numpy fp32 mirror of the
CMA-ES scalar and of the CEM mean stays inside the radii on every tail_ref input family, and mistaken variants do not."""
import numpy as np
import pytest

from oracle import planner as opl
from tests import pi_tail_ref as pr
from tests import tail_ref as tr

f32 = np.float32
HNU = 40
FAMILIES = [f for f in tr.FAMILIES if not f.startswith("demo")]   # the baselines have no demonstration


def _weights(rews, temp):
    std = rews.std(dtype=f32)
    std = f32(1.0) if std < 1e-4 else std
    mean = rews.mean(dtype=f32)
    return opl.softmax(((rews - mean) / std / f32(temp)).astype(f32)), mean, std


def _cma_mirror(w, Y, mu, sigma, variant=None):
    d = (Y - mu[None]).astype(f32)
    V = (w[:, None] * (d * d).astype(f32)).astype(f32).sum(axis=0, dtype=f32)
    roots = V if variant == "no_sqrt" else np.sqrt(V).astype(f32)
    return max(f32(roots.mean(dtype=f32)) * f32(sigma), f32(1e-3))


@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("N", [1, 7, 63, 1025])
def test_cma_sigma_mirror_within_radius(fam, N):
    f = tr.make_family(fam, N, seed=3)
    Y, mu = tr.make_samples(N, HNU, seed=3)
    sigma, temp = 0.7, 0.1
    w, mean, std = _weights(f["rews"], temp)
    ref = tr.reference(f["rews"], temp, Y0s=Y, mu=mu)
    tr.check_stats(ref, f["rews"], mean, std, tr.numpy_depth(N), fam)
    wb = tr.weight_bounds(ref, tr.numpy_depth(N), mean, std)
    want, _ = pr.cma_sigma_reference(ref, sigma)
    rad = pr.cma_sigma_radius(ref, Y, mu, wb["rho"], tr.numpy_depth(N) + 1, sigma, tr.numpy_depth(HNU))
    pr.check_scalar(_cma_mirror(w, Y, mu, sigma), want, rad, f"{fam} N={N}")
    assert rad <= 1e-4 * want, f"{fam} N={N}: radius {rad:.3e} is loose against sigma' = {want:.3e}"


def test_cma_sigma_radius_catches_mistakes():
    N = 1025
    f = tr.make_family("normal", N, seed=1)
    Y, mu = tr.make_samples(N, HNU, seed=1)
    w, mean, std = _weights(f["rews"], 1.0)
    ref = tr.reference(f["rews"], 1.0, Y0s=Y, mu=mu)
    wb = tr.weight_bounds(ref, tr.numpy_depth(N), mean, std)
    want, _ = pr.cma_sigma_reference(ref, 0.5)
    rad = pr.cma_sigma_radius(ref, Y, mu, wb["rho"], tr.numpy_depth(N) + 1, 0.5, tr.numpy_depth(HNU))
    new_mu = (w.astype(np.float64) @ Y.astype(np.float64)).astype(f32)
    for bad in (_cma_mirror(w, Y, mu, 0.5, "no_sqrt"), _cma_mirror(w, Y, new_mu, 0.5), _cma_mirror(w[::-1].copy(), Y, mu, 0.5)):
        assert abs(float(bad) - want) > rad


def test_cma_sigma_floor():
    """Y0s == mu everywhere: every root is 0 and sigma' is the floor exactly"""
    N = 64
    Y = np.full((N, HNU), 0.3, f32)
    f = tr.make_family("normal", N)
    ref = tr.reference(f["rews"], 0.1, Y0s=Y, mu=Y[0])
    want, roots = pr.cma_sigma_reference(ref, 0.9)
    assert want == 1e-3 and not roots.any()


@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("N", [1, 7, 10, 11, 1025])
def test_cem_mirror_within_radius(fam, N):
    f = tr.make_family(fam, N, seed=5)
    Y, _ = tr.make_samples(N, HNU, seed=5)
    w, _, _ = _weights(f["rews"], 0.1)
    idx = pr.cem_indices(w)
    assert len(idx) == min(N, 10) and len(set(idx.tolist())) == len(idx)
    got = Y[idx].mean(axis=0, dtype=f32)
    tr.check_columns(got, pr.cem_mean_reference(Y, idx), pr.cem_mean_radius(Y, idx), f"{fam} N={N}")
    if N > 10:
        wrong = np.argsort(w, kind="stable")[:10]          # ascending: the worst samples
        assert np.abs(Y[wrong].mean(axis=0, dtype=f32) - pr.cem_mean_reference(Y, idx)).max() > pr.cem_mean_radius(Y, idx).max()


def test_cem_tie_order():
    """equal weights: the highest index first (stable ascending argsort, reversed), zero weights included"""
    w = np.array([0.5, 0.0, 0.25, 0.25, 0.0, 0.0], f32)
    assert pr.cem_indices(w).tolist() == [0, 3, 2, 5, 4, 1]
