"""The float64 reference of the black-box objectives (tests/bbo_ref.py) on the CPU: the fp32 mirror of k_bbo's order meets the
bound on constructed families, four deliberate slips leave it, the C oracle equals the mirror bit for bit, and the measured
per-call constants of mbd_sincosf / mbd_expf still hold."""
import numpy as np
import pytest

from tests import bbo_oracle as bo
from tests import bbo_ref as br

f32 = np.float32
DIMS = (1, 2, 255, 256, 257, 800, 6912)
FNS = ("Ackley", "Rastrigin", "Levy")
FAMILIES = ("zero", "plus_one", "minus_one", "edges", "minimiser", "random")


def minimiser_Y(fn, dim):
    """Y whose X is the global minimiser (0 for Ackley / Rastrigin, 1 for Levy), rounded to fp32"""
    x_min, x_max = br.DOMAINS[fn]
    x = 1.0 if fn == "Levy" else 0.0
    return np.full(dim, (x - x_min) / (x_max - x_min) * 2 - 1, f32)


def family(name, fn, dim, N=5):
    rng = np.random.default_rng(dim * 31 + len(name))
    if name == "zero":
        Y = np.zeros((N, dim), f32)
    elif name == "plus_one":
        Y = np.ones((N, dim), f32)
    elif name == "minus_one":
        Y = -np.ones((N, dim), f32)
    elif name == "edges":
        Y = np.where(rng.random((N, dim)) < 0.5, f32(-1), f32(1)).astype(f32)
    elif name == "minimiser":
        Y = np.repeat(minimiser_Y(fn, dim)[None], N, axis=0)
        Y[1:] += (rng.standard_normal((N - 1, dim)) * 1e-3).astype(f32)
    else:
        Y = np.clip(rng.standard_normal((N, dim)), -1, 1).astype(f32)
    return Y.astype(f32)


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("fn", FNS)
def test_mirror_within_bound_and_oracle_bit_exact(orc, fn, dim):
    x_min, x_max = br.DOMAINS[fn]
    for fam in FAMILIES:
        Y = family(fam, fn, dim)
        got = br.objective_f32(fn, Y, x_min, x_max, orc.fmap)
        J64, rad = br.reference(fn, Y, x_min, x_max)
        br.check_J(got, J64, rad, f"{fn} dim={dim} {fam}")
        assert np.array_equal(bo.bbo_eval(fn, Y, x_min, x_max).view(np.uint32), got.view(np.uint32)), f"{fn} dim={dim} {fam}"


def test_minimiser_values(orc):
    """at the (fp32-rounded) global minimiser f is ~0: the reference and the bound agree with the closed form"""
    for fn in FNS:
        x_min, x_max = br.DOMAINS[fn]
        Y = minimiser_Y(fn, 800)[None]
        J64, rad = br.reference(fn, Y, x_min, x_max)
        assert abs(J64[0]) < 1e-3, (fn, J64)
        br.check_J(br.objective_f32(fn, Y, x_min, x_max, orc.fmap), J64, rad, fn)


@pytest.mark.parametrize("perturb,fns", [("drop", FNS), ("map", FNS), ("cos_x", ("Ackley", "Rastrigin")), ("levy_last", ("Levy",))])
def test_bound_notices_slips(orc, perturb, fns):
    """each deliberate slip leaves the bound on every sample of the random family (dim 800); for Levy's last term the last
    element is put at the clip edge (w = 2), where the middle-term formula differs from the last-term one by ~7"""
    for fn in fns:
        x_min, x_max = br.DOMAINS[fn]
        Y = family("random", fn, 800, N=16)
        if perturb == "levy_last":
            Y[:, -1] = 1.0
        J64, rad = br.reference(fn, Y, x_min, x_max)
        bad = br.objective_f32(fn, Y, x_min, x_max, orc.fmap, perturb=perturb).astype(np.float64)
        assert (np.abs(bad - J64) > rad).all(), f"{perturb} {fn}: {np.abs(bad - J64) / rad}"


def test_measured_constants_hold(orc):
    """the per-call constants the bound charges, re-measured over dense sweeps of the arguments the objectives reach"""
    a = np.linspace(-64.0, 64.0, 1 << 22).astype(f32)
    a64 = a.astype(np.float64)
    assert np.max(np.abs(orc.fmap("sin", a) - np.sin(a64))) <= br.SINCOS_ABS
    assert np.max(np.abs(orc.fmap("cos", a) - np.cos(a64))) <= br.SINCOS_ABS
    e = np.linspace(-2.5, 1.5, 1 << 21).astype(f32)
    ex = np.exp(e.astype(np.float64))
    assert np.max(np.abs(orc.fmap("exp", e) - ex) / ex) <= br.EXP_REL
