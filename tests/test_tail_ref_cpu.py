"""The float64 tail reference and its bounds (tests/tail_ref.py), checked without a GPU: the numpy fp32 mirror of the
planner (oracle/planner.py) must stay inside the bounds on every input family, and deliberately wrong variants of it must
not — so the bounds are tight enough to catch the mistakes a tail kernel can make before any kernel is run against them."""
import numpy as np
import pytest

from oracle import planner as opl
from tests import tail_ref as tr

f32 = np.float32
TEMPS = (0.01, 0.1, 1.0, 5.0)
SIZES = (1, 2, 63, 1025, 8193)
HNU = 40


def _mirror(rews, Y0s, temp, logpd=None, rew_xref=0.0, perturb=None):
    """oracle/planner.py::reverse_once_stats with its std exposed and one optional mistake:
    'ddof1' sample std, 'drop_last' the last sample left out, 'shift' every weight moved to the next index,
    'no_max' exp(logp) without subtracting the max, clamped like mbd_expf (0 below -87, argument capped at 88)"""
    rews = rews.astype(f32)
    N = rews.size
    keep = N - 1 if perturb == "drop_last" and N > 1 else N
    r = rews[:keep]
    std = r.std(dtype=f32, ddof=1 if perturb == "ddof1" and keep > 1 else 0)
    std = f32(1.0) if std < 1e-4 else std
    mean = r.mean(dtype=f32)
    logp = ((r - mean) / std / f32(temp)).astype(f32)
    if logpd is not None:
        pd = logpd[:keep]
        ld = (((pd - pd.max()).astype(f32) + f32(rew_xref) - mean) / std / f32(temp)).astype(f32)
        logp = np.where(ld > logp, ld, logp).astype(f32)
        logp = ((logp - logp.mean(dtype=f32)) / logp.std(dtype=f32) / f32(temp)).astype(f32)
    if perturb == "no_max":
        x = np.minimum(logp, f32(88.0))
        e = np.where(x < -87.0, f32(0), np.exp(x)).astype(f32)
        w = (e / e.sum(dtype=f32)).astype(f32)
    else:
        w = opl.softmax(logp)
    if keep < N:
        w = np.concatenate([w, np.zeros(N - keep, f32)])
    if perturb == "shift":
        w = np.roll(w, 1)
    Ybar = np.einsum("n,nj->j", w.astype(np.float64), Y0s.astype(np.float64)).astype(f32)
    return Ybar, mean, std, w


def _check_mirror(fam, N, temp, perturb=None):
    f = tr.make_family(fam, N, tie=(0, N - 1) if N > 1 else (0, 0))
    Y, Ybar_i = tr.make_samples(N, HNU)
    coef = tr.schedule_coef()
    ref = tr.reference(f["rews"], temp, f["logpd"], f["rew_xref"], Y, Ybar_i, coef)
    if perturb is None:
        # the oracle itself, exactly as the GPU tests use it
        Ybar, mean, w = opl.reverse_once_stats(f["rews"], Y, temp, logpd=f["logpd"], rew_xref=f["rew_xref"])
        std = f["rews"].std(dtype=f32)
        std = f32(1.0) if std < 1e-4 else std
    else:
        Ybar, mean, std, w = _mirror(f["rews"], Y, temp, f["logpd"], f["rew_xref"], perturb)
    out = tr.update_f32(Ybar, Ybar_i, coef)
    tr.check_step(ref, rews=f["rews"], Y0s=Y, Ybar_i=Ybar_i, coef=coef, mean_used=mean, std_used=std, weights=w,
                  Ybar_im1=out, depth=tr.numpy_depth(N), nruns=(N + 63) // 64, logpd=f["logpd"], rew_xref=f["rew_xref"],
                  what=f"{fam} N={N} temp={temp}")


@pytest.mark.parametrize("fam", tr.FAMILIES)
def test_fp32_mirror_within_bounds(fam):
    for N in SIZES:
        if N == 1 and fam.startswith("demo"):
            continue   # the demo re-normalisation divides by std(logp) = 0: undefined upstream as well (no guard there)
        for temp in TEMPS:
            _check_mirror(fam, N, temp)


def test_oracle_update_is_the_fp32_replay():
    """oracle/planner.py::update and the operation-order replay the sentinel tests compare with bit for bit agree"""
    _, alphas, alphas_bar, _ = opl.make_schedule(1e-4, 1e-2, 100)
    Y, Ybar_i = tr.make_samples(3, 300)
    a = opl.update(Ybar_i, Y[0], alphas, alphas_bar, 60)
    b = tr.update_f32(Y[0], Ybar_i, tr.schedule_coef(60, 100))
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("perturb", ["ddof1", "drop_last", "shift", "no_max"])
def test_bounds_reject_perturbed_mirror(perturb):
    caught = []
    for fam in tr.FAMILIES:
        for N in SIZES[1:]:
            for temp in TEMPS:
                try:
                    _check_mirror(fam, N, temp, perturb)
                except AssertionError:
                    caught.append((fam, N, temp))
    assert caught, f"no input family exposes the '{perturb}' mistake"
    # each mistake is visible on the plain normal family too, not only on a contrived edge
    assert any(c[0] == "normal" for c in caught) or perturb == "no_max", caught
    if perturb == "no_max":
        # subtracting the max only matters once logits exceed the exp range: temp 0.01 does that
        assert any(c[2] == 0.01 for c in caught), caught


def test_bounds_are_per_weight_not_relative_to_the_max():
    """a weight e^-20 .. e^-60 below the best one is still checked to 1e-4 of itself (a bound relative to the largest
    weight would accept anything there)"""
    f = tr.make_family("normal", 1025)
    Y, Ybar_i = tr.make_samples(1025, 8)
    ref = tr.reference(f["rews"], 0.1, Y0s=Y)
    wb = tr.weight_bounds(ref, tr.cta_depth(1025), float(np.mean(f["rews"].astype(np.float64))), ref["std"])
    small = np.flatnonzero((ref["delta"] < -20) & (ref["delta"] > -60))
    assert small.size > 0 and (wb["rho"][small] < 1e-4).all()


def test_guard_margin_of_the_generated_inputs():
    for N in (2, 63, 8193):
        for fam, guarded in (("guard_below", True), ("guard_above", False), ("constant", True), ("normal", False)):
            ref = tr.reference(tr.make_family(fam, N)["rews"], 0.1)
            assert ref["guarded"] == guarded
            assert ref["std"] == 0.0 or ref["std"] < 0.5e-4 or ref["std"] > 2e-4
