"""The CPU oracle's pushT physics step against the float64 reference with a radius per word (tests/pusht_ref.py), on the
constructed families of tests/pusht_families.py, at mu = 1 (shipped) and mu = 0, in both solver modes.  No GPU needed.

Bit equality between `k_pusht` and the oracle shows that they agree; this file shows that the oracle computes the documented
step (DESIGN.md §2, "Accuracy contract of the pushT step"): every word within K radii, the bound tight enough to matter, the
merged out-of-plane pyramid row equal to Brax's two rows, and both alternative `ORC_PT_*` readings detected."""
import numpy as np
import pytest

import mbd_b200
from mbd_b200.envs.pusht import PT
from oracle import oracle as orc
from tests import pusht_families as F
from tests import pusht_ref as X

K = 2.0
MUS = (1.0, 0.0)


def n_of(fam):
    return 129 if F.FAMILIES.index(fam) % 2 else 77


def table(mu):
    P = mbd_b200.envs.get_env("pushT").params.copy()
    P[PT["MU"]] = mu
    return P


@pytest.fixture(scope="module")
def cases():
    """{(mu, family): [(params, state, controls, reference)]}"""
    out = {}
    for mu in MUS:
        P = table(mu)
        for fam in F.FAMILIES:
            out[(mu, fam)] = [(P, st, u, X.step(P, st, u)) for st, u in F.build(fam, n_of(fam))]
    return out


def _oracle(P, st, u, mode, iters=None):
    return orc.pusht_rollout(X.solver_params(P, mode, iters=iters), st, u[:, None], want_final=True)["final"]


def ratio(got, ref, rad):
    """largest |got - value| / radius over the decided samples (0 where equal)"""
    ok = ~ref["undecided"]
    d = np.abs(got.astype(np.float64) - ref["value"])[ok]
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(d == 0, 0.0, d / rad[ok])
    return float(q.max()) if q.size else 0.0


def test_every_family_reaches_its_paths(cases):
    """each family reaches exactly the kernel paths it is built for; together they reach all of them, and the inside-box
    branch on both boxes"""
    seen, inside = set(), set()
    for (mu, fam), launches in cases.items():
        paths = {r["path"] for (_, _, _, r) in launches}
        assert paths == F.PATHS[fam], (mu, fam, paths)
        seen |= paths
        for (_, _, _, r) in launches:
            inside |= set(r["inside"])
    assert seen == set(X.PATHS)
    assert inside == {0, 1}


def test_exact_qp_and_the_merged_pyramid_row(cases):
    """the float64 QP meets its KKT conditions, and the kernel's 3-row form of a contact (the out-of-plane pair as one row
    with half the regulariser) has the same constraint force J^T x as Brax's 4-row pyramid"""
    for (mu, fam), launches in cases.items():
        for (_, _, _, r) in launches:
            assert r["kkt"] <= 1e-12, (mu, fam, r["kkt"])
            assert r["merge_gap"] <= 1e-12, (mu, fam, r["merge_gap"])


@pytest.mark.parametrize("mode", ["fixed", "prod"])
def test_oracle_within_the_bound(cases, mode):
    worst = {}
    for (mu, fam), launches in cases.items():
        und = np.mean([r["undecided"].mean() for (_, _, _, r) in launches])
        assert und <= F.UNDECIDED_CAP[fam], f"mu={mu} {fam}: {und:.3f} of the samples undecided"
        for P, st, u, ref in launches:
            q = ratio(_oracle(P, st, u, mode), ref, X.radius(ref, mode))
            worst[(mu, fam)] = max(worst.get((mu, fam), 0.0), q)
            assert q <= K, f"{mode} mu={mu} {fam}: |oracle - value| = {q:.3g} radii"
    print(mode, {k: round(v, 3) for k, v in worst.items()})
    assert max(worst.values()) > 0.5          # the radius is not simply huge
    for mu in MUS:     # the tie family straddles the face choice on half its launches; no other family is undecided
        und = np.mean([r["undecided"].mean() for (_, _, _, r) in cases[(mu, "tie")]])
        assert 0.45 <= und <= F.UNDECIDED_CAP["tie"], und


def test_truncation_constant(cases):
    """the production-mode truncation radius is the stated constant C_TRUNC = 4 x the largest ratio |production - fixed
    point| / unit truncation radius over every family; pin the measurement it was taken from.  The substep chains reach
    larger ratios (tests/test_pusht_horizon_ref_cpu.py::test_truncation_constant_along_the_chains pins TRUNC_MEASURED, the
    largest over both), still below C_TRUNC"""
    worst = 0.0
    for (mu, fam), launches in cases.items():
        for P, st, u, ref in launches:
            d = np.abs(_oracle(P, st, u, "prod").astype(np.float64) - _oracle(P, st, u, "fixed"))
            with np.errstate(divide="ignore", invalid="ignore"):
                q = np.where(d == 0, 0.0, d / ref["trunc"])
            worst = max(worst, float(q[~ref["undecided"]].max(initial=0.0)))
    print("largest truncation ratio", worst)
    assert 0.5 * X.TRUNC_FAMILIES <= worst <= X.TRUNC_FAMILIES and X.C_TRUNC == 4.0 * X.TRUNC_FAMILIES
    assert X.TRUNC_FAMILIES <= X.TRUNC_MEASURED < X.C_TRUNC


def test_the_bound_is_not_vacuous(cases):
    """every radius of a decided sample is finite and below its family's cap, and its largest velocity radius is a small
    fraction of its largest velocity change; with no row, 99 % of the words are within 256 u of their value; on the face
    contacts (the first four launches per slider pose) within 2^17 u — the soft contact (k = 2770 / s^2 on a penetration
    known to 1e-7 m) amplifies the input rounding"""
    for (mu, fam), launches in cases.items():
        for (_, st, _, ref) in launches:
            ok = ~ref["undecided"]
            r = ref["radius"][ok]
            assert np.isfinite(r).all(), f"mu={mu} {fam}: infinite radius"
            assert r.size == 0 or r.max() <= F.RADIUS_CAP[fam], f"mu={mu} {fam}: radius {r.max():.3g}"
            dqd = np.abs(ref["value"][ok, 8:13] - st[8:13].astype(np.float64)).max(1)
            rel = ref["radius"][ok, 8:13].max(1) / np.maximum(dqd, 1e-30)
            assert rel.size == 0 or rel.max() <= F.REL_CAP[fam], f"mu={mu} {fam}: velocity radius {rel.max():.3g} of the change"
    words = [0, 1, 2, 3, 4, 8, 9, 10, 11, 12]

    def rel(ref):
        v = np.abs(ref["value"][:, words])
        return (ref["radius"][:, words] / (X.U * np.maximum(v, 1e-30)))[v > 0]

    for mu in MUS:
        free = np.concatenate([rel(r) for (_, _, _, r) in cases[(mu, "free")]])
        assert np.percentile(free, 99) < 256, np.percentile(free, 99)
        for fam, per in (("box0", 8), ("box1", 10)):
            ls = cases[(mu, fam)]
            faces = np.concatenate([rel(ls[p * per + k][3]) for p in range(2) for k in range(4)])
            assert np.percentile(faces, 99) < 2.0 ** 17, (mu, fam, np.percentile(faces, 99))


# the two non-default readings of oracle/pusht_oracle.c; each must leave the bound on some family
VARIANTS = {"ORC_PT_REG_INVWEIGHT": 1, "ORC_PT_CONTACT_MIDPOINT": 0}


@pytest.mark.parametrize("switch", list(VARIANTS))
def test_every_alternative_reading_is_detected(cases, tmp_path, switch):
    lib = orc.build_variant({switch: VARIANTS[switch]}, str(tmp_path / "variant.so"))
    old, orc._LIB = orc._LIB, lib
    try:
        worst, where = 0.0, None
        for (mu, fam), launches in cases.items():
            for P, st, u, ref in launches:
                q = ratio(_oracle(P, st, u, "fixed"), ref, X.radius(ref, "fixed"))
                if q > worst:
                    worst, where = q, (mu, fam)
    finally:
        orc._LIB = old
    print(switch, worst, where)
    assert worst > K, f"{switch}={VARIANTS[switch]} stays within {worst:.3g} radii ({where})"
