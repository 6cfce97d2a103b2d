"""The tiny-operand families (tests/tiny_families.py) on the CPU: each reaches its site and band in the float64 reference's own
intermediate values, and the CPU oracle is within K radii of the float64 step there (undecided samples held to one consistent
assignment of their branches, tests/xpbd_ref.py); the host harness of the RL acting step is within K radii of its float64
reference on observations within each band of their mean.  No GPU needed.  Run with -s for the site, band and largest ratio per family."""
import numpy as np
import pytest

from mbd_b200.blackbox.mbd_mnist import normal_host
from oracle import oracle as orc
from tests import tiny_families as T
from tests import xpbd_ref as X
from tests.test_ppo_cpu import harness, host_act  # noqa: F401  (harness: the fixture of the host build)
from tests.test_rl_ref_cpu import check_act
from tests.test_sac_cpu import host_act as sac_host_act
from tests.test_sac_cpu import sac_harness  # noqa: F401

K = 2.0
N = 5


@pytest.fixture(scope="module")
def env(tmp_path_factory):
    return T.make_env(tmp_path_factory.mktemp("tiny"))


def cases(env, n=N):
    """[(family, band, state, actions, reference)]"""
    out = []
    for fam in T.FAMILIES:
        for band in T.SITE[fam][1]:
            for st, u in T.build(env, fam, band, n):
                out.append((fam, band, st, u, X.positional_step(env.blob, np.broadcast_to(st, (n,) + st.shape), u)))
    return out


def site_value(fam, ref):
    """[n] float64 operand of the family's site: the ball's first contact for the contact sites, the arm's joint otherwise"""
    d = ref["diag"][T.SITE[fam][0]]
    return d[:, 0, 0] if d.ndim == 3 else d[:, 1]


def ratio(got, ref, blob, states, actions):
    """largest |got - value| / radius: decided samples against the step, undecided ones against their best consistent
    assignment of branch outcomes"""
    ok = ~ref["undecided"]
    d = np.abs(got.astype(np.float64) - ref["value"])[ok]
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(d == 0, 0.0, d / ref["radius"][ok])
    worst = float(q.max()) if q.size else 0.0
    if (~ok).any():
        br = X.branch_outcomes(blob, states, actions, ref)
        assert not br["still"].any(), "an undecided sample the forced evaluations could not decide"
        best, _ = X.held_ratios(got[br["rows"]], br)
        worst = max(worst, float(best.max()))
    return worst


def test_families_reach_their_sites_and_bands(env):
    rows = []
    for fam, band, st, u, ref in cases(env):
        v = site_value(fam, ref)
        assert T.in_band(v, band).all(), f"{fam} {band}: operand {v[0]:.3g} not in the band"
        rows.append(f"{fam:9s} {T.SITE[fam][0]:20s} {band:10s} operand {v[0]:.4g}")
    print("\n" + "\n".join(rows))


def test_oracle_within_the_bound(env):
    rows = []
    for fam, band, st, u, ref in cases(env):
        assert np.isfinite(ref["value"]).all() and np.isfinite(ref["radius"]).all(), f"{fam} {band}: bound not finite"
        states = np.broadcast_to(st, (u.shape[0],) + st.shape)
        got = orc.xpbd_rollout(env.blob, st, u[:, None], want_final=True, nsub_override=1)["final"]
        assert np.isfinite(got).all()
        q = ratio(got, ref, env.blob, states, u)
        rows.append(f"{fam:9s} {band:10s} oracle {q:.3g} radii, {int(ref['undecided'].sum())} of {u.shape[0]} undecided")
        assert q <= K, f"{fam} {band}: {q:.3g} radii"
    print("\n" + "\n".join(rows))


@pytest.mark.parametrize("kind", ["ppo", "sac"])
def test_act_harness_within_the_bound(kind, harness, sac_harness):   # noqa: F811
    """the host harness of k_ppo_act / k_sac_act on observations within each band of their mean: finite and within K radii of
    the float64 acting step"""
    L = harness if kind == "ppo" else sac_harness
    rows = []
    for band, case in T.act_cases(kind, 33):
        O, nu, pol, mean, std, obs, key = case
        got = (host_act if kind == "ppo" else sac_host_act)(L, pol, mean, std, obs, normal_host(key, (obs.shape[0], nu)))
        assert all(np.isfinite(g).all() for g in got), f"{kind} {band}: not finite"
        r, _ = check_act(kind, case, got, f"{band}")
        rows.append(f"{kind} obs - mean {band:10s} {({k: round(v, 3) for k, v in r.items()})} radii")
    print("\n" + "\n".join(rows))
