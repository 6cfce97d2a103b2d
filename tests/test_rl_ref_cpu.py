"""The RL acting step, GAE and the observation statistics against the float64 reference with a radius per value (tests/rl_ref.py)
on the constructed families of tests/rl_families.py.  No GPU needed.

The host harnesses of include/mbd_ppo.h and include/mbd_sac.h (the header the kernels compile) and the float32 restatement of
k_ppo_gae (`ppo_ref.gae_kernel_f32`, bit-equal to the kernel) are held to K radii on every family; the radii are finite and below
a cap per family; and numpy mirrors of the three computations meet the bound unmutated and leave it under each deliberate mistake,
on the family named for it (DESIGN.md §2, "Accuracy contract of the RL acting step, GAE and statistics")."""
import numpy as np
import pytest

from mbd_b200.blackbox.mbd_mnist import normal_host
from mbd_b200.rl import networks as nets
from tests import ppo_ref
from tests import rl_families as F
from tests import rl_ref as X
from tests.test_ppo_cpu import harness, host_act  # noqa: F401  (harness: the fixture of the host build)
from tests.test_sac_cpu import host_act as sac_host_act
from tests.test_sac_cpu import sac_harness  # noqa: F401

K = 2.0
f32 = np.float32
B = 64
# largest radius / (1 + |value|) per family over both policies (measured: DESIGN.md §2), with headroom
RADIUS_CAP = {"mild": 2.0, "std_floor": 1.0, "obs_mean": 0.01, "floor": 1e-4, "loc": 1e-3, "wide": 1e-3, "raw": 1e-3, "cap": 1e-3}
GAE_RADIUS_CAP = 1e-3            # radius / (1 + |value|) of vs and of the advantages before the normalisation
NORM_RADIUS_CAP = {"offset": 0.5, "constant": np.inf}    # of the normalised advantages; elsewhere NORM_RADIUS_DEFAULT
NORM_RADIUS_DEFAULT = 1e-4


def check_act(kind, case, got, what=""):
    """largest |got - f64| / radius of (act, raw, logp) for one launch, asserting K"""
    O, nu, pol, mean, std, obs, key = case
    eps = normal_host(key, (obs.shape[0], nu))
    ref = X.act(kind, pol, mean, std, obs, eps, O, nu)
    out = {}
    for name, g in zip(("act", "raw", "logp"), got):
        q = X.ratio(g, ref[name])
        out[name] = float(q.max())
        assert out[name] <= K, f"{what} {kind} O={O} nu={nu} {name}: {out[name]:.3g} radii at {np.unravel_index(np.argmax(q), q.shape)}"
    return out, ref


# ---- the acting step --------------------------------------------------------------------------------------------------------------
def _host(kind, L, case):
    O, nu, pol, mean, std, obs, key = case
    eps = normal_host(key, (obs.shape[0], nu))
    return (host_act if kind == "ppo" else sac_host_act)(L, pol, mean, std, obs, eps)


@pytest.mark.parametrize("kind", ["ppo", "sac"])
def test_host_harness_within_the_bound(kind, harness, sac_harness):  # noqa: F811
    L = harness if kind == "ppo" else sac_harness
    for fam, cases in F.act_cases(kind, B).items():
        worst = {}
        for case in cases:
            r, _ = check_act(kind, case, _host(kind, L, case), fam)
            worst = {k: max(worst.get(k, 0.0), v) for k, v in r.items()}
        print(f"{kind} {fam:10s} largest |harness - f64| / radius {({k: round(v, 3) for k, v in worst.items()})}")


@pytest.mark.parametrize("kind", ["ppo", "sac"])
def test_act_radii_are_finite_and_capped(kind):
    for fam, cases in F.act_cases(kind, B).items():
        for O, nu, pol, mean, std, obs, key in cases:
            ref = X.act(kind, pol, mean, std, obs, normal_host(key, (B, nu)), O, nu)
            for name in ("act", "raw", "logp"):
                rel = ref[name].r / (1.0 + np.abs(ref[name].v))
                assert np.isfinite(ref[name].r).all(), f"{kind} {fam} {name}: a radius is not finite"
                assert rel.max() <= RADIUS_CAP[fam], f"{kind} {fam} O={O} nu={nu} {name}: radius {rel.max():.3g} (1 + |value|)"


def test_families_reach_the_branches():
    """the constructed inputs reach what they are named for: the swish cap on both sides, raw on both sides of the tanh cap and
    near 0, scale at its floor"""
    c = F.act_cases("ppo", B)
    pre = np.concatenate([np.concatenate([p.ravel() for p in X.act("ppo", *cs[2:6], normal_host(cs[6], (B, cs[1])), cs[0], cs[1])["pre"]])
                          for cs in c["cap"]])
    assert (pre < -80).any() and ((pre > -80) & (pre < -79)).any()
    raw = np.concatenate([X.act("ppo", *cs[2:6], normal_host(cs[6], (B, cs[1])), cs[0], cs[1])["raw"].v.ravel() for cs in c["raw"]])
    assert (np.abs(raw) < 1e-2).any() and ((np.abs(raw) > 2) & (np.abs(raw) < 20)).any()
    assert ((raw > 20) & (raw < 20.01)).any() and ((raw < 20) & (raw > 19.99)).any() and (raw < -20).any()
    sc = X.act("ppo", *c["floor"][0][2:6], normal_host(c["floor"][0][6], (B, 6)), 17, 6)["scale"].v
    assert np.abs(sc - 0.001).max() < 1e-12


# ---- the numpy fp32 mirror of the acting step, and its mistakes ------------------------------------------------------------------
def _sp32(x):
    return np.logaddexp(x, f32(0)).astype(f32)


def _tanh32(x, cap=40.0):
    e = np.exp(np.minimum(f32(2) * np.abs(x), f32(cap))).astype(f32)
    t = (f32(1) - f32(2) / (e + f32(1))).astype(f32)
    return np.where(x < 0, -t, t).astype(f32)


def mirror_act(kind, O, nu, pol, mean, std, obs, key, mistake=None):
    eps = normal_host(key, (obs.shape[0], nu))
    sizes = nets.policy_sizes(O, nu) if kind == "ppo" else nets.sac_policy_sizes(O, nu)
    layers = nets.unflatten(np.asarray(pol, f32), sizes)
    with np.errstate(over="ignore", invalid="ignore"):
        x = ((obs - mean) * std if mistake == "norm_mul" else (obs - mean) / std).astype(f32)
        for l, (W, b) in enumerate(layers):
            last = l + 1 == len(layers)
            x = (x @ W).astype(f32)
            if not (last and mistake == "no_last_bias"):
                x = (x + b).astype(f32)
            if not last:
                x = (x / (f32(1) + np.exp(-x))).astype(f32) if kind == "ppo" else np.maximum(x, f32(0))
        loc, s = x[:, :nu], x[:, nu:]
        scale = _sp32(s) + (f32(0) if mistake == "no_min_std" else f32(0.001))
        r = (eps * scale + loc).astype(f32)
        z = (r / scale - loc / scale).astype(f32)
        logpdf = (f32(-0.5) * (z * z) - (f32(X.HALF_LOG_2PI) + np.log(scale))).astype(f32)
        jf = f32(1) if mistake == "jac1" else f32(2)
        jac = (jf * (f32(X.LOG2) - r - _sp32(f32(2) * r if mistake == "sp_sign" else f32(-2) * r))).astype(f32)
        lp = (logpdf - jac).astype(f32)
        logp = (lp[:, :nu - 1] if mistake == "sum_nu1" else lp).sum(1, dtype=f32)
        act = _tanh32(r, 4.0 if mistake == "tanh_cap4" else 40.0)
    return act, r, logp


ACT_MISTAKES = {"no_last_bias": "floor", "no_min_std": "floor", "jac1": "raw", "sp_sign": "raw", "tanh_cap4": "raw",
                "norm_mul": "floor", "sum_nu1": "floor"}


def _family_max(kind, fam, mistake):
    worst = 0.0
    for case in F.act_cases(kind, B)[fam]:
        O, nu, pol, mean, std, obs, key = case
        ref = X.act(kind, pol, mean, std, obs, normal_host(key, (B, nu)), O, nu)
        got = mirror_act(kind, *case, mistake=mistake)
        worst = max(worst, max(float(X.ratio(g, ref[n]).max()) for g, n in zip(got, ("act", "raw", "logp"))))
    return worst


@pytest.mark.parametrize("kind", ["ppo", "sac"])
def test_act_mirror_meets_the_bound(kind):
    for fam in F.ACT_FAMILIES:
        w = _family_max(kind, fam, None)
        print(f"{kind} mirror {fam:10s} {w:.3f}")
        assert w <= K, f"{kind} {fam}: the unmutated mirror is {w:.3g} radii away"


@pytest.mark.parametrize("mistake", sorted(ACT_MISTAKES))
@pytest.mark.parametrize("kind", ["ppo", "sac"])
def test_act_mistake_leaves_the_bound(kind, mistake):
    fam = ACT_MISTAKES[mistake]
    w = _family_max(kind, fam, mistake)
    print(f"{kind} {mistake} on {fam}: {w:.3g} radii")
    assert w > K, f"{kind}: {mistake} stays within {w:.3g} radii on {fam}"


# ---- GAE --------------------------------------------------------------------------------------------------------------------------
def gae_mirror(c, mistake=None):
    """k_ppo_gae's recursion in numpy float32 (vectorised over the trajectories), then the kernel's normalisation
    (ppo_ref.gae_kernel_f32 is the kernel's exact order and the unmutated reference of this mirror)"""
    rew, disc, tr = F.gae_rows(c)
    g, lam, rs = f32(c["discount"]), f32(c["lam"]), f32(c["reward_scaling"])
    T = c["T"]
    r = (rew * rs).astype(f32)
    term = ((f32(1) - disc) * (f32(1) - tr)).astype(f32)
    if mistake == "swap":
        term, tr = tr, term
    tm = (f32(1) - tr).astype(f32)
    v = c["values"][:T]
    boot = c["values"][T - 1] if mistake == "boot_last" else c["values"][T]
    vs = np.zeros_like(v)
    acc, vnext = np.zeros_like(boot), boot
    for t in range(T - 1, -1, -1):
        delta = ((r[t] + g * (f32(1) - term[t]) * vnext - v[t]) * tm[t]).astype(f32)
        keep = f32(1) if mistake == "no_trunc_mask" else tm[t]
        acc = (delta + g * (f32(1) - term[t]) * keep * lam * acc).astype(f32)
        vs[t] = acc + v[t]
        vnext = v[t]
    vsn = np.concatenate([vs[1:], boot[None]], 0)
    adv = ((r + g * (f32(1) - term) * vsn - v) * tm).astype(f32)
    m = adv.mean(dtype=f32)
    sd = np.sqrt(((adv - m) ** 2).mean(dtype=f32))
    return vs, ((adv - m) / (sd + f32(1e-8))).astype(f32)


def gae_check(c, vs_got, adv_got, depth=None):
    """(largest ratio of vs, of the normalised advantages) against the float64 reference"""
    rew, disc, tr = F.gae_rows(c)
    vs, adv = X.gae(rew, disc, tr, c["values"], c["reward_scaling"], c["discount"], c["lam"])
    n, info = X.normalize_advantages(adv, X.gae_depth(c["mb"], c["T"]) if depth is None else depth)
    return float(X.ratio(vs_got, vs).max()), float(X.ratio(adv_got, n).max()), vs, adv, n, info


GAE_SHAPES = [(1, 1), (5, 7), (20, 31), (5, 33), (1, 1023), (5, 1024), (20, 1025), (5, 4096)]


def gae_case_list():
    out = []
    for fam in F.GAE_FAMILIES:
        for k, (T, mb) in enumerate(GAE_SHAPES if fam in ("mild", "offset", "constant") else GAE_SHAPES[:4]):
            out.append((fam, F.gae_case(fam, T, mb, seed=k, params=F.GAE_PARAMS[k % len(F.GAE_PARAMS)])))
    return out


def test_gae_restatement_within_the_bound():
    """ppo_ref.gae_kernel_f32 (k_ppo_gae's order; the GPU suite keeps the two bit-equal) on every family and shape"""
    worst = {}
    for fam, c in gae_case_list():
        vs32, adv32 = ppo_ref.gae_kernel_f32(c["reward"], c["disc"], c["trunc"], c["values"], c["traj"], c["B"], c["T"],
                                             c["reward_scaling"], c["discount"], c["lam"])
        qv, qa, vs, adv, n, info = gae_check(c, vs32, adv32)
        assert qv <= K and qa <= K, f"{fam} T={c['T']} mb={c['mb']}: vs {qv:.3g}, advantages {qa:.3g} radii"
        w = worst.setdefault(fam, [0.0, 0.0])
        w[0], w[1] = max(w[0], qv), max(w[1], qa)
        assert np.isfinite(vs.r).all() and np.isfinite(n.r).all()
        assert (vs.r / (1 + np.abs(vs.v))).max() <= GAE_RADIUS_CAP and (adv.r / (1 + np.abs(adv.v))).max() <= GAE_RADIUS_CAP
        if info["s_lo"] > 0.5 * info["std"]:     # the std is known; elsewhere only the numerator is (rl_ref.normalize_advantages)
            assert (n.r / (1 + np.abs(n.v))).max() <= NORM_RADIUS_CAP.get(fam, NORM_RADIUS_DEFAULT), \
                f"{fam}: normalised radius {(n.r / (1 + np.abs(n.v))).max():.3g}"
    for fam, (a, b) in worst.items():
        print(f"gae {fam:12s} largest ratio vs {a:.3f}  normalised advantages {b:.3f}")


GAE_MISTAKES = {"no_trunc_mask": "mild", "swap": "both", "boot_last": "none"}


def test_gae_mirror_meets_the_bound():
    for fam, c in gae_case_list():
        vs, adv = gae_mirror(c)
        qv, qa, *_ = gae_check(c, vs, adv, depth=X.gae_depth(c["mb"], c["T"]) + c["T"] * c["mb"])   # numpy's sum: any order
        assert qv <= K and qa <= K, f"{fam} T={c['T']} mb={c['mb']}: mirror vs {qv:.3g}, advantages {qa:.3g}"


@pytest.mark.parametrize("mistake", sorted(GAE_MISTAKES))
def test_gae_mistake_leaves_the_bound(mistake):
    fam = GAE_MISTAKES[mistake]
    w = 0.0
    for f, c in gae_case_list():
        if f == fam:
            vs, adv = gae_mirror(c, mistake)
            w = max(w, max(gae_check(c, vs, adv, depth=X.gae_depth(c["mb"], c["T"]) + c["T"] * c["mb"])[:2]))
    print(f"gae {mistake} on {fam}: {w:.3g} radii")
    assert w > K


def test_gae_constant_advantages_are_exact():
    """every advantage equal: the fp32 mean is exact and the normalised advantages are exactly 0 (the bound there is only
    the numerator's; rl_ref.normalize_advantages)"""
    c = F.gae_case("constant", 5, 1024)
    _, adv32 = ppo_ref.gae_kernel_f32(c["reward"], c["disc"], c["trunc"], c["values"], c["traj"], c["B"], c["T"],
                                      c["reward_scaling"], c["discount"], c["lam"])
    assert np.all(adv32 == 0)


# ---- statistics -------------------------------------------------------------------------------------------------------------------
ROWS = 256


def stats_mirror(state, x, mistake=None):
    """k_ppo_stat_partial / _final in numpy float64: chunk sums about the batch's first row, rows ascending, chunks in order,
    then the pairwise combination with the old state; std = clip(sqrt(sv / count)), both rounded once to fp32"""
    count, mean, sv = state
    x = np.asarray(x, np.float64)
    n = x.shape[0]
    c = x[0] if mistake != "old_shift" else mean
    s1 = np.zeros(x.shape[1])
    s2 = np.zeros(x.shape[1])
    for r0 in range(0, n, ROWS):
        d = x[r0:r0 + ROWS] - c
        a1, a2 = np.zeros_like(s1), np.zeros_like(s2)
        for row in d:
            a1, a2 = a1 + row, a2 + row * row
        s1, s2 = s1 + a1, s2 + a2
    new_count = count + n
    if mistake == "old_shift":                      # the parent's form: summed_var += S2 - (S1 / count) S1 about the old mean
        mu = s1 / new_count
        new_mean, new_sv = mean + mu, sv + (s2 - mu * s1)
    else:
        mb = s1 / n
        m2 = s2 - mb * s1
        delta = (c + mb) - mean
        new_mean = mean + delta * (n / new_count)
        if mistake == "old_mean_only":
            new_sv = sv + ((x - mean) ** 2).sum(0)
        else:
            new_sv = sv + m2 + delta * delta * (count * (n / new_count))
    denom = new_count - 1 if mistake == "n_minus_1" else new_count
    std = np.clip(np.sqrt(new_sv / denom), 1e-6, 1e6)
    return (new_count, new_mean, new_sv), new_mean.astype(f32), std.astype(f32)


STAT_SHAPES = {"mild": [(5, 300, 3), (128, 257, 2)], "offset": [(3, 1000, 3), (128, 600, 2)], "constant": [(4, 256, 3)],
               "wide": [(2, 513, 2)], "count": [(1, 1 << 20, 17)]}     # (O, rows, updates)


def stat_run(fam, fn, mistake=None):
    """largest ratio of the stored mean and std over the family's update sequences"""
    worst = 0.0
    for O, rows, updates in STAT_SHAPES[fam]:
        st = st_m = (0.0, np.zeros(O), np.zeros(O))
        for x in F.stat_batches(fam, O, rows, updates):
            st, ref = X.stats_update(st, x, -(-rows // ROWS))
            st_m, mean32, std32 = fn(st_m, x, mistake)
            worst = max(worst, float(X.ratio(mean32, ref["mean"]).max()), float(X.ratio(std32, ref["std"]).max()))
        if fam == "count":
            assert st[0] > 2 ** 24
    return worst


def test_stats_mirror_meets_the_bound():
    for fam in F.STAT_FAMILIES:
        w = stat_run(fam, stats_mirror)
        print(f"stats mirror {fam:9s} {w:.3f}")
        assert w <= K, f"{fam}: {w:.3g} radii"


STAT_MISTAKES = {"n_minus_1": "mild", "old_mean_only": "mild", "old_shift": "offset"}


@pytest.mark.parametrize("mistake", sorted(STAT_MISTAKES))
def test_stats_mistake_leaves_the_bound(mistake):
    fam = STAT_MISTAKES[mistake]
    w = stat_run(fam, stats_mirror, mistake)
    print(f"stats {mistake} on {fam}: {w:.3g} radii")
    assert w > K


def test_stats_radii_are_tight():
    """the stored words are the fp32 roundings of the float64 statistics: every radius within 1.01 u |value| plus 1e-12 of it"""
    for fam in F.STAT_FAMILIES:
        O, rows, updates = STAT_SHAPES[fam][0]
        st = (0.0, np.zeros(O), np.zeros(O))
        for x in F.stat_batches(fam, O, rows, updates):
            st, ref = X.stats_update(st, x, -(-rows // ROWS))
            for k in ("mean", "std"):
                assert np.all(ref[k].r <= 1.01 * X.U * np.abs(ref[k].v) + 1e-12 * (1 + np.abs(ref[k].v))), f"{fam} {k}"
