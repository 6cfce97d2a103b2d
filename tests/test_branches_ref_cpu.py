"""The samples the float64 references leave undecided, held to one of their branch outcomes.  No GPU needed.

Where a discontinuous predicate's margin is within its radius and its outcomes lie more than JUMP radii apart, the references
mark the sample `undecided`, and the other CPU files only bound how many there are.  A fp32 evaluation there may take
either outcome, but downstream of it computes that outcome's formula; so each undecided sample is held to K radii of ONE
consistent assignment of its gated predicates (tests/xpbd_ref.py `branch_outcomes`, tests/car2d_ref.py
`check_rollout_branches`, tests/pusht_ref.py `held_ratios`), on the oracle and the cases of the existing CPU files:
* one XPBD substep: xpbd_families x the shipped envs, contact_params and the twelve modelgen models;
* the XPBD substep chains and the relaunched horizons of tests/test_horizon_ref_cpu.py;
* the car2d families; the pushT families at mu = 1 and 0 in both solver modes.
Per family it prints undecided / held / unchecked, the largest held ratio and the median distance to the second-best
assignment in radii (large: the branch is identified, not just covered).  Then the forcing itself is checked (the decided
outcome forced reproduces the reference bit for bit; a contact site moves only its own link's words), and each of the
mistakes the hull accepts is shown to fail the new check while it passes the existing one."""
import numpy as np
import pytest

from tests import car2d_families as CF
from tests import car2d_ref as CX
from tests import horizon_ref as HR
from tests import pusht_families as PF
from tests import pusht_ref as PX
from tests import xpbd_families as F
from tests import xpbd_ref as X
from tests.test_car2d_ref_cpu import oracle_run as car_run
from tests.test_horizon_ref_cpu import CHAIN_MODELS, N_CHAIN, envs, horizons, memo, oracle_run  # noqa: F401  (fixtures)
from tests.test_pusht_ref_cpu import MUS, n_of, table
from tests.test_pusht_ref_cpu import _oracle as pusht_oracle
from tests.test_xpbd_ref_cpu import MODELS, N
from tests.test_xpbd_ref_cpu import _oracle_step as xpbd_oracle

K = 2.0
# largest fraction of a (model, family)'s undecided samples left unchecked (a forced evaluation gated a new site, or more
# than 2^MAX_BITS assignments).  Measured 0 on every case of this file; none may appear.
UNCHECKED_CAP = 0.0


@pytest.fixture(scope="module")
def xpbd_cases(tmp_path_factory):
    """{(model, family): [(blob, state, actions, reference)]}: the launches of tests/test_xpbd_ref_cpu.py"""
    tmp = tmp_path_factory.mktemp("models")
    out = {}
    for name in MODELS:
        env = F.make_env(name, tmp)
        for fam in F.FAMILIES:
            for st, u in F.build(env, fam, N):
                out.setdefault((name, fam), []).append((env.blob, st, u, X.positional_step(env.blob, np.broadcast_to(st, (N,) + st.shape), u)))
    return out


@pytest.fixture(scope="module")
def car_cases():
    """{family: [(x0, Y, xref)]}: the cases of tests/test_car2d_ref_cpu.py"""
    env = CF.car()
    out = {}
    for fam in CF.FAMILIES[:-1]:
        st, u = CF.one_step(fam, env.params)
        out[fam] = [(st, u[:, None], None)]
    out["demo"] = [(x0, Y, env.xref) for x0, Y in CF.rollouts(env.params, env.xref)]
    return out


@pytest.fixture(scope="module")
def pusht_cases():
    """{(mu, family): [(params, state, controls, reference)]}: the cases of tests/test_pusht_ref_cpu.py"""
    return {(mu, fam): [(table(mu), st, u, PX.step(table(mu), st, u)) for st, u in PF.build(fam, n_of(fam))]
            for mu in MUS for fam in PF.FAMILIES}


def _line(what, und, held, unchecked, worst, second):
    sec = f"{np.median(second):.3g}" if len(second) else "-"
    print(f"{what:38s} undecided {und:5d}  held {held:5d}  unchecked {unchecked:3d}  largest held {worst:6.3f}  "
          f"median second-best {sec}")


def _held(blob, states, actions, ref, got):
    """(held ratios, second-best distances, unchecked count) of the undecided rows of one launch"""
    if not ref["undecided"].any():
        return np.zeros(0), np.zeros(0), 0
    br = X.branch_outcomes(blob, states, actions, ref)
    best, second = X.held_ratios(np.asarray(got)[br["rows"]], br)
    ok = ~br["still"]
    return best[ok], second[ok], int((~ok).sum())


# ---------------------------------------------------------------------------------------------------------------------
# XPBD: one substep, the substep chains, the relaunched horizons
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def xpbd_held(xpbd_cases):
    """{(model, family): (undecided, held ratios, second-best, unchecked)} of the oracle's one-substep launches"""
    out = {}
    for (name, fam), launches in xpbd_cases.items():
        und, held, second, unc = 0, [], [], 0
        for blob, st, u, ref in launches:
            S = np.broadcast_to(st, (N,) + st.shape)
            b, s, c = _held(blob, S, u, ref, xpbd_oracle(blob, st, u))
            und, unc = und + int(ref["undecided"].sum()), unc + c
            held += list(b)
            second += list(s)
        out[(name, fam)] = (und, np.array(held), np.array(second), unc)
    return out


def test_xpbd_one_substep_undecided_held(xpbd_held):
    total = 0
    for (name, fam), (und, held, second, unc) in xpbd_held.items():
        if not und:
            continue
        total += und
        _line(f"xpbd {name} {fam}", und, len(held), unc, held.max(initial=0.0), second)
        assert unc <= UNCHECKED_CAP * und, f"{name} {fam}: {unc} of {und} undecided samples unchecked"
        assert held.max(initial=0.0) <= K, f"{name} {fam}: best assignment {held.max():.3g} radii"
    assert total > 50          # the undecided zone is populated


def test_xpbd_substep_chain_undecided_held(envs, memo):
    tot_und = 0
    for name in CHAIN_MODELS:
        env = envs[name]
        run = oracle_run(env.blob)
        nsub = int(env.blob.view(np.int32)[3])
        for fam in F.FAMILIES:
            und, held, second, unc = 0, [], [], 0
            for st, u in F.build(env, fam, N_CHAIN):
                ch = HR.substep_chain(run, st, u, nsub)
                prev, got = np.concatenate(ch[:-1]), np.concatenate(ch[1:])
                _, q, c, info = HR.step_ratios(memo, env.blob, prev, np.tile(u, (nsub, 1)), got)
                und, unc = und + info["undecided"], unc + c
                held += info["held"]
                second += info["second"]
            if und:
                tot_und += und
                _line(f"chain {name} {fam}", und, len(held), unc, max(held, default=0.0), second)
                assert unc <= UNCHECKED_CAP * und, f"{name} {fam}: {unc} of {und} unchecked"
                assert max(held, default=0.0) <= K, f"{name} {fam}: best assignment {max(held):.3g} radii"
    assert tot_und > 0


def test_xpbd_relaunched_horizon_undecided_held(horizons, memo):
    per = {}
    for name, label, H_, blob, st, Y, full, traj, xref, rel in horizons:
        prev, got, u = [], [], []
        for (b, t), ch in rel.items():
            prev += ch[:-1]
            got += ch[1:]
            u += [Y[b, t]] * (len(ch) - 1)
        _, q, c, info = HR.step_ratios(memo, blob, np.stack(prev), np.stack(u), np.stack(got))
        a = per.setdefault(name, [0, [], [], 0])
        a[0] += info["undecided"]
        a[1] += info["held"]
        a[2] += info["second"]
        a[3] += c
    for name, (und, held, second, unc) in per.items():
        if und:
            _line(f"horizon {name}", und, len(held), unc, max(held, default=0.0), second)
        assert unc <= UNCHECKED_CAP * max(und, 1), f"{name}: {unc} of {und} unchecked"
        assert max(held, default=0.0) <= K, f"{name}: best assignment {max(held):.3g} radii"
    assert per["gen0"][0] > 0


def test_forcing_the_decided_outcome_is_the_reference(xpbd_cases):
    """forcing every predicate instance to the outcome float64 took reproduces value and radius bit for bit on the decided
    samples; forcing a decided instance the other way is refused"""
    tried = 0
    for (name, fam), launches in xpbd_cases.items():
        for blob, st, u, ref in launches[:1]:
            S = np.broadcast_to(st, (N,) + st.shape)
            force = {k: v.astype(np.int8) for k, v in ref["outcomes"].items()}
            again = X.positional_step(blob, S, u, force)
            ok = ~ref["undecided"]
            assert np.array_equal(again["value"][ok], ref["value"][ok]), (name, fam)
            assert np.array_equal(again["radius"][ok], ref["radius"][ok]), (name, fam)
            tried += 1
    assert tried >= len(MODELS) * 3
    blob, st, u, ref = xpbd_cases[("humanoidrun", "F1")][0]
    key = ("dq.w >= 0",)
    with pytest.raises(ValueError):
        X.positional_step(blob, np.broadcast_to(st, (N,) + st.shape), u, {key: (~ref["outcomes"][key]).astype(np.int8)})


def test_a_contact_site_moves_only_its_own_link(xpbd_cases):
    """the per-link factorisation branch_outcomes relies on: the two outcomes of a contact site differ in no word outside
    its link (and do differ inside it)"""
    seen = 0
    for (name, fam), launches in xpbd_cases.items():
        for blob, st, u, ref in launches:
            if not ref["undecided"].any():
                continue
            S = np.broadcast_to(st, (N,) + st.shape)
            for key, mask in ref["sites"].items():
                i, l = np.argwhere(mask)[0]
                outs = []
                for v in (0, 1):
                    f = np.full(mask.shape, -1, np.int8)
                    f[i, l] = v
                    outs.append(X.positional_step(blob, S[i:i + 1], u[i:i + 1], {key: f[i:i + 1]})["value"][0])
                other = np.arange(outs[0].shape[0]) != l
                assert np.array_equal(outs[0][other], outs[1][other]), (name, fam, key)
                assert not np.array_equal(outs[0][l], outs[1][l]), (name, fam, key)
                seen += 1
    assert seen >= 10


# ---------------------------------------------------------------------------------------------------------------------
# car2d and pushT
# ---------------------------------------------------------------------------------------------------------------------
def test_car2d_undecided_held(car_cases):
    P = CF.car().params
    seen = 0
    for fam, launches in car_cases.items():
        und, best, second = 0, [], []
        for x0, Y, xref in launches:
            res = CX.check_rollout_branches(P, x0, Y, car_run(P, x0, Y, xref))
            und += res["undecided"]
            best += list(res["best"])
            second += list(res["second"])
        if und:
            seen += und
            _line(f"car2d {fam}", und, len(best), 0, max(best), second)
            assert max(best) <= K, f"{fam}: {max(best):.3g} radii from both outcomes"
    assert seen > 0


@pytest.mark.parametrize("mode", ["fixed", "prod"])
def test_pusht_undecided_held(pusht_cases, mode):
    seen = 0
    for (mu, fam), launches in pusht_cases.items():
        und, best, second = 0, [], []
        for P, st, u, ref in launches:
            if not ref["undecided"].any():
                continue
            b, s = PX.held_ratios(pusht_oracle(P, st, u, mode), ref, mode)
            und += len(b)
            best += list(b)
            second += list(s)
        if und:
            seen += und
            _line(f"pushT {mode} mu={mu} {fam}", und, len(best), 0, max(best), second)
            assert max(best) <= K, f"{mode} mu={mu} {fam}: {max(best):.3g} radii from every configuration"
    assert seen > 0


# ---------------------------------------------------------------------------------------------------------------------
# the check is not vacuous: mistakes the per-stage hull accepts, each failing the new check
# ---------------------------------------------------------------------------------------------------------------------
def _blend(br, j, got_row):
    """the midpoint of the two outcomes of every link with a site (the rest as computed)"""
    out = np.asarray(got_row, np.float64).copy()
    for l in range(out.shape[0]):
        ok = np.flatnonzero(br["valid"][j, :, l])
        if len(ok) > 1:
            out[l] = 0.5 * (br["value"][j, ok[0], l] + br["value"][j, ok[1], l])
    return out


def test_mistake_midpoint_blend(xpbd_cases, car_cases, pusht_cases):
    """the midpoint of the two outcomes (the static-friction impulse halved in the gated zone; the car halfway between q
    and q_new; the mean of pushT's two face configurations) is inside the hull the existing check accepts"""
    worst = {}
    for (name, fam), launches in xpbd_cases.items():
        for blob, st, u, ref in launches:
            if not ref["undecided"].any():
                continue
            S = np.broadcast_to(st, (N,) + st.shape)
            br = X.branch_outcomes(blob, S, u, ref)
            got = xpbd_oracle(blob, st, u).copy()
            for j, i in enumerate(br["rows"]):
                got[i] = _blend(br, j, got[i])
            assert HR.ratio(got, ref["value"], ref["radius"], np.broadcast_to(~ref["undecided"][:, None, None], got.shape)) <= K
            b, _ = X.held_ratios(got[br["rows"]], br)
            worst["xpbd"] = max(worst.get("xpbd", 0.0), float(b.min()))
    P = CF.car().params
    for fam, launches in car_cases.items():
        for x0, Y, xref in launches:
            o = car_run(P, x0, Y, xref)
            n, H, _ = Y.shape
            prev = np.concatenate([np.broadcast_to(np.reshape(x0, (-1, 1, 3)), (n, 1, 3)), o["traj"][:, :-1]], 1).reshape(-1, 3)
            ref = CX.step(P, prev, Y.reshape(-1, 2))
            und = ref["undecided"]
            if not und.any():
                continue
            traj = o["traj"].reshape(-1, 3).copy()
            traj[und] = (0.5 * (prev[und].astype(np.float64) + ref["new_value"][und])).astype(np.float32)
            best, _ = CX.held_steps(prev, traj, ref)
            worst["car2d"] = max(worst.get("car2d", 0.0), float(best.min()))
    for (mu, fam), launches in pusht_cases.items():
        for P, st, u, ref in launches:
            if not ref["undecided"].any() or len(ref["configs"]) < 2:
                continue
            got = pusht_oracle(P, st, u, "fixed").copy()
            und = ref["undecided"]
            got[und] = np.mean([c["value"][und] for c in ref["configs"]], 0).astype(np.float32)
            b, _ = PX.held_ratios(got, ref, "fixed")
            worst["pushT"] = max(worst.get("pushT", 0.0), float(b.min()))
    print("midpoint blend, smallest best-assignment distance (radii):", {k: round(v, 1) for k, v in worst.items()})
    assert set(worst) == {"xpbd", "car2d", "pushT"}
    for k, v in worst.items():
        assert v > K, f"{k}: the midpoint blend is within {v:.3g} radii of a consistent assignment"


def test_mistake_contact_test_split_between_stages(xpbd_cases):
    """dist < 0 decided separately in the position and the velocity stage.  A kernel that recomputes the predicate with
    another association order in each stage can take one outcome in each; this test stands in for it by splicing the two
    forced evaluations of a sample whose only site is one contact test: the link's positions and orientation from one
    outcome, its velocities from the other (the velocity stage acts on velocities only; the other outcome's project_xd
    velocities differ from the spliced kernel's by the position-stage change, which is within the radius at dist = 0).
    At dist = 0 the position stage is continuous (dl vanishes with dist), so only the split that collides in the position
    stage and not in the velocity stage leaves the velocity the position change implies uncorrected; that one must fail the
    new check somewhere"""
    worst = {}
    for (name, fam), launches in xpbd_cases.items():
        for blob, st, u, ref in launches:
            keys = [k for k in ref["sites"] if k[0] == "dist < 0"]
            if not keys:
                continue
            S = np.broadcast_to(st, (N,) + st.shape)
            br = X.branch_outcomes(blob, S, u, ref)
            got = xpbd_oracle(blob, st, u)
            for j, i in enumerate(br["rows"]):
                for key in keys:
                    for l in np.flatnonzero(ref["sites"][key][i]):
                        if X.instances(ref["sites"], i, got.shape[1]) != [(key, l)]:
                            continue
                        v0, v1 = br["value"][j, 0], br["value"][j, 1]
                        for split, (pq, vw) in (("position collides", (v1, v0)), ("velocity collides", (v0, v1))):
                            fake = got[i].astype(np.float64)
                            fake[l, :7], fake[l, 7:] = pq[l, :7], vw[l, 7:]
                            b, _ = X.held_ratios(fake[None], dict(rows=[i], value=br["value"][j:j + 1], radius=br["radius"][j:j + 1],
                                                                  valid=br["valid"][j:j + 1], whole=br["whole"][j:j + 1]))
                            worst[split] = max(worst.get(split, 0.0), float(b[0]))
    print("contact test split between the stages, largest best-assignment distance (radii):",
          {k: round(v, 2) for k, v in worst.items()})
    assert "position collides" in worst, "no sample whose only site is one contact test"
    assert worst["position collides"] > K


# ---------------------------------------------------------------------------------------------------------------------
# constructed states for the sites no family reaches: a hinge at pi (the atan2 cut of a spring or a finite limit) and a
# link spun at 1e7 rad/s about z (dq.w within its radius after one substep)
# ---------------------------------------------------------------------------------------------------------------------
CUT_CASES = [("hopper", 2, 0), ("walker2d", 5, 0), ("humanoidrun", 3, 1), ("halfcheetah", 3, 0)]   # (model, link, dof)
SPIN_CASES = [("humanoidrun", 0), ("humanoidrun", 1), ("ant", 0), ("cartpole", 1)]                # (model, link)
N_SITE = 16
SPIN = 1e7
SPIN_AXIS = (0.0, 0.0, 1.0)


def _parents(blob):
    L = int(blob.view(np.int32)[X.B.H_NLINK])
    return blob.view(np.int32)[X.B.HDR_WORDS + X.B.F_PARENT * X.B.MAXL:][:L]


@pytest.fixture(scope="module")
def site_cases(tmp_path_factory):
    """[(label, kind, blob, state, actions, reference)]: kind 'cut' (the hinge (link, dof) at its reference + pi, at rest)
    or 'spin' (the reset pose at rest, one link spinning at SPIN rad/s about SPIN_AXIS)"""
    tmp = tmp_path_factory.mktemp("sites")
    out = []
    for name, l, k in CUT_CASES:
        env = F.make_env(name, tmp)
        (qi, d), = [(qi, d) for (l_, k_, qi, d) in F._hinges(env.sys, env._links) if (l_, k_) == (l, k)]
        q = env.sys.init_q.astype(np.float64).copy()
        q[qi] = env.sys.ref(d) + np.pi
        st = F._init(env, q, np.zeros(env.sys.qd_size()))
        u = F.actions(env.action_size, N_SITE, 3)
        out.append((f"{name} hinge {l}.{k} at pi", "cut", env.blob, st, u,
                    X.positional_step(env.blob, np.broadcast_to(st, (N_SITE,) + st.shape), u)))
    for name, l in SPIN_CASES:
        env = F.make_env(name, tmp)
        st = F._init(env, env.sys.init_q, np.zeros(env.sys.qd_size())).copy()
        st[l, 7:10] = np.multiply(SPIN_AXIS, SPIN)
        u = F.actions(env.action_size, N_SITE, 3)
        out.append((f"{name} link {l} spun", "spin", env.blob, st, u,
                    X.positional_step(env.blob, np.broadcast_to(st, (N_SITE,) + st.shape), u)))
    return out


def test_constructed_sites_held(site_cases):
    """every constructed case gates the site it is built for on every sample; a cut sample goes through the whole-sample
    enumeration; the oracle is held to one assignment and the other is far"""
    kinds = set()
    for label, kind, blob, st, u, ref in site_cases:
        want = ("atan2 cut (spring)", "atan2 cut (limit)") if kind == "cut" else ("dq.w >= 0",)
        gated = [key for key in ref["sites"] if key[0] in want]
        assert gated and ref["undecided"].any(), f"{label}: {sorted(ref['sites'])}"
        kinds |= {key[0] for key in gated}
        br = X.branch_outcomes(blob, np.broadcast_to(st, (N_SITE,) + st.shape), u, ref)
        assert not br["still"].any(), f"{label}: {int(br['still'].sum())} unchecked"
        assert br["whole"].all() == (kind == "cut")
        best, second = X.held_ratios(xpbd_oracle(blob, st, u)[br["rows"]], br)
        _line(label, len(best), len(best), 0, best.max(), second)
        assert best.max() <= K, f"{label}: best assignment {best.max():.3g} radii"
        assert np.median(second) > K, f"{label}: the branch is not identified"
    assert kinds == {"atan2 cut (spring)", "atan2 cut (limit)", "dq.w >= 0"}


def test_cut_and_dq_w_sites_factorise(site_cases):
    """forcing one site changes words only where branch_outcomes assumes: a dq.w site its own link; a limit cut (joint
    solve) its link and the parent; a spring cut (acceleration update: the link's and the parent's angular velocity, then
    every joint that reads either) its link, the parent, the grandparent and the children of both"""
    for label, kind, blob, st, u, ref in site_cases:
        par = _parents(blob)
        kids = lambda l: set(np.flatnonzero(par == l).tolist())   # noqa: E731
        S = np.broadcast_to(st, (1,) + st.shape)
        for key, mask in ref["sites"].items():
            l = int(np.flatnonzero(mask[0])[0])
            outs = []
            for v in (0, 1):
                f = np.full((1, mask.shape[1]), -1, np.int8)
                f[0, l] = v
                outs.append(X.positional_step(blob, S, u[:1], {key: f})["value"][0])
            moved = set(np.flatnonzero((outs[0] != outs[1]).any(-1)).tolist())
            p = int(par[l])
            if key[0] == "dq.w >= 0":
                allowed = {l}
            elif key[0] == "atan2 cut (limit)":
                allowed = {l, p}
            else:
                allowed = {l, p} | kids(l) | (kids(p) if p >= 0 else set()) | ({int(par[p])} if p >= 0 else set())
            allowed.discard(-1)
            assert l in moved and moved <= allowed, f"{label} {key}: link {l} moved {sorted(moved)}, allowed {sorted(allowed)}"


def test_mistake_dq_w_sign_in_one_component(site_cases):
    """project_xd's dq.w sign taken from the other branch in one component of w only: the kernel's own result with one
    component of w replaced by the other branch's (the component for which that lands farthest from both), on the samples
    whose two branches differ in at least two components of w (where they differ in one, that flip is the consistent
    one).  The existing check does not look at these samples; this one must find each far from both consistent outcomes"""
    worst = np.inf
    for label, kind, blob, st, u, ref in site_cases:
        if kind != "spin":
            continue
        S = np.broadcast_to(st, (N_SITE,) + st.shape)
        br = X.branch_outcomes(blob, S, u, ref)
        got = xpbd_oracle(blob, st, u)[br["rows"]].astype(np.float64)
        l = int(np.flatnonzero(ref["sites"][("dq.w >= 0",)][br["rows"][0]])[0])
        for j in range(len(br["rows"])):
            d = [(np.abs(got[j, l] - br["value"][j, a, l]) / br["radius"][j, a, l]).max() for a in (0, 1)]
            near, far = (0, 1) if d[0] <= d[1] else (1, 0)
            sep = np.abs(br["value"][j, near, l, 7:10] - br["value"][j, far, l, 7:10]) / np.maximum(
                br["radius"][j, near, l, 7:10], br["radius"][j, far, l, 7:10])
            if (sep > 2 * K).sum() < 2:
                continue        # the branches differ in one component of w only: flipping it is the consistent flip
            dist = []
            for c in (7, 8, 9):
                fake = got.copy()
                fake[j, l, c] = br["value"][j, far, l, c]
                dist.append(float(X.held_ratios(fake, br)[0][j]))
            worst = min(worst, max(dist))
            assert max(dist) > K, f"{label} sample {j}: a one-component dq.w flip is within {max(dist):.3g} radii"
    print("dq.w sign in one component, smallest best-assignment distance (radii):", round(worst, 1))
    assert np.isfinite(worst), "no sample whose dq.w branches differ in two components of w"
