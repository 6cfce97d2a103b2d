"""The CPU oracle's rollout loop against the float64 horizon reference (tests/horizon_ref.py).  No GPU needed.

tests/test_xpbd_ref_cpu.py holds one substep from a constructed state and one reward.  This file holds the loop around
them, every piece teacher-forced on the oracle's own fp32 states:
* the substep chain: s_k = rollout(nsub_override = k).final against positional_step(s_{k-1}, u), k = 1 .. n_frames, on
  every family state of every shipped positional env, the contact fixture and random models;
* the env-step chain at H = 50 (and H = 60 for humanoidtrack, past the 50 demo rows): the state after every step from
  prefix runs, each prefix run's rewss equal to the full run's bit for bit; every step's reward, the tracked positions,
  the return (from the exact fp32 rewards and from the float64 rewards) and the demo log-density;
* along the horizon, for a few samples: every substep of every env step relaunched one substep at a time from the
  state the loop reached, ending on the loop's own next state bit for bit and each substep within the bound.
Then each slip of the loop that the oracle and the kernels could share is shown to leave the bound on some case."""
import numpy as np
import pytest

import mbd_b200
from mbd_b200.model import blob as B
from oracle import oracle as orc
from tests import horizon_ref as HR
from tests import xpbd_families as F

K = 2.0
N_CHAIN = 33             # samples per family state in the substep chain
N_HORIZON = 16           # samples per start in the env-step chain
N_RELAUNCH = 3           # of which relaunched substep by substep along the horizon
H = 50
CHAIN_MODELS = F.SHIPPED + ["contact_params"] + [f"gen{s}" for s in F.MODELGEN_SEEDS]
# the random models other than gen0 and gen100 blow up to inf / NaN within 50 env steps under random actions (gen2, for
# one, from every start): they take part in the substep chain only
HORIZON_MODELS = F.SHIPPED + ["contact_params", "gen0", "gen100"]

# largest fraction of undecided substeps (tests/xpbd_ref.py: a branch within its radius whose outcomes differ by more
# than JUMP radii) along the chains.  Measured with the oracle (bit-identical to every kernel), then rounded up; the
# measurement is given beside each cap.  Every (model, family) not listed measured 0.  The states of a chain leave the
# constructed corners, so these are not the one-substep caps of tests/xpbd_families.py (contact_params, for one, is
# decided everywhere after one substep and not after five).
CHAIN_UNDECIDED = {("ant", "F1"): 0.01,                 # measured 0.0091: the feet rest on the floor in the reset pose
                   ("ant", "F2"): 0.03,                 # 0.0242
                   ("ant", "F3"): 0.0015,               # 0.0008; 0.0014 at 129 samples per state (the GPU test's n)
                   ("hopper", "F1"): 0.001,             # 0 here; 0.00097 at 129 samples
                   ("walker2d", "F2"): 0.0015,          # 0 here; 0.00078 at 129 samples, 0.0013 (2 of 1540) at 77
                   ("humanoidstandup", "F1"): 0.005,    # 0.0043: lies on the floor
                   ("humanoidstandup", "F2"): 0.005,    # 0.0043
                   ("humanoidstandup", "F3"): 0.01,     # 0.0087
                   ("humanoidstandup", "F4"): 0.015,    # 0.0119
                   ("halfcheetah", "F6"): 0.001}        # 0.0003
CHAIN_UNDECIDED_F5 = 0.03                               # contacts at the floor: largest 0.026 (humanoidrun)
# along the horizon, per model over every start (N_RELAUNCH samples x H steps x n_frames substeps); the largest fraction
# measured beside each cap.  gen0 (14 links, 18 contacts) falls onto the floor within a few steps and stays there.
HORIZON_UNDECIDED = {"humanoidrun": 0.05,               # 0.0429
                     "humanoidstandup": 0.06,           # 0.0552
                     "humanoidtrack": 0.05,             # 0.0493
                     "hopper": 0.003,                   # 0.0020
                     "walker2d": 0.012,                 # 0.0100
                     "ant": 0.012,                      # 0.0107
                     "halfcheetah": 0.008,              # 0.0071
                     "cartpole": 0.0,                   # 0
                     "contact_params": 0.006,           # 0.0053
                     "gen0": 0.36,                      # 0.3489
                     "gen100": 0.005}                   # 0.0044


def chain_undecided_cap(model, fam):
    return CHAIN_UNDECIDED.get((model, fam), CHAIN_UNDECIDED_F5 if fam == "F5" else 0.0)


def oracle_run(blob):
    ntrack = int(np.asarray(blob).view(np.int32)[5])

    def run(st, Y, nsub=0, xref=None):
        return orc.xpbd_rollout(blob, st, Y, xref=xref, want_rewss=True, want_final=True, want_track=ntrack > 0,
                                nsub_override=nsub)
    return run


def horizon_actions(nu, n, H_, seed):
    """a different action per sample and step: N(0, 0.7) clipped to the control range, sample 0 saturated at +-37 (bang-bang
    at the control limits, the sample most likely to blow up, see horizon_ref.finite_samples)"""
    rng = np.random.default_rng(seed)
    Y = np.clip(rng.normal(size=(n, H_, nu)) * 0.7, -1.0, 1.0)
    Y[0] = np.where(rng.random((H_, nu)) < 0.5, -37.0, 37.0)
    return Y.astype(np.float32)


def starts(env, name):
    """the reset pose at rest (not for the random models, whose init_q is not a resting pose) and the first state of every
    family the model has"""
    sys = env.sys
    out = []
    if not name.startswith("gen"):
        out.append(("reset", np.ascontiguousarray(env.pipeline_init(sys.init_q, np.zeros(sys.qd_size())).raw, dtype=np.float32)))
    for fam in F.FAMILIES:
        b = F.build(env, fam, 8)
        if b:
            out.append((fam, b[0][0]))
    return out


def horizon_starts(env, name, run, xref):
    """(label, state, demo) of the env-step chain: every start of `starts` with the env's demo, and for a tracking env also
    the reset pose against a demo 2-8 cm off sample 0's own tracked path (the shipped demo is more than 0.5 m from random
    rollouts after a few steps, where every term of the log-density sits at its clip)"""
    out = [(label, st, xref) for label, st in starts(env, name)]
    if xref is not None:
        st = out[0][1]
        tk = run(st, horizon_actions(env.action_size, 2, xref.shape[1], 999)[1:])["track"][0]
        off = np.linspace(0.02, 0.08, xref.shape[0])[:, None, None] * np.float32([1.0, -0.5, 0.3])
        out.append(("own demo", st, (tk.transpose(1, 0, 2) + off).astype(np.float32)))
    return out


@pytest.fixture(scope="module")
def memo():
    return HR.StepMemo()


@pytest.fixture(scope="module")
def envs(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("models")
    return {name: F.make_env(name, tmp) for name in CHAIN_MODELS}


@pytest.fixture(scope="module")
def horizons(envs):
    """[(model, start, H, blob, st, Y, full, traj, xref, relaunched {(b, t): [s^0 .. s^nsub]})]"""
    out = []
    for name in HORIZON_MODELS:
        env = envs[name]
        run = oracle_run(env.blob)
        nsub = int(env.blob.view(np.int32)[3])
        xref = env.xref if name == "humanoidtrack" else None
        for si, (label, st, xr) in enumerate(horizon_starts(env, name, run, xref)):
            for H_ in ((H, 60) if xr is not None else (H,)):
                Y = horizon_actions(env.action_size, N_HORIZON, H_, 1000 + si)
                full, traj = HR.env_step_chain(run, st, Y, xr)
                prev = HR.previous_states(st, traj)
                ok = HR.finite_samples(traj)
                assert ok[1:].all(), f"{name} {label}: samples {np.flatnonzero(~ok)} left the finite range"
                rel = {}
                for b in np.flatnonzero(ok)[:N_RELAUNCH]:
                    for t in range(H_):
                        ch = HR.relaunch_chain(run, prev[b, t], Y[b, t], nsub)
                        assert HR.same_bits(ch[-1], traj[b, t]), f"{name} {label}: relaunched step {t} of sample {b}"
                        rel[(b, t)] = ch
                out.append((name, label, H_, env.blob, st, Y, full, traj, xr, rel))
    return out


def relaunch_ratio(memo, blob, Y, rel, shift=0):
    """every relaunched substep against positional_step of its predecessor under the actions of step t + shift"""
    prev, got, u = [], [], []
    for (b, t), ch in rel.items():
        tt = min(max(t + shift, 0), Y.shape[1] - 1)
        prev += ch[:-1]
        got += ch[1:]
        u += [Y[b, tt]] * (len(ch) - 1)
    return HR.step_ratio(memo, blob, np.stack(prev), np.stack(u), np.stack(got)), len(u)


# ---------------------------------------------------------------------------------------------------------------------
# the substep chain
# ---------------------------------------------------------------------------------------------------------------------
def test_substep_chain_within_the_bound(envs, memo):
    rep = {}
    for name in CHAIN_MODELS:
        env = envs[name]
        run = oracle_run(env.blob)
        nsub = int(env.blob.view(np.int32)[3])
        for fam in F.FAMILIES:
            worst, und, tot = 0.0, 0, 0
            for i, (st, u) in enumerate(F.build(env, fam, N_CHAIN)):
                ch = HR.substep_chain(run, st, u, nsub)
                prev, got = np.concatenate(ch[:-1]), np.concatenate(ch[1:])
                q, nu_ = HR.step_ratio(memo, env.blob, prev, np.tile(u, (nsub, 1)), got)
                assert q <= K, f"{name} {fam}[{i}]: substep chain {q:.3g} radii"
                worst, und, tot = max(worst, q), und + nu_, tot + len(prev)
            if tot:
                rep[(name, fam)] = (worst, und / tot)
                assert und <= chain_undecided_cap(name, fam) * tot, f"{name} {fam}: {und} of {tot} substeps undecided"
    print("substep chain, (largest ratio, undecided fraction):", {k: (round(a, 3), round(b, 4)) for k, (a, b) in rep.items()})
    assert max(a for a, _ in rep.values()) > 0.05          # the oracle is not simply the float64 value


# ---------------------------------------------------------------------------------------------------------------------
# the env-step chain
# ---------------------------------------------------------------------------------------------------------------------
def test_horizon_outputs_within_the_bound(horizons):
    rep = {}
    for name, label, H_, blob, st, Y, full, traj, xref, _ in horizons:
        res = HR.check_horizon(blob, st, Y, full, traj, xref)
        for k, v in res.items():
            assert v <= K, f"{name} {label} H={H_} {k}: {v:.3g} radii"
        rep[(name, label, H_)] = max(res.values())
    print("env-step chain, largest ratio:", {k: round(v, 3) for k, v in rep.items()})
    assert {h[2] for h in horizons if h[0] == "humanoidtrack"} == {50, 60}


def test_relaunched_substeps_along_the_horizon(horizons, memo):
    rep = {}
    for name, label, H_, blob, st, Y, full, traj, xref, rel in horizons:
        (q, und), tot = relaunch_ratio(memo, blob, Y, rel)
        rep[(name, label, H_)] = (q, und / tot)
        assert q <= K, f"{name} {label} H={H_}: {q:.3g} radii"
        assert und <= HORIZON_UNDECIDED[name] * tot, f"{name} {label}: {und} of {tot} substeps undecided"
    print("relaunched substeps, (largest ratio, undecided fraction):", {k: (round(a, 3), round(b, 4)) for k, (a, b) in rep.items()})


def test_humanoidtrack_reads_the_last_demo_row_past_href(horizons):
    """at H = 60 > href = 50 the check accepts the clamped log-density and not the one that wraps round to row t - 50;
    against the shipped demo and its own-path demo the terms are not all at their clip"""
    seen = 0
    for name, label, H_, blob, st, Y, full, traj, xref, _ in horizons:
        if H_ != 60:
            continue
        if label == "own demo":
            lp = HR.logpd(blob, traj, xref, rows=np.arange(H_) % xref.shape[1])
            assert HR.ratio(full["logpd"], lp.v, lp.r) > K, label
            seen += 1
    assert seen == 1
    assert all(h[6]["logpd"].max() > -0.95 for h in horizons if h[1] == "own demo"), "every term at its clip"


# ---------------------------------------------------------------------------------------------------------------------
# the check is not vacuous: each slip the oracle and the kernels could share leaves the bound on some case
# ---------------------------------------------------------------------------------------------------------------------
def _worst(horizons, fn, names=None):
    w = 0.0
    for h in horizons:
        if names is None or h[0] in names:
            q = fn(*h)
            w = max(w, q if q is not None else 0.0)
    return w


def test_slip_actions_shifted_by_one_step(horizons, memo):
    for shift in (1, -1):
        w = _worst(horizons, lambda name, label, H_, blob, st, Y, full, traj, xref, rel:
                   relaunch_ratio(memo, blob, Y, rel, shift)[0][0])
        assert w > K, f"actions of step t{shift:+d}: {w:.3g} radii"


def test_slip_xref_row_t_plus_one(horizons):
    def f(name, label, H_, blob, st, Y, full, traj, xref, rel):
        lp = HR.logpd(blob, traj, xref, rows=HR.xref_rows(H_ + 1, xref.shape[1])[1:])
        return HR.ratio(full["logpd"], lp.v, lp.r)
    assert _worst(horizons, f, {"humanoidtrack"}) > K


def test_slip_pre_and_post_step_reward_swapped(horizons):
    """the run envs' reward on s_{t-1} instead of s_t, and humanoidtrack's on s_t instead of s_{t-1}"""
    from tests import xpbd_ref as X

    def f(name, label, H_, blob, st, Y, full, traj, xref, rel):
        n = traj.shape[0]
        prev = HR.previous_states(st, traj)
        if name == "humanoidtrack":
            r = X.reward_pre(blob, traj.reshape((-1,) + traj.shape[2:]))
        else:
            r = X.reward_post(blob, prev.reshape((-1,) + prev.shape[2:]))
        return HR.ratio(full["rewss"], r.v.reshape(n, -1), r.r.reshape(n, -1))
    for names in (("humanoidrun", "humanoidstandup", "hopper", "walker2d", "cartpole"), ("humanoidtrack",)):
        for nm in names:
            assert _worst(horizons, f, {nm}) > K, nm


def test_slip_ant_x_before_after_the_first_substep(horizons):
    from tests import xpbd_ref as X

    def f(name, label, H_, blob, st, Y, full, traj, xref, rel):
        keys = list(rel)
        before = np.stack([rel[k][1] for k in keys])
        after = np.stack([rel[k][-1] for k in keys])
        r = X.reward_ant(blob, before, after, np.stack([Y[b, t] for b, t in keys]))
        got = np.array([full["rewss"][b, t] for b, t in keys])
        return HR.ratio(got, r.v, r.r)
    for nm in ("ant", "halfcheetah"):
        assert _worst(horizons, f, {nm}) > K, nm


def test_slip_return_over_H_minus_one(horizons):
    def f(name, label, H_, blob, st, Y, full, traj, xref, rel):
        ret = HR.mean_return(full["rewss"], count=H_ - 1)
        return HR.ratio(full["rews"], ret.v, ret.r)
    assert _worst(horizons, f) > K


def test_slip_logpd_over_ntrack_only(horizons):
    def f(name, label, H_, blob, st, Y, full, traj, xref, rel):
        lp = HR.logpd(blob, traj, xref, count=int(blob.view(np.int32)[5]))
        return HR.ratio(full["logpd"], lp.v, lp.r)
    assert _worst(horizons, f, {"humanoidtrack"}) > K


def test_reference_pins_the_loop_constants():
    """the substeps per env step the chains above run: humanoidtrack 5, the run envs 7, ant 10, halfcheetah 16, hopper /
    walker2d 20; humanoidtrack tracks 5 links over 50 demo rows, so H = 60 reads past the last one"""
    want = dict(humanoidtrack=5, humanoidrun=7, humanoidstandup=7, ant=10, halfcheetah=16, hopper=20, walker2d=20)
    for name, nf in want.items():
        assert int(mbd_b200.envs.get_env(name).blob.view(np.int32)[3]) == nf, name
    env = mbd_b200.envs.get_env("humanoidtrack")
    assert env.xref.shape == (5, 50, 3) and int(env.blob.view(np.int32)[B.H_NTRACK]) == 5
