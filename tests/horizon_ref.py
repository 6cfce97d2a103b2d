"""Float64 reference of a whole rollout horizon, on top of the one-substep reference of tests/xpbd_ref.py.

What runs in production is `n_frames` substeps per env step over H env steps (upstream utils.py:14-20,
mbd_planner.py:109): the state is carried from substep to substep and from step to step, step t uses the actions
Y[:, t], the per-step reward is taken before, after, or before and after the step, the return is sum_t r_t / H and the
demo log-density of humanoidtrack is a mean over (ntrack, H).  This module holds every piece of that loop to float64 with
the running error bounds of xpbd_ref, always teacher-forced on the implementation's own fp32 states (exact inputs):

* `step_rewards`: the reward of step t from the states of the rollout itself, `reward_post(s_t)` for the run envs,
  hopper / walker2d and cartpole, `reward_pre(s_{t-1})` for humanoidtrack, `reward_ant(s_{t-1}, s_t, u_t)` for ant and
  halfcheetah;
* `mean_return`: sum_t r_t / H of given fp32 rewards, radius gamma_H sum|r_t| / H plus one rounding; `return_of` the same
  from float64 rewards that carry their own radii;
* `logpd`: humanoidtrack.py:98-106, -mean over (k, t) of (clip(|x_k(s_t) - xref[k, t]|, 0, 0.5) / 0.5)^2.  Step t
  reads row min(t, href - 1): for H > href the last row is held.  That clamp is this project's extension (SURVEY F9);
  upstream only defines H <= href;
* `substep_chain` / `env_step_chain` / `relaunch_chain`: the loops the tests drive through a `run` callable (the CPU
  oracle or `ops.rollout`), returning what the references above are compared with.

A free-running bound over several substeps is not attempted: two correct fp32 rollouts may part at a contact.
"""
from __future__ import annotations

import numpy as np

from mbd_b200.model import blob as B
from tests import xpbd_ref as X
from tests.xpbd_ref import R

CLIP = 0.5     # humanoidtrack.py:103


def _flat(a, n, H):
    return np.ascontiguousarray(a, dtype=np.float32).reshape((n * H,) + a.shape[2:])


def _nh(x, n, H):
    return R(x.v.reshape(n, H), x.r.reshape(n, H))


def previous_states(s0, traj):
    """[n, H, L, 13]: the state before step t (s0 for t = 0, traj[:, t - 1] after), s0 [L, 13] or per sample [n, L, 13]"""
    traj = np.asarray(traj, dtype=np.float32)
    n = traj.shape[0]
    start = np.broadcast_to(np.asarray(s0, dtype=np.float32).reshape((-1, 1) + traj.shape[2:]), (n, 1) + traj.shape[2:])
    return np.concatenate([start, traj[:, :-1]], 1)


def step_rewards(blob, s0, traj, Y):
    """R [n, H]: the reward of every step of a rollout from its own states.  traj [n, H, L, 13] is the state after step t,
    s0 the start ([L, 13] or [n, L, 13]), Y [n, H, nu] the actions of each step."""
    m = X.Model(blob)
    traj = np.asarray(traj, dtype=np.float32)
    n, H = traj.shape[:2]
    prev = previous_states(s0, traj)
    if m.reward == B.REWARD_HUMANOIDTRACK:
        r = X.reward_pre(blob, _flat(prev, n, H))
    elif m.reward == B.REWARD_ANT:
        r = X.reward_ant(blob, _flat(prev, n, H), _flat(traj, n, H), _flat(np.asarray(Y, np.float32), n, H))
    else:
        r = X.reward_post(blob, _flat(traj, n, H))
    return _nh(r, n, H)


def mean_return(rewss, count=None):
    """sum_t r_t / count (count = H) of given fp32 per-step rewards [n, H]: gamma_H sum|r| for the sum, one rounding for
    the division"""
    r = np.asarray(rewss, dtype=np.float32).astype(np.float64)
    H = r.shape[1]
    return X.fsum([R(r[:, t]) for t in range(H)]) / float(H if count is None else count)


def return_of(rew, count=None):
    """sum_t r_t / count (count = H) of float64 per-step rewards R [n, H] with their radii"""
    H = rew.v.shape[1]
    return X.fsum([R(rew.v[:, t], rew.r[:, t]) for t in range(H)]) / float(H if count is None else count)


def xref_rows(H, href):
    """the demo row step t reads: min(t, href - 1)"""
    return np.minimum(np.arange(H), href - 1)


def track_positions(blob, traj):
    """the tracked link origins of every step, (value, radius) [n, H, ntrack, 3]"""
    traj = np.asarray(traj, dtype=np.float32)
    n, H = traj.shape[:2]
    v, r = X.track_positions(blob, _flat(traj, n, H))
    return v.reshape((n, H) + v.shape[1:]), r.reshape((n, H) + r.shape[1:])


def logpd(blob, traj, xref, rows=None, count=None):
    """humanoidtrack.py:98-106 over a horizon: 0 - sum_{k, t} (clip(|x_k(s_t) - xref[k, rows[t]]|, 0, .5) / .5)^2 / count
    with rows = xref_rows(H, href) and count = ntrack * H.  traj [n, H, L, 13], xref [ntrack, href, 3] -> R [n].
    Each term: the difference, the sum of three squares (gamma_3), sqrt, the clip (Lipschitz) and the exact scaling by 2,
    the square; then gamma_(ntrack H) for the sum of all terms in any order and one rounding for the division."""
    m = X.Model(blob)
    traj = np.asarray(traj, dtype=np.float32)
    n, H = traj.shape[:2]
    xref = np.asarray(xref, dtype=np.float32).astype(np.float64)
    rows = xref_rows(H, xref.shape[1]) if rows is None else rows
    x = X.link_origins(blob, _flat(traj, n, H))
    terms = []
    for k, l in enumerate(m.track):
        d = tuple(R(x[i].v[:, l].reshape(n, H), x[i].r[:, l].reshape(n, H)) - xref[k, rows, i][None, :] for i in range(3))
        q = X.exact_scale(X.rmin(X.sqrt(X.dot(d, d)), CLIP), 1.0 / CLIP)
        sq = q * q
        terms += [R(sq.v[:, t], sq.r[:, t]) for t in range(H)]
    return -(X.fsum(terms) / float(m.ntrack * H if count is None else count))


# ---------------------------------------------------------------------------------------------------------------------
# comparison
# ---------------------------------------------------------------------------------------------------------------------
def ratio(got, value, radius, mask=None):
    """largest |got - value| / radius over the masked entries: 0 where equal, inf where the radius is 0 and they differ or
    where `got` is not finite"""
    d = np.abs(np.asarray(got, dtype=np.float64) - value)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(d == 0, 0.0, d / radius)
    q = np.where(np.isfinite(d), q, np.inf)
    if mask is not None:
        q = q[mask]
    return float(q.max()) if q.size else 0.0


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32)
    return a.shape == b.shape and bool(np.array_equal(a.view(np.uint32), b.view(np.uint32)))


class StepMemo:
    """xpbd_ref.positional_step per sample row, memoised on the exact input words (blob, state, actions).  The reference is a
    pure function of its inputs, so implementations that hand it the same fp32 words (every kernel variant, every n) share
    one evaluation; rows seen for the first time are evaluated together."""

    def __init__(self):
        self.rows = {}
        self.branch_rows = {}

    def branches(self, blob, states, actions):
        """the forced-branch outcomes (xpbd_ref.branch_outcomes) of every undecided row -> [(row index, (value [A, L, 13],
        radius, valid [A, L], whole, still, nsites))], memoised like the step itself"""
        states = np.ascontiguousarray(states, dtype=np.float32)
        actions = np.ascontiguousarray(actions, dtype=np.float32)
        _, _, und = self(blob, states, actions)
        tag = np.ascontiguousarray(blob, dtype=np.uint32).tobytes()
        keys = {i: (tag, states[i].tobytes(), actions[i].tobytes()) for i in np.flatnonzero(und)}
        todo = {}
        for i, k in keys.items():
            if k not in self.branch_rows:
                todo.setdefault(k, i)
        if todo:
            idx = list(todo.values())
            ref = X.positional_step(blob, states[idx], actions[idx])
            br = X.branch_outcomes(blob, states[idx], actions[idx], ref)
            for j, r in enumerate(br["rows"]):
                self.branch_rows[keys[idx[r]]] = (br["value"][j], br["radius"][j], br["valid"][j], bool(br["whole"][j]),
                                                  bool(br["still"][j]), int(br["nsites"][j]))
        return [(i, self.branch_rows[k]) for i, k in keys.items()]

    def __call__(self, blob, states, actions):
        """states [n, L, 13], actions [n, nu] -> (value [n, L, 13], radius [n, L, 13], undecided [n])"""
        states = np.ascontiguousarray(states, dtype=np.float32)
        actions = np.ascontiguousarray(actions, dtype=np.float32)
        tag = np.ascontiguousarray(blob, dtype=np.uint32).tobytes()
        keys = [(tag, s.tobytes(), a.tobytes()) for s, a in zip(states, actions)]
        first = {}
        for i, k in enumerate(keys):
            if k not in self.rows:
                first.setdefault(k, i)
        todo = list(first.values())
        if todo:
            ref = X.positional_step(blob, states[todo], actions[todo])
            for j, i in enumerate(todo):
                self.rows[keys[i]] = (ref["value"][j], ref["radius"][j], bool(ref["undecided"][j]))
        got = [self.rows[k] for k in keys]
        return np.stack([g[0] for g in got]), np.stack([g[1] for g in got]), np.array([g[2] for g in got], dtype=bool)


def step_ratio(memo, blob, prev, u, got):
    """teacher-forced check of one substep: got [n, L, 13] against positional_step(prev, u) -> (largest ratio over the
    decided samples, undecided count)"""
    value, radius, und = memo(blob, prev, u)
    ok = np.broadcast_to(~und[:, None, None], value.shape)
    return ratio(got, value, radius, ok), int(und.sum())


def step_ratios(memo, blob, prev, u, got):
    """step_ratio with the undecided samples held to their forced branches (xpbd_ref.held_ratios) -> (largest ratio over the
    decided samples, largest best-assignment ratio over the undecided ones, count still unchecked, dict(undecided, held
    [ratio per held sample], second [distance to the second-best assignment per held sample]))"""
    value, radius, und = memo(blob, prev, u)
    ok = np.broadcast_to(~und[:, None, None], value.shape)
    dec = ratio(got, value, radius, ok)
    held, second, unchecked = [], [], 0
    got = np.asarray(got)
    for i, (v, r, valid, whole, still, _) in memo.branches(blob, prev, u):
        if still:
            unchecked += 1
            continue
        br = dict(rows=[i], value=v[None], radius=r[None], valid=valid[None], whole=[whole])
        b, s = X.held_ratios(got[i][None], br)
        held.append(float(b[0]))
        second.append(float(s[0]))
    return dec, max(held, default=0.0), unchecked, dict(undecided=int(und.sum()), held=held, second=second)


# ---------------------------------------------------------------------------------------------------------------------
# the loops, through run(state [L, 13], Y [n, H, nu], nsub=0, xref=None) -> dict(final, rewss, rews, track, logpd) numpy
# ---------------------------------------------------------------------------------------------------------------------
def substep_chain(run, st, u, nsub):
    """[s_0, s_1, ..., s_nsub] with s_k = run(st, u, nsub=k).final: the state after k substeps of one env step, each of
    which the tests check against positional_step(s_{k-1}, u)"""
    n = u.shape[0]
    out = [np.broadcast_to(np.asarray(st, np.float32), (n,) + st.shape)]
    for k in range(1, nsub + 1):
        out.append(run(st, u[:, None], nsub=k)["final"])
    return out


def env_step_chain(run, st, Y, xref=None):
    """the full run (rewss, rews, final, track, logpd) and the state after every step from prefix runs H' = h.  Each prefix
    run's rewss must equal the full run's rewss[:, :h] bit for bit: that is what makes its final state the full run's
    s_h.  -> (full, traj [n, H, L, 13])"""
    n, H = Y.shape[:2]
    full = run(st, Y, xref=xref)
    traj = []
    for h in range(1, H + 1):
        o = run(st, np.ascontiguousarray(Y[:, :h]))
        assert same_bits(o["rewss"], full["rewss"][:, :h]), f"prefix run H' = {h}: rewss differ from the full run's"
        traj.append(o["final"])
    assert same_bits(traj[-1], full["final"]), "the H' = H prefix run's final state differs from the full run's"
    return full, np.stack(traj, 1)


def relaunch_chain(run, s_prev, u, nsub):
    """one env step from one fp32 state [L, 13], one substep per launch (n = 1, nsub = 1): [s^0, ..., s^nsub].  The
    recurrent state of the loop is the 13 words per link; if nothing else is carried, s^nsub is the state the loop reached"""
    out = [np.asarray(s_prev, np.float32)]
    for _ in range(nsub):
        out.append(run(out[-1], np.asarray(u, np.float32).reshape(1, 1, -1), nsub=1)["final"][0])
    return out


def finite_samples(traj):
    """[n]: the samples whose states stay finite over the whole horizon.  A random model driven bang-bang at its control
    limits can blow up to inf / NaN (every correct fp32 evaluation with it); there is nothing to bound after that."""
    t = np.asarray(traj, dtype=np.float32)
    return np.isfinite(t.reshape(t.shape[0], -1)).all(1)


def _rows_of(ok, a):
    return np.broadcast_to(ok.reshape((-1,) + (1,) * (np.ndim(a) - 1)), np.shape(a))


def check_horizon(blob, st, Y, full, traj, xref=None):
    """every horizon output of a run against its float64 value, from the run's own states, over the samples whose states
    stay finite -> dict(largest ratio per output)"""
    m = X.Model(blob)
    ok = finite_samples(traj)
    rew = step_rewards(blob, st, traj, Y)
    res = dict(rewss=ratio(full["rewss"], rew.v, rew.r, _rows_of(ok, rew.v)))
    ret = mean_return(full["rewss"])
    res["rews"] = ratio(full["rews"], ret.v, ret.r, ok)
    ret = return_of(rew)
    res["rews_f64"] = ratio(full["rews"], ret.v, ret.r, ok)
    if full.get("track") is not None and m.ntrack:
        tv, tr = track_positions(blob, traj)
        res["track"] = ratio(full["track"], tv, tr, _rows_of(ok, tv))
    if xref is not None:
        lp = logpd(blob, traj, xref)
        res["logpd"] = ratio(full["logpd"], lp.v, lp.r, ok)
    return res
