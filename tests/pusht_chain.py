"""pushT's rollout loop held to float64 substep by substep (tests/test_pusht_horizon_ref_cpu.py, tests/test_pusht_horizon_f64_gpu.py).

`pusht_body` (csrc/pusht.cuh) and `orc_pusht_rollout` clip an env step's control once and then run NSUB substeps with it.  A
launch with NSUB = 1 whose controls repeat each env step's control NSUB times therefore runs the very substeps of the shipped
NSUB = 5 launch, and with `want_traj` it returns the state after every substep: row 5t + 4 of its trajectory is row t of the
shipped one, bit for bit.  Each substep k is then held to `pusht_ref.step(P with NSUB = 1, s_{k-1}, u_k)` of the
implementation's own state before it (teacher forcing), with the radius of the solver mode.

The starts reach contact on purpose: random controls leave the pusher in free flight most of the time, so every start also
runs a scripted push toward the slider, generated closed loop at test-build time and replayed open loop.
"""
from __future__ import annotations

import numpy as np

from mbd_b200 import prng
from mbd_b200.envs.pusht import PT
from tests import horizon_ref as HR
from tests import pusht_families as F
from tests import pusht_ref as X

NSUB = 5                    # pushT.py:20, the NSUB of the shipped parameter table
H = 50
# the starts: reset poses (the goal words differ, the physics does not; each seed pushes with its own offset) and one state
# per contact family (pusht_families.build(family, .)[index]); "corner" is the pusher on the diagonal of a re-entrant corner
RESETS = {0: (-0.05, 0.02), 1: (0.05, -0.02), 2: (0.02, 0.05)}
FAMILY_STARTS = {"box0": ("box0", 0), "both": ("both", 0), "corner": ("both", 2), "limits_both": ("limits_both", 0),
                 "theta": ("theta", 4), "speeds": ("speeds", 0)}
PUSH_OFFSET = (-0.05, 0.02)
START_LABELS = [f"reset{s}" for s in RESETS] + list(FAMILY_STARTS)


def starts(env):
    """[(label, state [16] float32, offset of its scripted push)]"""
    out = [(f"reset{s}", env.reset(prng.split(prng.PRNGKey(s))[1]).pipeline_state.raw.copy(), off) for s, off in RESETS.items()]
    out += [(label, F.build(fam, 4)[i][0], PUSH_OFFSET) for label, (fam, i) in FAMILY_STARTS.items()]
    return out


def substep_controls(Y, nsub=NSUB):
    """[..., H, 2] -> [..., H * nsub, 2]: each env step's control once per substep"""
    return np.repeat(np.asarray(Y, np.float32), nsub, axis=-2)


def slider_com(P, st):
    """the slider's centre of mass in the world: its origin plus R(theta) (CX, CY)"""
    th = float(st[4])
    cx, cy = float(P[PT["CX"]]), float(P[PT["CY"]])
    return np.array([st[2] + np.cos(th) * cx - np.sin(th) * cy, st[3] + np.sin(th) * cx + np.cos(th) * cy])


def scripted_push(step, P, st, offset, H_=H):
    """[H_, 2] float32: the unit vector from the pusher to the slider's COM plus `offset`, recomputed every env step on the
    state that step(state [16], u [2]) -> state [16] (one env step of the shipped table) reaches"""
    s = np.asarray(st, np.float32)
    out = []
    for _ in range(H_):
        d = slider_com(P, s) - s[:2].astype(np.float64)
        u = (d / np.linalg.norm(d) + np.asarray(offset)).astype(np.float32)
        out.append(u)
        s = step(s, u)
    return np.stack(out)


def sequences(step, P, st, offset, seed):
    """the control sequences [2, H, 2] replayed from one start: the scripted push and a random one (pusht_families.controls:
    N(0, 1.2) draws, the first steps saturated at +-1 and +-37, so the clip acts)"""
    return np.stack([scripted_push(step, P, st, offset), F.controls(H, seed)])


def previous(st, traj):
    """[n, K, 16]: the state before each substep (st for the first)"""
    traj = np.asarray(traj, np.float32)
    start = np.broadcast_to(np.asarray(st, np.float32), (traj.shape[0], 1, 16))
    return np.concatenate([start, traj[:, :-1]], 1)


class StepMemo:
    """pusht_ref.step per (table, state, control), memoised on the exact input words: every implementation that hands it the same
    fp32 words (the oracle, k_pusht at every n) shares one evaluation"""

    def __init__(self):
        self.rows = {}
        self.evaluated = 0

    def __call__(self, P, states, u):
        """states [m, 16], u [m, 2] -> dict(value, radius (fixed point), trunc [m, 16], undecided [m], path [m], impulse [m, 5]: the
        velocity change of the constraint impulse)"""
        P = np.ascontiguousarray(P, np.float32)
        states = np.ascontiguousarray(states, np.float32).reshape(-1, 16)
        u = np.ascontiguousarray(u, np.float32).reshape(-1, 2)
        tag = P.tobytes()
        got = []
        for s, a in zip(states, u):
            key = (tag, s.tobytes(), a.tobytes())
            if key not in self.rows:
                r = X.step(P, s, a[None])
                imp = r["configs"][0]["impulse"][0]
                self.rows[key] = (r["value"][0], r["radius"][0], r["trunc"][0], bool(r["undecided"][0]), r["path"], imp)
                self.evaluated += 1
            got.append(self.rows[key])
        return dict(value=np.stack([g[0] for g in got]), radius=np.stack([g[1] for g in got]),
                    trunc=np.stack([g[2] for g in got]), undecided=np.array([g[3] for g in got]),
                    path=np.array([g[4] for g in got]), impulse=np.stack([g[5] for g in got]))


def check(memo, P, mode, prev, got, u):
    """substeps got [m, 16] against pusht_ref.step(P, prev, u) -> dict(ratio (largest over the decided substeps), undecided
    [m], path [m], finite (every decided radius), rel (per decided substep with a constraint impulse: the smallest over the
    five velocities of radius / |velocity change of the impulse|; a substep that dropped its impulse leaves the bound where
    this is below 1 / K), ref)"""
    ref = memo(P, prev, u)
    rad = X.radius(ref, mode)
    ok = ~ref["undecided"]
    q = HR.ratio(got, ref["value"], rad, np.broadcast_to(ok[:, None], rad.shape))
    imp = np.abs(ref["impulse"])
    with np.errstate(divide="ignore", invalid="ignore"):
        rel = np.where(imp > 0, rad[:, 8:13] / imp, np.inf).min(1)[ok & (imp.max(1) > 0)]
    return dict(ratio=q, undecided=ref["undecided"], path=ref["path"], finite=bool(np.isfinite(rad[ok]).all()), rel=rel,
                ref=ref)


def truncation_ratio(prod, fixed, ref):
    """largest |production - fixed point| / unit truncation radius over the decided substeps (pusht_ref.C_TRUNC's measure)"""
    ok = ~ref["undecided"]
    return HR.ratio(prod, np.asarray(fixed, np.float64), ref["trunc"], np.broadcast_to(ok[:, None], ref["trunc"].shape))

