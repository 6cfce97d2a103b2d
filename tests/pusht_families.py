"""Constructed pushT states for the float64 check of one physics step (tests/pusht_ref.py), shared by the CPU and GPU tests.

A family is a list of launches (state [16] float32, controls [n, 2] float32): one state shared by every sample of a launch
and a batch of controls (N(0, 1.2) draws, saturated +-1 and +-37, so |u| > 1 is clipped).  Pusher positions are placed in
the slider's body frame and carried to the world by the slider pose.  The T (include/mbd_pusht.h, assets/pusht.json): box 0
is the bar x in [-0.15, 0.15], |y| <= 0.05, box 1 the crossbar x in [-0.15, -0.05], |y| <= 0.15; pusher radius 0.05,
limits [-1, 1] on the four slides, none on the hinge.
  free            no row
  box0, box1      one contact on every face and exposed corner of one box, 1e-3 from a corner (normal poorly determined)
  both            the pusher in the T's re-entrant corners: 6 rows, pt_solve<8>
  limits          1-4 violated slide limits on both sides, no contact: pt_solve<4> through the general branch
  limits_contact  1 or 2 limits plus one contact: pt_solve<4> / pt_solve<8>
  limits_both     3-4 limits plus both contacts: 9-10 rows, pt_solve<12>
  deep            centre inside a box, both branches of the face choice px < py
  tie             centre inside a box on the diagonal px = py (the face choice straddles)
  depths          penetration 1e-5 .. 2e-3 around solimp's mid * width = 5e-4 and width = 1e-3
  speeds          60 rad/s spin (centrifugal), 5 m/s approach, 3 m/s sliding
  theta           slider angle +-10, 1e2, 1e3 rad (the hinge has no limit)
"""
from __future__ import annotations

import numpy as np

FAMILIES = ["free", "box0", "box1", "both", "limits", "limits_contact", "limits_both", "deep", "tie", "depths", "speeds", "theta"]
# the kernel paths each family must reach (tests/pusht_ref.py diagnostics), and the largest undecided fraction allowed
PATHS = {"free": {"none"}, "box0": {"fast4-box0"}, "box1": {"fast4-box1"}, "both": {"solve8"}, "limits": {"solve4"},
         "limits_contact": {"solve4", "solve8"}, "limits_both": {"solve12"}, "deep": {"fast4-box0", "fast4-box1"},
         "tie": {"fast4-box0", "fast4-box1"}, "depths": {"fast4-box0"}, "speeds": {"fast4-box0", "fast4-box1"},
         "theta": {"fast4-box0", "fast4-box1"}}
UNDECIDED_CAP = {f: 0.0 for f in FAMILIES}
UNDECIDED_CAP["tie"] = 0.55         # the face choice at px = py (half the launches): the two normals differ by 90 degrees
# largest radius of any output word (m, m/s) per family, and of a sample's largest velocity radius relative to its largest
# velocity change |qd' - qd| (so no family counts as checked while a step without its contact impulse would pass).  The
# largest radii are those of the pushers 7e-4 m off a corner, where the friction rows' activity is uncertain and the
# force bound takes the hull over the active sets the solve may cross (tests/pusht_ref.py)
RADIUS_CAP = {"free": 1e-5, "box0": 0.2, "box1": 0.5, "both": 0.05, "limits": 1e-4, "limits_contact": 2e-3,
              "limits_both": 0.02, "deep": 2e-3, "tie": 1e-3, "depths": 1e-3, "speeds": 0.01, "theta": 2e-3}
REL_CAP = {"free": 1e-4, "box0": 0.1, "box1": 0.25, "both": 0.1, "limits": 1e-4, "limits_contact": 2e-3,
           "limits_both": 0.01, "deep": 2e-3, "tie": 2e-3, "depths": 2e-3, "speeds": 1e-3, "theta": 5e-3}
# largest fraction of samples whose production solve (TOL 1e-6) hits the 100-sweep cap (ITERS 100 and 200 differ), and
# whose TOL = 0 solve is not at a fixed point after 4000 sweeps (ITERS 4000 and 8000 differ: Gauss-Seidel in fp32 cycles
# between neighbouring words on the dependent rows of a contact).  Measured (the oracle and the kernel agree bit for bit)
# over mu = 1 and mu = 0, rounded up.
SWEEP_CAP = {"free": 0.0, "box0": 0.01, "box1": 0.03, "both": 0.75, "limits": 0.0, "limits_contact": 0.0,
             "limits_both": 0.0, "deep": 0.2, "tie": 0.25, "depths": 0.0, "speeds": 0.0, "theta": 0.03}
NOT_FIXED_CAP = {"free": 0.0, "box0": 0.02, "box1": 0.03, "both": 0.1, "limits": 0.0, "limits_contact": 0.02,
                 "limits_both": 0.15, "deep": 0.04, "tie": 0.08, "depths": 0.01, "speeds": 0.0, "theta": 0.01}
GOAL = (-0.4, 0.4, np.pi)


def controls(n, seed):
    rng = np.random.default_rng(seed)
    a = rng.normal(size=(n, 2)) * 1.2
    a[0], a[1] = (1.0, 1.0), (-1.0, -1.0)
    a[2], a[3] = (37.0, -37.0), (-37.0, 0.3)
    return a.astype(np.float32)


def state(pusher, slider=(0.0, 0.0, 0.0), local=True, qd=(0.0,) * 5):
    """q | qd [16] float32: the pusher at `pusher` in the slider's body frame (local) or in the world"""
    x, y, th = slider
    px, py = pusher
    if local:
        c, s = np.cos(np.float64(np.float32(th))), np.sin(np.float64(np.float32(th)))
        px, py = x + c * px - s * py, y + s * px + c * py
    st = np.zeros(16)
    st[0:5] = (px, py, x, y, th)
    st[5:8] = GOAL
    st[8:13] = qd
    return st.astype(np.float32)


def _states(family, rng):
    v = lambda: tuple(rng.uniform(-0.5, 0.5, 5) * (1, 1, 1, 1, 4))   # noqa: E731
    poses = [(0.2, -0.1, 0.3), (-0.1, 0.3, -1.2)]
    out = []
    if family == "free":
        out += [state((0.5, 0.5), (-0.3, -0.2, 0.4), False, v()), state((-0.6, 0.7), (0.2, 0.1, -2.0), False, v())]
    elif family == "box0":
        for pose in poses:
            for p in [(0.07, 0.096), (0.07, -0.096), (0.196, 0.0), (0.196, -0.03), (0.18, 0.08), (0.18, -0.08),
                      (0.1507, 0.0507), (0.1507, -0.0507)]:
                out.append(state(p, pose, True, v()))
    elif family == "box1":
        for pose in poses:
            for p in [(-0.196, 0.12), (-0.196, -0.13), (-0.1, 0.196), (-0.1, -0.196), (-0.004, 0.12), (-0.004, -0.12),
                      (-0.18, 0.18), (-0.02, -0.18), (-0.1507, -0.1507), (-0.0493, 0.1507)]:
                out.append(state(p, pose, True, v()))
    elif family == "both":
        for pose in poses:
            for p in [(-0.02, 0.08), (-0.02, -0.08), (-0.03, 0.07), (-0.01, 0.09)]:
                out.append(state(p, pose, True, v()))
    elif family == "limits":
        out += [state((-0.5, 0.5), (1.01, 0.0, 0.2), False, v()), state((0.2, -1.005), (-1.02, 0.3, 0.0), False, v()),
                state((-1.01, 0.5), (1.005, -1.01, 2.0), False, v()), state((1.01, -1.005), (-1.01, 1.02, 1.0), False, v())]
    elif family == "limits_contact":
        out += [state((0.196, 0.0), (1.005, 0.3, 0.0), True, v()), state((-0.1, 0.196), (1.005, 0.3, 0.0), True, v()),
                state((0.07, -0.096), (-0.3, -1.01, 0.0), True, v()), state((-0.1, -0.196), (-1.004, 0.2, 0.0), True, v())]
    elif family == "limits_both":
        out += [state((-0.01, 0.09), (1.03, 1.02, 0.0), True, v()), state((-0.01, 0.09), (1.03, 0.95, 0.0), True, v()),
                state((-0.02, -0.08), (-1.03, -1.02, 0.0), True, v())]
    elif family == "deep":
        for pose in poses:
            for p in [(0.1, 0.02), (0.13, 0.0), (0.06, -0.03), (-0.1, 0.12), (-0.06, 0.12), (-0.12, -0.13)]:
                out.append(state(p, pose, True, v()))
    elif family == "tie":
        for pose in poses:
            for p in [(0.12, 0.02), (-0.08, 0.13)]:
                out.append(state(p, pose, True, v()))
    elif family == "depths":
        for d in (-1e-5, -3e-4, -5e-4, -7e-4, -1e-3, -2e-3):
            out.append(state((0.2 + d, 0.0), (0.1, -0.2, 0.4), True, v()))
    elif family == "speeds":
        out += [state((0.196, 0.0), (0.1, 0.0, 0.2), True, (0.0, 0.0, 0.0, 0.0, 60.0)),
                state((-0.1, 0.196), (0.0, 0.1, -0.4), True, (0.3, -0.2, 0.1, 0.2, -60.0)),
                state((0.07, 0.096), (0.0, 0.0, 0.0), True, (0.0, -5.0, 0.0, 0.0, 0.0)),
                state((0.07, -0.096), (0.0, 0.0, 0.0), True, (3.0, 0.5, 0.0, 0.0, 0.0))]
    elif family == "theta":
        for th in (10.0, -10.0, 1e2, -1e2, 1e3, -1e3):
            out.append(state((0.07, 0.096), (0.2, -0.1, th), True, v()))
            out.append(state((-0.196, 0.12), (-0.2, 0.1, th), True, v()))
    else:
        raise ValueError(family)
    return out


def build(family, n, seed=0):
    """the launches of one family: [(state [16], controls [n, 2])]"""
    rng = np.random.default_rng(seed + FAMILIES.index(family))
    return [(s, controls(n, 100 * seed + 7 * i + FAMILIES.index(family))) for i, s in enumerate(_states(family, rng))]
