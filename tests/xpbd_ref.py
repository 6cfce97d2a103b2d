"""Float64 reference of ONE Brax-positional substep (`positional_step`, DESIGN.md §2) with a running error bound.

The rollout kernels and the CPU oracle are fp32 restatements of the same step with one fixed association order; bit
equality between them says nothing about whether either computes the documented step.  This module evaluates the step
from its equations in float64 on the same fp32 inputs and carries, next to every value, a radius: a first-order bound on
how far ANY correct fp32 evaluation of the step may lie from the float64 value (Wilkinson-style running error analysis,
vectorised over samples and links).  Every blob word and every state word is an exact input (radius 0); the header's fp32
`inv_dt` / `two_inv_dt` / `half_dt` are used as stored.

Error model, u = 2^-24:
* `+ - * /` and `sqrt` round once: |fl(x) - x| <= u|x| (plus 2^-149 for the subnormal range).  An FMA rounds once, so the
  model over-counts it; that only widens the bound.
* a sum or dot product of k terms costs gamma_k * sum|terms| on top of the terms' own radii, which makes the bound
  independent of the association order;
* `rotate(v, q)` is charged (4.5 |q.r| + 4 |q.r|^2) |v| for the quaternion's radius (the map is quadratic in q: a radial
  perturbation a q moves R(q) v by at most 4|a||v|, a tangential one t by 2|t||v|) and gamma_32 |v| for rounding, which covers both the matrix form and the
  v + 2s(u x v) + 2u x (u x v) form the kernels use;
* `atan2` costs (x.r + y.r) / (hypot(x, y) - x.r - y.r) propagated plus ATAN2_ULP ulps (tests/test_fp32_device_gpu.py proves
  ATAN2_ULP for `mbd_atan2f` on the device build for every quotient inside the device division's domain); `cos` costs COS_ABS_ERR;
* `sqrt(x)` propagates min(x.r / sqrt(x), sqrt(x.r)): the derivative form, or the Hoelder form below x ~ x.r;
* a normalised fp32 vector has components in [-1 - 8u, 1 + 8u]; every value is intersected with such an interval where one
  is known (`clip_interval`), which keeps a direction whose norm is not much larger than its radius finite.  Where the
  step scales a direction by a magnitude proportional to the norm (joint translation and alignment, friction tangents) the
  product is evaluated as the continuous map it is, e.g. P = n dl = -e / W with W inside [im_c + im_p + eps, that + |r|^2],
  plus 8 roundings for the operations folded away.

Branches: where the margin of a discontinuous predicate is within its radius, the result is the interval hull of both
outcomes; when the two outcomes differ by more than JUMP times the radius, that predicate instance is a gated SITE and the
sample is marked `undecided`.  Predicates: the static-friction test |dl_t| < mu |dl|, the sinking gate v_n_old <= 0, the
contact test dist < 0 (the normal velocity impulse does not vanish with dl), the `dq.w >= 0` sign of project_xd, and the
atan2 branch cut at +-pi where the angle feeds a spring or a finite limit.  Clamps, min and |.| are Lipschitz and need no
gate.  A fp32 evaluation whose margin is within the radius may take either outcome, and downstream of it computes that
outcome's formula, so an undecided sample is held to the evaluations with its sites FORCED (`positional_step(force=)`,
`branch_outcomes`): it must lie within K radii of one consistent assignment of outcomes.  The contact test is one variable
per (link, contact slot), read by both the position stage and the velocity stage.

`reward_*` evaluate the per-step rewards the kernels compute (upstream humanoidrun.py:46-51, humanoidstandup.py:50-56,
hopper.py:57-65, walker2d.py:56-61, cartpole.py:44, humanoidtrack.py:87-106, ant [brax-recalled]) on a given fp32 state,
with the same arithmetic.
"""
from __future__ import annotations

import numpy as np

from mbd_b200.model import blob as B

U = 2.0 ** -24
ETA = 2.0 ** -149
ATAN2_ULP = 4.0          # max ulp error of mbd_atan2f; tests/test_fp32_device_gpu.py::test_atan2_exhaustive proves it on the
                         # device build for every quotient (max 2.454 with the quotient's rounding), test_fp32_spec.py samples the host
COS_ABS_ERR = 2.5e-7     # max absolute error of mbd_sincosf on |x| <= 1200 (max 9.32e-8 over every float32 there,
                         # tests/test_fp32_device_gpu.py::test_unary_exhaustive)
EPS = float(np.float32(1e-6))   # XPBD regulariser (ORC_EPS default)
ROT_GRAD = 4.5   # |d(R(q) v)/dq| <= (4|radial| + 2|tangential|) |v| <= sqrt(20) |v| near |q| = 1
ROT_ROUND = 32


def gamma(k):
    return k * U / (1.0 - k * U)


class R:
    """value + radius, arrays of one shape ([n, L] in the step)"""
    __slots__ = ("v", "r")

    def __init__(self, v, r=None):
        self.v = np.asarray(v, dtype=np.float64)
        self.r = np.zeros_like(self.v) if r is None else np.asarray(r, dtype=np.float64)

    def __neg__(self):
        return R(-self.v, self.r)

    def __add__(self, o):
        o = _c(o)
        return _round(self.v + o.v, self.r + o.r)

    __radd__ = __add__

    def __sub__(self, o):
        o = _c(o)
        return _round(self.v - o.v, self.r + o.r)

    def __rsub__(self, o):
        return _c(o) - self

    def __mul__(self, o):
        o = _c(o)
        return _round(self.v * o.v, _m(np.abs(self.v), o.r) + _m(np.abs(o.v), self.r) + _m(self.r, o.r))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = _c(o)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = self.v / o.v
            den = np.abs(o.v) - o.r
            rp = np.where(den > 0, (self.r + np.abs(v) * o.r) / np.where(den > 0, den, 1.0), np.inf)
        return _round(v, rp)

    def __rtruediv__(self, o):
        return _c(o) / self


def _m(a, b):
    """a * b for radii, with 0 * inf = 0 (an exact zero times an unbounded quantity is still exactly zero)"""
    with np.errstate(invalid="ignore"):
        return np.where((a == 0) | (b == 0), 0.0, a * b)


def _c(x):
    return x if isinstance(x, R) else R(x)


def _round(v, rp):
    return R(v, rp + U * (np.abs(v) + rp) + ETA)


def exact_scale(x, s):
    """x * s for a power of two s (no rounding)"""
    return R(x.v * s, x.r * abs(s))


def where(m, a, b):
    a, b = _c(a), _c(b)
    return R(np.where(m, a.v, b.v), np.where(m, a.r, b.r))


def fsum(terms):
    terms = [_c(t) for t in terms]
    v = sum(t.v for t in terms)
    rp = sum(t.r for t in terms)
    a = sum(np.abs(t.v) for t in terms)
    k = len(terms)
    return R(v, rp + gamma(k) * (a + rp) + k * ETA)


def sqrt(x):
    v = np.sqrt(np.maximum(x.v, 0.0))
    with np.errstate(divide="ignore", invalid="ignore"):
        rp = np.where(v > 0, np.minimum(x.r / np.where(v > 0, v, 1.0), np.sqrt(x.r)), np.sqrt(x.r))
    return _round(v, rp)


def rabs(x):
    return R(np.abs(x.v), x.r)


def clamp(x, lo, hi):
    """Lipschitz: the radius carries over"""
    return R(np.clip(x.v, lo, hi), x.r)


def rmin(a, b):
    a, b = _c(a), _c(b)
    return R(np.minimum(a.v, b.v), np.maximum(a.r, b.r))


def atan2(y, x):
    """value, radius and the branch-cut flag (x < 0 with y's sign undecided: the angle is +pi or -pi)"""
    v = np.arctan2(y.v, x.v)
    h = np.hypot(x.v, y.v)
    d = h - (x.r + y.r)
    with np.errstate(divide="ignore", invalid="ignore"):
        rp = np.where(d > 0, (x.r + y.r) / np.where(d > 0, d, 1.0), np.pi)
    cut = (x.v < 0) & (np.abs(y.v) <= y.r)
    rp = rp + ATAN2_ULP * (2 * U * (np.abs(v) + rp) + ETA)
    return R(v, rp), cut


def dot(a, b):
    return fsum([x * y for x, y in zip(a, b)])


def cross(a, b):
    return (fsum([a[1] * b[2], -(a[2] * b[1])]), fsum([a[2] * b[0], -(a[0] * b[2])]), fsum([a[0] * b[1], -(a[1] * b[0])]))


def vadd(a, b):
    return tuple(x + y for x, y in zip(a, b))


def vsub(a, b):
    return tuple(x - y for x, y in zip(a, b))


def vscale(a, s):
    return tuple(x * s for x in a)


def vwhere(m, a, b):
    return tuple(where(m, x, y) for x, y in zip(a, b))


def qmul(a, b):
    """Hamilton product (w, x, y, z)"""
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return (fsum([aw * bw, -(ax * bx), -(ay * by), -(az * bz)]),
            fsum([aw * bx, ax * bw, ay * bz, -(az * by)]),
            fsum([aw * by, -(ax * bz), ay * bw, az * bx]),
            fsum([aw * bz, ax * by, -(ay * bx), az * bw]))


def conj(q):
    return (q[0], -q[1], -q[2], -q[3])


def pure(v):
    return (R(np.zeros_like(v[0].v)), v[0], v[1], v[2])


def qnormalize(q):
    """q / |q|: the map's Jacobian is the projection (I - q^ q^T) / |q|, so an input perturbation of 2-norm d moves every
    component by at most d / |q|; the rounding of |q| (sum of four squares, sqrt, reciprocal) and of the scaling is
    gamma_8 relative"""
    nv = np.sqrt(sum(c.v * c.v for c in q))
    d = np.sqrt(sum(c.r * c.r for c in q))
    with np.errstate(divide="ignore", invalid="ignore"):
        prop = np.where(nv > d, d / np.where(nv > d, nv - d, 1.0), np.inf)
    return tuple(R(c.v / nv, prop + gamma(8) * (np.abs(c.v) / nv + prop) + 8 * ETA) for c in q)


def rot_matrix(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def rotate(v, q):
    """R(q) v for a (nearly) unit quaternion: the polynomial map R(q) = (1 - 2|u|^2) I + 2 u u^T + 2 s [u]x, which is
    what every restatement of math.rotate evaluates; its bound is stated in the module docstring"""
    v, q = tuple(_c(c) for c in v), tuple(_c(c) for c in q)
    M = rot_matrix([c.v for c in q])
    vv = [c.v for c in v]
    nv = np.sqrt(sum(c * c for c in vv)) + sum(c.r for c in v)
    qr = np.sqrt(sum(c.r * c.r for c in q))
    out = []
    for i in range(3):
        val = sum(M[i][j] * vv[j] for j in range(3))
        rp = sum(_m(np.abs(M[i][j]), v[j].r) for j in range(3)) + _m(nv, ROT_GRAD * qr + 4.0 * qr * qr)
        out.append(R(val, rp + gamma(ROT_ROUND) * (nv + rp) + 8 * ETA))
    return tuple(out)


def inv_rotate(v, q):
    return rotate(v, conj(q))


def clip_interval(x, lo, hi):
    """intersection of [x.v - x.r, x.v + x.r] with [lo, hi], an interval every fp32 evaluation is known to stay in"""
    a = np.maximum(x.v - x.r, lo)
    b = np.minimum(x.v + x.r, hi)
    a, b = np.where(a <= b, a, lo), np.where(a <= b, b, hi)
    keep = (x.v - x.r >= lo) & (x.v + x.r <= hi)
    return R(np.where(keep, x.v, 0.5 * (a + b)), np.where(keep, x.r, 0.5 * (b - a)))


def normalize(a):
    """(a / |a| with the zero guard, |a|).  Every component of a normalised fp32 vector lies in [-1 - 8u, 1 + 8u]; where
    the norm is not much larger than its radius that interval is what is known about the direction."""
    c = sqrt(dot(a, a))
    ok = c.v > c.r
    safe = R(np.where(ok, c.v, 1.0), np.where(ok, c.r, 0.0))
    inv = 1.0 / safe
    one = 1.0 + 8 * U
    n = tuple(clip_interval(R(np.where(ok, (x * inv).v, 0.0), np.where(ok, (x * inv).r, one)), -one, one) for x in a)
    return n, c


def extra(x, k):
    """k more roundings relative to |x|: the operations of the fp32 form that the float64 rewriting folded away"""
    return R(x.v, x.r + gamma(k) * (np.abs(x.v) + x.r))


JUMP = 16.0   # a branch whose two outcomes differ by less than JUMP times the radius is covered by their hull, not gated


def hull(x):
    """the interval hull of x and of 0: both outcomes of a branch that either adds x or adds nothing"""
    if isinstance(x, tuple):
        return tuple(hull(c) for c in x)
    return R(0.5 * x.v, 0.5 * np.abs(x.v) + x.r)


def norm_bound(v):
    """an upper bound of |v| for every fp32 evaluation"""
    return np.sqrt(sum(c.v * c.v for c in v)) + sum(c.r for c in v)


def other_reading(a):
    """the angle on the other side of the atan2 branch cut: a - 2 pi sign(a), with a's radius"""
    return R(a.v - 2 * np.pi * np.sign(a.v), a.r)


def dead_zone(a, cut, lo, hi, decide):
    """a - clip(a, lo, hi): exactly 0 where a is inside the band by more than its radius.  At an atan2 branch cut both
    +-pi readings must give 0, otherwise the reading is a gated site: decide(within, natural) picks it."""
    def excess(x):
        e = _round(x.v - np.clip(x.v, lo, hi), x.r)
        inside = (x.v - x.r > lo) & (x.v + x.r < hi)
        return R(np.where(inside, 0.0, e.v), np.where(inside, 0.0, e.r)), inside
    e, inside = excess(a)
    e_alt, alt_inside = excess(other_reading(a))
    keep = decide(cut & ~(inside & alt_inside), np.ones_like(cut, dtype=bool))
    return where(keep, e, e_alt)


# ---------------------------------------------------------------------------------------------------------------------
# model
# ---------------------------------------------------------------------------------------------------------------------
class Model:
    def __init__(self, blob):
        blob = np.ascontiguousarray(blob, dtype=np.uint32)
        self.f = blob.view(np.float32).astype(np.float64)
        self.i = blob.view(np.int32)
        self.L, self.nu = int(self.i[B.H_NLINK]), int(self.i[B.H_NU])
        self.reward = int(self.i[B.H_REWARD])
        self.ntrack = int(self.i[B.H_NTRACK])
        self.track = [int(self.i[B.H_TRACK0 + k]) for k in range(self.ntrack)]
        h = self.f
        self.dt, self.inv_dt, self.half_dt, self.two_inv_dt = h[B.H_DT], h[B.H_INV_DT], h[B.H_HALF_DT], h[B.H_TWO_INV_DT]
        self.vel_damp, self.ang_damp = h[B.H_VEL_DAMP], h[B.H_ANG_DAMP]
        self.scale_pos, self.scale_ang = h[B.H_SCALE_POS], h[B.H_SCALE_ANG]
        self.collide_scale, self.elasticity = h[B.H_COLLIDE_SCALE], h[B.H_ELASTICITY]
        self.g = (h[B.H_GX], h[B.H_GY], h[B.H_GZ])
        self.rw = h[B.H_RW0:B.H_RW0 + 4]

    def lf(self, field):
        o = B.HDR_WORDS + field * B.MAXL
        return self.f[o:o + self.L]

    def li(self, field):
        o = B.HDR_WORDS + field * B.MAXL
        return self.i[o:o + self.L]

    def lf3(self, field):
        return tuple(self.lf(field + a) for a in range(3))

    def lf4(self, field):
        return tuple(self.lf(field + a) for a in range(4))


def _const(shape, vals):
    return tuple(R(np.broadcast_to(c, shape).copy()) for c in vals)


def _gather(vec, idx, default):
    """vec[:, idx] per component, `default` where idx < 0"""
    ok = idx >= 0
    j = np.where(ok, idx, 0)
    return tuple(R(np.where(ok, c.v[:, j], d), np.where(ok, c.r[:, j], 0.0)) for c, d in zip(vec, default))


def _children(m):
    return [m.li(B.F_CHILD0 + c) for c in range(B.MAXCHILD)]


def _child_terms(vec_list_of_links, m):
    """for every link, the per-child values (0 where the child slot is empty)"""
    out = []
    for ch in _children(m):
        ok = ch >= 0
        j = np.where(ok, ch, 0)
        out.append(tuple(R(np.where(ok, c.v[:, j], 0.0), np.where(ok, c.r[:, j], 0.0)) for c in vec_list_of_links))
    return out


def euler(j, parity):
    """joint angles of R(j) = Rx(psi) Ry(theta) Rz(phi) in the joint frame, their instantaneous axes (parent joint frame),
    r10 / r20 and the branch-cut flags"""
    w, x, y, z = j
    r00 = fsum([1.0, exact_scale(y * y, -2), exact_scale(z * z, -2)])
    r01 = exact_scale(fsum([x * y, -(w * z)]), 2)
    r02 = exact_scale(fsum([x * z, w * y]), 2)
    r12 = exact_scale(fsum([y * z, -(w * x)]), 2)
    r22 = fsum([1.0, exact_scale(x * x, -2), exact_scale(y * y, -2)])
    r10 = exact_scale(fsum([x * y, w * z]), 2)
    r20 = exact_scale(fsum([x * z, -(w * y)]), 2)
    psi, c0 = atan2(-r12, r22)
    cth2 = fsum([r00 * r00, r01 * r01])
    cth = sqrt(cth2)
    theta, c1 = atan2(r02, cth)
    phi, c2 = atan2(-r01, r00)
    zero = R(np.zeros_like(w.v))
    lon, _ = normalize((zero, r22, -r12))
    ax0 = (R(np.ones_like(w.v)), zero, zero)
    ax2 = (r02 * parity, r12 * parity, r22 * parity)
    return dict(ang=(psi, theta, phi * parity), cut=(c0, c1, c2), ax=(ax0, lon, ax2), r10=r10, r20=r20, cth2=cth2.v)


def _slide_axis(k, parity, a_p, shape):
    e = [0.0, 0.0, 0.0]
    e[k] = 1.0
    ev = _const(shape, e)
    if k == 2:
        ev = (ev[0], ev[1], R(np.broadcast_to(parity, shape).copy()))
    return rotate(ev, a_p)


# ---------------------------------------------------------------------------------------------------------------------
# one substep
# ---------------------------------------------------------------------------------------------------------------------
SITES = ("static friction", "sinking gate", "dist < 0", "dq.w >= 0", "atan2 cut (spring)", "atan2 cut (limit)")


def positional_step(blob, states, actions, force=None, strict=True):
    """states [n, L, 13] fp32, actions [n, nu] fp32 -> dict(value [n, L, 13], radius [n, L, 13], undecided [n],
    reasons {predicate: [n] mask}, sites {site: [n, L] mask}, diag {name: [n, L] or [n, L, MAXCON] float64})

    A site is one predicate instance: (predicate, contact slot) for the three contact predicates, (predicate, dof) for the
    two atan2 cuts, (predicate,) for dq.w; its masks are per (sample, link).  `sites` holds the gated instances that made
    a sample undecided, and `outcomes` the outcome every instance took.  `force` maps a site to an int8 array [n, L]: -1
    leaves the instance free, 0 / 1 take the outcome False / True (for a cut, True is the angle atan2 computes and False
    the other reading a - 2 pi sign(a)).  A forced outcome replaces the hull where the instance is gated; where its margin
    is within its radius but the outcomes are closer than JUMP radii, the hull stays (the contact test still takes the
    forced outcome in the position stage: it covers both).  Forcing an instance whose margin is outside its radius to the
    outcome float64 does not take is an error (with strict=False it is recorded in `infeasible` [n, L] and the decided
    outcome is taken: another forced site decided this one); forcing it to that outcome changes nothing."""
    m = Model(blob)
    states = np.asarray(states, dtype=np.float32).astype(np.float64)
    actions = np.asarray(actions, dtype=np.float32).astype(np.float64)
    n, L = states.shape[0], m.L
    shape = (n, L)
    reasons = {}
    sites = {}
    outcomes = {}
    infeasible = np.zeros(shape, dtype=bool)
    force = {} if force is None else force
    # float64 values of the operands of the exact square roots and divisions (tests/tiny_families.py): the squared norms the
    # step takes square roots of and the contact depth it divides
    diag = {}

    def gate(name, mask, key=None):
        """marks the samples where a discontinuous predicate is within its radius and its outcomes jump"""
        mask = np.broadcast_to(mask, shape)
        reasons[name] = reasons.get(name, np.zeros(n, dtype=bool)) | mask.any(axis=-1)
        if key is not None and mask.any():
            sites[key] = sites.get(key, np.zeros(shape, dtype=bool)) | mask

    def forced(key, within, natural):
        """(outcome, forced mask) of a predicate instance: float64's own outcome `natural` unless `force` takes one where
        the margin is `within` its radius"""
        within = np.broadcast_to(within, shape)
        natural = np.broadcast_to(natural, shape)
        f = force.get(key)
        if f is None:
            outcomes[key] = natural
            return natural, np.zeros(shape, dtype=bool)
        f = np.broadcast_to(np.asarray(f, dtype=np.int8), shape)
        bad = (f >= 0) & ~within & ((f == 1) != natural)
        infeasible[...] |= bad
        if bad.any() and strict:
            raise ValueError(f"{key} forced against a decided outcome at {np.argwhere(bad)[:4].tolist()}")
        fm = (f >= 0) & within
        out = np.where(fm, f == 1, natural)
        outcomes[key] = out
        return out, fm

    def decide(key, gated, natural):
        """the outcome of a predicate instance gated on `gated` (within its radius, outcomes over JUMP radii apart)"""
        out, fm = forced(key, gated, natural)
        gate(key[0], gated & ~fm, key)
        return out

    def col(k):
        return R(states[:, :, k].copy())

    p, q, w, v = (col(0), col(1), col(2)), (col(3), col(4), col(5), col(6)), (col(7), col(8), col(9)), (col(10), col(11), col(12))
    p_prev, q_prev = p, q
    ident = (1.0, 0.0, 0.0, 0.0)
    par = m.li(B.F_PARENT)
    ndof = m.li(B.F_NDOF)
    jointed = ndof > 0
    smask = m.li(B.F_SLIDE)
    has_slide = smask != 0
    parity = m.lf(B.F_PARITY)
    PQ, JQ = m.lf4(B.F_PQ), m.lf4(B.F_JQ)
    RC, RP = m.lf3(B.F_RC), m.lf3(B.F_RP)
    im_c, im_p, ii_p = m.lf(B.F_INV_MASS), m.lf(B.F_PINV_MASS), m.lf(B.F_PINV_INERTIA)
    zero = R(np.zeros(shape))

    def dof(k, d):
        return m.lf(B.F_DOF0 + k * B.DOF_STRIDE + d)

    # ---- acceleration update: joint torques (motor, passive spring / damper, constraint_ang_damping), slide forces
    qp = _gather(q, par, ident)
    wp = _gather(w, par, (0.0, 0.0, 0.0))
    a_p = qmul(qp, PQ)
    a_c = qmul(q, JQ)
    ea = euler(qmul(conj(a_p), a_c), parity)
    diag["cth2 (acceleration)"] = ea["cth2"]
    jd = inv_rotate(vsub(w, wp), a_p)
    cad = m.lf(B.F_ANG_DAMP)
    rcw_s = rotate(RC, q)
    d_s = vsub(vadd(p, rcw_s), _const(shape, RP))
    va_s = vadd(v, cross(w, rcw_s))
    tq_terms = [[c * (-cad)] for c in jd]
    fw_terms = [[], [], []]
    for k in range(B.MAXDOF):
        exists = ndof > k
        is_slide = exists & (((smask >> k) & 1) == 1)
        a_id = m.li(B.F_DOF0 + k * B.DOF_STRIDE + B.D_ACT)
        u = actions[:, np.where(a_id >= 0, a_id, 0)]
        u = np.where(a_id >= 0, u, 0.0)
        tau = R(np.clip(u, dof(k, B.D_CLO), dof(k, B.D_CHI))) * dof(k, B.D_GEAR)
        tau = where(exists & (a_id >= 0), tau, 0.0)
        stiff, damp = dof(k, B.D_STIFF), dof(k, B.D_DAMP)
        ak = _slide_axis(k, parity, a_p, shape)
        f = fsum([tau, -(dot(d_s, ak) * stiff), -(dot(va_s, ak) * damp)])
        vel = dot(ea["ax"][k], jd)
        keep = decide(("atan2 cut (spring)", k), ea["cut"][k] & exists & ~is_slide & (stiff != 0), np.ones(shape, dtype=bool))
        t = fsum([tau, -(where(keep, ea["ang"][k], other_reading(ea["ang"][k])) * stiff), -(vel * damp)])
        hinge = exists & ~is_slide
        for i in range(3):
            tq_terms[i].append(where(hinge, ea["ax"][k][i] * t, 0.0))
            fw_terms[i].append(where(is_slide, ak[i] * f, 0.0))
    tq = tuple(fsum(t) for t in tq_terms)
    Fw = tuple(fsum(t) for t in fw_terms)
    T = rotate(tq, a_p)
    T = vwhere(has_slide, vadd(T, cross(rcw_s, Fw)), T)
    T = vwhere(jointed, T, (zero, zero, zero))
    Fa = vwhere(has_slide, vscale(Fw, m.lf(B.F_INV_MASS)), (zero, zero, zero))

    # ---- semi-implicit Euler
    acc = []
    kids = _child_terms(T, m)
    for i in range(3):
        acc.append(fsum([T[i]] + [-c[i] for c in kids]))
    w = tuple(fsum([w[i] * m.ang_damp, acc[i] * m.dt]) for i in range(3))
    al = tuple(where(has_slide, Fa[i] + m.g[i], m.g[i]) for i in range(3))
    v = tuple(fsum([v[i] * m.vel_damp, al[i] * m.dt]) for i in range(3))
    q = qnormalize(tuple(a + b for a, b in zip(q, qmul(pure(vscale(w, m.half_dt)), q))))
    p = tuple(fsum([p[i], v[i] * m.dt]) for i in range(3))
    w_before, v_before = w, v

    # ---- joint position solve: XPBD, one Jacobi pass over the joints
    pp = _gather(p, par, (0.0, 0.0, 0.0))
    qp = _gather(q, par, ident)
    rpw = rotate(RP, qp)
    rcw = rotate(RC, q)
    e = vsub(vadd(p, rcw), vadd(pp, rpw))
    a_p = qmul(qp, PQ)
    for k in range(B.MAXDOF):
        is_slide = (ndof > k) & (((smask >> k) & 1) == 1)
        if not is_slide.any():
            continue
        ak = _slide_axis(k, parity, a_p, shape)
        x = clamp(dot(e, ak), dof(k, B.D_LO), dof(k, B.D_HI))
        e = vwhere(is_slide, tuple(fsum([e[i], -(ak[i] * x)]) for i in range(3)), e)
    # P = n dl with n = e / |e|, dl = -|e| / (w_p + w_c + eps): P = -e / W, where W depends on the direction only through
    # |r x n|^2, so it stays inside [im_c + im_p + eps, that + |rc|^2 + ii_p |rp|^2] even where the direction is unknown
    diag["anchor2"] = dot(e, e).v
    nrm, c = normalize(e)
    crc, crp = cross(rcw, nrm), cross(rpw, nrm)
    W = fsum([im_p, dot(crp, crp) * ii_p, im_c, dot(crc, crc), EPS])
    w_lo = im_c + im_p + EPS
    W = clip_interval(W, w_lo * (1 - 16 * U), (w_lo + norm_bound(rcw) ** 2 + ii_p * norm_bound(rpw) ** 2) * (1 + 16 * U))
    P = tuple(extra(-x / W, 8) for x in e)
    dp_c = vscale(P, im_c)
    dq_c = tuple(exact_scale(x, 0.5) for x in qmul(pure(cross(rcw, P)), q))
    dp_p = vscale(P, -im_p)
    dq_p = tuple(exact_scale(x, -0.5) * ii_p for x in qmul(pure(cross(rpw, P)), qp))
    a_c = qmul(q, JQ)
    ea = euler(qmul(conj(a_p), a_c), parity)
    diag["cth2 (joint solve)"] = ea["cth2"]
    err = []
    for k in range(B.MAXDOF):
        is_slide = ((smask >> k) & 1) == 1
        used = jointed & ~is_slide & ((k == 0) | (ndof > 1))      # a 1-dof joint aligns its axis instead of using angles 1, 2
        ek = dead_zone(ea["ang"][k], ea["cut"][k] & used, dof(k, B.D_LO), dof(k, B.D_HI),
                       lambda within, nat, k=k: decide(("atan2 cut (limit)", k), within, nat))
        err.append(where(is_slide, ea["ang"][k], ek))
    one = ndof == 1
    dqj3 = tuple(fsum([ea["ax"][k][i] * err[k] for k in range(3)]) for i in range(3))
    dqj = vwhere(one, (err[0], -ea["r20"], ea["r10"]), dqj3)
    dq = rotate(dqj, a_p)
    # Pa = na dla with na = dq / |dq|, dla = -|dq| / ((1 + ii_p) |na|^2 + eps) and |na|^2 = 1 +- 8u: Pa = -dq / D
    D = R(1.0 + ii_p + EPS, (1.0 + ii_p) * 8 * U)
    Pa = tuple(extra(-x / D, 8) for x in dq)
    dqa_c = tuple(exact_scale(x, 0.5) for x in qmul(pure(Pa), q))
    dqa_p = tuple(exact_scale(x, -0.5) * ii_p for x in qmul(pure(Pa), qp))
    z3, z4 = (zero,) * 3, (zero,) * 4
    dpc = vwhere(jointed, vscale(dp_c, m.scale_pos), z3)
    dpp = vwhere(jointed, vscale(dp_p, m.scale_pos), z3)
    dqc = vwhere(jointed, tuple(fsum([a * m.scale_pos, b * m.scale_ang]) for a, b in zip(dq_c, dqa_c)), z4)
    dqp = vwhere(jointed, tuple(fsum([a * m.scale_pos, b * m.scale_ang]) for a, b in zip(dq_p, dqa_p)), z4)
    kp, kq = _child_terms(dpp, m), _child_terms(dqp, m)
    p = tuple(fsum([p[i], dpc[i]] + [c[i] for c in kp]) for i in range(3))
    q = qnormalize(tuple(fsum([q[i], dqc[i]] + [c[i] for c in kq]) for i in range(4)))

    # ---- plane contacts (sphere / cap centres against z = 0) + static friction
    ncon = m.li(B.F_NCON)
    im = im_c
    dp_acc = [[], [], []]
    dq_acc = [[], [], [], []]
    contacts = []
    for ci in range(B.MAXCON):
        active = ncon > ci
        if not active.any():
            break
        base = B.F_CON0 + ci * B.CON_STRIDE
        S = m.lf3(base)
        rad, mu = m.lf(base + 3), m.lf(base + 4)
        centre = vadd(p, rotate(S, q))
        dist = centre[2] - rad
        diag.setdefault("dist", []).append(np.where(active, dist.v, np.nan))
        near = active & (np.abs(dist.v) <= dist.r)
        coll, coll_fm = forced(("dist < 0", ci), near, dist.v < 0)   # one outcome for the position and velocity stages
        cp = (centre[0], centre[1], centre[2] - fsum([rad, exact_scale(dist, 0.5)]))
        r = vsub(cp, p)
        wn = fsum([im, r[0] * r[0], r[1] * r[1]])
        dl = where(coll, -dist / (wn + EPS), 0.0)
        # static friction: cancel the tangential travel of the contact point since the start of the substep
        pbar = vadd(p_prev, rotate(inv_rotate(r, q), q_prev))
        dxy = (cp[0] - pbar[0], cp[1] - pbar[1], zero)
        diag.setdefault("travel2", []).append(np.where(active & coll, dot(dxy, dxy).v, np.nan))
        # P_t = n_t dl_t with dl_t = -|dx| / (w_t + eps): P_t = -dx / W_t, W_t in [im + eps, im + eps + |r|^2]
        nt, ct = normalize(dxy)
        cr = cross(r, nt)
        Wt = clip_interval(fsum([im, dot(cr, cr), EPS]), (im + EPS) * (1 - 8 * U), (im + EPS + norm_bound(r) ** 2) * (1 + 16 * U))
        dlt = extra(ct / Wt, 4)
        margin = rabs(dl) * mu - dlt
        stat = coll & (margin.v > 0)
        Pt = tuple(extra(-x / Wt, 8) for x in dxy)
        either = active & coll & (np.abs(margin.v) <= margin.r) & (margin.r > 0)
        stat, fm = forced(("static friction", ci), either, stat)
        gated = either & (dlt.v > JUMP * dlt.r)
        gate("static friction", gated & ~fm, ("static friction", ci))
        Pt = vwhere(either & ~(fm & gated), hull(Pt), vwhere(stat, Pt, (zero,) * 3))
        Pt = (Pt[0], Pt[1], dl)
        dpl = vscale(Pt, im)
        dql = tuple(exact_scale(x, 0.5) for x in qmul(pure(cross(r, Pt)), q))
        for i in range(3):
            dp_acc[i].append(where(active, dpl[i], 0.0))
        for i in range(4):
            dq_acc[i].append(where(active, dql[i], 0.0))
        contacts.append((ci, active, cp, dl, coll, mu, near, coll_fm))
    if contacts:
        has_con = ncon > 0
        dpt = tuple(fsum(t) for t in dp_acc)
        dqt = tuple(fsum(t) for t in dq_acc)
        p = vwhere(has_con, tuple(fsum([p[i], dpt[i] * m.collide_scale]) for i in range(3)), p)
        q = vwhere(has_con, qnormalize(tuple(fsum([q[i], dqt[i] * m.collide_scale]) for i in range(4))), q)

    # ---- project_xd: velocities from the positional change
    v = tuple((p[i] - p_prev[i]) * m.inv_dt for i in range(3))
    dq = qmul(q, conj(q_prev))
    pos = decide(("dq.w >= 0",), (np.abs(dq[0].v) <= dq[0].r) & (dq[0].r > 0), dq[0].v >= 0)
    sgn = np.where(pos, m.two_inv_dt, -m.two_inv_dt)
    w = tuple(dq[i] * sgn for i in (1, 2, 3))

    # ---- velocity solve: dynamic friction, restitution, normal velocity of approaching contacts
    if contacts:
        dv_acc = [[], [], []]
        dw_acc = [[], [], []]
        v0, w0 = v, w
        for ci, active, cp, dl, coll, mu, near, coll_fm in contacts:
            r = vsub(cp, p)
            rel = vadd(v0, cross(w0, r))
            vn = rel[2]
            tvec = (rel[0], rel[1], zero)
            diag.setdefault("velocity2", []).append(np.where(active & coll, dot(tvec, tvec).v, np.nan))
            # P_d = -t min(fr, |v_t|) kd = -v_t s kd with s = min(fr / |v_t|, 1) in [0, 1]
            tdir, vtn = normalize(tvec)
            fr = rabs(dl) * mu * m.inv_dt
            full = fr.v - fr.r >= vtn.v + vtn.r
            ok = vtn.v - vtn.r > 0
            ratio = fr / R(np.where(ok, vtn.v, 1.0), np.where(ok, vtn.r, 0.0))
            s_ = clip_interval(rmin(ratio, 1.0), 0.0, 1.0)
            s_ = R(np.where(full, 1.0, np.where(ok, s_.v, 0.5)), np.where(full, 0.0, np.where(ok, s_.r, 0.5)))
            cr = cross(r, tdir)
            kd = 1.0 / clip_interval(fsum([im, dot(cr, cr), EPS]), (im + EPS) * (1 - 8 * U), (im + EPS + norm_bound(r) ** 2) * (1 + 16 * U))
            Pd = tuple(extra(-(x * s_) * kd, 8) for x in tvec)
            rel_old = vadd(v_before, cross(w_before, r))
            vn_old = rel_old[2]
            rest = rmin(-(vn_old * m.elasticity), 0.0)
            wn = fsum([im, r[0] * r[0], r[1] * r[1]])
            prz = fsum([-vn, rest]) * (1.0 / (wn + EPS))
            sink = decide(("sinking gate", ci), active & coll & (np.abs(vn_old.v) <= vn_old.r) & (vn_old.r > 0), vn_old.v <= 0)
            Pz = where(sink, prz, 0.0)
            Pv = (Pd[0], Pd[1], Pz)
            gated = near & (np.abs(Pz.v) > JUMP * Pz.r)
            gate("dist < 0", gated & ~coll_fm, ("dist < 0", ci))
            Pv = vwhere(near & ~(coll_fm & gated), tuple(hull(x) for x in Pv), vwhere(coll, Pv, (zero,) * 3))
            dvl = vscale(Pv, im)
            dwl = cross(r, Pv)
            for i in range(3):
                dv_acc[i].append(where(active, dvl[i], 0.0))
                dw_acc[i].append(where(active, dwl[i], 0.0))
        has_con = ncon > 0
        v = vwhere(has_con, tuple(fsum([v[i]] + dv_acc[i]) for i in range(3)), v)
        w = vwhere(has_con, tuple(fsum([w[i]] + dw_acc[i]) for i in range(3)), w)

    comps = list(p) + list(q) + list(w) + list(v)
    value = np.stack([c.v for c in comps], axis=-1)
    radius = np.stack([c.r for c in comps], axis=-1)
    undecided = np.zeros(n, dtype=bool)
    for m_ in reasons.values():
        undecided |= m_
    diag = {k: np.stack(v, axis=-1) if isinstance(v, list) else v for k, v in diag.items()}
    return dict(value=value, radius=radius, undecided=undecided, reasons=reasons, sites=sites, outcomes=outcomes,
                infeasible=infeasible, diag=diag)


# ---------------------------------------------------------------------------------------------------------------------
# undecided samples: the outcomes of their sites, forced
# ---------------------------------------------------------------------------------------------------------------------
MAX_BITS = 10    # at most 2^10 forced evaluations per sample; a sample needing more is left unchecked


def instances(sites, i, L):
    """[(site, link)] of sample i, links ascending"""
    return [(key, l) for l in range(L) for key in sorted(sites) if sites[key][i, l]]


def branch_outcomes(blob, states, actions, ref):
    """the undecided samples of ref = positional_step(blob, states, actions) under assignments of their sites.

    After the joint solve, the contact stage, project_xd and the velocity solve act on one link at a time, so a link's 13
    words depend only on its own contact and dq.w sites: pass a forces bit j of a to the j-th site of EVERY link, and one
    pass gives each link its outcome under assignment a (2^(largest site count of a link) passes).  An atan2 cut couples
    links through the acceleration update and the joint solve, so a sample with a cut site is enumerated as a whole: bit j
    to the sample's j-th site.
    -> dict(rows [m] sample indices, value / radius [m, A, L, 13], valid [m, A, L] (a is an assignment of link l's own sites,
    or every a for a whole-sample enumeration), whole [m], still [m] (a forced evaluation gated a new site, or more than
    MAX_BITS sites: unchecked), nsites [m]).  An assignment under which one forced site decides another against its forced
    outcome (the sinking gate of a contact forced not to collide, say) is infeasible and not valid."""
    m = Model(blob)
    L = m.L
    states = np.asarray(states, dtype=np.float32)
    actions = np.asarray(actions, dtype=np.float32)
    rows = np.flatnonzero(ref["undecided"])
    sites = ref["sites"]
    info = []
    for i in rows:
        inst = instances(sites, i, L)
        whole = any(key[0].startswith("atan2") for key, _ in inst)
        if whole:
            bit = {(key, l): j for j, (key, l) in enumerate(inst)}
            nb = len(inst)
        else:
            bit, cnt = {}, [0] * L
            for key, l in inst:
                bit[(key, l)] = cnt[l]
                cnt[l] += 1
            nb = max(cnt)
        info.append((whole, bit, nb, len(inst)))
    A = 1 << min(max([nb for _, _, nb, _ in info if nb <= MAX_BITS], default=0), MAX_BITS)
    M = len(rows)
    value = np.full((M, A, L, 13), np.nan)
    radius = np.full((M, A, L, 13), np.nan)
    valid = np.zeros((M, A, L), dtype=bool)
    still = np.array([nb > MAX_BITS for _, _, nb, _ in info], dtype=bool)
    for nb in sorted({nb for _, _, nb, _ in info if nb <= MAX_BITS}):
        g = [j for j, x in enumerate(info) if x[2] == nb]
        for a in range(1 << nb):
            force = {}
            for gj, j in enumerate(g):
                for (key, l), b in info[j][1].items():
                    f = force.setdefault(key, np.full((len(g), L), -1, dtype=np.int8))
                    f[gj, l] = (a >> b) & 1
            out = positional_step(blob, states[rows[g]], actions[rows[g]], force, strict=False)
            for gj, j in enumerate(g):
                value[j, a], radius[j, a] = out["value"][gj], out["radius"][gj]
                still[j] |= bool(out["undecided"][gj])
                whole, bit = info[j][0], info[j][1]
                bad = out["infeasible"][gj]
                if whole:
                    valid[j, a] = not bad.any()
                else:
                    cnt = np.zeros(L, dtype=int)
                    for (_, l) in bit:
                        cnt[l] += 1
                    valid[j, a] = (a < (1 << cnt)) & ~bad
    return dict(rows=rows, value=value, radius=radius, valid=valid, whole=np.array([x[0] for x in info], dtype=bool),
                still=still, nsites=np.array([x[3] for x in info], dtype=int))


def _word_ratio(got, value, radius):
    d = np.abs(np.asarray(got, dtype=np.float64) - value)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(d == 0, 0.0, d / radius)
    return np.where(np.isfinite(d), q, np.inf)


def held_ratios(got, br):
    """got [m, L, 13] (the rows of `br`) -> (best [m], second [m]): the largest ratio of the sample to its best consistent
    assignment (each link's minimum over its own assignments, or the minimum over whole-sample assignments), and the same
    for the second-best assignment of the link (or sample) where it is closest (inf with a single assignment)"""
    got = np.asarray(got)
    M = len(br["rows"])
    best, second = np.zeros(M), np.full(M, np.inf)
    for j in range(M):
        q = _word_ratio(got[j][None], br["value"][j], br["radius"][j]).max(-1)        # [A, L]
        q = np.where(br["valid"][j], q, np.inf)
        if br["whole"][j]:
            per = np.sort(q.max(1))
            best[j] = per[0]
            second[j] = per[1] if len(per) > 1 else np.inf
        else:
            per = np.sort(q, axis=0)                                                  # [A, L]
            best[j] = per[0].max()
            multi = np.isfinite(per[1]) if len(per) > 1 else np.zeros(per.shape[1], bool)
            second[j] = per[1][multi].min() if multi.any() else np.inf
    return best, second


# ---------------------------------------------------------------------------------------------------------------------
# rewards on a given fp32 state [n, L, 13]
# ---------------------------------------------------------------------------------------------------------------------
def _state(states):
    s = np.asarray(states, dtype=np.float32).astype(np.float64)
    col = lambda k: R(s[:, :, k].copy())   # noqa: E731
    return (col(0), col(1), col(2)), (col(3), col(4), col(5), col(6)), (col(7), col(8), col(9)), (col(10), col(11), col(12))


def _f32(x):
    return float(np.float32(x))


def link_origins(blob, states):
    """com.to_world: x.pos = x_i.pos - R(rot) com, per link"""
    m = Model(blob)
    p, q, _, _ = _state(states)
    return vsub(p, rotate(m.lf3(B.F_COM), q))


def _pick(vec, l):
    return tuple(R(c.v[:, l], c.r[:, l]) for c in vec)


def reward_post(blob, states):
    """per-step reward of humanoidrun, humanoidstandup, hopper / walker2d and cartpole on the post-step state -> R [n]"""
    m = Model(blob)
    x0 = _pick(link_origins(blob, states), 0)
    if m.reward == B.REWARD_HUMANOIDRUN:                        # humanoidrun.py:46-51
        dz = clamp(rabs(x0[2] - _f32(1.3)), -1.0, 1.0)
        return (x0[0] - dz) - rabs(x0[1]) * _f32(0.1)
    if m.reward == B.REWARD_HUMANOIDSTANDUP:                   # humanoidstandup.py:50-56
        return ((1.5 - clamp(rabs(x0[2] - _f32(1.3)), -2.0, 1.0)) - rabs(x0[0]) * _f32(0.1)) - rabs(x0[1]) * _f32(0.1)
    if m.reward == B.REWARD_HOPPER:                            # hopper.py:57-65 (RW0 = 1.0), walker2d.py:56-61 (RW0 = 1.1)
        return x0[0] - exact_scale(clamp(rabs(x0[2] - m.rw[0]), -1.0, 1.0), 0.5)
    if m.reward == B.REWARD_CARTPOLE:                          # cartpole.py:44: cos(q[1]) - |qd[0]|
        p, q, w, v = _state(states)
        n = q[0].v.shape[0]
        q0, q1 = _pick(q, 0), _pick(q, 1)
        a_p = qmul(q0, tuple(c[1] for c in m.lf4(B.F_PQ)))
        a_c = qmul(q1, tuple(c[1] for c in m.lf4(B.F_JQ)))
        ea = euler(qmul(conj(a_p), a_c), m.lf(B.F_PARITY)[1])
        psi = ea["ang"][0]
        c = R(np.cos(psi.v), psi.r + COS_ABS_ERR)
        rcw = rotate(tuple(np.full(n, c_[0]) for c_ in m.lf3(B.F_RC)), q0)
        va = vadd(_pick(v, 0), cross(_pick(w, 0), rcw))
        e0 = tuple(R(np.full(n, x)) for x in (1.0, 0.0, 0.0))
        axis = rotate(e0, tuple(R(np.full(n, c_[0])) for c_ in m.lf4(B.F_PQ)))
        return c - rabs(dot(va, axis))
    raise ValueError(f"reward kind {m.reward} has no post-step reward")


def reward_pre(blob, states):
    """humanoidtrack.py:87-96 on the PRE-step state: 1 + (-|xd.vel[0].x - 1.6| - |x.pos[0].z - 1.3| - 0.1 |x.pos[0].y|)"""
    m = Model(blob)
    p, q, w, v = _state(states)
    rc = rotate(m.lf3(B.F_COM), q)
    x0 = _pick(vsub(p, rc), 0)
    v0 = _pick(vadd(v, cross(rc, w)), 0)
    return 1.0 + ((-rabs(v0[0] - _f32(1.6)) - rabs(x0[2] - _f32(1.3))) - rabs(x0[1]) * _f32(0.1))


def track_positions(blob, states):
    """the tracked link origins [n, ntrack, 3] as (value, radius)"""
    m = Model(blob)
    x = link_origins(blob, states)
    val = np.stack([np.stack([x[i].v[:, l] for i in range(3)], -1) for l in m.track], 1)
    rad = np.stack([np.stack([x[i].r[:, l] for i in range(3)], -1) for l in m.track], 1)
    return val, rad


def logpd_one_step(blob, states, xref_row):
    """humanoidtrack.py:98-106 for a horizon of one: -mean_k (clip(|x_k - xref_k|, 0, 0.5) / 0.5)^2, xref_row [ntrack, 3]"""
    m = Model(blob)
    x = link_origins(blob, states)
    terms = []
    for k, l in enumerate(m.track):
        d = tuple(R(x[i].v[:, l], x[i].r[:, l]) - float(xref_row[k, i]) for i in range(3))
        nr = sqrt(dot(d, d))
        qk = exact_scale(rmin(nr, 0.5), 2.0)
        terms.append(qk * qk)
    return -(fsum(terms) / float(m.ntrack))


def reward_ant(blob, states_before, states_after, actions):
    """ant / halfcheetah [brax-recalled]: (x_after - x_before) / env_dt + healthy - w_ctrl * sum(u^2), u the action handed in"""
    m = Model(blob)
    xb = link_origins(blob, states_before)[0]
    xa = link_origins(blob, states_after)[0]
    u = np.asarray(actions, dtype=np.float32).astype(np.float64)
    ss = fsum([R(u[:, k]) * R(u[:, k]) for k in range(u.shape[1])])
    fwd = (R(xa.v[:, 0], xa.r[:, 0]) - R(xb.v[:, 0], xb.r[:, 0])) / m.rw[0]
    return (fwd + m.rw[1]) - ss * m.rw[2]
