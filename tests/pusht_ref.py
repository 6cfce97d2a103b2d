"""Float64 reference of ONE pushT physics step (DESIGN.md §7a, include/mbd_pusht.h) with a radius per output word.

`k_pusht` and oracle/pusht_oracle.c are two fp32 copies of one association order, compared bit for bit; a slip present in
both passes that comparison.  This module evaluates the step from its equations in float64 on the same fp32 inputs (the
parameter table, the state q | qd [16] and the clipped controls) and gives every output word a radius that bounds any
correct fp32 evaluation of it.  It shares the value-plus-radius class `R`, `gamma` and the error model of tests/xpbd_ref.py:
u = 2^-24, one rounding per `+ - * / sqrt`, gamma_k * sum|terms| for a sum or dot of k terms, and COS_ABS_ERR for
`mbd_sincosf` (tests/test_fp32_spec.py::test_sincos proves it up to |x| = 1200).

The step, written from the equations rather than from either fp32 copy:
* mass matrix: the full 5x5 M(theta) of the pusher (mass m_p on two slides) and the slider (mass m, Izz about the COM I, body
  COM c rotated to r = R(theta) c): the slider block is [[m, 0, -m r_y], [0, m, m r_x], [-m r_y, m r_x, I + m |r|^2]].  The
  QP's inverse mass is np.linalg.inv of the M whose masses are the reciprocals of the stored inverse words (IMP, IMS, IIS),
  the integration solves (M + dt D) with the stored MP, MS, IS, all with np.linalg;
* qf_smooth = gear * u - D qd + the centrifugal force m w^2 r of the offset COM on the two slides (the hinge row has none);
* rows: joint limits (side, pos = min(q - lo, hi - q)); one sphere-box contact per box (closest point outside, the nearest
  face when the centre is inside, contact point midway between the surfaces) with the 4-sided pyramid AS BRAX STATES IT:
  n - mu t, n + mu t and the out-of-plane pair n - mu z, n + mu z, whose in-plane Jacobian is n twice, each with the full
  regulariser;
* solimp (power 2) imp(pos), aref = -b vel - k imp pos, R = (1 - imp) / imp * diag(J M^-1 J^T);
* the QP min 1/2 x^T (J M^-1 J^T + R) x + x^T (J M^-1 qf - aref), x >= 0, solved exactly (NNLS on the Cholesky factor,
  polished on its active set, KKT checked in float64); the Hessian is SPD, so x and J^T x are unique;
* semi-implicit Euler: qd += dt (M + dt D)^-1 (qf + J^T x), q += dt qd.

Radius.  Part 1, building the system in fp32.  The kernel solves the 3-row form of a contact (the out-of-plane pair merged
into one row with half the regulariser; its multiplier is the sum of the pair's, which are equal at the minimiser by
symmetry), so the perturbation analysis runs on that system A x = -b: every entry of J (geometry), of M^-1 (its entries are
(1/m) delta + (1/I) g g^T with g = (r_y, -r_x, 1): gamma_4 of their magnitude plus the propagated radius of r), of
A = J M^-1 J^T (two dot products: gamma_3 then gamma_5), of the regularised diagonal and of b carries a radius.  If x~ solves
the LCP (A~, b~) then it solves the LCP (A, b~ + dA x~): for a strongly monotone LCP (lambda = lambda_min(A) > 0, float64,
per sample) two solutions for right-hand sides q and q' satisfy lambda |x - x'|^2 <= (x - x')^T A (x - x') = -(x - x')^T (q - q')
- x^T w' - x'^T w <= |x - x'| |q - q'|, so |x~ - x|_2 <= (|rb|_2 + |rA (|x| + e)|_2) / lambda; with |rA x~| <= |rA |x|| +
|rA|_F e this solves to e <= (|rb| + |rA |x||) / (lambda - |rA|_F).  That normwise bound is the fallback; the radius
used is componentwise.  The solution of an LCP with an SPD matrix is piecewise linear in its right-hand side: on the piece
with active set S', dx = -A_S'S'^-1 dq_S' and dF = J_S'^T dx.  Integrated along the segment from b to b~ + eps + dA x~,
|x~ - x| <= Gx |dq| and |J^T (x~ - x)| <= GF |dq|, with Gx, GF the elementwise maxima of |A_S'S'^-1| and |J_S'^T A_S'S'^-1|
over the active sets the segment can cross, and |dq| <= t0 + C |x~ - x| solved as the least nonnegative solution of
(I - C Gx) dq = t0 (valid while |C Gx|_inf < 1).  A first pass takes every S'; rows whose multiplier exceeds its bound stay
active on the whole segment, rows at 0 whose residual exceeds its bound stay inactive, and a second pass takes only the sets
between those.  GF does not charge the force for the null space of J^T that the dependent rows of a contact leave in x.
Part 2, the solver.
* Fixed-point mode (TOL = 0, ITERS = 4000): the kernel stops after a sweep in which no row changed, i.e. J^T dx rounded to
  exactly 0 in all five components, which (short of an exact cancellation of five fp32 sums) means every dx_i = 0.  At such a
  point a row with x_i > 0 kept x_i = fl(x_i - fl(res_i) / D_i), so |res_i| <= u (1 + 4u) D~_i x_i; a row at 0 had res_i >= 0;
  and res_i is the residual (A~ x~ + b~)_i up to gamma_{m+2} (|b~_i| + sum_j |A~_ij| |x~_j|).  So x~ solves the LCP
  (A~, b~ + eps) exactly with |eps_i| <= rho_i(|x~|), and eps joins rb above: e <= (|rb| + |rA |x|| + |rho(|x|)|) /
  (lambda - |rA|_F - |rho'|), rho' the coefficient of e in rho(|x| + e).  Everything is computed from the inputs and the
  float64 solution; the kernel's multipliers are not needed.  The premise fails where J^T dx can round to exactly 0 with
  dx != 0: at mu = 0 the three rows of a contact are identical, and a sweep that moves the multipliers along the null space
  of J^T stops the solver there; and where 4000 sweeps do not reach a fixed point at all.  For those samples the radius is
  not proven; the tests still hold them to K radii and report how close they come.
* Production mode (TOL = 1e-6, ITERS = 100): the solver stops once a sweep moved the force J^T x by <= TOL * |J^T x|_inf.  No
  derivation of the remaining distance survives the dependent rows of a contact (the iteration matrix on the 3 rows of a
  contact has a unit eigenvalue along the null space of J^T), so the truncation radius is a STATED CONSTANT: C_TRUNC * TOL *
  |F|_inf on every component of the force F = J^T x, C_TRUNC = 4 x the largest |production - fixed point| / (TOL |F|_inf
  pushed through the integration) measured over all families (tests/pusht_families.py); along the substep chains of
  tests/pusht_chain.py the largest is 1.76 x less than C_TRUNC (TRUNC_MEASURED below).
The force radius is |J_:k|_2 e + sum_i rJ_ik (|x_i| + e) + gamma_{m+1} (|qf_k| + sum_i |J_ik x_i|); the integration
charges the solve of (M + dt D) its Gaussian-elimination backward error gamma_12 |M| (the elimination of the two slides
first, the kernel's closed form, has |L||U| = |M|) plus the radii of its entries, then one rounding per `qd + dt qdd`.

Branches: the contact test dist < 0, the limit test pm < 0 and its side pmin < pmax, the inside/outside test d2 > 0 (in fp32
d2 > 0 exactly when |lx| > hx or |ly| > hy), the face choice px < py and the signs of lx, ly on the face normal are decided
per launch (every sample of a launch shares the state).  Where a margin is within its radius, every combination of outcomes
is evaluated and the result is their interval hull; a sample whose outcomes differ by more than JUMP radii in some word is
`undecided`.  The solimp branches x < mid and x > 1 are continuous (both outcomes meet at the boundary): their hull is taken
locally and never makes a sample undecided.

Diagnostics per sample: the kernel's row count (3 per contact) and the path it takes: "none", "fast4-box0" / "fast4-box1"
(the register fast path: one contact, no limit), "solve4" / "solve8" / "solve12" (the general branch, pt_solve<NRP>).
"""
from __future__ import annotations

import itertools

import numpy as np
from scipy.optimize import nnls

from mbd_b200.envs.pusht import PT
from tests.xpbd_ref import COS_ABS_ERR, JUMP, U, R, fsum, gamma, normalize, sqrt

PI_F = float(np.float32(np.pi))
PATHS = ("none", "fast4-box0", "fast4-box1", "solve4", "solve8", "solve12")
# production-mode truncation: C_TRUNC * TOL * |J^T x|_inf on every force component, a measured constant (module docstring):
# 4 x the largest ratio measured over every family at mu = 1 and mu = 0 (2833, mu = 0 limits plus one contact;
# tests/test_pusht_ref_cpu.py::test_truncation_constant pins it).  Over the families and the substep chains of
# tests/pusht_chain.py together the largest ratio is 6577 (tests/test_pusht_horizon_ref_cpu.py pins it): mu = 0, the pusher
# pressed into the re-entrant corner by the scripted push from the `speeds` start, both contacts active (solve8), where
# Gauss-Seidel contracts so slowly that a sweep moving the force by TOL |F| still leaves it 6.6e-3 |F| from the fixed point.
# C_TRUNC is kept: 1.76 x that figure
TRUNC_FAMILIES = 2900.0
TRUNC_MEASURED = 6600.0
C_TRUNC = 4.0 * TRUNC_FAMILIES


def _f(P, name, k=0):
    return float(P[PT[name] + k])


def solver_params(P, mode, nsub=1, iters=None):
    """the parameter table with NSUB and the solver mode: 'fixed' (TOL = 0, ITERS = 4000) or 'prod' (the shipped TOL, 100)"""
    P = np.array(P, dtype=np.float32)
    P[PT["NSUB"]] = nsub
    if mode == "fixed":
        P[PT["TOL"]], P[PT["ITERS"]] = 0.0, 4000 if iters is None else iters
    else:
        P[PT["TOL"]], P[PT["ITERS"]] = np.float32(1e-6), 100 if iters is None else iters
    return P


# ---------------------------------------------------------------------------------------------------------------------
# per-launch geometry (the state is shared by every sample of a launch)
# ---------------------------------------------------------------------------------------------------------------------
class _Gates:
    """decides discontinuous predicates; records those whose margin is within its radius and, for an enumerated
    configuration, forces their outcome"""

    def __init__(self, forced=None):
        self.forced = forced or {}
        self.straddle = []
        self.inside = []          # boxes whose contact took the centre-inside branch

    def lt0(self, name, m):
        """m < 0 (m an R scalar)"""
        if name in self.forced:
            return self.forced[name]
        if abs(float(m.v)) <= float(m.r) and float(m.r) > 0:
            self.straddle.append(name)
        return bool(m.v < 0)


def _rot(c, s, x, y):
    """R(theta) (x, y)"""
    return fsum([c * x, -(s * y)]), fsum([s * x, c * y])


def _clamp_excess(x, h):
    """(clamp(x, -h, h), x - clamp(x, -h, h)): inside the band by more than the radius the clamp returns x itself and the
    excess is an exact 0; outside it by more than the radius the clamp is the exact bound"""
    if abs(x.v) + x.r < h:
        return x, R(0.0)
    if abs(x.v) - x.r > h:
        cl = R(np.sign(x.v) * h)
        return cl, x - cl
    cl = R(np.clip(x.v, -h, h), x.r)
    return cl, x - cl


def _contact(P, b, q, s, c, g):
    """sphere-box geometry of box b: dict(n (world normal, box -> sphere), rho (arm from the slider origin), dist), or the
    gate outcomes that lead there"""
    B = [_f(P, "BOX0", 4 * b + k) for k in range(4)]
    rp = _f(P, "RP")
    bx, by = _rot(c, s, B[0], B[1])
    bx, by = q[2] + bx, q[3] + by
    dx, dy = q[0] - bx, q[1] - by
    lx, ly = fsum([c * dx, s * dy]), fsum([c * dy, -(s * dx)])          # R(theta)^T d
    (clx, ex), (cly, ey) = _clamp_excess(lx, B[2]), _clamp_excess(ly, B[3])
    mx, my = R(abs(lx.v) - B[2], lx.r), R(abs(ly.v) - B[3], ly.r)
    margin = mx if mx.v >= my.v else my          # d2 > 0 in fp32 exactly when |lx| > hx or |ly| > hy
    if g.lt0(f"box{b} d2 > 0", R(-margin.v, margin.r)):
        (nlx, nly), d = normalize((ex, ey))
        dist = d - rp
        sx, sy = clx, cly
    else:
        g.inside.append(b)
        px = R(B[2] - abs(lx.v), lx.r) + 0.0
        py = R(B[3] - abs(ly.v), ly.r) + 0.0
        if g.lt0(f"box{b} px < py", px - py):
            sg = -1.0 if g.lt0(f"box{b} lx < 0", lx) else 1.0
            nlx, nly = R(sg), R(0.0)
            dist = -px - rp
            sx, sy = R(sg * B[2]), cly
        else:
            sg = -1.0 if g.lt0(f"box{b} ly < 0", ly) else 1.0
            nlx, nly = R(0.0), R(sg)
            dist = -py - rp
            sx, sy = clx, R(sg * B[3])
    nx, ny = _rot(c, s, nlx, nly)
    half = dist * 0.5
    ax, ay = B[0] + (sx + nlx * half), B[1] + (sy + nly * half)
    rx, ry = _rot(c, s, ax, ay)
    return dict(n=(nx, ny), rho=(rx, ry), dist=dist)


def _dir_row(k, dx, dy):
    """Jacobian (pusher x, y | slider x, y, theta) of the relative velocity of the contact point along (dx, dy)"""
    rx, ry = k["rho"]
    return [dx, dy, -dx, -dy, -fsum([rx * dy, -(ry * dx)])]


def geometry(P, st, forced=None):
    """the rows of one launch: dict(rows3 = [(J [5 R], pos R, rscale, tag)] in the kernel's order, rows4 = the same with the
    pyramid's out-of-plane pair as two rows, act (per box), nlim, path, straddle)"""
    g = _Gates(forced)
    q = [R(float(v)) for v in st[:8]]
    th = float(st[4])
    s, c = R(np.sin(th), COS_ABS_ERR), R(np.cos(th), COS_ABS_ERR)
    rows3, rows4 = [], []
    nlim = 0
    for k in range(4):
        lo, hi = _f(P, "LIM0", 2 * k), _f(P, "LIM0", 2 * k + 1)
        pmin, pmax = q[k] - lo, hi - q[k]
        pm = R(min(pmin.v, pmax.v), max(pmin.r, pmax.r))        # min is Lipschitz; the side matters only when active
        if g.lt0(f"lim{k} active", pm):
            low = g.lt0(f"lim{k} side", pmin - pmax)
            pm = pmin if low else pmax
            J = [R(0.0)] * 5
            J[k] = R(1.0 if low else -1.0)
            rows3.append((J, pm, 1.0, f"lim{k}"))
            rows4.append((J, pm, 1.0, f"lim{k}"))
            nlim += 1
    mu = _f(P, "MU")
    act = []
    for b in range(2):
        k = _contact(P, b, q, s, c, g)
        a = g.lt0(f"box{b} dist < 0", k["dist"])
        act.append(a)
        if not a:
            continue
        nx, ny = k["n"]
        tx, ty = -ny, nx
        r0 = _dir_row(k, nx - mu * tx, ny - mu * ty)
        r1 = _dir_row(k, nx + mu * tx, ny + mu * ty)
        rn = _dir_row(k, nx, ny)
        rows3 += [(r0, k["dist"], 1.0, f"box{b}"), (r1, k["dist"], 1.0, f"box{b}"), (rn, k["dist"], 0.5, f"box{b}")]
        rows4 += [(r0, k["dist"], 1.0, f"box{b}"), (r1, k["dist"], 1.0, f"box{b}"), (rn, k["dist"], 1.0, f"box{b}"),
                  (rn, k["dist"], 1.0, f"box{b}")]
    nr = len(rows3)
    if nr == 0:
        path = "none"
    elif nlim == 0 and act[0] != act[1]:
        path = "fast4-box0" if act[0] else "fast4-box1"
    else:
        path = "solve4" if nr <= 4 else ("solve8" if nr <= 8 else "solve12")
    return dict(rows3=rows3, rows4=rows4, path=path, nrows=nr, straddle=g.straddle, inside=g.inside, s=s, c=c, q=q)


# ---------------------------------------------------------------------------------------------------------------------
# the exact QP
# ---------------------------------------------------------------------------------------------------------------------
def qp_exact(A, b):
    """argmin 1/2 x^T A x + b^T x over x >= 0 for an SPD A, and the largest KKT violation relative to the problem's scale"""
    m = len(b)
    L = np.linalg.cholesky(A)
    x, _ = nnls(L.T, -np.linalg.solve(L, b), maxiter=50 * m)

    def polish(S):
        xs = np.zeros(m)
        if S.any():
            xs[S] = np.linalg.solve(A[np.ix_(S, S)], -b[S])
        return xs

    def kkt(x):
        w = A @ x + b
        sc = np.abs(b).max() + (np.abs(A) @ np.abs(x)).max() + 1e-300
        return max(0.0, -x.min(), -w.min(), np.abs(w * x).max() / (sc * (np.abs(x).max() + 1e-300))) / sc

    best = polish(x > 0)
    if kkt(best) > 1e-12:
        for S in itertools.product([False, True], repeat=m):   # at most 2^12 active sets: only if the polish fails
            xs = polish(np.array(S))
            if kkt(xs) <= 1e-12:
                best = xs
                break
    return best, kkt(best)


# ---------------------------------------------------------------------------------------------------------------------
# one step
# ---------------------------------------------------------------------------------------------------------------------
def _mass(P, rx, ry, inv):
    """5x5 mass matrix at the slider's COM offset (rx, ry): from the stored inverse words (inv=True, the QP's M) or from the
    stored masses plus dt * D (the integration's M + dt D)"""
    if inv:
        mp, m, I = 1.0 / _f(P, "IMP"), 1.0 / _f(P, "IMS"), 1.0 / _f(P, "IIS")
        dd = np.zeros(5)
    else:
        mp, m, I = _f(P, "MP"), _f(P, "MS"), _f(P, "IS")
        dd = _f(P, "DT") * np.array([_f(P, k) for k in ("DPX", "DPY", "DSX", "DSY", "DSTH")])
    M = np.zeros((5, 5))
    M[0, 0] = M[1, 1] = mp
    M[2, 2] = M[3, 3] = m
    M[2, 4] = M[4, 2] = -m * ry
    M[3, 4] = M[4, 3] = m * rx
    M[4, 4] = I + m * (rx * rx + ry * ry)
    return M + np.diag(dd)


def _imp_aref(P, pos, vel):
    """solimp (power 2) impedance and reference acceleration; the branches x < mid, x > 1 are continuous, their hull is
    taken where x is within its radius of the switch"""
    dmin, dmax, width, mid = (_f(P, k) for k in ("DMIN", "DMAX", "WIDTH", "MID"))
    x = R(abs(pos.v), pos.r) / width
    a = (x * x) * (1.0 / mid)
    b = 1.0 - (1.0 - x) * (1.0 - x) * (1.0 / (1.0 - mid))

    def lin(y):
        d = dmin + y * (dmax - dmin)
        return R(np.clip(d.v, dmin, dmax), d.r)

    da, db = lin(a), lin(b)
    imp = da if x.v < mid else db
    if abs(x.v - mid) <= x.r:
        lo, hi = min(da.v - da.r, db.v - db.r), max(da.v + da.r, db.v + db.r)
        imp = R(0.5 * (lo + hi), 0.5 * (hi - lo))
    if x.v > 1.0:
        imp = R(dmax)
    if abs(x.v - 1.0) <= x.r:
        lo, hi = min(imp.v - imp.r, dmax), max(imp.v + imp.r, dmax)
        imp = R(0.5 * (lo + hi), 0.5 * (hi - lo))
    aref = -(vel * _f(P, "KB")) - (imp * _f(P, "KK")) * pos
    return imp, aref


def _one_config(P, st, u, geo):
    n = u.shape[0]
    s, c, q = geo["s"], geo["c"], geo["q"]
    qd = [R(float(v)) for v in st[8:16]]
    dt = _f(P, "DT")
    CX, CY = _f(P, "CX"), _f(P, "CY")
    rx, ry = _rot(c, s, CX, CY)
    ms = _f(P, "MS")
    w = qd[4]
    mw2 = (w * w) * ms
    f = [R(u[:, 0]) * _f(P, "GEAR0") - qd[0] * _f(P, "DPX"), R(u[:, 1]) * _f(P, "GEAR1") - qd[1] * _f(P, "DPY"),
         mw2 * rx - qd[2] * _f(P, "DSX"), mw2 * ry - qd[3] * _f(P, "DSY"), -(w * _f(P, "DSTH"))]
    fv = np.stack([np.broadcast_to(t.v, (n,)) for t in f], 1)
    fr = np.stack([np.broadcast_to(t.r, (n,)) for t in f], 1)

    # ---- inverse mass of the QP and its radius: (1/m) delta + (1/I) g g^T, g = (r_y, -r_x, 1)
    Mi = np.linalg.inv(_mass(P, float(rx.v), float(ry.v), inv=True))
    ims, iIs = _f(P, "IMS"), _f(P, "IIS")
    gv = np.array([0.0, 0.0, abs(float(ry.v)), abs(float(rx.v)), 1.0])
    gr = np.array([0.0, 0.0, float(ry.r), float(rx.r), 0.0])
    rMi = np.zeros((5, 5))                                        # the pusher's IMP: a stored word, used as is
    sl = slice(2, 5)
    base = np.diag([0, 0, ims, ims, 0.0]) + iIs * np.outer(gv, gv)
    rMi[sl, sl] = (gamma(4) * base + iIs * (np.outer(gr, gv) + np.outer(gv, gr) + np.outer(gr, gr)))[sl, sl]

    # ---- the two forms of the rows
    def mats(rows):
        m = len(rows)
        J = np.array([[float(t.v) for t in r[0]] for r in rows]).reshape(m, 5)
        rJ = np.array([[float(t.r) for t in r[0]] for r in rows]).reshape(m, 5)
        return J, rJ

    rows3, rows4 = geo["rows3"], geo["rows4"]
    m3, m4 = len(rows3), len(rows4)
    out = {}
    Mint = _mass(P, float(rx.v), float(ry.v), inv=False)
    Minti = np.linalg.inv(Mint)
    # radius of the entries of M + dt D (one rounding per operation of its assembly)
    ms_, Is = _f(P, "MS"), _f(P, "IS")
    a_ = -(ry * ms_)
    b_ = rx * ms_
    J3 = (fsum([rx * rx, ry * ry]) * ms_ + Is) + dt * _f(P, "DSTH")
    rMint = np.zeros((5, 5))
    rMint[0, 0] = gamma(2) * Mint[0, 0]
    rMint[1, 1] = gamma(2) * Mint[1, 1]
    rMint[2, 2] = gamma(2) * Mint[2, 2]
    rMint[3, 3] = gamma(2) * Mint[3, 3]
    rMint[2, 4] = rMint[4, 2] = float(a_.r)
    rMint[3, 4] = rMint[4, 3] = float(b_.r)
    rMint[4, 4] = float(J3.r)

    if m4 == 0:
        F = np.zeros((n, 5))
        rF = np.zeros((n, 5))
        x3 = np.zeros((n, 0))
        out["kkt"] = 0.0
        out["merge_gap"] = 0.0
        Fscale = np.zeros(n)
    else:
        J4, _ = mats(rows4)
        J3m, rJ3 = mats(rows3)
        qdv = np.array([float(t.v) for t in qd[:5]])

        def system(rows, J, rJ):
            MiJ = J @ Mi                                       # rows of (M^-1 J^T)^T
            A = J @ Mi @ J.T
            m = len(rows)
            imp, aref = [], []
            for i, (Jr, pos, rsc, _) in enumerate(rows):
                vel = fsum([Jr[k] * qd[k] for k in range(5)])
                im, ar = _imp_aref(P, pos, vel)
                imp.append(im)
                aref.append(ar)
            rMiJ = np.abs(rJ) @ np.abs(Mi) + np.abs(J) @ rMi + gamma(3) * (np.abs(J) @ np.abs(Mi))
            rA = np.abs(J) @ rMiJ.T + rJ @ np.abs(MiJ).T + gamma(5) * (np.abs(J) @ np.abs(MiJ).T)
            D = np.zeros(m)
            rD = np.zeros(m)
            for i, (_, _, rsc, _) in enumerate(rows):
                arr = R(A[i, i], rA[i, i])
                d = arr + ((1.0 - imp[i]) / imp[i] * rsc) * arr
                D[i], rD[i] = float(d.v), float(d.r)
            Areg = A.copy()
            Areg[np.diag_indices(m)] = D
            rAreg = rA.copy()
            rAreg[np.diag_indices(m)] = rD
            Mif = fv @ Mi.T                                    # [n, 5]
            rMif = fr @ np.abs(Mi).T + np.abs(fv) @ rMi.T + gamma(3) * (np.abs(fv) @ np.abs(Mi).T)
            bq = Mif @ J.T                                     # [n, m]
            rb = rMif @ np.abs(J).T + np.abs(Mif) @ rJ.T + gamma(5) * (np.abs(Mif) @ np.abs(J).T)
            arv = np.array([float(a.v) for a in aref])
            arr_ = np.array([float(a.r) for a in aref])
            bq = bq - arv
            rb = rb + arr_ + U * (np.abs(bq) + rb)
            return Areg, rAreg, bq, rb, D, rD

        A4, _, b4, _, _, _ = system(rows4, J4, np.zeros_like(J4))
        A3, rA3, b3, rb3, D3, rD3 = system(rows3, J3m, rJ3)
        x4 = np.zeros((n, m4))
        x3s = np.zeros((n, m3))
        kk = 0.0
        for i in range(n):
            x4[i], e1 = qp_exact(A4, b4[i])
            x3s[i], e2 = qp_exact(A3, b3[i])
            kk = max(kk, e1, e2)
        out["kkt"] = kk
        F = x4 @ J4
        F3 = x3s @ J3m
        Fscale = np.abs(F).max(1)
        out["merge_gap"] = float(np.max(np.abs(F3 - F) / np.maximum(Fscale, 1e-30)[:, None])) if n else 0.0
        # the kernel's multipliers: the 3-row form of the float64 minimiser (the out-of-plane pair summed)
        x3 = np.zeros((n, m3))
        j = 0
        for i, r in enumerate(rows3):
            x3[:, i] = x4[:, j]
            if r[2] == 0.5:
                x3[:, i] += x4[:, j + 1]
                j += 1
            j += 1
        lam = float(np.linalg.eigvalsh(A3).min())
        rAF = float(np.linalg.norm(rA3))
        ax = np.abs(x3)
        tA = np.linalg.norm(ax @ rA3.T, axis=1)
        trb = np.linalg.norm(rb3, axis=1)
        Aabs = np.abs(A3) + rA3
        gm = gamma(m3 + 2)
        rho0 = U * (1 + 4 * U) * (D3 + rD3) * ax + gm * ((np.abs(b3) + rb3) + ax @ Aabs.T)
        rho1 = U * (1 + 4 * U) * (D3 + rD3) + gm * Aabs.sum(1)
        den = lam - rAF - float(np.linalg.norm(rho1))
        with np.errstate(divide="ignore"):
            e = np.where(den > 0, (trb + tA + np.linalg.norm(rho0, axis=1)) / max(den, 1e-300), np.inf)
        rF = (np.linalg.norm(J3m, axis=0)[None, :] * e[:, None] + (ax + e[:, None]) @ rJ3
              + gamma(m3 + 1) * (np.abs(fv) + ax @ np.abs(J3m)))
        # componentwise, along the path: x~ solves the LCP (A, q~) with q~ = b~ + eps + dA x~, and the solution of an LCP with
        # an SPD matrix is piecewise linear in q: on the piece with active set S', dx = -A_S'S'^-1 dq_S' and dF = J_S'^T dx.
        # So |x~ - x| <= Gx |dq| and |F~ - F| <= GF |dq|, Gx / GF the elementwise maxima of |A_S'S'^-1| / |J_S'^T A_S'S'^-1|
        # over the active sets the path can cross, |dq| <= t0 + C |x~ - x| (rb, rho and rA |x~| at |x~| <= |x| + |dx|).
        # Stage 1 takes every S'; rows whose multiplier or residual exceeds its stage-1 bound keep their status on the whole
        # path, so stage 2 takes only the sets between the surely active rows and those plus the uncertain ones.
        stable = np.zeros(n, bool)
        w3 = x3 @ A3.T + b3
        C = rA3 + gm * Aabs + np.diag(U * (1 + 4 * U) * (D3 + rD3))
        gains = {}

        def gain(sure, unc):
            key = (sure.tobytes(), unc.tobytes())
            if key not in gains:
                Gx, GF = np.zeros((m3, m3)), np.zeros((5, m3))
                ui = np.flatnonzero(unc)
                for bits in itertools.product([False, True], repeat=len(ui)):
                    Sp = sure.copy()
                    Sp[ui[np.array(bits, bool)]] = True
                    if not Sp.any():
                        continue
                    Ai = np.linalg.inv(A3[np.ix_(Sp, Sp)])
                    Gx[np.ix_(Sp, Sp)] = np.maximum(Gx[np.ix_(Sp, Sp)], np.abs(Ai))
                    GF[:, Sp] = np.maximum(GF[:, Sp], np.abs(J3m[Sp].T @ Ai))
                gains[key] = (Gx, GF)
            return gains[key]

        none, every = np.zeros(m3, bool), np.ones(m3, bool)
        for i in range(n):
            t0 = rb3[i] + gm * (np.abs(b3[i]) + rb3[i]) + C @ ax[i]

            def dq_of(Gx):
                Mx = C @ Gx
                if np.abs(Mx).sum(1).max() >= 0.5:
                    return None
                return np.linalg.solve(np.eye(m3) - Mx, t0)     # = sum_k Mx^k t0 >= 0, the least solution of dq >= t0 + Mx dq

            Gx, GF = gain(none, every)
            dq = dq_of(Gx)
            if dq is None:
                continue                                           # keep the normwise bound
            dx = Gx @ dq
            sure = x3[i] > dx
            unc = ~sure & ~((x3[i] == 0) & (w3[i] > np.abs(A3) @ dx + dq))
            Gx2, GF2 = gain(sure, unc)
            dq2 = dq_of(Gx2)
            if dq2 is not None:
                Gx, GF, dq = Gx2, GF2, dq2
            stable[i] = not unc.any()
            rF[i] = GF @ dq + (ax[i] + Gx @ dq) @ rJ3 + gamma(m3 + 1) * (np.abs(fv[i]) + ax[i] @ np.abs(J3m))
        out["lam"] = lam
        out["e"] = e
        out["stable"] = stable
    ftot = fv + F
    rftot = fr + rF
    # ---- (M + dt D) qdd = ftot: the solve's backward error gamma_12 |M| plus the radii of M's entries
    qdd = ftot @ Minti.T
    dM = (rMint + gamma(12) * np.abs(Mint)).T
    rq = (rftot + np.abs(qdd) @ dM) @ np.abs(Minti).T
    rq = (rftot + (np.abs(qdd) + rq) @ dM) @ np.abs(Minti).T       # |qdd~| <= |qdd| + first-order radius
    qdd_r = [R(qdd[:, k], rq[:, k]) for k in range(5)]
    # unit truncation radius: TOL * |F|_inf on every force component, through the same solve
    tol = _f(P, "TOL")
    tF = np.repeat((tol * Fscale)[:, None], 5, 1)
    tq = tF @ np.abs(Minti).T * (1 + 1e-6)
    value = np.zeros((n, 16))
    radius = np.zeros((n, 16))
    trunc = np.zeros((n, 16))
    value[:] = st.astype(np.float64)
    for k in range(5):
        v1 = qd[k] + qdd_r[k] * dt
        p1 = q[k] + v1 * dt
        value[:, 8 + k], radius[:, 8 + k] = v1.v, v1.r
        value[:, k], radius[:, k] = p1.v, p1.r
        trunc[:, 8 + k] = tq[:, k] * dt * (1 + 4 * U)
        trunc[:, k] = trunc[:, 8 + k] * dt * (1 + 4 * U)
    out.update(value=value, radius=radius, trunc=trunc, x3=x3, F=F, impulse=dt * (F @ Minti.T))
    return out


def step(P, st, u):
    """one physics step of pushT for one fp32 state [16] and fp32 controls [n, 2] (clipped here like the kernel) ->
    dict(value [n, 16], radius_fixed, trunc_unit [n, 16], undecided [n], path, nrows, straddle, kkt, merge_gap, configs: per
    enumerated gate outcome, among others the velocity change of the constraint impulse, impulse [n, 5] = dt (M + dt D)^-1 J^T x)"""
    P = np.asarray(P, dtype=np.float32).astype(np.float64)
    st = np.asarray(st, dtype=np.float32).astype(np.float64)
    u = np.clip(np.asarray(u, dtype=np.float32).astype(np.float64), -1.0, 1.0)
    geo = geometry(P, st)
    names = list(dict.fromkeys(geo["straddle"]))
    outs, geos = [], []
    for vals in itertools.product([False, True], repeat=len(names)):
        forced = dict(zip(names, vals))
        gg = geometry(P, st, forced) if names else geo
        new = [x for x in gg["straddle"] if x not in forced]
        assert not new, f"gates {new} only straddle under another outcome"
        geos.append(gg)
        outs.append(_one_config(P, st, u, gg))
    o0 = outs[0] if len(outs) == 1 else None
    if o0 is not None:
        value, radius, trunc = o0["value"], o0["radius"], o0["trunc"]
        undecided = np.zeros(u.shape[0], bool)
    else:
        lo = np.min([o["value"] - o["radius"] for o in outs], 0)
        hi = np.max([o["value"] + o["radius"] for o in outs], 0)
        value, radius = 0.5 * (lo + hi), 0.5 * (hi - lo)
        trunc = np.max([o["trunc"] for o in outs], 0)
        undecided = np.zeros(u.shape[0], bool)
        for a, b in itertools.combinations(outs, 2):
            jump = np.abs(a["value"] - b["value"]) > JUMP * np.maximum(a["radius"], b["radius"])
            undecided |= jump.any(1)
    return dict(value=value, radius=radius, trunc=trunc, undecided=undecided, path=geo["path"], nrows=geo["nrows"], inside=geo["inside"],
                paths={g["path"] for g in geos}, straddle=names, kkt=max(o["kkt"] for o in outs),
                merge_gap=max(o["merge_gap"] for o in outs), configs=outs)


def radius(ref, mode):
    """the radius of a solver mode: fixed point, or fixed point + C_TRUNC x the unit truncation radius"""
    return ref["radius"] if mode == "fixed" else ref["radius"] + C_TRUNC * ref["trunc"]


# ---------------------------------------------------------------------------------------------------------------------
# reward (pushT.py:50-62) on a given fp32 state, and the return
# ---------------------------------------------------------------------------------------------------------------------
def reward(states):
    """states [..., >= 8] fp32 -> R of the per-step reward 1 - (|goal - slider| + |theta_g - theta| / pi + max(|pusher -
    slider| - 0.2, 0)), pi and 0.2 as the fp32 constants the kernel uses"""
    s = np.asarray(states, dtype=np.float32).astype(np.float64)
    q = [R(s[..., k]) for k in range(8)]
    gx, gy = q[5] - q[2], q[6] - q[3]
    px, py = q[0] - q[2], q[1] - q[3]
    dps = sqrt(fsum([px * px, py * py])) - float(np.float32(0.2))
    d = R(np.maximum(dps.v, 0.0), dps.r)
    ang = q[7] - q[4]
    return 1.0 - ((sqrt(fsum([gx * gx, gy * gy])) + R(np.abs(ang.v), ang.r) / PI_F) + d)


def mean_return(rewss):
    """sum_t r_t / H of given fp32 per-step rewards [n, H]: gamma_H sum|r| for the sum, one rounding for the division"""
    r = np.asarray(rewss, dtype=np.float32).astype(np.float64)
    H = r.shape[1]
    tot = fsum([R(r[:, t]) for t in range(H)])
    return tot / float(H)


# ---------------------------------------------------------------------------------------------------------------------
# undecided samples: held to one enumerated configuration
# ---------------------------------------------------------------------------------------------------------------------
def held_ratios(got, ref, mode):
    """got [n, 16] against every enumerated gate configuration of ref = step(...) in a solver mode -> (best [u], second [u])
    over the u undecided samples: the largest ratio to the nearest configuration, and to the next-nearest (inf with one)"""
    und = ref["undecided"]
    g = np.asarray(got, dtype=np.float64)[und]
    per = []
    for cfg in ref["configs"]:
        d = np.abs(g - cfg["value"][und])
        with np.errstate(divide="ignore", invalid="ignore"):
            q = np.where(d == 0, 0.0, d / radius(cfg, mode)[und])
        per.append(np.where(np.isfinite(d), q, np.inf).max(1))
    per = np.sort(np.stack(per), axis=0)
    return per[0], (per[1] if len(per) > 1 else np.full(len(g), np.inf))
