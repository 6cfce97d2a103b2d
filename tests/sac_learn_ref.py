"""Float64 contract of the fused SAC update (include/mbd_sac_learn.h, DESIGN.md §2): the gradients of the three losses carried with
radii to every dW, db and the log alpha gradient, and Adam / Polyak given an fp32 gradient.

The forward passes use tests/rl_ref.py's running-error arithmetic (dense units, ReLU, the NormalTanh head).  The backward pass
extends it:
* a backward matvec d_in = W d_out is charged |W| r_out plus gamma_{nout+1} of every term's magnitude;
* a ReLU derivative whose pre-activation lies within its radius of 0 may take either branch: the radius becomes |value| + radius
  (the union of 0 and the propagated value);
* the actor seed is -1 into the critic that gives the min; where the two critics' Q lie within their radii of each other either
  critic may be picked, and both seeds get radius 1 (the union of 0 and -1);
* dW = sum_b In_b D_b / N is charged the inputs' radii through |D| and |In|, gamma_{n+1} of the magnitudes and the division's rounding.
The values are float64 evaluations of the formulas; `check_grads` also holds them to sac_ref.grads64 (torch autograd in float64).

Adam (torch's formula, capturable) and Polyak are checked given the implementation's own fp32 gradient against float64 Adam and
Polyak of that gradient, with the fp32 constants 0.1f, 0.999f, 0.001f charged as inputs with radii.
"""
from __future__ import annotations

import math

import numpy as np

from mbd_b200.rl import networks as nets
from tests import rl_ref
from tests.rl_ref import EXP_REL
from tests.xpbd_ref import ETA, R, U, exact_scale, gamma

f32 = np.float32
H = 256
K = 2.0                 # the contract holds results to K radii, as tests/rl_ref.py
ALPHA_LR = 3e-4


def _w(a):
    return np.asarray(a, f32).astype(np.float64)


def _cols(x: R, a, b) -> R:
    return R(x.v[:, a:b], x.r[:, a:b])


def _cat(a: R, b: R) -> R:
    return R(np.concatenate([a.v, b.v], 1), np.concatenate([a.r, b.r], 1))


def q_layers(q, O, nu, c):
    """[(W, b)] of critic c in float64 (the layer-major buffer)"""
    out = []
    for l, (W, b) in enumerate(nets.sac_q_unflatten(np.asarray(q, f32), nets.sac_q_sizes(O, nu))):
        out.append((_w(W[c]), _w(b[c, 0])))
    return out


def mlp(x: R, layers):
    """(pre-activations of the hidden layers, their ReLU outputs, the output) with radii"""
    pre, hs = [], []
    for l, (W, b) in enumerate(layers):
        x = rl_ref.dense(x, W, b)
        if l + 1 < len(layers):
            pre.append(x)
            x = rl_ref.relu(x)
            hs.append(x)
    return pre, hs, x


def back(W, d: R, pre: R | None) -> R:
    """d @ W^T (W [nin, nout], d [n, nout]) with the ReLU derivative of `pre` (None: no mask)"""
    aW = np.abs(W)
    v = d.v @ W.T
    prop = d.r @ aW.T
    k = W.shape[1] + 1
    r = prop + gamma(k) * ((np.abs(d.v) + d.r) @ aW.T) + k * ETA
    if pre is None:
        return R(v, r)
    on = pre.v > 0
    unsure = (np.abs(pre.v) <= pre.r) & (pre.r > 0)
    r = np.where(unsure, np.abs(v) + r, np.where(on, r, 0.0))
    return R(np.where(on, v, 0.0), r)


def wgrad(In: R, D: R, N: int) -> R:
    """sum_b In[b] (x) D[b] / N with the bias row (In = 1) appended: [nin + 1, nout]"""
    n = In.v.shape[0]
    In = _cat(In, R(np.ones((n, 1))))
    aI, aD = np.abs(In.v), np.abs(D.v)
    v = In.v.T @ D.v / N
    prop = (In.r.T @ aD + aI.T @ D.r + In.r.T @ D.r) / N
    r = prop + gamma(n + 1) * ((aI + In.r).T @ (aD + D.r)) / N
    return R(v, r + U * (np.abs(v) + r) + (n + 2) * ETA)


def _sigmoid(s: R) -> R:
    v = 1.0 / (1.0 + np.exp(-np.clip(s.v, -700, 700)))
    return R(v, 0.25 * s.r + (EXP_REL + 3.0) * U * (v + 0.25 * s.r) + ETA)


def _rowsum(x: R) -> R:
    k = x.v.shape[1]
    return R(x.v.sum(1), x.r.sum(1) + gamma(k) * (np.abs(x.v) + x.r).sum(1) + k * ETA)


def _mean_rows(x: R, n: int) -> R:
    """sum over the rows (any order) / n"""
    s = R(x.v.sum(), x.r.sum() + gamma(n) * (np.abs(x.v) + x.r).sum() + n * ETA)
    return s / float(n)


def contract(policy, q, target_q, log_alpha, mean, std, rows, eps, O, nu, reward_scaling, discounting) -> dict:
    """the three gradients as R in the parameters' flat layouts (policy [P], q [Q], alpha [1]) and the three losses"""
    rows = np.asarray(rows, f32)
    eps = np.asarray(eps, f32).astype(np.float64)
    n = rows.shape[0]
    obs, action = rows[:, :O], rows[:, O:O + nu].astype(np.float64)
    reward, discount = rows[:, O + nu].astype(np.float64), rows[:, O + nu + 1].astype(np.float64)
    next_obs, trunc = rows[:, O + nu + 2:2 * O + nu + 2], rows[:, 2 * O + nu + 2].astype(np.float64)
    x, xn = rl_ref.normalize(obs, mean, std), rl_ref.normalize(next_obs, mean, std)
    pl = [(_w(W), _w(b)) for W, b in nets.unflatten(np.asarray(policy, f32), nets.sac_policy_sizes(O, nu))]
    la = float(f32(np.asarray(log_alpha).reshape(-1)[0]))
    av = math.exp(la)
    alpha = R(np.float64(av), EXP_REL * U * av + ETA)
    # the target
    _, _, ln = mlp(xn, pl)
    _, tc, lpc_j, _, _ = rl_ref.head(_cols(ln, 0, nu), _cols(ln, nu, 2 * nu), eps[1])
    lpc = _rowsum(lpc_j)
    qt = [mlp(_cat(xn, tc), q_layers(target_q, O, nu, c))[2] for c in range(2)]
    qt0, qt1 = R(qt[0].v[:, 0], qt[0].r[:, 0]), R(qt[1].v[:, 0], qt[1].r[:, 0])
    qmin = R(np.minimum(qt0.v, qt1.v), np.maximum(qt0.r, qt1.r))
    rs, dg = float(f32(reward_scaling)), float(f32(discounting))
    target = R(reward) * rs + (R(discount) * dg) * (qmin - alpha * lpc)
    # the policy on x and its heads
    ppre, ph, lg = mlp(x, pl)
    loc, s = _cols(lg, 0, nu), _cols(lg, nu, 2 * nu)
    _, _, lpa_j, _, _ = rl_ref.head(loc, s, eps[0])
    _, tp, lpp_j, scale, _ = rl_ref.head(loc, s, eps[2])
    lpa, lpp = _rowsum(lpa_j), _rowsum(lpp_j)
    # the critics on (x, action) and on (x, tanh raw_p)
    m = 1.0 - trunc
    cin, ain = _cat(x, R(action)), _cat(x, tp)
    crit, act = [], []
    for c in range(2):
        L = q_layers(q, O, nu, c)
        crit.append((L,) + mlp(cin, L))
        act.append(mlp(ain, L))
    qa = [R(a[2].v[:, 0], a[2].r[:, 0]) for a in act]
    gq = np.zeros(nets.sac_q_num_params(O, nu))
    rq = np.zeros_like(gq)
    errs = []
    for c in range(2):
        L, pre, hs, qv = crit[c]
        err = (R(qv.v[:, 0], qv.r[:, 0]) - target) * m
        errs.append(err)
        d3 = err * m
        d3 = R(d3.v[:, None], d3.r[:, None])
        d2 = back(L[2][0], d3, pre[1])
        d1 = back(L[1][0], d2, pre[0])
        for l, (In, D) in enumerate(((cin, d1), (hs[0], d2), (hs[1], d3))):
            g = wgrad(In, D, 2 * n)
            nin, nout = g.v.shape[0] - 1, g.v.shape[1]
            off = _q_off(O, nu, l)
            wsl = slice(off + c * nin * nout, off + (c + 1) * nin * nout)
            bsl = slice(off + 2 * nin * nout + c * nout, off + 2 * nin * nout + (c + 1) * nout)
            gq[wsl], rq[wsl] = g.v[:nin].ravel(), g.r[:nin].ravel()
            gq[bsl], rq[bsl] = g.v[nin], g.r[nin]
    # the actor: seeds, the action gradient through the critics, the head, the policy
    pick0 = qa[0].v <= qa[1].v
    tie = np.abs(qa[0].v - qa[1].v) <= qa[0].r + qa[1].r
    gA = None
    for c in range(2):
        L = crit[c][0]
        pre, _, _ = act[c]
        seed = R(np.where(pick0 == (c == 0), -1.0, 0.0)[:, None], np.where(tie, 1.0, 0.0)[:, None])
        d2 = back(L[2][0], seed, pre[1])
        d1 = back(L[1][0], d2, pre[0])
        ga = back(L[0][0][O:], d1, None)
        gA = ga if gA is None else gA + ga
    t = tp
    g = gA * (1.0 - t * t) + alpha * exact_scale(t, 2.0)
    dloc = g
    ds = (g * R(eps[2]) - alpha / scale) * _sigmoid(s)
    dp3 = _cat(dloc, ds)
    dp2 = back(pl[2][0], dp3, ppre[1])
    dp1 = back(pl[1][0], dp2, ppre[0])
    gp, rp = [], []
    for In, D in ((x, dp1), (ph[0], dp2), (ph[1], dp3)):
        gw = wgrad(In, D, n)
        gp.append(gw.v.ravel())
        rp.append(gw.r.ravel())
    aterm = -lpa - (-0.5 * nu)
    ga = alpha * _mean_rows(R(aterm.v[:, None], aterm.r[:, None]), n)
    e2 = errs[0] * errs[0] + errs[1] * errs[1]
    closs = exact_scale(_mean_rows(R(e2.v[:, None], e2.r[:, None]), n), 0.25)
    qmin_a = R(np.minimum(qa[0].v, qa[1].v), np.maximum(qa[0].r, qa[1].r))
    at = alpha * lpp - qmin_a
    aloss = _mean_rows(R(at.v[:, None], at.r[:, None]), n)
    return dict(policy=R(np.concatenate(gp), np.concatenate(rp)), q=R(gq, rq), alpha=R(np.atleast_1d(ga.v), np.atleast_1d(ga.r)),
                losses=R(np.array([ga.v, closs.v, aloss.v]), np.array([ga.r, closs.r, aloss.r])))


def _q_off(O, nu, l):
    sizes = nets.sac_q_sizes(O, nu)
    return sum(2 * (i * o + o) for i, o in sizes[:l])


# ---- Adam and Polyak given an fp32 gradient -----------------------------------------------------------------------------------------
def _c32(x: float) -> R:
    """an fp32 constant of the implementation standing for the exact x"""
    return R(np.float64(x), abs(float(f32(x)) - x) + ETA)


def _sqrt(x: R) -> R:
    v = np.sqrt(np.maximum(x.v, 0.0))
    lo = np.maximum(x.v - x.r, 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        prop = np.where(lo > 0, x.r / (np.sqrt(lo) + v), np.sqrt(x.r))
    return R(v, prop + U * (v + prop) + ETA)


def adam(p, m, v, g, lr, t: int):
    """torch.optim.Adam's step t (float64 values of the formula on the fp32 inputs p, m, v, g; lr the fp32 word) with the radius of
    the fp32 evaluation: (p, m, v) as R"""
    p, m, v, g = (R(_w(a)) for a in (p, m, v, g))
    lr = float(f32(lr))
    mm = m + _c32(0.1) * (g - m)
    vv = v * _c32(0.999) + _c32(0.001) * (g * g)
    b1, b2 = 1.0 - 0.9 ** t, 1.0 - 0.999 ** t
    bc1 = R(np.float64(b1), U * b1 + 64 * 2.0 ** -53)       # float64 pow by squaring, rounded to fp32
    bc2 = R(np.float64(b2), U * b2 + 64 * 2.0 ** -53)
    step = R(np.float64(lr)) / bc1
    denom = _sqrt(vv) / _sqrt(bc2) + _c32(1e-8)
    return p - step * (mm / denom), mm, vv


def polyak(target, q_new, tau):
    return R(_w(target)) + float(f32(tau)) * (R(_w(q_new)) - R(_w(target)))
