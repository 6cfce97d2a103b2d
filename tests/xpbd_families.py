"""Input families for the float64 check of one positional substep (tests/xpbd_ref.py), shared by the CPU and the GPU tests.

Each family is a list of (state [L, 13] float32, actions [n, nu] float32): one constructed state, shared by every sample of
a launch, and a batch of different actions.  States come from `kinematics.pipeline_init` on chosen joint coordinates,
or from direct edits of such a state.
  F1 nominal       reset pose, joint rates +-2 rad/s
  F2 open joints   child links displaced by 1e-3..1e-2 m and turned 0.05 rad off their joint
  F3 limits        every limited hinge at lo -+ 1e-2 and hi -+ 1e-2
  F4 Euler corners the middle angle of every 2-/3-dof joint at 0, 1e-4 and +-(pi/2 - 0.05)
  F5 contacts      the lowest contact at dist -1e-2, -1e-4, +1e-4; at rest, small / large tangential travel, approaching
                   and separating
  F6 slide dofs    planar roots and carts inside, at and beyond their slide limits, moving along and across the rail
  F7 far away      F1 translated by (100, -50, 0) m
Every family's actions mix N(0, 0.7) draws (clipped), saturated +-1 and +-37 (far outside ctrl_range).
"""
from __future__ import annotations

import os

import numpy as np

from mbd_b200.model import blob as B

FIX = os.path.join(os.path.dirname(__file__), "fixtures")
SHIPPED = ["humanoidrun", "humanoidstandup", "humanoidtrack", "hopper", "walker2d", "ant", "halfcheetah", "cartpole"]
MODELGEN_SEEDS = [0, 1, 2, 3, 4, 5, 100, 101, 102, 103, 104, 105]   # 100.. are 11-link trees
FAMILIES = ["F1", "F2", "F3", "F4", "F5", "F6", "F7"]
# largest absolute radius of any output word (m, m/s, rad/s, quaternion units) per family: the check must not pass on any
# plausible value.  F4 holds joints 0.05 rad from gimbal lock, F7 states 100 m from the origin (7.6e-6 m fp32 resolution,
# divided by dt in project_xd); the other families stay far below their cap.
RADIUS_CAP = {"F1": 0.05, "F2": 0.05, "F3": 0.5, "F4": 2.0, "F5": 0.5, "F6": 0.1, "F7": 1.0}


def undecided_cap(model, family):
    """largest fraction of undecided samples (tests/xpbd_ref.py: a branch within its radius whose two outcomes differ by
    more than JUMP radii) a (model, family) may have"""
    if model == "contact_params":
        return 0.0            # the constructed model (F8): every family decided
    if family == "F5":
        return 0.025          # contacts placed at the floor: static-friction cone and dist = 0 within the radius
    if model == "ant" and family in ("F1", "F2"):
        return 0.08           # ant's feet rest on the floor in its reset pose, so its F1 / F2 states are contact states too
    if model == "humanoidstandup" and family == "F3":
        return 0.01           # lies on the floor: same reason
    if family in ("F1", "F2", "F7"):
        return 0.01
    return 0.0                # F3, F4, F6: margins far above the radii


def make_env(name, tmpdir):
    """a shipped env by name, 'contact_params' (tests/fixtures/contact_params.xml) or 'gen<seed>' (tests/modelgen.py)"""
    import mbd_b200
    if name == "contact_params":
        return mbd_b200.envs.GenericPositionalEnv(os.path.join(FIX, "contact_params.xml"), n_frames=5)
    if name.startswith("gen"):
        from tests import modelgen
        seed = int(name[3:])
        xml, _ = modelgen.random_model(seed, links=11 if seed >= 100 else 0)
        p = os.path.join(str(tmpdir), f"gen{seed}.xml")
        with open(p, "w") as f:
            f.write(xml)
        return mbd_b200.envs.GenericPositionalEnv(p, n_frames=3)
    return mbd_b200.envs.get_env(name)


def actions(nu, n, seed):
    rng = np.random.default_rng(seed)
    a = np.clip(rng.normal(size=(n, nu)) * 0.7, -1.0, 1.0)
    a[0], a[1] = 1.0, -1.0
    a[2], a[3] = 37.0, -37.0
    a[4, ::2] = 37.0
    return a.astype(np.float32)


def _hinges(sys, links):
    """(link, k, q index, dof index) of every hinge dof of the simulated links"""
    out = []
    for l in links:
        t = sys.link_types[l]
        if t == "f":
            continue
        qs, ds = int(sys.link_q_start[l]), int(sys.link_dof_start[l])
        for k in range(int(t)):
            if not sys.dof_is_slide[ds + k]:
                out.append((l, k, qs + k, ds + k))
    return out


def _base(env, rng):
    sys = env.sys
    q = sys.init_q.astype(np.float64).copy()
    for (_, _, qi, _) in _hinges(sys, env._links):
        q[qi] += rng.uniform(-0.05, 0.05)
    qd = rng.uniform(-2.0, 2.0, size=sys.qd_size())
    return q, qd


def _init(env, q, qd):
    return np.ascontiguousarray(env.pipeline_init(q, qd).raw, dtype=np.float32)


def _qmul(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return np.array([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw])


def _rot(v, q):
    w, u = q[0], q[1:]
    t = 2 * np.cross(u, v)
    return v + w * t + np.cross(u, t)


def contact_dists(blob, st):
    """dist of every contact of a state, float64"""
    bi, bf = blob.view(np.int32), blob.view(np.float32).astype(np.float64)
    L = int(bi[B.H_NLINK])
    lf = lambda f, l: bf[B.HDR_WORDS + f * B.MAXL + l]   # noqa: E731
    out = []
    for l in range(L):
        for ci in range(int(bi[B.HDR_WORDS + B.F_NCON * B.MAXL + l])):
            base = B.F_CON0 + ci * B.CON_STRIDE
            s = np.array([lf(base + a, l) for a in range(3)])
            c = st[l, 0:3].astype(np.float64) + _rot(s, st[l, 3:7].astype(np.float64))
            out.append(c[2] - lf(base + 3, l))
    return np.array(out)


def build(env, family, n, seed=0):
    """the launches of one family on one env ([] where the model has nothing the family exercises)"""
    sys, links = env.sys, env._links
    rng = np.random.default_rng(seed)
    acts = lambda k: actions(env.action_size, n, seed * 100 + k)   # noqa: E731
    q0, qd0 = _base(env, rng)
    out = []
    if family == "F1":
        out.append(_init(env, q0, qd0))
        qd1 = np.where(rng.random(qd0.size) < 0.5, -2.0, 2.0)
        out.append(_init(env, q0, qd1))
    elif family == "F2":
        st = _init(env, q0, qd0).astype(np.float64)
        par = env.blob.view(np.int32)[B.HDR_WORDS + B.F_PARENT * B.MAXL:][:len(links)]
        for l in range(len(links)):
            if par[l] < 0:
                continue
            d = rng.normal(size=3)
            st[l, 0:3] += d / np.linalg.norm(d) * rng.uniform(1e-3, 1e-2)
            a = rng.normal(size=3)
            a /= np.linalg.norm(a)
            qr = np.concatenate([[np.cos(0.025)], a * np.sin(0.025)])
            qn = _qmul(qr, st[l, 3:7])
            st[l, 3:7] = qn / np.linalg.norm(qn)
        if (par >= 0).any():
            out.append(st.astype(np.float32))
    elif family == "F3":
        lim = [(qi, d) for (_, _, qi, d) in _hinges(sys, links) if np.all(np.abs(sys.dof_limit[d]) < 1e3) and sys.dof_limit[d, 1] > sys.dof_limit[d, 0]]
        if lim:
            for side, sgn in ((0, -1), (0, 1), (1, -1), (1, 1)):
                q = q0.copy()
                for qi, d in lim:
                    q[qi] = sys.ref(d) + sys.dof_limit[d, side] + sgn * 1e-2
                out.append(_init(env, q, qd0))
    elif family == "F4":
        mids = [(qi, d) for (l, k, qi, d) in _hinges(sys, links) if k == 1 and sys.link_types[l] in "23"]
        if mids:
            for th in (0.0, 1e-4, np.pi / 2 - 0.05, -(np.pi / 2 - 0.05)):
                q = q0.copy()
                for qi, d in mids:
                    q[qi] = sys.ref(d) + th
                out.append(_init(env, q, qd0))
    elif family == "F5":
        if sys.contacts:
            st0 = _init(env, q0, np.zeros_like(qd0))
            vels = [(0, 0, 0), (1e-3, 0, 0), (2.0, 0.5, 0), (0.1, 0, -0.5), (0.1, 0, 0.5)]
            for d in (-1e-2, -1e-4, 1e-4):
                st = st0.astype(np.float64)
                st[:, 2] -= contact_dists(env.blob, st0).min() - d
                for vel in vels:
                    s = st.copy()
                    s[:, 7:10] = 0.0
                    s[:, 10:13] = vel
                    out.append(s.astype(np.float32))
    elif family == "F6":
        sl = [(l, k, int(sys.link_q_start[l]) + k, int(sys.link_dof_start[l]) + k) for l in links if sys.link_types[l] != "f"
              for k in range(int(sys.link_types[l])) if sys.dof_is_slide[int(sys.link_dof_start[l]) + k]]
        if sl:
            for where in ("inside", "at", "beyond"):
                q = q0.copy()
                qd = qd0.copy()
                for (_, _, qi, d) in sl:
                    lo, hi = sys.dof_limit[d]
                    if np.isfinite(hi) and abs(hi) < 1e3:
                        x = {"inside": 0.5 * hi, "at": hi, "beyond": hi + 0.05}[where]
                    else:
                        x = {"inside": 0.0, "at": 0.3, "beyond": -0.3}[where]
                    q[qi] = sys.ref(d) + x
                    qd[d] = 1.0
                st = _init(env, q, qd)
                out.append(st)
                across = st.astype(np.float64)
                for (l, _, _, d) in sl:
                    ax = np.abs(sys.dof_axis[d])
                    perp = np.eye(3)[int(np.argmin(ax + np.array([0, 0, 0.5])))]   # a world axis off the rail (z last: gravity)
                    across[links.index(l), 10:13] += 0.3 * perp
                out.append(across.astype(np.float32))
    elif family == "F7":
        st = _init(env, q0, qd0).astype(np.float64)
        st[:, 0:3] += np.array([100.0, -50.0, 0.0])
        out.append(st.astype(np.float32))
    else:
        raise ValueError(family)
    return [(s, acts(i)) for i, s in enumerate(out)]
