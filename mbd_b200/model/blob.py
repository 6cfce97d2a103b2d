"""Packs a compiled `System` into the flat 4-byte-word model blob of include/mbd_model.h.

All derived constants (anchor lever arms relative to the COM, composed parent-side joint
frames, exp() damping factors) are computed here in float64 and rounded once to float32,
so the CUDA kernel and the CPU oracle start from bit-identical constants.
"""
from __future__ import annotations

import numpy as np

from . import mjcf
from .mjcf import System

# ---- mirror of include/mbd_model.h (checked against the C side in tests/test_abi.py) ----
MAGIC = 0x4D424431
MAXL, MAXCHILD, MAXDOF, MAXCON, MAXTRACK = 16, 4, 3, 6, 8
DOF_STRIDE, CON_STRIDE = 8, 5
H_MAGIC, H_NLINK, H_NU, H_NFRAMES, H_REWARD, H_NTRACK, H_TRACK0 = 0, 1, 2, 3, 4, 5, 6
H_DT = H_TRACK0 + MAXTRACK
(H_INV_DT, H_GX, H_GY, H_GZ, H_VEL_DAMP, H_ANG_DAMP, H_SCALE_POS, H_SCALE_ANG, H_COLLIDE_SCALE,
 H_ELASTICITY, H_HALF_DT, H_TWO_INV_DT, H_RW0) = range(H_DT + 1, H_DT + 14)
HDR_WORDS = 64
F_PARENT, F_NDOF, F_CHILD0 = 0, 1, 2
F_MASS = F_CHILD0 + MAXCHILD
F_INV_MASS, F_PINV_MASS, F_PINV_INERTIA, F_COM = F_MASS + 1, F_MASS + 2, F_MASS + 3, F_MASS + 4
F_RC = F_COM + 3
F_JQ = F_RC + 3
F_RP = F_JQ + 4
F_PQ = F_RP + 3
F_PARITY = F_PQ + 4
F_ANG_DAMP = F_PARITY + 1
F_SLIDE = F_ANG_DAMP + 1
F_DOF0 = F_SLIDE + 1
F_NCON = F_DOF0 + MAXDOF * DOF_STRIDE
F_CON0 = F_NCON + 1
NFIELDS = F_CON0 + MAXCON * CON_STRIDE
D_STIFF, D_DAMP, D_LO, D_HI, D_ACT, D_GEAR, D_CLO, D_CHI = range(8)
BLOB_WORDS = HDR_WORDS + NFIELDS * MAXL
STATE_STRIDE = 13

REWARD_HUMANOIDRUN, REWARD_HUMANOIDTRACK, REWARD_HOPPER, REWARD_HUMANOIDSTANDUP, REWARD_ANT, REWARD_CARTPOLE = 0, 1, 2, 3, 4, 5

_BIG = 3.0e38  # stands in for +-inf limits (keeps the arithmetic NaN-free)


def pack(sys: System, n_frames: int, reward: int, links=None, track_links=(), reward_params=(0, 0, 0, 0)) -> np.ndarray:
    """Returns the uint32 blob.  `links` optionally restricts the simulated links (humanoidtrack
    drops the 5 cosmetic, dynamically decoupled *_ref bodies, SURVEY App. B)."""
    if sys.custom["spring_inertia_scale"] != 1.0:
        raise NotImplementedError("only spring_inertia_scale == 1 (identity rotational inertia) is supported")
    # Brax positional: mass = link.inertia.mass ** (1 - spring_mass_scale)
    mass_exp = 1.0 - float(sys.custom["spring_mass_scale"])
    if links is None:
        links = list(range(sys.num_links()))
    L = len(links)
    if L > MAXL:
        raise NotImplementedError(f"{L} links > {MAXL}")
    remap = {old: new for new, old in enumerate(links)}
    f = np.zeros(BLOB_WORDS, dtype=np.float32)
    u = f.view(np.uint32)
    i32 = f.view(np.int32)

    def lf(field, l):
        return HDR_WORDS + field * MAXL + l

    u[H_MAGIC] = MAGIC
    i32[H_NLINK], i32[H_NU], i32[H_NFRAMES], i32[H_REWARD] = L, sys.act_size(), n_frames, reward
    i32[H_NTRACK] = len(track_links)
    for k in range(MAXTRACK):
        i32[H_TRACK0 + k] = remap[track_links[k]] if k < len(track_links) else -1
    dt = float(sys.dt)
    f[H_DT], f[H_INV_DT] = dt, 1.0 / dt
    f[H_GX:H_GZ + 1] = sys.gravity
    f[H_VEL_DAMP] = np.exp(sys.custom["vel_damping"] * dt)
    f[H_ANG_DAMP] = np.exp(sys.custom["ang_damping"] * dt)
    f[H_SCALE_POS], f[H_SCALE_ANG] = sys.custom["joint_scale_pos"], sys.custom["joint_scale_ang"]
    f[H_COLLIDE_SCALE], f[H_ELASTICITY] = sys.custom["collide_scale"], sys.custom["elasticity"]
    f[H_HALF_DT], f[H_TWO_INV_DT] = 0.5 * dt, 2.0 / dt
    f[H_RW0:H_RW0 + 4] = reward_params

    # unused lanes: parent -1, ndof -1 marks "no link"
    for l in range(MAXL):
        i32[lf(F_PARENT, l)] = -1
        i32[lf(F_NDOF, l)] = -1
        for c in range(MAXCHILD):
            i32[lf(F_CHILD0 + c, l)] = -1
        f[lf(F_JQ, l)] = 1.0
        f[lf(F_PQ, l)] = 1.0
        f[lf(F_PARITY, l)] = 1.0
        f[lf(F_MASS, l)] = 1.0
        f[lf(F_INV_MASS, l)] = 1.0

    act_of_dof = {int(q): a for a, q in enumerate(sys.act_qd_id)}
    for old in links:
        sl = sys.dof_is_slide[sys.dof_link == old]
        if np.any(sl):
            # slide dofs: planar roots (hopper / walker2d / halfcheetah) and the cartpole cart — always on a link whose
            # parent is the world, and always BEFORE the hinges of the same link (the slide axes then live in the fixed
            # parent-side joint frame); that is the only arrangement the step implements
            if sys.link_parents[old] >= 0:
                raise NotImplementedError("slide joints are only supported on links whose parent is the world")
            if np.any(np.diff(sl.astype(int)) > 0):
                raise NotImplementedError("slide joints must precede the hinge joints of their link")
    for new, old in enumerate(links):
        par_old = sys.link_parents[old]
        if par_old >= 0 and par_old not in remap:
            raise ValueError("link subset must be closed under parents")
        par = remap[par_old] if par_old >= 0 else -1
        typ = sys.link_types[old]
        ndof = 0 if typ == "f" else int(typ)
        i32[lf(F_PARENT, new)] = par
        i32[lf(F_NDOF, new)] = ndof
        kids = [remap[c] for c in links if sys.link_parents[c] == old]
        if len(kids) > MAXCHILD:
            raise NotImplementedError("too many children")
        for c, k in enumerate(sorted(kids)):
            i32[lf(F_CHILD0 + c, new)] = k
        m = float(sys.mass[old]) ** mass_exp
        f[lf(F_MASS, new)], f[lf(F_INV_MASS, new)] = m, 1.0 / m
        f[lf(F_PINV_MASS, new)] = 1.0 / (float(sys.mass[par_old]) ** mass_exp) if par_old >= 0 else 0.0
        f[lf(F_PINV_INERTIA, new)] = 1.0 if par_old >= 0 else 0.0
        com = sys.com[old]
        for a in range(3):
            f[lf(F_COM + a, new)] = com[a]
        f[lf(F_ANG_DAMP, new)] = sys.custom["constraint_ang_damping"]
        f[lf(F_PARITY, new)] = sys.joint_parity[old]
        if ndof > 0:
            d0_ = int(sys.link_dof_start[old])
            i32[lf(F_SLIDE, new)] = sum(1 << k for k in range(ndof) if sys.dof_is_slide[d0_ + k])
            rc = sys.joint_pos[old] - com
            jq = sys.joint_rot[old]
            # parent side: link.transform.do(link.joint), lever arm from the parent's COM
            anchor_p = sys.link_pos[old] + mjcf.rotate(sys.joint_pos[old], sys.link_rot[old])
            pcom = sys.com[par_old] if par_old >= 0 else np.zeros(3)
            rp = anchor_p - pcom
            pq = mjcf.quat_mul(sys.link_rot[old], jq)
            pq = pq / np.linalg.norm(pq)
            for a in range(3):
                f[lf(F_RC + a, new)] = rc[a]
                f[lf(F_RP + a, new)] = rp[a]
            for a in range(4):
                f[lf(F_JQ + a, new)] = jq[a]
                f[lf(F_PQ + a, new)] = pq[a]
            d0 = int(sys.link_dof_start[old])
            for k in range(MAXDOF):
                base = F_DOF0 + k * DOF_STRIDE
                if k < ndof:
                    d = d0 + k
                    f[lf(base + D_STIFF, new)] = sys.dof_stiffness[d]
                    f[lf(base + D_DAMP, new)] = sys.dof_damping[d]
                    f[lf(base + D_LO, new)] = max(sys.dof_limit[d, 0], -_BIG)
                    f[lf(base + D_HI, new)] = min(sys.dof_limit[d, 1], _BIG)
                    a_id = act_of_dof.get(d, -1)
                    i32[lf(base + D_ACT, new)] = a_id
                    if a_id >= 0:
                        if sys.act_bias_q[a_id] != 0 or sys.act_bias_qd[a_id] != 0 or sys.act_gain[a_id] != 1:
                            raise NotImplementedError("only motor actuators (gain 1, no bias)")
                        f[lf(base + D_GEAR, new)] = sys.act_gear[a_id]
                        f[lf(base + D_CLO, new)] = max(sys.act_ctrl_range[a_id, 0], -_BIG)
                        f[lf(base + D_CHI, new)] = min(sys.act_ctrl_range[a_id, 1], _BIG)
                else:
                    # non-existent dof: constrained to angle 0, no actuator, no spring
                    i32[lf(base + D_ACT, new)] = -1
        cons = [c for c in sys.contacts if c["link"] == old]
        if len(cons) > MAXCON:
            raise NotImplementedError("too many contacts on one link")
        i32[lf(F_NCON, new)] = len(cons)
        for ci, c in enumerate(cons):
            if np.abs(c["plane_pos"]).max() != 0 or not np.allclose(c["plane_normal"], [0, 0, 1]):
                raise NotImplementedError("only the z=0 ground plane is supported")
            base = F_CON0 + ci * CON_STRIDE
            s = c["pos"] - com
            for a in range(3):
                f[lf(base + a, new)] = s[a]
            f[lf(base + 3, new)] = c["radius"]
            f[lf(base + 4, new)] = c["friction"]
    return u.copy()
