"""Input families that put the operand of one exact square root or division of the positional substep into one magnitude band
below 2^-101, shared by tests/test_tiny_operands_cpu.py and tests/test_tiny_operands_gpu.py.

The fp32 spec's MBD_SQRT / MBD_RCP / MBD_DIV are correctly rounded on the device for tiny operands only through their exact
pre-scaling (include/mbd_fp32.h); the float64 families of tests/xpbd_families.py never send an operand there.  Tiny position
differences need positions near the world origin and a step that is exact in fp32 around them, so these families run on a
model of their own (MODEL_XML): a free ball on the floor, with its contact at its centre, and 10 arms above it in the humanoid's
tree (11 links, so every rollout kernel runs it, the packed one included), no gravity, and zero actions.  All rotations are the identity, so every rotate and quaternion product of the step is exact, and the
velocities, anchors and depths below are the only small quantities.

  travel     the ball in the floor 2^-10 deep, moving sideways by c per substep: the static-friction tangent sqrt(dx^2 + dy^2)
             and the division of that travel (dlt = -ct / (w_t + eps))
  velocity   the same with c chosen so that the tangential velocity after the position solve, |v_t|^2, lands in the band
  anchor     the first arm's joint anchor c off the ball's (links near the origin): `normalize` of the anchor error
  depth      the ball exactly on the floor, dist = 0 (dl = -dist / (w + eps)).  Its nonzero bands are out of reach: dist is the
             difference of two float32 near the ball's radius, so it is 0 or at least 2^-27 in magnitude.
  gimbal     the first arm's joint exactly at gimbal lock (r00 = r01 = 0: the `cth` square root of 0).  Its nonzero bands are
             not tested: near-unit float32 quaternions whose device r00 is 0 and r01^2 is just below 2^-101 exist, but they
             are not constructed here.
Bands: exactly 0, subnormal, [2^-126, 2^-113) and [2^-113, 2^-101), of the operand the site takes the square root of or
divides (the squared norm for a square root, the dividend for the depth).
"""
from __future__ import annotations

import os

import numpy as np

BANDS = {"zero": (0.0, 0.0), "subnormal": (2.0 ** -149, 2.0 ** -126), "low": (2.0 ** -126, 2.0 ** -113),
         "high": (2.0 ** -113, 2.0 ** -101)}
# a square root's operand is a sum of two squares of components c: c^2 well inside each band
SQUARE_C = {"zero": 0.0, "subnormal": 2.0 ** -69, "low": 2.0 ** -60, "high": 2.0 ** -54}
# a dividend in the middle of each band (log scale)
LINEAR = {"zero": 0.0, "subnormal": 1.5 * 2.0 ** -138, "low": 1.5 * 2.0 ** -120, "high": 1.5 * 2.0 ** -107}
FAMILIES = ("travel", "velocity", "anchor", "depth", "gimbal")
# family -> (diagnostic of tests/xpbd_ref.positional_step, its bands)
SITE = {"travel": ("travel2", tuple(BANDS)), "velocity": ("velocity2", tuple(BANDS)), "anchor": ("anchor2", tuple(BANDS)),
        "depth": ("dist", ("zero",)), "gimbal": ("cth2 (acceleration)", ("zero",))}

# the humanoid's tree (11 links, 7 parents, the root free): what every rollout kernel, the packed one included, can run
PARENT = (-1, 0, 1, 2, 3, 2, 5, 0, 7, 0, 9)
NDOF = (0, 2, 2, 1, 1, 1, 1, 2, 1, 2, 1)
ARM = 0.5
_HEAD = """<mujoco model="tiny_operands">
  <compiler angle="degree" inertiafromgeom="true"/>
  <option timestep="0.004" gravity="0 0 0"/>
  <custom>
    <numeric data="0" name="spring_mass_scale"/>
    <numeric data="1" name="spring_inertia_scale"/>
  </custom>
  <default>
    <joint armature="0" damping="0.5" limited="true"/>
    <geom conaffinity="0" contype="0" density="1000"/>
    <motor ctrllimited="true" ctrlrange="-1 1"/>
  </default>
  <worldbody>
    <geom conaffinity="1" contype="0" name="floor" pos="0 0 0" size="40 40 1" type="plane"/>
"""


def _model_xml():
    """a free ball with its contact at its centre, and 10 arms in the humanoid's tree, each a sphere ARM above its parent with
    hinges about x (and y): every joint frame is the identity"""
    def body(l, ind):
        pad = "  " * ind
        if l == 0:
            out = [f'{pad}<body name="l0" pos="0 0 0.125">', f'{pad}  <joint name="root" type="free" limited="false" damping="0"/>',
                   f'{pad}  <geom name="g0" type="sphere" size="0.125" contype="1" friction="1 0.1 0.1"/>']
        else:
            out = [f'{pad}<body name="l{l}" pos="0 0 {ARM}">']
            for k, ax in list(zip(range(NDOF[l]), ("1 0 0", "0 1 0"))):
                out.append(f'{pad}  <joint name="j{l}_{k}" axis="{ax}" range="-{30 + 90 * k} {30 + 90 * k}"/>')
            out.append(f'{pad}  <geom name="g{l}" type="sphere" size="0.0625"/>')
        for c in range(len(PARENT)):
            if PARENT[c] == l:
                out += body(c, ind + 1)
        return out + [f"{pad}</body>"]
    motors = [f'    <motor gear="10" joint="j{l}_{k}"/>' for l in range(1, len(PARENT)) for k in range(NDOF[l])]
    return _HEAD + "\n".join(body(0, 2)) + "\n  </worldbody>\n  <actuator>\n" + "\n".join(motors) + "\n  </actuator>\n</mujoco>\n"


MODEL_XML = _model_xml()
DT = 0.004
RADIUS = 0.125


def make_env(tmpdir):
    import mbd_b200
    p = os.path.join(str(tmpdir), "tiny_operands.xml")
    with open(p, "w") as f:
        f.write(MODEL_XML)
    return mbd_b200.envs.GenericPositionalEnv(p, n_frames=1)


def _subtree_parents(l):
    out, grew = {l}, True
    while grew:
        grew = False
        for c in range(len(PARENT)):
            if PARENT[c] in out and c not in out:
                out.add(c)
                grew = True
    return out


def state(z=RADIUS + 0.25, v=(0.0, 0.0), anchor=0.0, arm_q=(1.0, 0.0, 0.0, 0.0)):
    """[11, 13] float32: the ball at (0, 0, z) moving sideways at v, every arm ARM above its parent and moving with it; link 1
    and its subtree offset by (anchor, anchor, 0), link 1 turned by arm_q"""
    L = len(PARENT)
    st = np.zeros((L, 13), np.float32)
    st[:, 3] = 1.0
    for l in range(L):
        st[l, 2] = np.float32(z) if l == 0 else st[PARENT[l], 2] + np.float32(ARM)
        assert st[l, 2] - (np.float32(ARM) if l else 0) == (st[PARENT[l], 2] if l else np.float32(z))   # exact anchors in z
    for l in _subtree_parents(1):
        st[l, 0:2] = anchor
    st[1, 3:7] = arm_q
    st[:, 10] = v[0]
    st[:, 11] = v[1]
    return st


def in_band(x, band):
    lo, hi = BANDS[band]
    x = np.abs(np.asarray(x, np.float64))
    return (x == 0) if band == "zero" else (x >= lo) & (x < hi)


def _velocity_for(band, env):
    """the sideways speed of the ball whose tangential velocity after the position solve has its square in the band"""
    from tests import xpbd_ref as X
    if band == "zero":
        return 0.0
    lo, hi = BANDS[band]
    target = np.sqrt(lo * hi)
    c = np.sqrt(target / 2.0)
    for _ in range(4):   # the velocity stage sees a fixed fraction of the travel: two corrections land it in the band
        st = state(z=RADIUS - 2.0 ** -10, v=(c / DT, c / DT))
        got = X.positional_step(env.blob, st[None], np.zeros((1, env.action_size), np.float32))["diag"]["velocity2"][0, 0, 0]
        c *= np.sqrt(target / got)
    return c / DT


def build(env, family, band, n):
    """[(state [11, 13], actions [n, nu])] of one family in one band: zero actions (a motor would turn the ball through the arm's
    reaction and end the exactness the families rely on)"""
    u = np.zeros((n, env.action_size), np.float32)
    if family == "travel":
        c = SQUARE_C[band]
        st = state(z=RADIUS - 2.0 ** -10, v=(c / DT, c / DT))
    elif family == "velocity":
        s = _velocity_for(band, env)
        st = state(z=RADIUS - 2.0 ** -10, v=(s, s))
    elif family == "anchor":
        st = state(anchor=SQUARE_C[band])
    elif family == "depth":
        st = state(z=RADIUS)
    elif family == "gimbal":
        st = state(arm_q=(0.5, 0.5, 0.5, 0.5))
    else:
        raise ValueError(family)
    return [(st, u)]



# ---- the RL acting step: obs - mean in each band --------------------------------------------------------------------------------
def _tiny(rng, band, shape):
    if band == "zero":
        return np.zeros(shape, np.float32)
    if band == "subnormal":
        v = rng.integers(1, 1 << 23, shape).astype(np.uint32).view(np.float32)
    else:
        lo, hi = np.log2(BANDS[band][0]), np.log2(BANDS[band][1])
        v = np.exp2(rng.uniform(lo + 1, hi - 1, shape)).astype(np.float32)
    return (v * rng.choice(np.float32([-1.0, 1.0]), shape)).astype(np.float32)


def act_cases(kind, B, seed=0):
    """[(band, (O, nu, policy, mean, std, obs, key))] for k_ppo_act / k_sac_act: the mild family of tests/rl_families.py with
    every observation's difference from its mean in the band; the even columns have mean 0 (in the subnormal band, subnormal
    observations), the odd ones a mean in the band too"""
    from tests import rl_families as RF
    out = []
    for k, band in enumerate(BANDS):
        O, nu, pol, mean, std, obs, key = RF._case(kind, 17, 6, B, seed + k, "mild")
        rng = np.random.default_rng(seed + 100 + k)
        mean = _tiny(rng, band, (O,))
        mean[::2] = 0.0
        obs = (mean + _tiny(rng, band, (B, O))).astype(np.float32)
        assert in_band(obs.astype(np.float64) - mean.astype(np.float64), band).all()
        out.append((band, (O, nu, pol, mean, std, obs, key)))
    return out
