"""VecEnv — a batch of environments of one kind, each with its own state, reset and stepped together on the device.

The device counterpart of `jax.vmap(env.reset)(keys)` / `jax.vmap(env.step)(states, actions)` and of Brax's
`AutoResetWrapper(EpisodeWrapper(env, episode_length, action_repeat=1))`, the interface RL training stands on.  A step is two
launches (mbd_vec_step, include/mbd_b200.h): the env's rollout kernel with H = 1 from every env's own state, then one thread per env
that computes the observation (float64 kinematics, include/mbd_kin64.h), done, the episode counters and the auto-reset.  Every
buffer is owned here and fixed, so a step can be captured in a CUDA graph:

    venv = VecEnv(get_env("hopper"), num_envs=4096)
    st = venv.reset(prng.split(prng.PRNGKey(0), 4096))
    st = venv.step(actions)                      # float32 cuda [B, Nu]
    st.obs, st.reward, st.done, st.truncation, st.steps, st.raw

Each env class is the specification: reset / step / obs / done reproduce the host `env.reset` / `env.step` of one state (raw state
and reward bit for bit, observations within one float32 ulp), see DESIGN.md §5e.

The xpbd envs can step every env with its own friction and actuator strength (DESIGN.md §5k):

    venv.set_model_factors(friction=f, gear=g)  # scalars or [B] arrays; env b is scaled_env(env, f[b], g[b])

or draw new factors at every episode of every env, inside the step (domain randomisation, DESIGN.md §5n):

    venv.set_domain_randomization((0.5, 1.5), (0.7, 1.3), keys)   # episode e of env b: dr_factors(keys[b], e, ...)
"""
from __future__ import annotations

import copy
import dataclasses
import os
from typing import Optional

import numpy as np
import torch

from .. import _lib, ops, prng
from ..model import blob as blob_mod
from .ant import Ant
from .base import PipelineEnv
from .car2d import Car2d
from .cartpole import Cartpole
from .generic import GenericPositionalEnv
from .halfcheetah import HalfCheetah
from .hopper import Hopper
from .humanoidtrack import HumanoidTrack
from .pusht import PushT

# include/mbd_kin64.h
K64_MAXL, K64_MAXQ, K64_SIM, K64_LS, K64_DS = 16, 64, 8, 32, 5
K64_LINK = K64_SIM + K64_MAXL
K64_DOF = K64_LINK + K64_MAXL * K64_LS
K64_INITQ = K64_DOF + K64_MAXQ * K64_DS
K64_WORDS = K64_INITQ + K64_MAXQ
_L = dict(TYPE=0, QS=1, DS=2, PARENT=3, SIMIDX=4, POS=5, ROT=8, JPOS=12, JROT=15, COM=19, PARITY=22, SPOS=23, SROT=26)


def pack_kin64(env: PipelineEnv) -> np.ndarray:
    """the float64 kinematics table of include/mbd_kin64.h for an xpbd env (its model, simulated links and cosmetic init poses)"""
    sys = env.sys
    L, nq, nqd = sys.num_links(), sys.q_size(), sys.qd_size()
    if L > K64_MAXL or nq > K64_MAXQ or nqd > K64_MAXQ:
        raise ValueError(f"model too large for the vector env: {L} links, nq {nq}, nqd {nqd}")
    links = list(env._links)
    T = np.zeros(K64_WORDS, np.float64)
    T[0:5] = L, nq, nqd, len(links), 1.0 if os.environ.get("MBD_FREE_QUAT_NORMALIZE", "1") != "0" else 0.0
    T[K64_SIM:K64_SIM + len(links)] = links
    spos, srot = env._static_x[0].astype(np.float32), env._static_x[1].astype(np.float32)
    for l in range(L):
        o = K64_LINK + l * K64_LS
        T[o + _L["TYPE"]] = -1 if sys.link_types[l] == "f" else int(sys.link_types[l])
        T[o + _L["QS"]], T[o + _L["DS"]], T[o + _L["PARENT"]] = sys.link_q_start[l], sys.link_dof_start[l], sys.link_parents[l]
        T[o + _L["SIMIDX"]] = links.index(l) if l in links else -1
        T[o + _L["POS"]:o + _L["POS"] + 3] = sys.link_pos[l]
        T[o + _L["ROT"]:o + _L["ROT"] + 4] = sys.link_rot[l]
        T[o + _L["JPOS"]:o + _L["JPOS"] + 3] = sys.joint_pos[l]
        T[o + _L["JROT"]:o + _L["JROT"] + 4] = sys.joint_rot[l]
        T[o + _L["COM"]:o + _L["COM"] + 3] = sys.com[l]
        T[o + _L["PARITY"]] = sys.joint_parity[l]
        T[o + _L["SPOS"]:o + _L["SPOS"] + 3] = spos[l]
        T[o + _L["SROT"]:o + _L["SROT"] + 4] = srot[l]
    for d in range(nqd):
        o = K64_DOF + d * K64_DS
        T[o:o + 3] = sys.dof_axis[d]
        T[o + 3] = 1.0 if sys.dof_is_slide[d] else 0.0
        T[o + 4] = sys.ref(d)
    T[K64_INITQ:K64_INITQ + nq] = sys.init_q
    return T


@dataclasses.dataclass
class _Spec:
    kind: int
    obs_layout: int
    done_rule: int
    nq: int
    nqd: int
    nu: int
    state_words: int
    obs_size: int
    reset: np.ndarray          # the MBD_VEC_RT_* table (float32)


def _reset_table(kind: str, nq: int, lo=0.0, hi=0.0, sigma=0.0, q0=None, off=None) -> np.ndarray:
    rt = np.zeros(_lib.VEC_RT_Q + 2 * nq, np.float32)
    rt[0], rt[1], rt[2], rt[3] = _lib.VEC_RESET[kind], np.float32(lo), np.float32(hi), np.float32(sigma)
    if q0 is not None:
        rt[_lib.VEC_RT_Q:_lib.VEC_RT_Q + len(q0)] = q0
    if off is not None:
        rt[4] = 1.0
        rt[_lib.VEC_RT_Q + nq:_lib.VEC_RT_Q + nq + len(off)] = off
    return rt


def env_spec(env) -> _Spec:
    """what the vector env needs to know about a host env: kind, obs layout, done rule, sizes and the reset table.  Each entry
    restates that env class's reset / _get_obs / step (the class is the specification)."""
    if isinstance(env, PushT):
        q0 = np.float32([0.1, -0.15, 0.0, 0.0, 0.0, -0.4, 0.4, np.pi])              # pushT.py:22-38; q[5:] = U * scale + offset
        scale = np.float32([0, 0, 0, 0, 0, 0.2, 0.2, np.pi / 4])
        rt = _reset_table("pusht", 16, q0=q0)
        rt[_lib.VEC_RT_Q + 16:_lib.VEC_RT_Q + 24] = scale
        return _Spec(_lib.VEC_PUSHT, _lib.VEC_OBS["state"], _lib.VEC_DONE_PUSHT, 16, 0, 2, 16, 16, rt)
    if isinstance(env, Car2d):
        return _Spec(_lib.VEC_CAR2D, _lib.VEC_OBS["state"], _lib.VEC_DONE_ZERO, 3, 0, 2, 3, 3, _reset_table("const", 3, q0=env.x0))
    if not isinstance(env, PipelineEnv):
        raise TypeError(f"no vector env for {type(env).__name__}")
    sys = env.sys
    nq, nqd = sys.q_size(), sys.qd_size()
    q0 = sys.init_q.astype(np.float32)
    done = _lib.VEC_DONE_ZERO
    layout = _lib.VEC_OBS["qqd"]
    if isinstance(env, HumanoidTrack):
        rt, done = _reset_table("none", nq, q0=q0), _lib.VEC_DONE_COUNTER
    elif isinstance(env, Hopper):        # hopper.py / walker2d.py
        s = env._reset_noise_scale
        rt, layout = _reset_table("uniform", nq, -s, s, q0=q0), _lib.VEC_OBS["hopper"]
    elif isinstance(env, Ant):           # ant.py / half_cheetah.py [brax-recalled]
        s = env._reset_noise_scale
        rt = _reset_table("normal", nq, -s, s, s, q0=q0)
        layout = _lib.VEC_OBS["skip1" if isinstance(env, HalfCheetah) else "skip2"]
    elif isinstance(env, Cartpole):
        rt = _reset_table("uniform", nq, -0.01, 0.01, q0=q0, off=np.float32([0.0, np.pi] + [0.0] * (nq - 2)))
    elif isinstance(env, GenericPositionalEnv):
        rt = _reset_table("uniform", nq, -env._reset_noise, env._reset_noise, q0=q0)
    else:                                # humanoidrun.py / humanoidstandup.py
        rt = _reset_table("uniform", nq, -0.01, 0.01, q0=q0)
    skip = {_lib.VEC_OBS["skip2"]: 2, _lib.VEC_OBS["skip1"]: 1}.get(layout, 0)
    return _Spec(_lib.VEC_XPBD, layout, done, nq, nqd, sys.act_size(), len(env._links) * 13, nq - skip + nqd, rt)


def factor_column(value, B: int, name: str) -> np.ndarray:
    """a model factor as float32 [B]: a scalar (every env) or a [B] array; ValueError unless every value is finite and >= 0"""
    if isinstance(value, torch.Tensor):
        value = value.detach().cpu().numpy()
    v = np.asarray(value, dtype=np.float64)
    if v.ndim == 0:
        v = np.full(B, v)
    if v.shape != (B,):
        raise ValueError(f"{name} must be a scalar or an array of shape ({B},) (got shape {v.shape})")
    with np.errstate(over="ignore"):
        f = v.astype(np.float32)
    if not (np.isfinite(f).all() and (f >= 0).all()):
        raise ValueError(f"{name} factors must be finite and >= 0 (got {v.tolist()})")
    return f


def dr_range(friction_range, gear_range) -> np.ndarray:
    """mbd_vec_dr.range: float32 [flo, fhi, glo, ghi]; ValueError unless each range is a pair of finite values >= 0 with lo <= hi
    (in float32, as the kernel reads them)"""
    out = []
    for name, r in (("friction_range", friction_range), ("gear_range", gear_range)):
        try:
            v = np.asarray(r, dtype=np.float64)
        except (TypeError, ValueError):
            raise ValueError(f"{name} must be a pair (lo, hi) (got {r!r})") from None
        if v.shape != (2,):
            raise ValueError(f"{name} must be a pair (lo, hi) (got {r!r})")
        with np.errstate(over="ignore"):
            f = v.astype(np.float32)
        if not (np.isfinite(f).all() and (f >= 0).all()):
            raise ValueError(f"{name} must be finite and >= 0 (got {v.tolist()})")
        if f[0] > f[1]:
            raise ValueError(f"{name} needs lo <= hi (got {v.tolist()})")
        out += [f[0], f[1]]
    return np.float32(out)


def dr_factors(key, episode: int, friction_range, gear_range):
    """(f, g): the model factors of episode `episode` of an env with DR key `key` (DESIGN.md §5n), the specification of the vector
    env's draw: kf, kg = split(fold_in(key, episode)); f = uniform(kf, (1,), flo, fhi)[0]; g = uniform(kg, (1,), glo, ghi)[0]"""
    r = dr_range(friction_range, gear_range)
    kf, kg = prng.split(prng.fold_in(key, episode))
    return prng.uniform(kf, (1,), r[0], r[1])[0], prng.uniform(kg, (1,), r[2], r[3])[0]


def scaled_env(env: PipelineEnv, friction: float = 1.0, gear: float = 1.0) -> PipelineEnv:
    """the specification of a vector env stepped with model factors (friction, gear): a host env of the same class whose every
    contact friction is fl(mu * friction) and every actuator gear fl(gear_a * gear), in float32 as the kernel forms them, with its
    device model rebuilt from that `sys`.  Its blob differs from env's in exactly those words."""
    if not isinstance(env, PipelineEnv):
        raise ValueError(f"model factors exist for the xpbd envs only, not {type(env).__name__}")
    fr, gr = factor_column(friction, 1, "friction")[0], factor_column(gear, 1, "gear")[0]
    sys = env.sys
    contacts = [dict(c, friction=float(np.float32(np.float32(c["friction"]) * fr))) for c in sys.contacts]
    act_gear = np.array([float(np.float32(np.float32(g) * gr)) for g in sys.act_gear], dtype=np.float64)
    out = copy.copy(env)
    out.sys = dataclasses.replace(sys, contacts=contacts, act_gear=act_gear)
    out.blob = blob_mod.pack(out.sys, out._n_frames, out.reward_kind, links=out._links, track_links=tuple(out.track_links),
                             **out._pack_kwargs())
    out._models = {}
    return out


@dataclasses.dataclass
class VecState:
    """views on the VecEnv's buffers (overwritten by the next reset / step / set_state)"""
    obs: torch.Tensor          # [B, O]
    reward: torch.Tensor       # [B]
    done: torch.Tensor         # [B] float32
    truncation: torch.Tensor   # [B] float32 (episode wrapper: 1 where the episode ended by its length only)
    steps: torch.Tensor        # [B] float32: env steps since the last reset
    raw: torch.Tensor          # xpbd [B, Lsim, 13]; pushT [B, 16] = q | qd; car2d [B, 3]


class VecEnv:
    def __init__(self, env, num_envs: int, episode_length: Optional[int] = None, device: Optional[torch.device] = None):
        _lib.require_gpu()
        self.env = env
        self.num_envs = B = int(num_envs)
        if not 1 <= B <= _lib.VEC_MAX_B:
            raise ValueError(f"num_envs must be in 1..{_lib.VEC_MAX_B}")
        self.episode_length = 0 if episode_length is None else int(episode_length)
        self.spec = sp = env_spec(env)
        self.device = dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        f32 = dict(device=dev, dtype=torch.float32)
        S, O = sp.state_words, sp.obs_size
        self.state, self.next_state, self.first_state = (torch.zeros((B, S), **f32) for _ in range(3))
        self.actions = torch.zeros((B, sp.nu), **f32)
        self.obs, self.first_obs = torch.zeros((B, O), **f32), torch.zeros((B, O), **f32)
        self.reward, self.done, self.truncation, self.steps = (torch.zeros(B, **f32) for _ in range(4))
        self._reset_tab = torch.as_tensor(sp.reset, device=dev)
        self._model = self._params = self._kin = None
        if sp.kind == _lib.VEC_XPBD:
            with torch.cuda.device(dev):
                self._model = env.device_model(dev)
            self._kin = torch.as_tensor(pack_kin64(env), device=dev)
        else:
            with torch.cuda.device(dev):
                p = env.device_params()
            self._params = p[0] if isinstance(p, tuple) else p
        P = _lib.VecPlan()
        P.kind, P.B, P.obs_layout, P.done_rule, P.episode_length = sp.kind, B, sp.obs_layout, sp.done_rule, self.episode_length
        P.nq, P.nqd, P.nu = sp.nq, sp.nqd, sp.nu
        P.model = self._model._h if self._model is not None else None
        P.params_dev = self._params.data_ptr() if self._params is not None else None
        P.kin_dev = self._kin.data_ptr() if self._kin is not None else None
        P.reset_dev = self._reset_tab.data_ptr()
        for name in ("state", "next_state", "first_state", "actions", "obs", "first_obs", "reward", "done", "truncation", "steps"):
            setattr(P, name + "_dev", getattr(self, name).data_ptr())
        self.plan = P
        self.factors: Optional[torch.Tensor] = None   # [B, 2] friction | gear factors once set_model_factors gave any
        self.dr: Optional[_lib.VecDr] = None            # domain randomisation (set_domain_randomization): the mbd_vec_dr
        self.dr_keys: Optional[torch.Tensor] = None   # [B, 2] DR keys and [B] episode counts it points to
        self.dr_episodes: Optional[torch.Tensor] = None

    def set_model_factors(self, friction=None, gear=None) -> None:
        """step env b with every contact friction scaled by friction[b] and every actuator gear by gear[b] (xpbd envs): env b then
        steps as the nominal VecEnv of scaled_env(env, friction[b], gear[b]), bit for bit.  Each argument is a scalar or a [B]
        array of finite values >= 0; an omitted one is 1.  Both omitted: the nominal model (the kernels of a VecEnv without
        factors).  The [B, 2] table is written in place, so a captured graph keeps reading the current values."""
        if self.spec.kind != _lib.VEC_XPBD:
            raise ValueError("model factors exist for the positional (xpbd) envs only")
        B = self.num_envs
        fr = factor_column(1.0 if friction is None else friction, B, "friction")
        gr = factor_column(1.0 if gear is None else gear, B, "gear")
        self.dr = None   # fixed factors end domain randomisation
        if friction is None and gear is None:
            self.plan.factors_dev = None
            return
        self._factor_table()
        self.factors.copy_(torch.from_numpy(np.stack([fr, gr], axis=1)))

    def set_domain_randomization(self, friction_range, gear_range, keys) -> None:
        """domain randomisation (xpbd envs, DESIGN.md §5n): every episode of env b steps with factors drawn from its DR key keys[b]
        and its episode count, (f, g) = dr_factors(keys[b], e, friction_range, gear_range); env b in episode e steps as the nominal
        VecEnv of scaled_env(env, f, g), bit for bit.  keys: uint32 [B, 2] (numpy or cuda, as in reset).  It takes effect at the next
        reset, which zeroes the episode counts and writes episode 0's factors; each auto-reset draws the next episode's.  `factors`
        holds the current table and `dr_episodes` the counts.  reset / step then launch mbd_vec_reset_dr / mbd_vec_step_dr with
        `dr`; code that launches ops.vec_step itself passes `venv.dr`.  set_model_factors ends it."""
        if self.spec.kind != _lib.VEC_XPBD:
            raise ValueError("domain randomisation exists for the positional (xpbd) envs only")
        r = dr_range(friction_range, gear_range)
        k = self._key_bits(keys).clone()   # owned: a later write to the caller's tensor does not change the draws
        self._factor_table()
        if self.dr_episodes is None:
            self.dr_episodes = torch.zeros(self.num_envs, device=self.device, dtype=torch.int32)
        self.dr_keys = k
        dr = _lib.VecDr()
        dr.keys_dev, dr.episodes_dev = k.data_ptr(), self.dr_episodes.data_ptr()
        dr.range[:] = [float(x) for x in r]
        self.dr = dr

    def _factor_table(self):
        """the [B, 2] factor table (allocated once, 1 everywhere) and the plan's pointer to it"""
        if self.factors is None:
            self.factors = torch.ones((self.num_envs, 2), device=self.device, dtype=torch.float32)
        self.plan.factors_dev = self.factors.data_ptr()

    def _key_bits(self, keys) -> torch.Tensor:
        """uint32 [B, 2] keys (numpy, or a cuda tensor of uint32 / int32 bits) as an int32 device tensor; the shape is checked first"""
        shape = tuple(keys.shape) if isinstance(keys, torch.Tensor) else np.shape(keys)
        if shape != (self.num_envs, 2) or (isinstance(keys, torch.Tensor) and keys.dtype not in (torch.uint32, torch.int32)):
            raise ValueError(f"keys must be uint32 [{self.num_envs}, 2]")
        if isinstance(keys, torch.Tensor):
            return keys.to(self.device).contiguous().view(torch.int32)
        return torch.as_tensor(np.ascontiguousarray(keys, dtype=np.uint32).view(np.int32), device=self.device)

    # ---- the batched env API -------------------------------------------------------------------------------------------------
    def _view(self) -> VecState:
        raw = self.state.view(self.num_envs, -1, 13) if self.spec.kind == _lib.VEC_XPBD else self.state
        return VecState(self.obs, self.reward, self.done, self.truncation, self.steps, raw)

    def reset(self, keys) -> VecState:
        """vmap(env.reset)(keys): keys uint32 [B, 2] (numpy, or a cuda tensor of uint32 / int32 bits)"""
        k = self._key_bits(keys)
        with torch.cuda.device(self.device):
            ops.vec_reset(self.plan, k, self.dr)
        return self._view()

    def step(self, actions: Optional[torch.Tensor] = None) -> VecState:
        """vmap(env.step)(states, actions) (+ the episode wrapper and auto-reset when episode_length is set).  actions float32 cuda
        [B, Nu]; None (or the VecEnv's own `actions` buffer) steps with what the buffer holds — the form a CUDA graph captures."""
        if actions is not None and actions.data_ptr() != self.actions.data_ptr():
            self.actions.copy_(actions)
        with torch.cuda.device(self.device):
            ops.vec_step(self.plan, self.dr)
        return self._view()

    def set_state(self, raw) -> VecState:
        """start every env at the given states ([B, ...] in the layout of PipelineState.raw / pushT's q|qd / car2d's x); they also
        become the states the auto-reset returns to"""
        t = torch.as_tensor(np.asarray(raw, dtype=np.float32)) if not isinstance(raw, torch.Tensor) else raw
        self.state.copy_(t.reshape(self.num_envs, -1))
        with torch.cuda.device(self.device):
            ops.vec_set_state(self.plan)
        return self._view()

    def world_poses(self):
        """x.pos [B, L, 3], x.rot [B, L, 4] of every link (xpbd envs), as PipelineState.x of the host env"""
        if self.spec.kind != _lib.VEC_XPBD:
            raise ValueError("world poses exist for the positional (xpbd) envs only")
        L = self.env.sys.num_links()
        pos = torch.empty((self.num_envs, L, 3), device=self.device)
        rot = torch.empty((self.num_envs, L, 4), device=self.device)
        with torch.cuda.device(self.device):
            ops.vec_world_poses(self.plan, pos, rot)
        return pos, rot

    def pipeline_state(self, b: int):
        """host pipeline state of env b (for the render tools, e.g. io.brax_json)"""
        raw = self.state[b].cpu().numpy()
        if self.spec.kind == _lib.VEC_XPBD:
            return self.env._make_pipeline_state(raw.reshape(-1, 13))
        if self.spec.kind == _lib.VEC_PUSHT:
            return self.env.pipeline_init(raw[:8], raw[8:])
        return raw
