"""The vector env without a GPU: the ABI's refusals, the float64 kinematics header (include/mbd_kin64.h) built for the host against
the host env's kinematics, and the restatement of the episode wrapper / auto-reset rules.

Kinematics bound, per element: |dev - host| <= 1 float32 ulp of the host value, or <= 1e-12.  Both sides evaluate the same float64
expressions in the same order and round once to float32; only the last float64 bits of libm / BLAS may differ."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from mbd_b200 import _lib
from mbd_b200.envs import get_env
from mbd_b200.envs import vec as vec_mod
from mbd_b200.model import kinematics
from oracle import oracle as orc
from tests.vecenv_ref import wrapper_step

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
XPBD_ENVS = ["humanoidrun", "humanoidstandup", "humanoidtrack", "hopper", "walker2d", "cartpole", "ant", "halfcheetah"]
_f32p, _f64p = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double)


# ---- ABI ---------------------------------------------------------------------------------------------------------------------------
def _plan(**kw):
    P = _lib.VecPlan()
    P.kind, P.B, P.obs_layout, P.done_rule, P.episode_length, P.nq, P.nqd, P.nu = _lib.VEC_PUSHT, 4, _lib.VEC_OBS["state"], 2, 0, 16, 0, 2
    P.params_dev = P.reset_dev = 0x1000
    for name in ("state", "next_state", "first_state", "actions", "obs", "first_obs", "reward", "done", "truncation", "steps"):
        setattr(P, name + "_dev", 0x1000)
    for k, v in kw.items():
        setattr(P, k, v)
    return P


REJECT = [
    (dict(B=0), "B must be"), (dict(B=_lib.VEC_MAX_B + 1), "B must be"), (dict(kind=7), "unknown env kind"),
    (dict(steps_dev=None), "a buffer is missing"), (dict(first_obs_dev=None), "a buffer is missing"), (dict(reset_dev=None), "a buffer is missing"),
    (dict(model=0x2000), "takes no model"), (dict(params_dev=None), "needs its parameter table"),
    (dict(kind=_lib.VEC_XPBD, params_dev=None, obs_layout=0, nq=7, nqd=6), "needs a model"),
    (dict(kind=_lib.VEC_XPBD, model=0x2000, kin_dev=0x3000, obs_layout=0, nq=7, nqd=6), "takes no car2d"),
    (dict(obs_layout=0), "unknown obs layout"), (dict(obs_layout=9), "unknown obs layout"),
    (dict(kind=_lib.VEC_XPBD, params_dev=None, model=0x2000, kin_dev=0x3000, obs_layout=4, nq=7, nqd=6), "unknown obs layout"),
    (dict(nq=3), "nq / nqd"), (dict(done_rule=5), "unknown done rule"), (dict(episode_length=-1), "episode_length < 0"),
    (dict(kind=_lib.VEC_XPBD, params_dev=None, model=0x2000, kin_dev=0x3000, obs_layout=0, nq=28, nqd=27, done_rule=1, episode_length=5),
     "time-counter done"),
]


@pytest.mark.parametrize("fields,msg", REJECT, ids=[m + "-" + ",".join(f) for f, m in REJECT])
@pytest.mark.parametrize("entry", ["mbd_vec_step", "mbd_vec_set_state", "mbd_vec_reset", "mbd_vec_world_poses"])
def test_plan_rejected_before_cuda(fields, msg, entry):
    L = _lib.lib()
    P = _plan(**fields)
    if entry == "mbd_vec_reset":
        rc = L.mbd_vec_reset(ctypes.byref(P), ctypes.c_void_p(0x4000), None)
    elif entry == "mbd_vec_world_poses":
        rc = L.mbd_vec_world_poses(ctypes.byref(P), ctypes.c_void_p(0x4000), ctypes.c_void_p(0x4000), None)
    else:
        rc = getattr(L, entry)(ctypes.byref(P), None)
    assert rc == -1
    err = L.mbd_last_error().decode()
    assert err.startswith(entry) and msg in err, err


def test_reset_needs_keys_and_world_poses_need_xpbd():
    L = _lib.lib()
    P = _plan()
    assert L.mbd_vec_reset(ctypes.byref(P), None, None) == -1 and "keys is NULL" in L.mbd_last_error().decode()
    assert L.mbd_vec_world_poses(ctypes.byref(P), ctypes.c_void_p(0x4000), ctypes.c_void_p(0x4000), None) == -1
    assert "xpbd envs only" in L.mbd_last_error().decode()


def test_kinematics_table_size_agrees():
    assert vec_mod.K64_WORDS == _lib.K64_WORDS


# ---- float64 kinematics ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kin(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("kin64") / "libkin64_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "host_kin64", "kin64_harness.cpp"), "-o", so], check=True,
                   env={**os.environ, "CC": "", "CXX": ""})
    return ctypes.CDLL(so)


def _within(dev, host, what):
    """the per-element bound; returns the bit-exact fraction"""
    dev, host = np.asarray(dev, np.float32).ravel(), np.asarray(host, np.float32).ravel()
    err = np.abs(dev.astype(np.float64) - host.astype(np.float64))
    ok = (err <= np.spacing(np.abs(host)).astype(np.float64)) | (err <= 1e-12)
    assert ok.all(), f"{what}: {np.count_nonzero(~ok)} elements beyond 1 ulp, worst {err.max():.3g}"
    return float(np.mean(dev.view(np.uint32) == host.view(np.uint32)))


def _configs(env, n, seed):
    sys = env.sys
    rng = np.random.default_rng(seed)
    q = (sys.init_q + rng.uniform(-0.6, 0.6, (n, sys.q_size()))).astype(np.float32)
    qd = rng.uniform(-2.0, 2.0, (n, sys.qd_size())).astype(np.float32)
    return q, qd


def _dev_init(kin, T, q, qd, nsim):
    st = np.zeros((q.shape[0], nsim, 13), np.float32)
    q, qd = np.ascontiguousarray(q), np.ascontiguousarray(qd)
    kin.kin64_pipeline_init(T.ctypes.data_as(_f64p), q.shape[0], q.ctypes.data_as(_f32p), qd.ctypes.data_as(_f32p), st.ctypes.data_as(_f32p))
    return st


def _dev_state(kin, T, env, st):
    n = st.shape[0]
    L, nq, nqd = env.sys.num_links(), env.sys.q_size(), env.sys.qd_size()
    q, qd = np.zeros((n, nq), np.float32), np.zeros((n, nqd), np.float32)
    pos, rot = np.zeros((n, L, 3), np.float32), np.zeros((n, L, 4), np.float32)
    st = np.ascontiguousarray(st, np.float32)
    kin.kin64_state(T.ctypes.data_as(_f64p), n, st.ctypes.data_as(_f32p), q.ctypes.data_as(_f32p), qd.ctypes.data_as(_f32p),
                    pos.ctypes.data_as(_f32p), rot.ctypes.data_as(_f32p))
    return q, qd, pos, rot


@pytest.mark.parametrize("env_name", XPBD_ENVS)
def test_kin64_pipeline_init_and_inverse_match_host(kin, env_name, capsys):
    env = get_env(env_name)
    T = vec_mod.pack_kin64(env)
    q, qd = _configs(env, 24, seed=5)
    st = _dev_init(kin, T, q, qd, len(env._links))
    host_st = np.stack([kinematics.pipeline_init(env.sys, q[i], qd[i], links=env._links) for i in range(len(q))])
    fr = {"pipeline_init": _within(st, host_st, "pipeline_init")}
    # the states of a short oracle rollout from the init pose, plus the random configurations above
    raw0 = kinematics.pipeline_init(env.sys, env.sys.init_q, np.zeros(env.sys.qd_size()), links=env._links)
    Y0s = np.clip(np.random.default_rng(2).normal(size=(6, 4, env.action_size)), -1, 1).astype(np.float32)
    fin = np.stack([orc.xpbd_rollout(env.blob, raw0, Y0s[:, :h], want_final=True)["final"] for h in range(1, 5)]).reshape(-1, *raw0.shape)
    states = np.concatenate([host_st, fin])
    dq, dqd, dpos, drot = _dev_state(kin, T, env, states)
    hs = [env._make_pipeline_state(s) for s in states]
    fr["q"] = _within(dq, np.stack([h.q for h in hs]), "q")
    fr["qd"] = _within(dqd, np.stack([h.qd for h in hs]), "qd")
    fr["x.pos"] = _within(dpos, np.stack([h.x.pos for h in hs]), "x.pos")
    assert np.array_equal(drot, np.stack([h.x.rot for h in hs]))
    with capsys.disabled():
        print(f"\n  {env_name}: bit-exact fraction " + ", ".join(f"{k} {v:.4f}" for k, v in fr.items()))


# ---- episode wrapper / auto-reset restatement ---------------------------------------------------------------------------------------
def test_wrapper_rules_on_scripted_done_patterns():
    ep = 3
    done, steps = np.zeros(3, np.float32), np.zeros(3, np.float32)
    # env 0 never ends by itself, env 1 ends at its 2nd step, env 2 ends at every step
    env_done_seq = [[0, 0, 1], [0, 1, 1], [0, 0, 1], [0, 0, 1], [0, 0, 1]]
    got = []
    for ed in env_done_seq:
        done, trunc, steps, reset = wrapper_step(done, steps, np.float32(ed), ep)
        got.append((done.tolist(), trunc.tolist(), steps.tolist(), reset.tolist()))
    assert got[0] == ([0, 0, 1], [0, 0, 0], [1, 1, 1], [False, False, True])
    assert got[1] == ([0, 1, 1], [0, 0, 0], [2, 2, 1], [False, True, True])
    assert got[2] == ([1, 0, 1], [1, 0, 0], [3, 1, 1], [True, False, True])    # env 0 truncated at the episode length
    assert got[3] == ([0, 0, 1], [0, 0, 0], [1, 2, 1], [False, False, True])
    assert got[4] == ([0, 1, 1], [0, 1, 0], [2, 3, 1], [False, True, True])     # env 1: length reached, not done by itself
    # no wrapper: done is the env's, steps count, nothing resets
    d, t, s, r = wrapper_step(np.float32([1, 0]), np.float32([4, 4]), np.float32([1, 0]), 0)
    assert d.tolist() == [1, 0] and t.tolist() == [0, 0] and s.tolist() == [5, 5] and not r.any()
