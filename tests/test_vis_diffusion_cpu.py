"""The diffusion-process page (mbd_b200.scripts.vis_diffusion) without a GPU: the document builder against a literal restatement
of the reference's `dumps` (scripts/vis_diffusion.py:27-112) walking `BraxLikeSystem`, on rollouts from `utils.rollout_states`;
the argument handling (car2d refused, a missing mu_0ts.npy, the rollout cache and its hash)."""
import json
import os

import numpy as np
import pytest

from mbd_b200 import utils
from mbd_b200.envs import get_env
from mbd_b200.envs.base import State
from mbd_b200.io import brax_json
from mbd_b200.io.brax_json import GEOM_TYPE_NAMES, BraxLikeSystem, _tolist
from mbd_b200.scripts import vis_diffusion as vd

K, H = 3, 4
plot_interval = 10


def _to_dict(geom):
    """brax.io.json._to_dict on a geom, with this package's number format (`brax_json._tolist`)"""
    return {k: (_tolist(v) if isinstance(v, np.ndarray) else v) for k, v in geom.items()}


def ref_dumps(sys, statess, env_name) -> dict:
    """scripts/vis_diffusion.py:27-112, restated line for line on numpy; `d` starts from the system part of brax_json.to_dict"""
    d = {"link_names": list(sys.link_names), "opt": {"timestep": sys.dt}, "dt": sys.dt}

    link_names = [n or f"link {i}" for i, n in enumerate(sys.link_names)]
    link_names += ["world"]

    link_geoms = {}
    for id_ in range(sys.ngeom):
        link_idx = int(sys.geom_bodyid[id_]) - 1
        rgba = sys.geom_rgba[id_]
        geom = {
            "name": GEOM_TYPE_NAMES[int(sys.geom_type[id_])],
            "link_idx": link_idx,
            "pos": sys.geom_pos[id_],
            "rot": sys.geom_quat[id_],
            "rgba": rgba,
            "size": sys.geom_size[id_],
        }
        link_geoms.setdefault(link_names[link_idx], []).append(_to_dict(geom))

    all_link_geoms = {}
    all_link_names = []
    traj_len = len(statess[0])
    for k in range(traj_len):
        for _, (name, geoms) in enumerate(link_geoms.items()):
            name = f"{name}_{k}" if k > 0 else name
            geoms_new = []
            for geom in geoms:
                geom_new = geom.copy()
                if "world" in name:
                    geom_new["link_idx"] = -1
                elif "goal" in name:
                    geom_new["rgba"] = [0.0, 1.0, 0.0, 1.0]
                elif "_ref" in name:
                    if "torso" in name or "thigh" in name:
                        geom_new["link_idx"] = geom["link_idx"] + k * (len(link_names) - 1)
                        a = k / traj_len * 0.8 + 0.2
                        geom_new["rgba"] = [(1 - a), 1.0, (1 - a), 1.0]
                    else:
                        geom_new["rgba"] = [1.0, 1.0, 1.0, 0.0]
                else:
                    geom_new["link_idx"] = geom["link_idx"] + k * (len(link_names) - 1)
                    a = k / traj_len * 0.8 + 0.2
                    geom_new["rgba"] = [1, (1 - a), (1 - a), 1.0]
                geoms_new.append(geom_new)
            all_link_geoms[name] = geoms_new
            all_link_names.append(name)
    d["geoms"] = all_link_geoms
    d["link_names"] = all_link_names

    if env_name == "pushT":
        statess_new = []
        for states in statess:
            states_new = []
            for i, state in enumerate(states):
                pipeline_state = state
                pipeline_state = pipeline_state.replace(
                    x=pipeline_state.x.replace(pos=pipeline_state.x.pos + np.float32([0.0, 0.0, i * 0.01 / 50]))
                )
                states_new.append(pipeline_state)
            statess_new.append(states_new)
        statess = statess_new
    pos_list, rot_list = [], []
    for states in statess:
        pos_list.append(np.concatenate([s.x.pos for s in states]))
        rot_list.append(np.concatenate([s.x.rot for s in states]))
    for state in statess[-1]:
        pos_list.append(np.concatenate([state.x.pos] * traj_len))
        rot_list.append(np.concatenate([state.x.rot] * traj_len))
    d["states"] = {"x": {"pos": _tolist(np.stack(pos_list)), "rot": _tolist(np.stack(rot_list))}}
    return d


def _host_step(env):
    """a host stand-in for env.step (the real one runs the CUDA kernel): the action nudges the actuated coordinates"""
    rng = np.random.default_rng(3)
    nq = env.sys.q_size()

    def step(state, u):
        q = np.asarray(state.pipeline_state.q, np.float64) + rng.normal(size=nq) * 0.02
        q[-len(u):] += 0.05 * np.asarray(u, np.float64)
        ps = env.pipeline_init(q, np.zeros(env.sys.qd_size()))
        return State(ps, None, 0.0, 0.0)
    return step


def _rollouts(env):
    step = _host_step(env)
    rng = np.random.default_rng(0)
    ps0 = env.pipeline_init(env.sys.init_q, np.zeros(env.sys.qd_size()))
    state = State(ps0, None, 0.0, 0.0)
    us = rng.uniform(-1, 1, size=(K, H, env.action_size)).astype(np.float32)
    statess = [utils.rollout_states(step, state, us[k]) for k in range(K)]
    pos = np.stack([np.stack([np.asarray(ps.x.pos, np.float32) for ps in states]) for states in statess])
    rot = np.stack([np.stack([np.asarray(ps.x.rot, np.float32) for ps in states]) for states in statess])
    return statess, pos, rot


@pytest.mark.parametrize("name", ["hopper", "pushT", "humanoidtrack"])
def test_document_matches_the_reference_dumps(name):
    env = get_env(name)
    statess, pos, rot = _rollouts(env)
    assert pos.shape[:2] == (K, H)
    got = json.loads(json.dumps(brax_json.diffusion_to_dict(env.sys, pos, rot, env.dt, lift=name == "pushT")))
    want = json.loads(json.dumps(ref_dumps(BraxLikeSystem(env.sys, env.dt), statess, name)))
    assert got == want

    # the rules, spelled out
    L = env.sys.num_links()
    names = list(env.sys.link_names)
    assert len(got["states"]["x"]["pos"]) == K + H
    assert np.asarray(got["states"]["x"]["pos"]).shape == (K + H, H * L, 3)
    assert got["link_names"] == list(got["geoms"]) and len(got["link_names"]) % H == 0
    base = got["link_names"][:len(got["link_names"]) // H]
    assert "world" in base and set(base) <= set(names) | {"world"}
    assert got["link_names"] == [n if k == 0 else f"{n}_{k}" for k in range(H) for n in base]
    for k in range(H):
        a = k / H * 0.8 + 0.2
        for n in names + ["world"]:
            key = n if k == 0 else f"{n}_{k}"
            if key not in got["geoms"]:
                continue
            for g in got["geoms"][key]:
                l = names.index(n) if n in names else -1
                if n == "world":
                    assert g["link_idx"] == -1
                elif "goal" in n:
                    assert g["link_idx"] == l and g["rgba"] == [0.0, 1.0, 0.0, 1.0]
                elif "_ref" in n and ("torso" in n or "thigh" in n):
                    assert g["link_idx"] == l + k * L and g["rgba"] == [1 - a, 1.0, 1 - a, 1.0]
                elif "_ref" in n:
                    assert g["link_idx"] == l and g["rgba"] == [1.0, 1.0, 1.0, 0.0]
                else:
                    assert g["link_idx"] == l + k * L and g["rgba"] == [1.0, 1 - a, 1 - a, 1.0]
    # the last H frames play the final rollout: every copy on that step's pose (pushT lifted by i * 0.01 / 50)
    fp = np.asarray(got["states"]["x"]["pos"])
    for t in range(H):
        want_t = pos[-1, t].astype(np.float32) + (np.float32([0, 0, t * 0.01 / 50]) if name == "pushT" else np.float32(0))
        np.testing.assert_allclose(fp[K + t].reshape(H, L, 3), np.broadcast_to(want_t, (H, L, 3)), atol=1e-6)
    if name == "pushT":
        assert any("goal" in n for n in names)
    if name == "humanoidtrack":
        assert any("_ref" in n and "torso" in n for n in names) and any("_ref" in n and "thigh" not in n and "torso" not in n for n in names)


def test_car2d_is_refused(tmp_path):
    with pytest.raises(SystemExit, match="car2d"):
        vd.main(["--env_name", "car2d", "--path", str(tmp_path)])


def test_missing_iterates_say_run_the_planner(tmp_path):
    with pytest.raises(SystemExit, match="run the planner first"):
        vd.main(["--env_name", "hopper", "--path", str(tmp_path)])


def test_iterates_prepend_the_random_iterate(tmp_path):
    from mbd_b200 import prng
    from mbd_b200.blackbox.mbd_mnist import normal_host
    mu = np.random.default_rng(1).uniform(-1, 1, size=(5, 7, 3)).astype(np.float32)
    np.save(tmp_path / "mu_0ts.npy", mu)
    us = vd.load_iterates(str(tmp_path), 3)
    assert us.shape == (6, 7, 3)
    np.testing.assert_array_equal(us[1:], mu)
    np.testing.assert_array_equal(us[0], normal_host(prng.PRNGKey(0), (7, 3)))


def test_rollout_cache_follows_the_inputs(tmp_path, monkeypatch):
    env = get_env("hopper")
    calls = []

    def fake(env_, state, us):
        calls.append(us.copy())
        K_, H_ = us.shape[:2]
        L = env_.sys.num_links()
        return np.full((K_, H_, L, 3), len(calls), np.float32), np.full((K_, H_, L, 4), len(calls), np.float32)

    monkeypatch.setattr(vd, "device_rollouts", fake)
    cache = str(tmp_path / "rollouts.npz")
    us = np.zeros((2, 3, env.action_size), np.float32)
    p1, _ = vd.rollouts("hopper", env, us, cache=cache)
    assert len(calls) == 1 and os.path.exists(cache)
    p2, _ = vd.rollouts("hopper", env, us, cache=cache)           # same inputs: loaded
    assert len(calls) == 1 and np.array_equal(p1, p2)
    us[1, 2, 0] = 0.5                                             # a changed iterate: rebuilt
    p3, _ = vd.rollouts("hopper", env, us, cache=cache)
    assert len(calls) == 2 and p3[0, 0, 0, 0] == 2
    with np.load(cache) as z:
        assert str(z["hash"]) == vd.inputs_hash("hopper", us)


def test_script_writes_the_page_from_the_cache(tmp_path, monkeypatch):
    """end to end without a GPU: the rollouts come from the cache, the page embeds the document"""
    env = get_env("hopper")
    mu = np.random.default_rng(2).uniform(-1, 1, size=(2, 4, env.action_size)).astype(np.float32)
    np.save(tmp_path / "mu_0ts.npy", mu)
    us = vd.load_iterates(str(tmp_path), env.action_size)
    L = env.sys.num_links()
    pos = np.random.default_rng(3).normal(size=(3, 4, L, 3)).astype(np.float32)
    rot = np.random.default_rng(4).normal(size=(3, 4, L, 4)).astype(np.float32)
    np.savez(tmp_path / "rollouts.npz", pos=pos, rot=rot, hash=np.array(vd.inputs_hash("hopper", us)))
    monkeypatch.setattr(vd, "device_rollouts", None)              # must not be needed
    out = vd.main(["--env_name", "hopper", "--path", str(tmp_path)])
    page = open(out).read()
    doc = json.dumps(brax_json.diffusion_to_dict(env.sys, pos, rot, env.dt))
    assert page == brax_json.page(doc, vd.HEIGHT)
