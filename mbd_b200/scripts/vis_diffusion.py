"""Render the diffusion process — counterpart of upstream mbd/scripts/vis_diffusion.py.

    python -m mbd_b200.scripts.vis_diffusion --env_name humanoidtrack

Reads results/{env}/mu_0ts.npy (written by `python -m mbd_b200.planners.mbd_planner`), prepends the random iterate
normal(PRNGKey(0), (Hsample, Nu)) and rolls every iterate out from env.reset(split(PRNGKey(0))[1]), recording the pipeline state
before each of the Hsample steps.  The page results/{env}/render_diffusion.html shows one frame per iterate with all of its poses
at once, then plays the final trajectory (`brax_json.diffusion_to_dict`).

The rollouts of all iterates are ONE launch of the recorded rollout kernel (`ops.rollout(..., want_traj=True)`, pushT
`ops.pusht_rollout(..., want_traj=True)`); the world poses of the K * Hsample raw states come from the vector env's float64
epilogue (`VecEnv.set_state` + `VecEnv.world_poses`), the same numbers `env.step` returns.  pushT's poses are planar kinematics of q,
derived on the host with `env.pipeline_init` (cheap next to the page itself, see DESIGN.md §5h).

The reference caches its rollouts in rollouts.pkl and never invalidates that file.  Here they go to rollouts.npz together with a
hash of what they were computed from (env name, the iterates); a cache whose hash differs from the inputs is rebuilt.
car2d has no geoms to draw (the reference's script fails on it too) and is refused.
"""
from __future__ import annotations

import argparse
import hashlib
import os
import sys
from typing import Optional

import numpy as np
import torch

from .. import _lib, ops, prng, utils

HEIGHT = 500   # vis_diffusion.py:141


def normal_iterate(H: int, nu: int) -> np.ndarray:
    """jax.random.normal(PRNGKey(0), (Hsample, Nu)) in the current threefry layout (vis_diffusion.py:23-24)"""
    from ..blackbox.mbd_mnist import normal_host
    return normal_host(prng.PRNGKey(0), (H, nu))


def load_iterates(path: str, nu: int) -> np.ndarray:
    """the random iterate followed by mu_0ts [Ndiffuse-1, Hsample, Nu] -> [K, Hsample, Nu] (Hsample from the array's shape)"""
    mu_0ts = np.load(os.path.join(path, "mu_0ts.npy")).astype(np.float32)
    if mu_0ts.ndim != 3 or mu_0ts.shape[2] != nu:
        raise SystemExit(f"{path}/mu_0ts.npy has shape {mu_0ts.shape}; expected (iterates, Hsample, {nu})")
    return np.concatenate([normal_iterate(mu_0ts.shape[1], nu)[None], mu_0ts], axis=0)


def inputs_hash(env_name: str, us: np.ndarray) -> str:
    h = hashlib.sha256()
    h.update(env_name.encode())
    h.update(np.asarray(us.shape, np.int64).tobytes())
    h.update(np.ascontiguousarray(us, np.float32).tobytes())
    return h.hexdigest()


def world_poses(env, raw: torch.Tensor):
    """x.pos [N, L, 3], x.rot [N, L, 4] (float32 numpy) of N raw xpbd states [N, Lsim, 13] on the device, through the vector env's
    world-pose epilogue in chunks of at most VEC_MAX_B states (cosmetic links keep their init pose, as in _make_pipeline_state)"""
    from ..envs.vec import VecEnv
    N = raw.shape[0]
    B = min(N, _lib.VEC_MAX_B)
    venv = VecEnv(env, num_envs=B, device=raw.device)
    pos, rot = [], []
    for b0 in range(0, N, B):
        chunk = raw[b0:b0 + B]
        if chunk.shape[0] < B:    # the last chunk is padded with copies of its first state
            chunk = torch.cat([chunk, chunk[:1].expand(B - chunk.shape[0], *chunk.shape[1:])])
        venv.set_state(chunk.reshape(B, -1))
        p, r = venv.world_poses()
        pos.append(p.cpu().numpy())
        rot.append(r.cpu().numpy())
    return np.concatenate(pos)[:N], np.concatenate(rot)[:N]


def rollout_states_device(env, raw0: torch.Tensor, us: torch.Tensor) -> torch.Tensor:
    """[K, H, Lsim, 13]: the raw state before each of the H steps of every iterate us [K, H, Nu] (one launch, xpbd envs)"""
    K, H, _ = us.shape
    out = ops.rollout(env.device_model(), raw0, us, want_traj=True)
    return torch.cat([raw0[None, None].expand(K, 1, *raw0.shape), out["traj"][:, :H - 1]], dim=1)


def device_rollouts(env, state, us: np.ndarray):
    """pos [K, H, L, 3], rot [K, H, L, 4]: the world poses of the pipeline state before each of the H steps of every iterate us[k],
    all K rollouts in one launch"""
    K, H, _ = us.shape
    if env.kind == "xpbd":
        m = env.device_model()
        raw0 = torch.as_tensor(np.asarray(state.pipeline_state.raw, np.float32), device=m.device)
        before = rollout_states_device(env, raw0, torch.as_tensor(np.ascontiguousarray(us, np.float32), device=m.device))
        pos, rot = world_poses(env, before.reshape(K * H, *raw0.shape))
        L = pos.shape[1]
        pos, rot = pos.reshape(K, H, L, 3), rot.reshape(K, H, L, 4)
        pos[:, 0], rot[:, 0] = state.pipeline_state.x.pos, state.pipeline_state.x.rot    # the start state as the env holds it
        ref = getattr(env, "ref_body_idx", None)
        if ref is not None:
            # humanoidtrack.step puts the *_ref bodies on the reference trajectory at the time counter of the pre-step state
            # (humanoidtrack.py:63-82); the state before step t >= 1 came from the state with counter done0 + t - 1
            d0 = int(np.int32(state.done))
            for t in range(1, H):
                tt = min(d0 + t - 1, env.xref.shape[1] - 1)
                for i, idx in enumerate(ref):
                    pos[:, t, idx] = env.xref[i, tt]
        return pos, rot
    if env.kind == "pusht":
        P = env.device_params()
        x0 = torch.as_tensor(np.asarray(state.pipeline_state.raw, np.float32), device=P.device)
        out = ops.pusht_rollout(P, x0, torch.as_tensor(np.ascontiguousarray(us, np.float32), device=P.device), want_traj=True)
        raws = torch.cat([x0[None, None].expand(K, 1, x0.numel()), out["traj"][:, :H - 1]], dim=1).cpu().numpy()
        pos = np.empty((K, H, 3, 3), np.float32)
        rot = np.empty((K, H, 3, 4), np.float32)
        for k in range(K):
            for t in range(H):
                ps = env.pipeline_init(raws[k, t, :8], raws[k, t, 8:])
                pos[k, t], rot[k, t] = ps.x.pos, ps.x.rot
        return pos, rot
    raise SystemExit(f"no world poses for env kind {env.kind!r}")


def host_rollouts(env, state, us: np.ndarray):
    """the same poses stepped one env.step at a time (vis_diffusion.py:115-139 `render_us` per iterate)"""
    pos, rot = [], []
    for k in range(us.shape[0]):
        rollout = utils.rollout_states(env.step, state, us[k])
        pos.append(np.stack([np.asarray(ps.x.pos, np.float32) for ps in rollout]))
        rot.append(np.stack([np.asarray(ps.x.rot, np.float32) for ps in rollout]))
    return np.stack(pos), np.stack(rot)


def rollouts(env_name: str, env, us: np.ndarray, cache: Optional[str] = None, host: bool = False):
    """(pos, rot) of every iterate, from `cache` (rollouts.npz) when its hash matches the inputs; otherwise computed and saved"""
    key = inputs_hash(env_name, us)
    if cache is not None and os.path.exists(cache):
        with np.load(cache) as z:
            if str(z["hash"]) == key:
                print("loaded rollouts")
                return z["pos"], z["rot"]
    rng = prng.PRNGKey(0)
    rng, rng_reset = prng.split(rng)
    state_init = env.reset(rng_reset)
    pos, rot = (host_rollouts if host else device_rollouts)(env, state_init, us)
    if cache is not None:
        tmp = cache + f".tmp{os.getpid()}.npz"
        np.savez(tmp, pos=pos, rot=rot, hash=np.array(key))
        os.replace(tmp, cache)
        print("saved rollouts")
    return pos, rot


def render_page(env_name: str, env, pos, rot) -> str:
    import json
    from ..io import brax_json
    doc = brax_json.diffusion_to_dict(env.sys, pos, rot, env.dt, lift=env_name == "pushT")
    return brax_json.page(json.dumps(doc), HEIGHT)


def default_path(env_name: str) -> str:
    import mbd_b200
    return f"{mbd_b200.__path__[0]}/../results/{env_name}"


def main(argv=None) -> str:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--env_name", default="humanoidtrack")
    ap.add_argument("--path", default=None, help="directory of mu_0ts.npy and of the outputs (default results/{env_name})")
    ap.add_argument("--host", action="store_true", help="step the rollouts one env.step at a time instead of one launch")
    args = ap.parse_args(argv)
    if args.env_name == "car2d":
        raise SystemExit("vis_diffusion: car2d has no geoms to render (its state is a point); choose a Brax-visualizable env")
    path = args.path or default_path(args.env_name)
    if not os.path.exists(os.path.join(path, "mu_0ts.npy")):
        raise SystemExit(f"vis_diffusion: {path}/mu_0ts.npy not found; run the planner first: "
                         f"python -m mbd_b200.planners.mbd_planner --env_name {args.env_name}")
    from ..envs import get_env
    env = get_env(args.env_name)
    us = load_iterates(path, env.action_size)
    pos, rot = rollouts(args.env_name, env, us, cache=os.path.join(path, "rollouts.npz"), host=args.host)
    out = os.path.join(path, "render_diffusion.html")
    with open(out, "w") as f:
        f.write(render_page(args.env_name, env, pos, rot))
    return out


if __name__ == "__main__":
    main(sys.argv[1:])
