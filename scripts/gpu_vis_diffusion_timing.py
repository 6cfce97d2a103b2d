"""Cost of the diffusion-process page (python -m mbd_b200.scripts.vis_diffusion) on the current GPU.

humanoidrun, K = 300 iterates (the random one + 299 synthetic mu_0ts rows) of Hsample = 50 steps, the poses before each step:
  - device path, each part timed on its own (wall clock after a synchronize, best of REPS after a warm-up):
      rollout      one launch of the recorded rollout kernel (ops.rollout(..., want_traj=True)) and the state rows before each step;
      world_poses  the K * H raw states through VecEnv.set_state + VecEnv.world_poses (chunks of at most VEC_MAX_B) and the copy back;
      json         brax_json.diffusion_to_dict + json.dumps + the page;
  - host path: the reference's loop, one env.step per step (vis_diffusion.py:115-139), once, on HOST_ITERATES iterates (all K by
    default), with the same JSON part.
The GPU name and power limit are read in the same run.  pushT's host pose derivation (env.pipeline_init per state) is timed too.
    python scripts/gpu_vis_diffusion_timing.py [out.json] [host_iterates]   (default profiles/h100_vis_diffusion.json, all)"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mbd_b200 import prng  # noqa: E402
from mbd_b200.envs import get_env  # noqa: E402
from mbd_b200.io import brax_json  # noqa: E402
from mbd_b200.scripts import vis_diffusion as vd  # noqa: E402

K, H, REPS = 300, 50, 3


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")])) if out.strip() else {}


def best(fn, reps=REPS):
    fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return min(ts), r


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join("profiles", "h100_vis_diffusion.json")
    host_k = int(sys.argv[2]) if len(sys.argv) > 2 else K
    res = dict(gpu=gpu_info(), env="humanoidrun", K=K, H=H, reps=REPS)
    env = get_env("humanoidrun")
    rng = np.random.default_rng(0)
    us = np.concatenate([vd.normal_iterate(H, env.action_size)[None],
                         rng.uniform(-1, 1, size=(K - 1, H, env.action_size)).astype(np.float32)])
    state = env.reset(prng.split(prng.PRNGKey(0))[1])
    m = env.device_model()
    raw0 = torch.as_tensor(np.asarray(state.pipeline_state.raw, np.float32), device=m.device)
    us_t = torch.as_tensor(us, device=m.device)

    t_roll, before = best(lambda: vd.rollout_states_device(env, raw0, us_t))
    t_world, (pos, rot) = best(lambda: vd.world_poses(env, before.reshape(K * H, *raw0.shape)))
    pos, rot = pos.reshape(K, H, -1, 3), rot.reshape(K, H, -1, 4)
    t_all, _ = best(lambda: vd.device_rollouts(env, state, us))

    def page(p, r):
        return brax_json.page(json.dumps(brax_json.diffusion_to_dict(env.sys, p, r, env.dt)), vd.HEIGHT)
    t_json, doc = best(lambda: page(pos, rot))
    res["device"] = dict(rollout_s=round(t_roll, 4), world_poses_s=round(t_world, 4), rollouts_total_s=round(t_all, 4),
                         json_s=round(t_json, 3), total_s=round(t_all + t_json, 3), page_bytes=len(doc))
    print(res["device"], flush=True)

    t0 = time.perf_counter()
    hs = []
    for k0 in range(0, host_k, 10):
        hs.append(vd.host_rollouts(env, state, us[k0:min(k0 + 10, host_k)]))
        print(f"host: {k0 + len(hs[-1][0])} iterates in {time.perf_counter() - t0:.1f} s", flush=True)
    t_host = time.perf_counter() - t0
    hpos, hrot = np.concatenate([h[0] for h in hs]), np.concatenate([h[1] for h in hs])
    same = bool(np.array_equal(hpos.view(np.uint32), pos[:host_k].view(np.uint32)) and
                np.array_equal(hrot.view(np.uint32), rot[:host_k].view(np.uint32)))
    res["host"] = dict(iterates=host_k, rollouts_s=round(t_host, 2), per_step_ms=round(t_host / (host_k * H) * 1e3, 3),
                       rollouts_all_K_s=round(t_host * K / host_k, 2), poses_bit_identical_to_device=same)
    res["host"]["total_s"] = round(res["host"]["rollouts_all_K_s"] + t_json, 2)
    print(res["host"], flush=True)

    penv = get_env("pushT")
    pstate = penv.reset(prng.split(prng.PRNGKey(0))[1])
    pus = rng.uniform(-1, 1, size=(K, H, 2)).astype(np.float32)
    t_pt, _ = best(lambda: vd.device_rollouts(penv, pstate, pus))
    res["pusht_device_rollouts_s"] = round(t_pt, 4)
    print({"pusht_device_rollouts_s": res["pusht_device_rollouts_s"]}, flush=True)

    os.makedirs(os.path.dirname(out_path) or ".", exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
