"""Time per control step of the receding-horizon controller (python -m mbd_b200.planners.mbd_mpc) on the current GPU.

For every case (env, Nsample x Hsample, Nwarm = 10) at B = 1 and B = 8 seeds:
  - device: the graph-replayed loop (Controller.run), one replay of the captured warm control step per control step;
  - host:   the host-driven loop of the same arithmetic (Controller.run_host_driven): eager steps, the plan copied to the host, a host
            env.step per seed, the warm start, keys and step counter written with torch;
  - step:   one batched diffusion step alone (graph replay), so that a control step can be read as Nwarm steps + the rest.
The two loops alternate REPS times in one process; each reports the best wall time of control steps 1 ... NSTEP - 1 (synchronised
at both ends) divided by NSTEP - 1.  Both loops must give the same actions, rewards and states bit for bit.  The closed-loop mean
reward of every seed is reported.  The GPU name and power limit are read in the same run.
    python scripts/gpu_mpc_timing.py [out.json]   (default profiles/h100_mpc.json)"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mbd_b200.planners import mbd_mpc  # noqa: E402
from mbd_b200.planners.mbd_mpc import Args, Controller  # noqa: E402

CASES = [("car2d", 64, 40), ("hopper", 1024, 50), ("humanoidrun", 1024, 50)]
NWARM, NDIFFUSE, NSTEP, REPS = 10, 20, 21, 3
TEMPS = [0.1, 0.05, 0.3, 0.2, 0.15, 0.5, 0.08, 1.0]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")])) if out.strip() else {}


def args_list(env_name, N, H, B):
    return [Args(seed=s, env_name=env_name, Nsample=N, Hsample=H, Ndiffuse=NDIFFUSE, Nwarm=NWARM, Nstep=NSTEP, not_render=True,
                 disable_recommended_params=True, temp_sample=TEMPS[s % 8]) for s in range(B)]


def step_ms(ctl, reps=20):
    """one batched diffusion step, graph-replayed (the controller's engine, before its run)"""
    e = ctl.engine
    e.capture()
    best = float("inf")
    for _ in range(3):
        e.set_step(NDIFFUSE - 1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(min(reps, NDIFFUSE - 1)):
            e.step()
        torch.cuda.synchronize()
        best = min(best, (time.perf_counter() - t0) / min(reps, NDIFFUSE - 1))
    e.graph = None
    return best * 1e3


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join("profiles", "h100_mpc.json")
    res = dict(gpu=gpu_info(), Nwarm=NWARM, Ndiffuse=NDIFFUSE, Nstep=NSTEP, reps=REPS,
               timed="best over reps of the wall time of control steps 1 .. Nstep - 1, divided by Nstep - 1", cases=[])
    for env_name, N, H in CASES:
        for B in (1, 8):
            al = args_list(env_name, N, H, B)
            env = mbd_mpc._prepare(al, batch=True)
            t_step = step_ms(Controller(env, al))
            dev_t, host_t, same = [], [], True
            for _ in range(REPS):
                c = Controller(env, args_list(env_name, N, H, B))
                r = c.run(log_every=10 ** 9)
                dev_t.append(c.warm_seconds / (NSTEP - 1))
                h = Controller(env, args_list(env_name, N, H, B), host=True)
                q = h.run_host_driven()
                host_t.append(h.warm_seconds / (NSTEP - 1))
                same = same and all(np.array_equal(getattr(r, f).view(np.uint32), getattr(q, f).view(np.uint32))
                                    for f in ("actions", "rewards", "states", "rew_hist"))
            row = dict(env=env_name, Nsample=N, Hsample=H, B=B, diffusion_step_ms=round(t_step, 4),
                       device_ms_per_control_step=round(min(dev_t) * 1e3, 3), host_ms_per_control_step=round(min(host_t) * 1e3, 3),
                       speedup=round(min(host_t) / min(dev_t), 2), bit_identical=bool(same),
                       closed_loop_reward_per_seed=[round(float(x), 5) for x in r.reward])
            print(row, flush=True)
            res["cases"].append(row)
    os.makedirs(os.path.dirname(out_path) or ".", exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
