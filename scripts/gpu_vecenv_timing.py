"""Cost of one vector-env step (mbd_b200.envs.vec.VecEnv) on the current GPU.

For humanoidrun, hopper, ant and pushT at B in {1, 256, 4096, 16384}:
  - step_us: one captured step (launch (1), the physics, + launch (2), the epilogue) replayed from a CUDA graph, CUDA events over
    REPS replays after a warm-up;
  - epilogue_us: launch (2) alone, captured and timed the same way through mbd_vec_set_state, which runs the same kernel body
    (observation from the float64 kinematics, the per-env stores; first_state / first_obs instead of the episode bookkeeping);
    physics_us = step_us - epilogue_us;
  - env-steps/s = B / step_us.
Plus the host `env.step` loop of one env (B = 1) for comparison.  The GPU name and power limit are read in the same run.
    python scripts/gpu_vecenv_timing.py [out.json]     (default profiles/h100_vecenv.json)"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mbd_b200 import ops, prng  # noqa: E402
from mbd_b200.envs import get_env  # noqa: E402
from mbd_b200.envs.vec import VecEnv  # noqa: E402

ENVS = ["humanoidrun", "hopper", "ant", "pushT"]
SIZES = [1, 256, 4096, 16384]
REPS = 50


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")])) if out.strip() else {}


def timed(fn, reps=REPS):
    for _ in range(5):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / reps


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join("profiles", "h100_vecenv.json")
    res = dict(gpu=gpu_info(), reps=REPS, rows=[], host_loop=[])
    for name in ENVS:
        env = get_env(name)
        for B in SIZES:
            venv = VecEnv(env, B)
            venv.reset(prng.split(prng.PRNGKey(0), B))
            venv.actions.uniform_(-1, 1)
            venv.step()
            g = torch.cuda.CUDAGraph()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
                venv.step()
            torch.cuda.current_stream().wait_stream(s)
            step_us = timed(g.replay)
            g2 = torch.cuda.CUDAGraph()
            with torch.cuda.stream(s), torch.cuda.graph(g2, stream=s):
                ops.vec_set_state(venv.plan)
            torch.cuda.current_stream().wait_stream(s)
            epi_us = timed(g2.replay)
            row = dict(env=name, B=B, step_us=round(step_us, 2), epilogue_us=round(epi_us, 2),
                       physics_us=round(step_us - epi_us, 2), epilogue_share=round(epi_us / step_us, 3),
                       env_steps_per_s=round(B / step_us * 1e6))
            print(row, flush=True)
            res["rows"].append(row)
        st = env.reset(prng.PRNGKey(0))
        a = np.zeros(env.action_size, np.float32)
        for _ in range(3):
            st = env.step(st, a)
        t0 = time.perf_counter()
        for _ in range(20):
            st = env.step(st, a)
        host_us = (time.perf_counter() - t0) / 20 * 1e6
        res["host_loop"].append(dict(env=name, B=1, step_us=round(host_us, 1)))
        print(res["host_loop"][-1], flush=True)
    os.makedirs(os.path.dirname(out_path) or ".", exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
