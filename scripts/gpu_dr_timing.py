"""Domain randomisation of the vector env (DESIGN.md §5n) on the current GPU: what drawing new factors at every auto-reset costs.

One captured VecEnv step (episode_length 10, so a tenth of the envs auto-reset and draw at every step) replayed from a CUDA graph, with
domain randomisation (ranges [0.5, 1.5] x [0.7, 1.3]) against a fixed [B, 2] factor table (§5k's per-env-model arm), for hopper and
humanoidrun at B in {1, 256, 4096, 16384}; CUDA events over 50 replays, the two arms alternated, the best of 3 and the spread
(max - min) / min of each arm reported.  The GPU name and power limit are read in the same run.
    python scripts/gpu_dr_timing.py [out.json]     (default profiles/h100_dr.json)"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mbd_b200 import prng  # noqa: E402
from mbd_b200.envs import get_env  # noqa: E402
from mbd_b200.envs.vec import VecEnv  # noqa: E402
from mbd_b200.rl.ppo import dr_keys  # noqa: E402
from scripts.gpu_vecenv_timing import gpu_info, timed  # noqa: E402

ENVS = ["hopper", "humanoidrun"]
SIZES = [1, 256, 4096, 16384]
EPISODE = 10


def captured_step(env, B, dr: bool):
    venv = VecEnv(env, B, EPISODE)
    if dr:
        venv.set_domain_randomization((0.5, 1.5), (0.7, 1.3), dr_keys(0, B))
    else:
        rng = np.random.default_rng(B)
        venv.set_model_factors(friction=rng.uniform(0.5, 1.5, B), gear=rng.uniform(0.7, 1.3, B))
    keys = prng.split(prng.PRNGKey(0), B)
    venv.reset(keys)
    venv.steps.copy_(torch.arange(B, device=venv.device) % EPISODE)   # stagger the episodes: B / 10 auto-resets at every step
    venv.actions.uniform_(-1, 1)
    venv.step()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        venv.step()
    torch.cuda.current_stream().wait_stream(s)
    return venv, g


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join("profiles", "h100_dr.json")
    rows = []
    for name in ENVS:
        env = get_env(name)
        for B in SIZES:
            (v0, g0), (v1, g1) = captured_step(env, B, False), captured_step(env, B, True)
            t0, t1 = [], []
            for _ in range(3):   # alternated, best of 3
                t0.append(timed(g0.replay))
                t1.append(timed(g1.replay))
            torch.cuda.synchronize()
            draws = int(v1.dr_episodes.sum().item())
            row = dict(env=name, B=B, fixed_us=round(min(t0), 2), dr_us=round(min(t1), 2), ratio=round(min(t1) / min(t0), 3),
                       fixed_spread=round((max(t0) - min(t0)) / min(t0), 3), dr_spread=round((max(t1) - min(t1)) / min(t1), 3),
                       draws_in_run=draws)
            print(row, flush=True)
            rows.append(row)
            del v0, v1, g0, g1
    res = dict(gpu=gpu_info(), timed=f"graph-replayed VecEnv step, episode_length {EPISODE} with staggered episodes, CUDA events over "
                                     "50 replays, fixed factors and DR alternated, best of 3; spread = (max - min) / min of the 3",
               steps=rows)
    os.makedirs(os.path.dirname(out_path) or ".", exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
