"""Time per control step of the path-integral baselines as receding-horizon controllers (python -m mbd_b200.planners.pi_mpc) on the
current GPU, and the closed-loop comparison with model-based diffusion the controllers exist for.

Timing.  For every case (env, Nsample x Hsample, Nwarm = 10), method (mppi, cma-es, cem) and B = 1 and 8 seeds:
  - device: the graph-replayed loop (Controller.run), one replay of the captured warm control step per control step;
  - host:   the host-driven loop of the same arithmetic (Controller.run_host_driven): eager steps, the plan copied to the host, a host
            env.step per seed, the warm start, keys, sigma rows and step counter written with torch;
  - step:   one batched baseline step alone (graph replay), so that a control step can be read as Nwarm steps + the rest.
The two loops alternate REPS times in one process; each reports the best wall time of control steps 1 ... NSTEP - 1 (synchronised
at both ends) divided by NSTEP - 1.  Both loops must give the same actions, rewards, states, rew_hist and sigmas bit for bit.

Comparison.  Per env, mbd and every baseline at sigma_warm 1.0, 0.3 and 0.1 run the same 8 seeds as one batch at equal Nsample,
Hsample, Nwarm and Nstep (mbd_b200/scripts/run_mpc.py builds the Args); the closed-loop mean reward of every seed, the sigma every
seed's last control step ended with and the zero-action plant from the same reset states are reported.
The GPU name and power limit are read in the same run.
    python scripts/gpu_pi_mpc_timing.py [out.json]   (default profiles/h100_mpc_pi.json)"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mbd_b200  # noqa: E402
from mbd_b200.planners import pi_mpc  # noqa: E402
from mbd_b200.planners.pi_mpc import Args, Controller  # noqa: E402
from mbd_b200.scripts import run_mpc  # noqa: E402

CASES = [("hopper", 1024, 50), ("humanoidrun", 1024, 50)]
METHODS = ("mppi", "cma-es", "cem")
NWARM, NREFINE, NSTEP, REPS = 10, 20, 21, 3
TEMPS = [0.1, 0.05, 0.3, 0.2, 0.15, 0.5, 0.08, 1.0]
SIGMA_WARMS = (1.0, 0.3, 0.1)
CMP = dict(Nsolve=100, Nwarm=10, Nstep=50)
FIELDS = ("actions", "rewards", "states", "rew_hist", "sigmas")


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")])) if out.strip() else {}


def args_list(env_name, method, N, H, B):
    return [Args(seed=s, env_name=env_name, update_method=method, Nsample=N, Hsample=H, Nrefine=NREFINE, Nwarm=NWARM, Nstep=NSTEP,
                 not_render=True, disable_recommended_params=True, temp_sample=TEMPS[s % 8]) for s in range(B)]


def step_ms(ctl, reps=19):
    """one batched baseline step, graph-replayed (the controller's engine, before its run)"""
    e = ctl.engine
    e.capture()
    best = float("inf")
    for _ in range(3):
        e.set_step(NREFINE - 1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(min(reps, NREFINE - 1)):
            e.step()
        torch.cuda.synchronize()
        best = min(best, (time.perf_counter() - t0) / min(reps, NREFINE - 1))
    e.graph = None
    return best * 1e3


def timing_row(env_name, method, N, H, B):
    al = args_list(env_name, method, N, H, B)
    env = pi_mpc._prepare(al, batch=True)
    t_step = step_ms(Controller(env, al))
    dev_t, host_t, same = [], [], True
    for _ in range(REPS):
        c = Controller(env, args_list(env_name, method, N, H, B))
        r = c.run(log_every=10 ** 9)
        dev_t.append(c.warm_seconds / (NSTEP - 1))
        h = Controller(env, args_list(env_name, method, N, H, B), host=True)
        q = h.run_host_driven()
        host_t.append(h.warm_seconds / (NSTEP - 1))
        same = same and all(np.array_equal(getattr(r, f).view(np.uint32), getattr(q, f).view(np.uint32)) for f in FIELDS)
    return dict(env=env_name, method=method, Nsample=N, Hsample=H, B=B, baseline_step_ms=round(t_step, 4),
                device_ms_per_control_step=round(min(dev_t) * 1e3, 3), host_ms_per_control_step=round(min(host_t) * 1e3, 3),
                speedup=round(min(host_t) / min(dev_t), 2), bit_identical=bool(same))


def comparison(env_name, N, H):
    """closed-loop reward of the 8 seeds per algorithm, the baselines at every sigma_warm, and the zero-action plant"""
    r5 = lambda x: [round(float(v), 5) for v in x]   # noqa: E731
    rows, s0 = [], None
    for algo, sw in [("mbd", None)] + [(m, s) for m in METHODS for s in SIGMA_WARMS]:
        a = run_mpc.Args(env_name=env_name, Nsample=N, Hsample=H, sigma_warm=1.0 if sw is None else sw, **CMP)
        res, per = run_mpc.run_controllers(algo, a)
        s0 = res.states[:, 0]
        row = dict(env=env_name, algo=algo, sigma_warm=sw, reward_mean=round(float(res.reward.mean()), 4),
                   reward_std=round(float(res.reward.std()), 4), reward_per_seed=r5(res.reward),
                   ms_per_control_step=round(per * 1e3, 3))
        if res.sigmas is not None:
            row["last_sigma_per_seed"] = [float(f"{v:.4g}") for v in res.sigmas[:, -1]]
        print(row, flush=True)
        rows.append(row)
    zero = run_mpc.zero_action_rewards(mbd_b200.envs.get_env(env_name), s0, CMP["Nstep"])
    rows.append(dict(env=env_name, algo="zero", sigma_warm=None, reward_mean=round(float(zero.mean()), 4),
                     reward_std=round(float(zero.std()), 4), reward_per_seed=r5(zero)))
    print(rows[-1], flush=True)
    return rows


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join("profiles", "h100_mpc_pi.json")
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing here can be measured without one")
    res = dict(gpu=gpu_info(), Nwarm=NWARM, Nrefine=NREFINE, Nstep=NSTEP, reps=REPS,
               timed="best over reps of the wall time of control steps 1 .. Nstep - 1, divided by Nstep - 1",
               comparison_shape=dict(seeds=list(run_mpc.SEEDS), **CMP), cases=[], comparison=[])
    for env_name, N, H in CASES:
        res["comparison"] += comparison(env_name, N, H)
    for env_name, N, H in CASES:
        for method in METHODS:
            for B in (1, 8):
                row = timing_row(env_name, method, N, H, B)
                print(row, flush=True)
                res["cases"].append(row)
    os.makedirs(os.path.dirname(out_path) or ".", exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
