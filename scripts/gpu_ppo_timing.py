"""Cost of PPO training (mbd_b200.rl.ppo) on the current GPU, and the learning runs the GPU learning test is calibrated on.

  - per training step at the reference's shapes (halfcheetah, ant): acting (U unroll graphs + the record launch), the observation
    statistics, and the learner (the permutations + E * num_minibatches SGD graphs), CUDA events around each part over STEPS steps
    after one warm-up step; env-steps/s of the whole step;
  - the acting step alone: k_ppo_act (one launch) against the same work in torch (MLP, torch.randn sampling, tanh and log-prob),
    each also followed by the vector env's step, at B in {128, 2048, 4096} (halfcheetah), REPEATS times.  The torch work is timed
    twice: launched eagerly from the host (bound by the host's launch rate at these sizes, so it measures that, not GPU time) and
    replayed from a CUDA graph of the same ops (the GPU time of that work);
  - learning: the check of tests/test_ppo_gpu.py::test_short_run_learns (tests/ppo_ref.learn_config), evaluation return before and
    after for seeds 0 .. 4;
  - one full reference-configuration halfcheetah run (50 M env steps, seed 3, python -m mbd_b200.rl.train_brax's table): its
    evaluation curve, the wall clock at every evaluation and in total.
The GPU name, power limit and SM clock are read in the same run.
    python scripts/gpu_ppo_timing.py [out.json]     (default profiles/h100_ppo.json)"""
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mbd_b200 import _lib, ops, prng  # noqa: E402
from mbd_b200.envs import get_env  # noqa: E402
from mbd_b200.envs.vec import VecEnv  # noqa: E402
from mbd_b200.rl import networks as nets  # noqa: E402
from mbd_b200.rl import ppo, train_brax  # noqa: E402
from tests import ppo_ref  # noqa: E402

STEPS = 3
REPEATS = 3


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")])) if out.strip() else {}


def ev():
    return torch.cuda.Event(enable_timing=True)


def step_split(name):
    cfg = train_brax.ppo_config(name)
    c = ppo.counts(1, cfg["num_envs"], cfg["batch_size"], cfg["num_minibatches"], cfg["unroll_length"], 2)
    tr = ppo.PPOTrainer(get_env(name), (STEPS + 1) * c.env_steps_per_training_step, cfg["episode_length"], cfg["num_envs"], 128,
                        cfg["learning_rate"], cfg["entropy_cost"], cfg["discounting"], 0, cfg["unroll_length"], cfg["batch_size"],
                        cfg["num_minibatches"], cfg["num_updates_per_batch"], 2, True, cfg["reward_scaling"], 0.3, 0.95)
    tr.capture()
    tr.training_step()
    acting = stats = learner = 0.0
    t0 = time.perf_counter()
    for _ in range(STEPS):
        e = [ev() for _ in range(4)]
        e[0].record()
        for _ in range(tr.U):
            tr._unroll_graph.replay()
        ops.ppo_act(tr.plan, _lib.PPO_RECORD)
        e[1].record()
        ops.ppo_obs_stats(tr.plan)
        e[2].record()
        tr._permutations()
        tr.mb_ctl[0:1].fill_(tr.nmb)
        for _ in range(tr.E * tr.nmb):
            tr._sgd_graph.replay()
        e[3].record()
        torch.cuda.synchronize()
        tr.step_index += 1
        acting += e[0].elapsed_time(e[1])
        stats += e[1].elapsed_time(e[2])
        learner += e[2].elapsed_time(e[3])
    wall = (time.perf_counter() - t0) / STEPS
    n = STEPS
    return dict(env=name, num_envs=tr.B, U=tr.U, T=tr.T, minibatch=tr.mb, sgd_steps=tr.E * tr.nmb, acting_ms=acting / n, stats_ms=stats / n,
                learner_ms=learner / n, step_ms=(acting + stats + learner) / n, wall_ms=wall * 1e3,
                env_steps_per_s=c.env_steps_per_training_step / wall)


def act_alone(B, reps=200):
    env = get_env("halfcheetah")
    venv = VecEnv(env, B, 1000)
    venv.reset(prng.split(prng.PRNGKey(0), B))
    O, nu = venv.spec.obs_size, venv.spec.nu
    sizes = nets.policy_sizes(O, nu)
    pol = torch.from_numpy(nets.init_params(prng.PRNGKey(1), sizes)).cuda()
    mean, std = torch.zeros(O, device="cuda"), torch.ones(O, device="cuda")
    keys = torch.zeros((reps + 10, 2), device="cuda", dtype=torch.int32)
    actor = ppo.Actor(venv, pol, mean, std, keys)
    layers = nets.unflatten(pol, sizes)

    def kernel():
        ops.ppo_act(actor.plan, _lib.PPO_EVAL)

    def eager():
        with torch.no_grad():
            logits = nets.mlp(nets.normalize(venv.obs, mean, std), layers)
            loc, s = logits.chunk(2, -1)
            raw = torch.randn_like(loc) * (torch.nn.functional.softplus(s) + nets.MIN_STD) + loc
            lp = nets.log_prob(logits, raw)
            venv.actions.copy_(torch.tanh(raw))
        return lp

    def step():
        ops.vec_step(venv.plan)

    for _ in range(10):
        eager()
        kernel()
        step()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        eager()
    gs = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gs):
        eager()
        step()

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        actor.ctl.zero_()
        a, b = ev(), ev()
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        actor.ctl.zero_()
        return a.elapsed_time(b) * 1e3 / reps

    cases = {"k_ppo_act_us": kernel, "k_ppo_act_plus_env_step_us": lambda: (kernel(), step()),
             "torch_eager_act_us": eager, "torch_eager_act_plus_env_step_us": lambda: (eager(), step()),
             "torch_graph_act_us": g.replay, "torch_graph_act_plus_env_step_us": gs.replay}
    out = {"B": B}
    for _ in range(REPEATS):
        for k, fn in cases.items():
            out.setdefault(k, []).append(timed(fn))
    return out


def learning(seeds=(0, 1, 2, 3, 4)):
    rows = []
    for seed in seeds:
        curve = []
        t0 = time.perf_counter()
        ppo.train(environment=ppo_ref.LEARN_ENV, progress_fn=lambda n, m: curve.append((n, m["eval/episode_reward"])),
                  **ppo_ref.learn_config(seed))
        rows.append(dict(seed=seed, curve=curve, seconds=time.perf_counter() - t0))
        print(rows[-1], flush=True)
    return rows


def full_run(name="halfcheetah"):
    cfg = train_brax.ppo_config(name)
    curve = []
    t0 = time.perf_counter()

    def progress(n, m):
        curve.append(dict(step=n, episode_return=m["eval/episode_reward"], wall_s=time.perf_counter() - t0))
        print(curve[-1], flush=True)

    ppo.train(environment=name, progress_fn=progress, **cfg)
    return dict(env=name, config=cfg, curve=curve, wall_s=time.perf_counter() - t0,
                train_s=curve[-1]["wall_s"] - curve[0]["wall_s"], setup_s=curve[0]["wall_s"])


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles", "h100_ppo.json")
    res = dict(gpu=gpu_info(), torch=torch.__version__, steps_timed=STEPS)
    res["training_step"] = [step_split(n) for n in ("halfcheetah", "ant")]
    print(res["training_step"], flush=True)
    res["acting"] = [act_alone(B) for B in (128, 2048, 4096)]
    print(res["acting"], flush=True)
    res["learning_check"] = dict(env=ppo_ref.LEARN_ENV, config=ppo_ref.learn_config(0), runs=learning())
    res["full_run"] = full_run()
    res["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
    with open(out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res)[:3000])


if __name__ == "__main__":
    main()
