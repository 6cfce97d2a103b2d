"""Cost of SAC training (mbd_b200.rl.sac) on the current GPU, and the learning runs the GPU learning test is calibrated on.

  - one hopper training step at the reference's shapes (128 envs, 64 updates of 512 rows, a ring of 2^20): acting (act + env step +
    record + statistics), sampling, and the 64 updates, CUDA events around each part over STEPS steps after warm-up;
  - k_sac_act (one launch) against the same work in torch (the 256-wide ReLU MLP, torch.randn sampling, tanh) and k_sac_sample against
    torch.randint + index_select + three torch.randn, both torch versions replayed from CUDA graphs, REPEATS times;
  - one evaluation (128 envs x 1000 steps);
  - learning: the check of tests/test_sac_gpu.py::test_short_run_learns (tests/sac_ref.learn_config), evaluation return before and
    after for seeds 0 .. 4;
  - the reference's hopper run (python -m mbd_b200.rl.train_sac's table): the first EPOCHS epochs measured, with their evaluations, and
    the full run's wall clock projected from them (labelled as a projection); `--full` runs all 19 epochs instead.
The GPU name, power limit and SM clock are read in the same run.
    python scripts/gpu_sac_timing.py [--full] [out.json]     (default profiles/h100_sac.json)"""
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
from mbd_b200.rl import sac, train_sac  # noqa: E402
from tests import sac_ref  # noqa: E402

STEPS = 20
REPEATS = 3
EPOCHS = 1


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")])) if out.strip() else {}


def ev():
    return torch.cuda.Event(enable_timing=True)


def trainer(cfg, steps):
    c = sac.counts(1 << 30, cfg["num_envs"], cfg["min_replay_size"], 2)
    return sac.SACTrainer(get_env("hopper"), c.prefill_env_steps + steps * cfg["num_envs"], cfg["episode_length"], cfg["num_envs"], 128,
                          cfg["learning_rate"], cfg["discounting"], 0, cfg["batch_size"], 2, True, cfg["reward_scaling"], 0.005,
                          cfg["min_replay_size"], cfg["max_replay_size"], cfg["grad_updates_per_step"])


def step_split():
    cfg = train_sac.sac_config("hopper")
    tr = trainer(cfg, STEPS + 5)
    tr.capture()
    tr.prefill()
    for _ in range(5):
        tr.training_step()
    acting = sampling = updates = 0.0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(STEPS):
        e = [ev() for _ in range(4)]
        e[0].record()
        tr._act_graph.replay()
        e[1].record()
        tr._sample_graph.replay()
        e[2].record()
        for _ in range(tr.G):
            tr._sgd_graph.replay()
        e[3].record()
        tr.step_index += 1
        torch.cuda.synchronize()
        acting += e[0].elapsed_time(e[1])
        sampling += e[1].elapsed_time(e[2])
        updates += e[2].elapsed_time(e[3])
    wall = (time.perf_counter() - t0) / STEPS
    t1 = time.perf_counter()
    ret = tr.evaluate()
    eval_s = time.perf_counter() - t1
    n = STEPS
    return dict(env="hopper", num_envs=tr.B, updates=tr.G, batch=tr.mb, capacity=tr.cap, acting_ms=acting / n, sampling_ms=sampling / n,
                updates_ms=updates / n, step_ms=(acting + sampling + updates) / n, wall_ms=wall * 1e3,
                env_steps_per_s=tr.B / wall, eval_s=eval_s, eval_envs=128, eval_steps=tr.episode_length, eval_return=ret)


def timed(fn, reps, reset=None):
    fn()
    torch.cuda.synchronize()
    if reset:
        reset()
    a, b = ev(), ev()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    if reset:
        reset()
    return a.elapsed_time(b) * 1e3 / reps


def act_alone(B, reps=200):
    venv = VecEnv(get_env("hopper"), B, 1000)
    venv.reset(prng.split(prng.PRNGKey(0), B))
    O, nu = venv.spec.obs_size, venv.spec.nu
    sizes = nets.sac_policy_sizes(O, nu)
    pol = torch.from_numpy(nets.init_params(prng.PRNGKey(1), sizes)).cuda()
    mean, std = torch.zeros(O, device="cuda"), torch.ones(O, device="cuda")
    keys = torch.zeros((reps + 10, 2), device="cuda", dtype=torch.int32)
    actor = sac.Actor(venv, pol, mean, std, keys)
    layers = nets.unflatten(pol, sizes)

    def torch_act():
        with torch.no_grad():
            logits = nets.relu_mlp(nets.normalize(venv.obs, mean, std), layers)
            loc, s = logits.chunk(2, -1)
            raw = torch.randn_like(loc) * (torch.nn.functional.softplus(s) + nets.MIN_STD) + loc
            venv.actions.copy_(torch.tanh(raw))

    for _ in range(3):
        torch_act()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        torch_act()
    out = {"B": B}
    for _ in range(REPEATS):
        out.setdefault("k_sac_act_us", []).append(timed(lambda: ops.sac_act(actor.plan, _lib.SAC_EVAL), reps, actor.ctl.zero_))
        out.setdefault("torch_graph_act_us", []).append(timed(g.replay, reps))
    return out


def sample_alone(reps=100):
    cfg = train_sac.sac_config("hopper")
    tr = trainer(cfg, reps + 50)
    tr.ring_ctl[1] = tr.cap
    G, mb, nu, R = tr.G, tr.mb, tr.nu, tr.R
    idx = torch.zeros(G * mb, device="cuda", dtype=torch.int64)
    out_rows = torch.zeros((G * mb, R), device="cuda")
    out_eps = torch.zeros((3, G, mb, nu), device="cuda")

    def torch_sample():
        torch.randint(0, tr.cap, (G * mb,), device="cuda", out=idx)
        torch.index_select(tr.ring, 0, idx, out=out_rows)
        out_eps.normal_()

    for _ in range(3):
        torch_sample()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        torch_sample()
    res = {}
    for _ in range(REPEATS):
        res.setdefault("k_sac_sample_us", []).append(timed(lambda: ops.sac_sample(tr.plan), reps, lambda: tr.sample_ctl[0:2].zero_()))
        res.setdefault("torch_graph_sample_us", []).append(timed(g.replay, reps))
    return res


def learning(seeds=(0, 1, 2, 3, 4)):
    rows = []
    for seed in seeds:
        curve = []
        t0 = time.perf_counter()
        sac.train(environment=sac_ref.LEARN_ENV, progress_fn=lambda n, m: curve.append((n, m["eval/episode_reward"])),
                  **sac_ref.learn_config(seed))
        rows.append(dict(seed=seed, curve=curve, seconds=time.perf_counter() - t0))
        print(rows[-1], flush=True)
    return rows


def hopper_run(full):
    cfg = train_sac.sac_config("hopper")
    full_c = sac.counts(cfg["num_timesteps"], cfg["num_envs"], cfg["min_replay_size"], cfg["num_evals"])
    run_cfg = dict(cfg)
    if not full:      # the same epochs as the reference's run (same key chain length per epoch), the first EPOCHS of them
        run_cfg.update(num_evals=EPOCHS + 1, num_timesteps=full_c.prefill_env_steps + EPOCHS * full_c.steps_per_epoch * cfg["num_envs"])
    curve = []
    t0 = time.perf_counter()

    def progress(n, m):
        curve.append(dict(step=n, episode_return=m["eval/episode_reward"], wall_s=time.perf_counter() - t0))
        print(curve[-1], flush=True)

    sac.train(environment="hopper", progress_fn=progress, **run_cfg)
    wall = time.perf_counter() - t0
    per_epoch = (curve[-1]["wall_s"] - curve[0]["wall_s"]) / (len(curve) - 1)
    out = dict(env="hopper", config=run_cfg, curve=curve, wall_s=wall, setup_and_first_eval_s=curve[0]["wall_s"],
               seconds_per_epoch=per_epoch)
    if not full:
        out["projection_full_run_s"] = curve[0]["wall_s"] + per_epoch * full_c.num_evals_after_init
        out["projection_note"] = (f"projected, not measured: set-up and the first evaluation plus {full_c.num_evals_after_init} epochs at the "
                                  f"measured {per_epoch:.1f} s per epoch (the run's key chain differs only in the number of epochs)")
    return out


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    full = "--full" in sys.argv
    out = args[0] if args else os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles", "h100_sac.json")
    res = dict(gpu=gpu_info(), torch=torch.__version__, steps_timed=STEPS)
    res["training_step"] = step_split()
    print(res["training_step"], flush=True)
    res["acting"] = [act_alone(B) for B in (128, 4096)]
    print(res["acting"], flush=True)
    res["sampling"] = sample_alone()
    print(res["sampling"], flush=True)
    res["learning_check"] = dict(env=sac_ref.LEARN_ENV, config=sac_ref.learn_config(0), runs=learning())
    res["hopper_run"] = hopper_run(full)
    res["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
    with open(out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res)[:3000])


if __name__ == "__main__":
    main()
