"""Times the fused SAC update (sac.FusedLearner, mbd_sac_update) against the torch learner on hopper at the reference's configuration,
and records what the fused learner learns.

* update: one graph-replayed update of each learner, alternating the two learners in one process (CUDA events, median of repeats);
* the per-launch breakdown of the fused update (torch.profiler's kernel times of k_sac_learn_rows and k_sac_learn_weights);
* training step: one training step (acting, sampling, 64 updates) of each learner, alternating;
* learning check: sac_ref.learn_config(seed) with learner="fused" for seeds 0 .. 9 and with the torch learner for seeds 5 .. 9 (the
  evaluation return before and after, the final log alpha and mean |Q|);
* --full: the reference's full hopper run (train_sac's table, seed 1) with the fused learner: wall clock and the evaluation curve.
  --budget=S stops it after the first epoch that ends past S seconds.
The GPU name, power limit and SM clock are read in the same run.
    python scripts/gpu_sac_learn_timing.py [--full [--budget=S]] [--no-learn] [out.json]     (default profiles/h100_sac_learn.json)"""
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mbd_b200.envs import get_env  # noqa: E402
from mbd_b200.rl import sac, train_sac  # noqa: E402
from tests import sac_ref  # noqa: E402

REPEATS = 7
STEPS = 10


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")])) if out.strip() else {}


def trainer(learner, steps):
    cfg = train_sac.sac_config("hopper")
    c = sac.counts(1 << 30, cfg["num_envs"], cfg["min_replay_size"], 2)
    tr = sac.SACTrainer(get_env("hopper"), c.prefill_env_steps + steps * cfg["num_envs"], cfg["episode_length"], cfg["num_envs"], 128,
                        cfg["learning_rate"], cfg["discounting"], 0, cfg["batch_size"], 2, True, cfg["reward_scaling"], 0.005,
                        cfg["min_replay_size"], cfg["max_replay_size"], cfg["grad_updates_per_step"], learner=learner)
    tr.capture()
    tr.prefill()
    tr.training_step()
    torch.cuda.synchronize()
    return tr


def ev():
    return torch.cuda.Event(enable_timing=True)


def time_update(tr):
    """ms of one graph-replayed update (the 64 updates of a sample, divided by 64)"""
    tr._sample_graph.replay()
    a, b = ev(), ev()
    a.record()
    for _ in range(tr.G):
        tr._sgd_graph.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / tr.G


def time_step(tr):
    a, b = ev(), ev()
    a.record()
    tr.training_step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def split_step(tr):
    """ms of the acting graph, the sampling graph and the 64 update replays of one training step"""
    e = [ev() for _ in range(4)]
    e[0].record()
    tr._act_graph.replay()
    e[1].record()
    tr._sample_graph.replay()
    e[2].record()
    for _ in range(tr.G):
        tr._sgd_graph.replay()
    e[3].record()
    torch.cuda.synchronize()
    tr.step_index += 1
    return dict(act_ms=e[0].elapsed_time(e[1]), sample_ms=e[1].elapsed_time(e[2]), updates_ms=e[2].elapsed_time(e[3]))


def launch_breakdown(tr):
    from torch.profiler import ProfilerActivity, profile
    tr._sample_graph.replay()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(tr.G):
            tr.sgd_step()               # eager launches, so that every kernel shows up on its own
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if "sac_learn" in e.key:
            us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            out[e.key] = dict(calls=e.count, mean_us=us / max(e.count, 1))
    return out


def med(x):
    x = sorted(x)
    return x[len(x) // 2]


def learning(seeds, learner="fused"):
    """the learning check's run for each seed: the return before and after, and the final log alpha and mean |Q| and |target Q|"""
    res = []
    for seed in seeds:
        cfg = sac_ref.learn_config(seed)
        t0 = time.perf_counter()
        tr = sac.SACTrainer(get_env(sac_ref.LEARN_ENV), cfg["num_timesteps"], cfg["episode_length"], cfg["num_envs"], 128,
                            cfg["learning_rate"], cfg["discounting"], seed, cfg["batch_size"], cfg["num_evals"],
                            cfg["normalize_observations"], cfg["reward_scaling"], 0.005, cfg["min_replay_size"], cfg["max_replay_size"],
                            cfg["grad_updates_per_step"], learner=learner)
        tr.capture()
        before = tr.evaluate()
        tr.prefill()
        for _ in range(tr.c.steps_per_epoch):
            tr.training_step()
        after = tr.evaluate()
        p = tr.params()
        res.append(dict(learner=learner, seed=seed, before=before, after=after, gain=after - before,
                        log_alpha=float(p["log_alpha"][0]), mean_abs_q=float(abs(p["q"]).mean()),
                        mean_abs_target_q=float(abs(p["target_q"]).mean()), seconds=time.perf_counter() - t0))
        print(res[-1], flush=True)
        del tr
    return res


def full_run(budget_s):
    """the reference's full hopper run (train_sac's table, seed 1) with the fused learner, epoch by epoch as sac.train runs it: the
    return after every epoch, its training time and log alpha.  The run stops after the first epoch that ends past budget_s
    (default: none), and the record says how many of the epochs it ran."""
    cfg = train_sac.sac_config("hopper")
    t_build = time.perf_counter()
    tr = sac.SACTrainer(get_env("hopper"), cfg["num_timesteps"], cfg["episode_length"], cfg["num_envs"], 128, cfg["learning_rate"],
                        cfg["discounting"], cfg["seed"], cfg["batch_size"], cfg["num_evals"], cfg["normalize_observations"],
                        cfg["reward_scaling"], 0.005, cfg["min_replay_size"], cfg["max_replay_size"], cfg["grad_updates_per_step"],
                        learner="fused")
    tr.capture()
    torch.cuda.synchronize()
    rec = dict(config=cfg, setup_s=time.perf_counter() - t_build, curve=[], epoch_s=[], epochs=tr.c.num_evals_after_init)
    t_run = time.perf_counter()
    r = tr.evaluate()
    tr.prefill()
    torch.cuda.synchronize()
    rec["prefill_and_first_eval_s"] = time.perf_counter() - t_run
    rec["curve"].append(dict(env_steps=0, ret=r))
    print(rec["curve"][-1], flush=True)
    while len(rec["epoch_s"]) < rec["epochs"]:
        t0 = time.perf_counter()
        for _ in range(tr.c.steps_per_epoch):
            tr.training_step()
        torch.cuda.synchronize()
        train_s = time.perf_counter() - t0
        r = tr.evaluate()
        rec["epoch_s"].append(time.perf_counter() - t0)
        rec["curve"].append(dict(env_steps=tr.env_steps(), ret=r, train_s=train_s, log_alpha=float(tr.learner.log_alpha[0])))
        print(rec["curve"][-1], flush=True)
        if time.perf_counter() - t_run > budget_s:
            break
    rec["epochs_run"] = len(rec["epoch_s"])
    rec["wall_s"] = time.perf_counter() - t_run
    rec["last_return"] = rec["curve"][-1]["ret"]
    return rec


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    out = args[0] if args else os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles",
                                            "h100_sac_learn.json")
    res = dict(gpu=gpu_info(), torch=torch.__version__)
    if "--full" in sys.argv:
        budget = float(next((a.split("=", 1)[1] for a in sys.argv if a.startswith("--budget=")), "1e9"))
        res["full_run"] = full_run(budget)
    else:
        trs = {k: trainer(k, 4 * REPEATS + 8) for k in ("torch", "fused")}
        upd = {k: [] for k in trs}
        step = {k: [] for k in trs}
        for _ in range(REPEATS):                 # alternate the two learners
            for k, tr in trs.items():
                upd[k].append(time_update(tr))
                step[k].append(time_step(tr))
        res["update_ms"] = {k: dict(median=med(v), all=v) for k, v in upd.items()}
        res["training_step_ms"] = {k: dict(median=med(v), all=v) for k, v in step.items()}
        res["training_step_split_ms"] = {k: split_step(tr) for k, tr in trs.items()}
        res["fused_launches"] = launch_breakdown(trs["fused"])
        res["update_speedup"] = res["update_ms"]["torch"]["median"] / res["update_ms"]["fused"]["median"]
        print(json.dumps(res)[:3000], flush=True)
        if "--no-learn" not in sys.argv:
            res["learning_check"] = learning(range(10))
            res["learning_check_torch"] = learning(range(5, 10), "torch")   # seeds 0 .. 4: profiles/h100_sac.json
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res)[:3000])


if __name__ == "__main__":
    main()
