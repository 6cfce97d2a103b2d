"""Worst-m scores and drawn members of the planner ensemble (DESIGN.md §5m) on the current GPU: what they cost, and what they do in
closed loop.

  - step: one graph-replayed batched MBD step with an ensemble of K in {3, 9, 16} members scored by the mean, by the worst member
    (worst = 1) and by the worst half (worst = K / 2); hopper and humanoidrun at 1024 samples x 50, B = 1 and 8 problems.  CUDA
    events over REPS replays, the arms alternated and the best of 3 kept for each;
  - draw: one graph-replayed warm control step of 8 hopper loops (1024 x 50, Nwarm 10) with K members drawn at every control step
    against the same K members fixed (the graphs differ by the draw launch alone), K in {3, 16}: the mean wall time of the warm
    control steps of a run, three runs per arm alternated, best kept;
  - closed loop on hopper with the settings of §5k / §5l (1024 x 50, Nsolve 100, Nwarm 10, Nstep 50, seeds 0..7, the 9 plants
    friction {0.5, 1.0, 1.5} x gear {0.7, 1.0, 1.3}), every algorithm planning four ways: §5l's gear ensemble scored by its worst
    member, and K = 4 members drawn at every control step from friction [0.5, 1.5] x gear [0.7, 1.3] scored by the mean, the
    worst member and the worst two.  §5l's gear-ensemble column of MBD is re-run and compared with profiles/h100_ensemble.json.
The GPU name and power limit are read in the same run.
    python scripts/gpu_ens_risk_timing.py [out.json [steps | closed [algo ...]]]     (default profiles/h100_ens_risk.json, all)
A part run (the step and draw timings, or the closed loop of some algorithms) adds its results to an existing out.json."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mbd_b200 import prng  # noqa: E402
from mbd_b200.envs import get_env  # noqa: E402
from mbd_b200.planners import mbd_mpc, pi_mpc  # noqa: E402
from mbd_b200.planners.engine import BatchedDiffusionEngine, key_chain, make_schedule  # noqa: E402
from mbd_b200.scripts import run_mpc  # noqa: E402
from scripts.gpu_vecenv_timing import REPS, gpu_info, timed  # noqa: E402

STEP_ENVS = ["hopper", "humanoidrun"]
KS = [3, 9, 16]
BS = [1, 8]
N, H = 1024, 50
ND = 3 * (5 + REPS) + 2          # every replay of the three timed rounds runs a real step (the counter never reaches 0)
FRICTION = [0.5, 1.0, 1.5]
GEAR = [0.7, 1.0, 1.3]
GEAR_ENSEMBLE = dict(plan_friction=(1.0, 1.0, 1.0), plan_gear=(0.7, 1.0, 1.3))
DRAWN = dict(plan_members=4, plan_friction_range=(0.5, 1.5), plan_gear_range=(0.7, 1.3))


def captured_engine(env, B, K, worst):
    """a B-problem batched MBD engine with K members in [0.7, 1.3] scored with ens_worst = worst, one step captured"""
    states, keys = [], []
    for s in range(B):
        rng, rng_reset = prng.split(prng.PRNGKey(s))
        states.append(env.reset(rng_reset))
        keys.append(key_chain(prng.split(rng)[0], ND))
    ens = np.random.default_rng(K).uniform(0.7, 1.3, (B, K, 2)).astype(np.float32)
    e = BatchedDiffusionEngine(env, N, H, [0.1] * B, False, states, ND, ensemble=ens, ens_worst=worst)
    _, al, ab, sg = make_schedule(1e-4, 1e-2, ND)
    e.load_schedule(keys, [sg] * B, [al] * B, [ab] * B)
    e.set_step(ND - 1)
    e.capture()
    return e


def step_rows():
    rows = []
    for name in STEP_ENVS:
        env = get_env(name)
        for B in BS:
            for K in KS:
                arms = {"mean": captured_engine(env, B, K, 0), "worst1": captured_engine(env, B, K, 1),
                        f"worst{K // 2}": captured_engine(env, B, K, K // 2)}
                t = {k: [] for k in arms}
                for _ in range(3):   # alternated, best of 3
                    for k, e in arms.items():
                        t[k].append(timed(e.graph.replay))
                for e in arms.values():
                    e.check_exchange()
                best = {k: min(v) for k, v in t.items()}
                row = dict(env=name, B=B, K=K, N=N, H=H, us={k: round(v, 2) for k, v in best.items()},
                           ratio_to_mean={k: round(v / best["mean"], 4) for k, v in best.items()},
                           spread_us={k: round(max(v) - min(v), 2) for k, v in t.items()})
                print(row, flush=True)
                rows.append(row)
                del arms
    return rows


def draw_rows(Nstep=21):
    """a warm control step with drawn members against the same control step with fixed members (8 hopper loops)"""
    rows = []
    for K in (3, 16):
        base = dict(env_name="hopper", Nsample=N, Hsample=H, Ndiffuse=100, Nwarm=10, Nstep=Nstep, not_render=True,
                    disable_recommended_params=True)
        arms = {"fixed": [mbd_mpc.Args(seed=s, plan_friction=(1.0,) * K, plan_gear=(1.0,) * K, **base) for s in range(8)],
                "drawn": [mbd_mpc.Args(seed=s, plan_members=K, plan_friction_range=(0.5, 1.5), plan_gear_range=(0.7, 1.3), **base)
                          for s in range(8)]}
        env = mbd_mpc._prepare(arms["fixed"], batch=True)
        mbd_mpc.check_args(arms["drawn"], True)
        t = {k: [] for k in arms}
        for _ in range(3):
            for k, al in arms.items():
                ctl = mbd_mpc.Controller(env, al)
                ctl.run()
                t[k].append(ctl.warm_seconds / (Nstep - 1) * 1e3)
                del ctl
        best = {k: min(v) for k, v in t.items()}
        row = dict(env="hopper", B=8, K=K, N=N, H=H, Nwarm=10, ms_per_warm_control_step={k: round(v, 3) for k, v in best.items()},
                   all_ms={k: [round(x, 3) for x in v] for k, v in t.items()}, ratio=round(best["drawn"] / best["fixed"], 4))
        print(row, flush=True)
        rows.append(row)
    return rows


def dump(res, out_path):
    os.makedirs(os.path.dirname(out_path) or ".", exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1)


def _run(algo, kw, plants, seeds):
    base = run_mpc.Args(env_name="hopper", Nsample=1024, Hsample=50, Nsolve=100, Nwarm=10, Nstep=50)
    al = []
    for f, g in plants:
        a = run_mpc.Args(**{**base.__dict__, "plant_friction": f, "plant_gear": g, **kw})
        al += run_mpc.mbd_args(a, seeds) if algo == "mbd" else run_mpc.pi_args(a, algo, seeds)
    mod = mbd_mpc if algo == "mbd" else pi_mpc
    t = time.perf_counter()
    ctl = mod.Controller(mod._prepare(al, batch=True), al)
    r = ctl.run()
    wall = time.perf_counter() - t
    rew = r.reward.reshape(len(plants), len(seeds))
    return dict(mean=[round(float(x.mean()), 4) for x in rew], std=[round(float(x.std()), 4) for x in rew],
                over_plants=round(float(rew.mean()), 4), per_seed=rew.round(5).tolist(),
                ms_per_warm_control_step=round(ctl.warm_seconds / 49 * 1e3, 2), wall_s=round(wall, 1))


def closed_loop(res, out_path, algos):
    """fills res["closed_loop_hopper"] for `algos` (and re-runs §5l's column with mbd), written after every run"""
    plants = [(f, g) for f in FRICTION for g in GEAR]
    seeds = run_mpc.SEEDS
    ways = {"gear_ensemble_worst1": dict(GEAR_ENSEMBLE, plan_worst=1), "drawn4_mean": dict(DRAWN),
            "drawn4_worst1": dict(DRAWN, plan_worst=1), "drawn4_worst2": dict(DRAWN, plan_worst=2)}
    out = dict(shape=dict(Nsample=1024, Hsample=50, Nsolve=100, Nwarm=10, Nstep=50, seeds=list(seeds)),
               plants=[dict(friction=f, gear=g) for f, g in plants],
               ways=dict(gear_ensemble_worst1="members (1, 0.7), (1, 1), (1, 1.3), scored by the worst member",
                         drawn4_mean="4 members drawn at every control step from friction [0.5, 1.5] x gear [0.7, 1.3], mean",
                         drawn4_worst1="the same draws, scored by the worst member",
                         drawn4_worst2="the same draws, scored by the mean of the worst two"),
               algos={})
    out["algos"] = res.get("closed_loop_hopper", {}).get("algos", {})
    res["closed_loop_hopper"] = {**res.get("closed_loop_hopper", {}), **out}
    out = res["closed_loop_hopper"]
    if "mbd" not in algos:
        return run_algos(res, out, out_path, algos, ways, plants, seeds)
    # §5l's MBD gear-ensemble column, re-run: the per-seed rewards of profiles/h100_ensemble.json
    prior = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles", "h100_ensemble.json")
    with open(prior) as f:
        old = json.load(f)["closed_loop_hopper"]["algos"]["mbd"]["gear_ensemble"]["per_seed"]
    again = _run("mbd", GEAR_ENSEMBLE, plants, seeds)
    out["rerun_5l_mbd_gear_ensemble"] = dict(per_seed=again["per_seed"], equal_to_h100_ensemble_json=again["per_seed"] == old)
    print("5l re-run equal:", again["per_seed"] == old, flush=True)
    dump(res, out_path)
    run_algos(res, out, out_path, algos, ways, plants, seeds)


def run_algos(res, out, out_path, algos, ways, plants, seeds):
    for algo in algos:
        out["algos"][algo] = {}
        for way, kw in ways.items():
            out["algos"][algo][way] = _run(algo, kw, plants, seeds)
            print(algo, way, out["algos"][algo][way]["mean"], out["algos"][algo][way]["ms_per_warm_control_step"], flush=True)
            dump(res, out_path)


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join("profiles", "h100_ens_risk.json")
    part = sys.argv[2] if len(sys.argv) > 2 else "all"
    algos = tuple(sys.argv[3:]) or ("mbd",) + run_mpc.BASELINES
    res = {}
    if os.path.exists(out_path):     # a part run adds to the results of the others
        with open(out_path) as f:
            res = json.load(f)
    if part in ("all", "steps"):
        res.update(gpu=gpu_info(), timed=f"graph-replayed batched MBD step (H = {H}), CUDA events over {REPS} replays, arms "
                                         "alternated, best of 3", steps=step_rows())
        dump(res, out_path)
        res["draw"] = draw_rows()
        dump(res, out_path)
    if part in ("all", "closed"):
        res.setdefault("gpu_closed_loop", []).append(gpu_info())
        closed_loop(res, out_path, algos)
    res["gpu_after"] = gpu_info()
    dump(res, out_path)


if __name__ == "__main__":
    main()
