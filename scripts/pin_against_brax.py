#!/usr/bin/env python
"""Pin the oracle's positional (XPBD) step against a REAL Brax — ready to run the day a Brax install is reachable.

The reference delegates all physics to Brax (un-vendored, un-pinned, not installable in the builder image or on the GPU box:
DESIGN.md section 2), so `oracle/mbd_oracle.c` restates Brax's published algorithm and every choice that could not be confirmed
sits behind a named compile-time switch (ORC_* at the top of that file).  This script closes the loop:

  python scripts/pin_against_brax.py --make-dump brax_dump.npz     # on ANY machine with jax + brax (+ the reference's assets):
        runs brax.positional.pipeline on upstream mbd/assets/humanoidrun.xml from the planner's seed-0 reset
        (mbd/envs/humanoidrun.py:19-32) and stores x_i.pos, x_i.rot, xd_i.ang, xd_i.vel after init and after each of
        --substeps pipeline steps under a fixed action, plus the model constants Brax compiled (masses, COMs, init_q)
        and jax.random known answers (normal / uniform / split of PRNGKey(0)).
  python scripts/pin_against_brax.py --compare brax_dump.npz       # here (no Brax needed):
        (1) model constants vs this repo's MJCF compiler, (2) PRNG known answers vs mbd_b200.prng / the oracle,
        (3) the oracle stepped substep by substep FROM BRAX'S OWN STATES (so errors do not compound), for every
        combination of the ORC_* switches: prints the per-stage max error of each combination, best first.
  python scripts/pin_against_brax.py --self-test                   # checks the machinery without Brax: a dump produced by a
        NON-default oracle variant must be identified as exactly that variant.

If `import brax` works in this process (e.g. a wheel under baseline/_ref), `--make-dump` and `--compare` can be chained:
  python scripts/pin_against_brax.py --make-dump /tmp/d.npz && python scripts/pin_against_brax.py --compare /tmp/d.npz
Exit code 0 with the line "PARITY UNPINNED: brax is not importable" when Brax is absent and --make-dump was requested.
"""
from __future__ import annotations

import argparse
import itertools
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
for extra in (os.path.join(ROOT, "baseline", "_ref"),):
    if os.path.isdir(extra):
        sys.path.insert(0, extra)

SWITCHES = {  # name -> candidate values (first = the default the CUDA kernels implement)
    "ORC_JOINT_PASSIVE_IN_ACCEL": [1, 0],
    "ORC_ANG_DAMP_IN_ACCEL": [1, 0],
    "ORC_STATIC_FRICTION_MU": [1, 0],
    "ORC_SINKING_GATE": [1, 0],
    "ORC_CONTACT_MIDPOINT": [1, 0],
    "ORC_TANGENT_EPS_FORM": [0, 1],
    "ORC_EPS_TANGENT": [1, 0],
    "ORC_EULER_ACOS": [0, 1],
    "ORC_EPS": ["1e-6f", "0.0f"],
}
PT_SWITCHES = {"ORC_PT_REG_INVWEIGHT": [0, 1], "ORC_PT_CONTACT_MIDPOINT": [1, 0]}   # oracle/pusht_oracle.c
FIELDS = [("x_i.pos", slice(0, 3)), ("x_i.rot", slice(3, 7)), ("xd_i.ang", slice(7, 10)), ("xd_i.vel", slice(10, 13))]


from oracle.oracle import build_variant  # noqa: E402  (shared with tests/test_xpbd_ref_cpu.py)


def step_states(lib, blob, states, action):
    """one positional step from EACH given state [K, L, 13] (states come from the reference dump: errors do not compound)"""
    from oracle import oracle as orc
    old = orc._LIB
    orc._LIB = lib
    try:
        out = [orc.xpbd_rollout(blob, st, action.reshape(1, 1, -1), want_final=True, nsub_override=1, nthreads=1)["final"][0] for st in states]
    finally:
        orc._LIB = old
    return np.stack(out)


def quat_err(a, b):
    """rotation quaternions are equal up to sign"""
    return np.minimum(np.abs(a - b).max(-1), np.abs(a + b).max(-1))


def compare(dump_path: str, limit: int = 0):
    import mbd_b200
    from mbd_b200 import prng
    d = np.load(dump_path)
    env = mbd_b200.envs.get_env("humanoidrun")
    print("== (1) model constants (brax.io.mjcf.load vs mbd_b200/model/mjcf.py) ==")
    for k, mine in (("mass", env.sys.mass), ("com", env.sys.com), ("init_q", env.sys.init_q)):
        if k in d:
            print(f"  {k:8s} max |diff| = {np.abs(np.asarray(d[k], np.float64) - mine).max():.3e}")
    print("== (2) PRNG known answers (jax.random vs mbd_b200.prng) ==")
    if "normal_key0" in d:
        from oracle import oracle as orc
        k0 = prng.PRNGKey(0)
        print("  split(PRNGKey(0))   equal:", bool(np.array_equal(np.asarray(d["split_key0"], np.uint32), prng.split(k0))),
              "(a mismatch here means jax_threefry_partitionable=True on the dumping side: DESIGN.md section 2)")
        print("  normal(PRNGKey(0),(8,)) bit-equal:", bool(np.array_equal(np.float32(d["normal_key0"]).view(np.uint32), orc.normal(k0, (8,)).view(np.uint32))))
        print("  uniform(PRNGKey(0),(8,)) bit-equal:", bool(np.array_equal(np.float32(d["uniform_key0"]).view(np.uint32),
                                                                         prng.uniform(k0, (8,)).view(np.uint32))))
    if "pusht_traj" in d:
        print("== (4) pushT, generalized backend (oracle/pusht_oracle.c vs brax.generalized.pipeline) ==")
        from oracle import oracle as orc
        pt = mbd_b200.envs.get_env("pushT")
        x0 = np.concatenate([np.float32(d["pusht_q0"]), np.zeros(8, np.float32)])
        acts = np.float32(d["pusht_actions"])[None]
        ref = np.float32(d["pusht_traj"])
        pt_rows = []
        with tempfile.TemporaryDirectory() as tmp:
            for ci, combo in enumerate(itertools.product(*PT_SWITCHES.values())):
                defs = dict(zip(PT_SWITCHES, combo))
                lib = build_variant(defs, os.path.join(tmp, f"pt{ci}.so"))
                old, orc._LIB = orc._LIB, lib
                try:
                    mine = orc.pusht_rollout(pt.params, x0, acts, want_traj=True, nthreads=1)["traj"][0]
                finally:
                    orc._LIB = old
                err = np.abs(mine - ref)
                pt_rows.append((float(err.max()), float(err[0].max()), defs))
        pt_rows.sort(key=lambda r: r[0])
        pt_default = {n: v[0] for n, v in PT_SWITCHES.items()}
        for tot, first, defs in pt_rows:
            tag = "DEFAULT (what the kernel implements)" if defs == pt_default else ", ".join(f"{k}={v}" for k, v in defs.items() if v != pt_default[k])
            print(f"  max |q, qd diff| = {tot:.3e}   after the first env step {first:.3e}   [{tag}]")
        print("  " + ("PINNED to 1e-3" if pt_rows[0][0] < 1e-3 else "NOT PINNED: the declared own choices (solver, regulariser diagonal, merged pyramid pair) or a "
                                                               "[brax-recalled] item of oracle/pusht_oracle.c differ — see its header"))
    print("== (3) positional step, stage by stage, from the dump's own states ==")
    states, action = np.float32(d["states"]), np.float32(d["action"])     # [K+1, L, 13], [Nu]
    names = list(SWITCHES)
    combos = list(itertools.product(*[SWITCHES[n] for n in names]))
    if limit:
        combos = combos[:limit]
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        for ci, combo in enumerate(combos):
            defs = dict(zip(names, combo))
            lib = build_variant(defs, os.path.join(tmp, f"v{ci}.so"))
            got = step_states(lib, env.blob, states[:-1], action)
            ref = states[1:]
            errs = {}
            for fname, sl in FIELDS:
                e = quat_err(got[..., sl], ref[..., sl]) if fname == "x_i.rot" else np.abs(got[..., sl] - ref[..., sl]).max(-1)
                errs[fname] = float(e.max())
            rows.append((max(errs.values()), defs, errs))
    rows.sort(key=lambda r: r[0])
    default = {n: SWITCHES[n][0] for n in names}
    for tot, defs, errs in rows[:8]:
        tag = "DEFAULT (what the kernels implement)" if defs == default else ", ".join(f"{k}={v}" for k, v in defs.items() if v != default[k])
        print(f"  max err {tot:.3e}   " + "  ".join(f"{k} {v:.2e}" for k, v in errs.items()) + f"   [{tag}]")
    best = rows[0]
    print("best combination:", {k: v for k, v in best[1].items() if v != default[k]} or "the default")
    print("PINNED" if best[0] < 1e-4 else "NOT PINNED: no switch combination reproduces the dump within 1e-4 — the restatement differs elsewhere "
          "(compare the first substep field by field; candidates: axis_angle_ang conventions, joint frame parity, com.inv_inertia)")
    return rows


def make_dump(path: str, substeps: int, ref_assets: str):
    try:
        import jax
        import jax.numpy as jp
        from brax.io import mjcf as bmjcf
        from brax.positional import pipeline as bpipe
    except Exception as e:  # noqa: BLE001
        print(f"PARITY UNPINNED: brax is not importable here ({e}).  Run this mode on a machine with jax + brax and copy the .npz back.")
        return 0
    sys_b = bmjcf.load(os.path.join(ref_assets, "humanoidrun.xml"))
    rng = jax.random.PRNGKey(0)
    rng, rng_reset = jax.random.split(rng)                 # mbd_planner.py:79
    r, r1, r2 = jax.random.split(rng_reset, 3)             # humanoidrun.py:21
    qpos = sys_b.init_q + jax.random.uniform(r1, (sys_b.q_size(),), minval=-0.01, maxval=0.01)
    qvel = jax.random.uniform(r2, (sys_b.qd_size(),), minval=-0.01, maxval=0.01)
    st = bpipe.init(sys_b, qpos, qvel)
    act = jp.clip(jax.random.normal(jax.random.PRNGKey(1), (sys_b.act_size(),)) * 0.8, -1, 1)

    def row(s):
        return np.concatenate([np.asarray(s.x_i.pos), np.asarray(s.x_i.rot), np.asarray(s.xd_i.ang), np.asarray(s.xd_i.vel)], axis=-1)
    states = [row(st)]
    for _ in range(substeps):
        st = bpipe.step(sys_b, st, act)
        states.append(row(st))
    # (4) pushT on the generalized backend (envs/pushT.py:16-20): q, qd after every env step of a scripted push
    extra = {}
    try:
        from brax.generalized import pipeline as gpipe
        sys_g = bmjcf.load(os.path.join(ref_assets, "pushT.xml"))
        q0 = np.zeros(8, np.float32); q0[:2] = [-0.21, 0.0]; q0[5:] = [-0.4, 0.4, np.pi]
        acts = np.float32([[1.0, 0.0]] * 4 + [[0.3, 0.8]] * 4 + [[-0.5, 0.2]] * 4)
        sg = gpipe.init(sys_g, jp.asarray(q0), jp.zeros(8))
        traj = []
        for a in acts:
            for _ in range(5):                                 # n_frames = 5
                sg = gpipe.step(sys_g, sg, jp.asarray(a))
            traj.append(np.concatenate([np.asarray(sg.q), np.asarray(sg.qd)]))
        extra = dict(pusht_q0=q0, pusht_actions=acts, pusht_traj=np.float32(traj))
    except Exception as e:  # noqa: BLE001
        print(f"pushT section skipped: {e}")
    k0 = jax.random.PRNGKey(0)
    np.savez(path, **extra, states=np.float32(states), action=np.float32(act), mass=np.asarray(sys_b.link.inertia.mass),
             com=np.asarray(sys_b.link.inertia.transform.pos), init_q=np.asarray(sys_b.init_q),
             split_key0=np.asarray(jax.random.split(k0)), normal_key0=np.asarray(jax.random.normal(k0, (8,))),
             uniform_key0=np.asarray(jax.random.uniform(k0, (8,))),
             versions=np.array([jax.__version__, __import__("brax").__version__]))
    print(f"wrote {path}: {len(states)} states of {states[0].shape}, jax {jax.__version__}, brax {__import__('brax').__version__}")
    return 0


def self_test():
    """a dump produced by a NON-default variant of the oracle must be identified as exactly that variant"""
    import mbd_b200
    from mbd_b200 import prng
    env = mbd_b200.envs.get_env("humanoidrun")
    q = env.sys.init_q.astype(np.float32); q[2] = 1.25   # feet on the floor: the contact switches matter
    st0 = env.pipeline_init(q, np.zeros(env.sys.qd_size(), np.float32)).raw
    action = np.clip(np.random.default_rng(0).normal(size=17) * 0.8, -1, 1).astype(np.float32)
    truth = {"ORC_SINKING_GATE": 0, "ORC_CONTACT_MIDPOINT": 0}
    with tempfile.TemporaryDirectory() as tmp:
        lib = build_variant(truth, os.path.join(tmp, "truth.so"))
        states = [st0]
        for _ in range(12):
            states.append(step_states(lib, env.blob, np.stack([states[-1]]), action)[0])
        path = os.path.join(tmp, "dump.npz")
        # a pushT trajectory from the oracle itself exercises section (4) of the comparison (difference exactly 0)
        from oracle import oracle as orc
        pt = mbd_b200.envs.get_env("pushT")
        q0 = np.zeros(8, np.float32); q0[:2] = [-0.21, 0.0]; q0[5:] = [-0.4, 0.4, np.pi]
        acts = np.float32([[1.0, 0.0]] * 4 + [[0.3, 0.8]] * 4)
        ptraj = orc.pusht_rollout(pt.params, np.concatenate([q0, np.zeros(8, np.float32)]), acts[None], want_traj=True)["traj"][0]
        np.savez(path, states=np.float32(states), action=action, pusht_q0=q0, pusht_actions=acts, pusht_traj=ptraj)
        SW = dict(SWITCHES)
        for k in list(SWITCHES):
            if k not in ("ORC_SINKING_GATE", "ORC_CONTACT_MIDPOINT", "ORC_TANGENT_EPS_FORM"):
                SWITCHES[k] = SWITCHES[k][:1]          # keep the grid small: 8 builds
        try:
            rows = compare(path)
        finally:
            SWITCHES.update(SW)
    default = {n: SW[n][0] for n in SW}
    err_of = lambda want: [r[0] for r in rows if all(r[1][k] == want.get(k, default[k]) for k in r[1])][0]   # noqa: E731
    ok = err_of(truth) == 0.0 and err_of({}) > 0.0     # the true variant reproduces the dump exactly, the default does not
    print("self-test:", "OK" if ok else f"FAILED (error of the true variant {err_of(truth)}, of the default {err_of({})})")
    return 0 if ok else 1


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--make-dump")
    ap.add_argument("--compare")
    ap.add_argument("--self-test", action="store_true")
    ap.add_argument("--substeps", type=int, default=10)
    ap.add_argument("--ref-assets", default=os.environ.get("MBD_REFERENCE_ASSETS"))
    a = ap.parse_args()
    if a.self_test:
        sys.exit(self_test())
    if a.make_dump:
        sys.exit(make_dump(a.make_dump, a.substeps, a.ref_assets))
    if a.compare:
        compare(a.compare)
        sys.exit(0)
    ap.print_help()
