"""Shard-size sweep of the rollout kernels: every kernel variant at the per-GPU shard sizes of a strong-scaling run
(8192 samples over 8 / 4 / 2 / 1 GPUs) — the data behind the auto-selector in choose_kernel (csrc/mbd_b200.cu).
Each variant is checked bit for bit against variant 2.  --lib loads another build of the library (e.g. an older commit's
libmbd_b200.so) instead of the tree's, so that two builds can be timed in alternating runs on one GPU.
    python scripts/gpu_shard_sweep.py [env] [out.json] [--lib PATH]"""
import argparse, json, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from mbd_b200 import build as b

ap = argparse.ArgumentParser()
ap.add_argument("env", nargs="?", default="humanoidrun")
ap.add_argument("out", nargs="?")
ap.add_argument("--lib", help="path of the libmbd_b200.so to load instead of the tree's build")
args = ap.parse_args()
if args.lib:
    b.OUT = os.path.abspath(args.lib); b.is_stale = lambda: False
import mbd_b200
from mbd_b200 import ops, prng

env = mbd_b200.envs.get_env(args.env)
st = torch.as_tensor(env.reset(prng.split(prng.PRNGKey(0))[1]).pipeline_state.raw, device="cuda:0")
m = ops.Model(env.blob)
key = np.uint32([1, 2]); H = 50; HNu = H * env.action_size
rows = []
for n in (256, 512, 1024, 2048, 4096, 8192):
    Y0s = torch.empty((n, HNu), device="cuda:0"); rews = torch.empty(n, device="cuda:0"); Yb = torch.zeros(HNu, device="cuda:0")
    ops.set_kernel_variant(2)
    ops.sample_rollout(m, st, key, n, 0, n, H, 0.88, Yb, Y0s, rews); torch.cuda.synchronize()
    ref = rews.cpu().numpy().copy()
    for v in (0, 1, 2, 3, 8):
        ops.set_kernel_variant(v)
        for _ in range(2): ops.sample_rollout(m, st, key, n, 0, n, H, 0.88, Yb, Y0s, rews)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20): ops.sample_rollout(m, st, key, n, 0, n, H, 0.88, Yb, Y0s, rews)
        e1.record(); torch.cuda.synchronize()
        rows.append(dict(env=args.env, n=n, variant=v, ms=e0.elapsed_time(e1) / 20, bit_identical=bool(np.array_equal(rews.cpu().numpy(), ref))))
        print(rows[-1], flush=True)
ops.set_kernel_variant(0)
if args.out:
    json.dump(rows, open(args.out, "w"), indent=1)
