"""Locates the first substep / link / field where the packed kernel (variant 8) leaves the scalar kernel (variant 2)."""
import os, sys
import numpy as np, torch
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import mbd_b200
from mbd_b200 import ops, prng
env = mbd_b200.envs.get_env(sys.argv[1] if len(sys.argv) > 1 else "humanoidrun")
st = env.reset(prng.split(prng.PRNGKey(0))[1]).pipeline_state.raw
m = env.device_model(torch.device("cuda:0"))
Y = np.clip(np.random.default_rng(11).normal(size=(45, 20, 17)) * 0.8, -1, 1).astype(np.float32)
T = lambda a: torch.as_tensor(a, device="cuda:0")
names = env.sys.link_names
F = ["p.x", "p.y", "p.z", "q.w", "q.x", "q.y", "q.z", "w.x", "w.y", "w.z", "v.x", "v.y", "v.z"]
def run(v, H, nsub):
    ops.set_kernel_variant(v)
    o = ops.rollout(m, T(st), T(Y[:, :H]), want_final=True, nsub_override=nsub)
    return o["final"].cpu().numpy()
found = False
for H in range(1, 21):
    for nsub in ([1, 2, 3, 4, 5, 6, 7] if H == 1 else [0]):
        a, b = run(8, H, nsub), run(2, H, nsub)
        d = a.view(np.uint32) != b.view(np.uint32)
        if d.any():
            idx = np.argwhere(d)
            print(f"first difference at H={H} nsub={nsub}: {len(idx)} words; samples {sorted(set(idx[:, 0]))}")
            for (n, l, f) in idx[:12]:
                print(f"  sample {n} link {names[l]} {F[f]}: packed {a[n, l, f]!r} scalar {b[n, l, f]!r}")
            found = True
            break
    if found:
        break
print("no difference" if not found else "done")
