"""Times the rollout-kernel variants at the headline size and checks they agree bit for bit."""
import os, sys
import numpy as np, torch
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import mbd_b200
from mbd_b200 import ops, prng
env = mbd_b200.envs.get_env("humanoidrun")
rng, rr = prng.split(prng.PRNGKey(0))
st = torch.as_tensor(env.reset(rr).pipeline_state.raw, device="cuda:0")
m = env.device_model()
key = np.uint32([1, 2])
res = {}
for n in (8192, 1024, 2048, 4096, 65536):
    H = 50
    Y0s = torch.empty((n, 850), device="cuda:0"); rews = torch.empty(n, device="cuda:0"); Yb = torch.zeros(850, device="cuda:0")
    for v in (1, 2, 3, 8):
        ops.set_kernel_variant(v)
        for _ in range(2):
            ops.sample_rollout(m, st, key, n, 0, n, H, 0.88, Yb, Y0s, rews)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            ops.sample_rollout(m, st, key, n, 0, n, H, 0.88, Yb, Y0s, rews)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 5
        res[(n, v)] = rews.cpu().numpy().copy()
        print(f"n={n} variant={v}: {ms:.3f} ms  {n*H/ms*1e3/1e6:.1f} M env-steps/s  same_as_v1={np.array_equal(res[(n,1)].view(np.uint32), res[(n,v)].view(np.uint32))}")
