"""Speed probe only (NOT bit-exact): the same kernels compiled with approximate div/sqrt, to size the
cost of the IEEE division / sqrt slow-path branches that split the instruction stream."""
import os, sys
import numpy as np, torch
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from mbd_b200 import build as b
if len(sys.argv) > 1:
    b.OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), sys.argv[1]); b.is_stale = lambda: False
import mbd_b200
from mbd_b200 import ops, prng
env = mbd_b200.envs.get_env("humanoidrun")
rng, rr = prng.split(prng.PRNGKey(0))
st = torch.as_tensor(env.reset(rr).pipeline_state.raw, device="cuda:0")
m = env.device_model(); key = np.uint32([1, 2])
for n in (8192, 4096):
    Y0s = torch.empty((n, 850), device="cuda:0"); rews = torch.empty(n, device="cuda:0"); Yb = torch.zeros(850, device="cuda:0")
    ref = None
    for v in (2, 3):
        ops.set_kernel_variant(v)
        for _ in range(2): ops.sample_rollout(m, st, key, n, 0, n, 50, 0.88, Yb, Y0s, rews)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5): ops.sample_rollout(m, st, key, n, 0, n, 50, 0.88, Yb, Y0s, rews)
        e1.record(); torch.cuda.synchronize()
        r = rews.cpu().numpy(); ref = r if ref is None else ref
        print(f"{sys.argv[1] if len(sys.argv)>1 else 'exact'} n={n} variant={v}: {e0.elapsed_time(e1)/5:.3f} ms  rew mean {rews.mean().item():.4f} same={np.array_equal(r, ref)}")
