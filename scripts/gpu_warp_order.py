"""Sensitivity of the v2 kernel to the slot -> link order (the SM arbiter issues the highest eligible warp id first)."""
import ctypes, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import mbd_b200
from mbd_b200 import ops, prng, _lib
env = mbd_b200.envs.get_env("humanoidrun")
rng, rr = prng.split(prng.PRNGKey(0))
st = torch.as_tensor(env.reset(rr).pipeline_state.raw, device="cuda:0")
key = np.uint32([1, 2]); n = 8192
Y0s = torch.empty((n, 850), device="cuda:0"); rews = torch.empty(n, device="cuda:0"); Yb = torch.zeros(850, device="cuda:0")
# links: 0 torso 1 lwaist 2 pelvis 3 rthigh 4 rshin 5 lthigh 6 lshin 7 ruarm 8 rlarm 9 luarm 10 llarm
ORDERS = {
    "default": None,
    "shins-top": [0, 8, 10, 7, 9, 1, 2, 3, 5, 4, 6],
    "thighs-top": [0, 8, 10, 7, 9, 1, 2, 4, 6, 3, 5],
    "reversed(critical lowest)": [4, 6, 3, 5, 2, 1, 9, 7, 10, 8, 0],
    "heavy-joints-top": [0, 8, 10, 2, 4, 6, 1, 7, 9, 3, 5],
    "legs-chain-top": [0, 8, 10, 7, 9, 1, 2, 5, 3, 6, 4],
    "link-order": list(range(11)),
}
ref = None
for name, order in ORDERS.items():
    m = ops.Model(env.blob)
    if order is not None:
        arr = (ctypes.c_int * 11)(*order)
        _lib.check(_lib.lib().mbd_model_set_warp_order(m.handle, arr, 11), "set order")
    for v in (8, 2):
        ops.set_kernel_variant(v)
        for _ in range(2): ops.sample_rollout(m, st, key, n, 0, n, 50, 0.88, Yb, Y0s, rews)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5): ops.sample_rollout(m, st, key, n, 0, n, 50, 0.88, Yb, Y0s, rews)
        e1.record(); torch.cuda.synchronize()
        r = rews.cpu().numpy(); ref = r if ref is None else ref
        print(f"{name:28s} variant={v}: {e0.elapsed_time(e1)/5:.3f} ms same={np.array_equal(r, ref)}")
