"""Per-phase cycle accounting of the v2 rollout kernel (instrumented build: run `python -m` nothing else needed, it compiles scripts/libmbd_prof.so itself; needs nvcc)."""
import ctypes, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from mbd_b200 import build as b
# instrumented build of the same sources (-DMBD_PROFILE_PHASES), kept apart from the product library
b.OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libmbd_prof.so")
b.NVCC_FLAGS = b.NVCC_FLAGS + ["-DMBD_PROFILE_PHASES"]
if not os.path.exists(b.OUT) or os.environ.get('MBD_PROF_REBUILD'):
    b.build(force=True)
b.is_stale = lambda: False
import mbd_b200
from mbd_b200 import ops, prng, _lib
env = mbd_b200.envs.get_env("humanoidrun")
rng, rr = prng.split(prng.PRNGKey(0))
st = torch.as_tensor(env.reset(rr).pipeline_state.raw, device="cuda:0")
m = env.device_model()
L = _lib.lib()
key = np.uint32([1, 2])
names = env.sys.link_names
for n in (int(os.environ.get("MBD_PROF_N", "8192")),):
    for v in ([int(x) for x in sys.argv[1:]] or [2, 8]):
        ops.set_kernel_variant(v)
        Y0s = torch.empty((n, 850), device="cuda:0"); rews = torch.empty(n, device="cuda:0"); Yb = torch.zeros(850, device="cuda:0")
        ops.sample_rollout(m, st, key, n, 0, n, 50, 0.88, Yb, Y0s, rews); torch.cuda.synchronize()
        L.mbd_prof_reset()
        ops.sample_rollout(m, st, key, n, 0, n, 50, 0.88, Yb, Y0s, rews); torch.cuda.synchronize()
        out = np.zeros((16, 8), np.uint64)
        L.mbd_prof_read(out.ctypes.data_as(ctypes.c_void_p))
        nc = (n + 63) // 64 if v >= 8 else (n + 31) // 32
        per = out[:11].astype(np.float64) / (nc * 350)
        print(f"\n== n={n} variant={v} (cycles per physics step, mean over CTAs) [A, wait, B, wait, C, wait, D, wait] total")
        for l in range(11):
            print(f"{names[l]:16s}", " ".join(f"{x:7.0f}" for x in per[l]), f"  | {per[l].sum():7.0f}")
