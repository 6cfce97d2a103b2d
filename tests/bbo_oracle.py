"""ctypes front end of tests/bbo_oracle.c, the CPU oracle of the black-box objectives (TEST INFRASTRUCTURE).

The library is compiled on first use into a temporary directory of this process with the CPU oracle's contraction rules
(gcc -O2 -ffp-contract=off -fno-fast-math -mfma, as oracle/Makefile), so the source tree is never written.
"""
from __future__ import annotations

import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_LIB = None

FNS = {"Ackley": 1, "Rastrigin": 2, "Levy": 3}


def lib():
    global _LIB
    if _LIB is None:
        tmp = tempfile.mkdtemp(prefix="bbo_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libbbo_oracle.so")
        cc = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"
        subprocess.run([cc, "-O2", "-std=gnu11", "-fPIC", "-shared", "-fvisibility=hidden", "-ffp-contract=off", "-fno-fast-math",
                        "-mfma", "-I" + os.path.join(_ROOT, "include"), "-o", so, os.path.join(_HERE, "bbo_oracle.c"), "-lm"],
                       check=True, capture_output=True)
        L = ctypes.CDLL(so)
        fp = ctypes.POINTER(ctypes.c_float)
        L.bbo_eval.argtypes = [ctypes.c_int, fp, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, fp]
        _LIB = L
    return _LIB


def bbo_eval(fn, Y0s, x_min: float, x_max: float) -> np.ndarray:
    """J = -f(Y0s[n]) [N] float32 in k_bbo's order; fn is a name of FNS or its MBD_BBO_* value"""
    fn = FNS.get(fn, fn)
    Y = np.ascontiguousarray(Y0s, dtype=np.float32)
    Y = Y.reshape(-1, Y.shape[-1])
    out = np.zeros(Y.shape[0], np.float32)
    fp = ctypes.POINTER(ctypes.c_float)
    rc = lib().bbo_eval(int(fn), Y.ctypes.data_as(fp), Y.shape[0], Y.shape[1], float(x_min), float(x_max), out.ctypes.data_as(fp))
    if rc != 0:
        raise ValueError(f"bbo_eval: unknown fn {fn}")
    return out
