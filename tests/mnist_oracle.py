"""ctypes front end of tests/mnist_oracle.c, the CPU restatement of the forward kernel after layer 1 (TEST INFRASTRUCTURE).

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


def lib():
    global _LIB
    if _LIB is None:
        tmp = tempfile.mkdtemp(prefix="mnist_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libmnist_oracle.so")
        cc = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"
        subprocess.run([cc, "-O2", "-std=gnu11", "-fPIC", "-shared", "-fvisibility=hidden", "-ffp-contract=off", "-fno-fast-math",
                        "-mfma", "-I" + os.path.join(_ROOT, "include"), "-o", so, os.path.join(_HERE, "mnist_oracle.c"), "-lm"],
                       check=True, capture_output=True)
        L = ctypes.CDLL(so)
        fp = ctypes.POINTER(ctypes.c_float)
        L.mnist_js.argtypes = [fp, fp, ctypes.POINTER(ctypes.c_uint8), ctypes.c_int, ctypes.c_int, fp]
        _LIB = L
    return _LIB


def js_from_z1(rows, z1, labels) -> np.ndarray:
    """Js [n] of parameter rows [n, 26506] from the layer-1 pre-activations z1 [n, M, 32] and the M labels, in the device's order"""
    rows = np.ascontiguousarray(rows, np.float32)
    z1 = np.ascontiguousarray(z1, np.float32)
    lab = np.ascontiguousarray(labels, np.uint8)
    n, M = z1.shape[0], z1.shape[1]
    assert rows.shape[0] == n and lab.shape[0] == M
    out = np.zeros(n, np.float32)
    fp = ctypes.POINTER(ctypes.c_float)
    lib().mnist_js(rows.ctypes.data_as(fp), z1.ctypes.data_as(fp), lab.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), n, M,
                   out.ctypes.data_as(fp))
    return out
