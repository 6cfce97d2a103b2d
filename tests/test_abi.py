"""The C-ABI library loads on a CPU-only box, exports every symbol include/mbd_b200.h declares,
agrees with the Python blob layout, and fails loudly (no CPU fallback) without a GPU."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from mbd_b200 import _lib
from mbd_b200.model import blob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions():
    src = open(os.path.join(ROOT, "include", "mbd_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mbd_[a-z0-9_]+)\s*\(", src)))


def test_exports_every_declared_symbol():
    L = _lib.lib()
    names = _declared_functions()
    assert len(names) >= 12
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/mbd_b200.h but not exported"
    assert sorted(_lib.EXPORTS) == names


def test_kernel_variant_accepts_only_the_kept_kernels():
    """mbd_set_kernel_variant takes auto (0) and the variants 1, 2, 3 and 8; every other value is MBD_EINVAL"""
    L = _lib.lib()
    try:
        for v in (0, 1, 2, 3, 8):
            assert L.mbd_set_kernel_variant(v) == 0, v
        for v in (4, 5, 6, 7, 9, 10):
            assert L.mbd_set_kernel_variant(v) == -1, v
    finally:
        L.mbd_set_kernel_variant(0)


def test_layout_matches_python_packer():
    out = np.zeros(64, np.int32)
    n = _lib.lib().mbd_layout_info(out.ctypes.data_as(_lib.c_i32p), 64)
    exp = blob.layout_words()
    assert n == len(exp)
    assert out[:n].tolist() == [int(np.array(v, dtype=np.uint32).view(np.int32)) if i == 0 else v for i, v in enumerate(exp)]


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    assert _lib.lib().mbd_device_count() == 0
    with pytest.raises(_lib.MbdError):
        _lib.require_gpu()
    from mbd_b200 import ops
    b = np.zeros(blob.BLOB_WORDS, np.uint32); b[0] = blob.MAGIC
    h = _lib.lib().mbd_model_create(b.ctypes.data_as(_lib.c_u32p), b.size)
    assert not h and b"no CUDA device" in _lib.lib().mbd_last_error()
    with pytest.raises(_lib.MbdError):
        ops.Model(b)


def test_bad_blob_rejected():
    b = np.zeros(blob.BLOB_WORDS, np.uint32)
    assert not _lib.lib().mbd_model_create(b.ctypes.data_as(_lib.c_u32p), b.size)
    assert not _lib.lib().mbd_model_create(b.ctypes.data_as(_lib.c_u32p), 5)


def test_product_does_not_import_oracle():
    """Only tests/, smoke() and bench.py may touch oracle/ — the package must not."""
    pkg = os.path.join(ROOT, "mbd_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt and "mbd_oracle" not in txt.replace("oracle/mbd_oracle.c", ""), os.path.join(dp, f)


def test_step_structs_match_the_ctypes_mirrors():
    """mbd_step_params / mbd_step_ctl / mbd_step_plan cross the ABI by pointer: sizeof and key offsets of the C structs
    (mbd_abi_sizes) equal those of the ctypes mirrors in mbd_b200/_lib.py"""
    import ctypes
    out = np.zeros(16, np.int32)
    n = _lib.lib().mbd_abi_sizes(out.ctypes.data_as(_lib.c_i32p), 16)
    P = _lib.StepPlan
    exp = [ctypes.sizeof(_lib.StepParams), 4 * _lib.STEP_CTL_WORDS, ctypes.sizeof(P), P.n_total.offset, P.xref_dev.offset, P.Y0s_dev.offset,
           P.P.offset, P.peer_base_ptrs.offset, P.timeout_cycles.offset, 16]
    assert n == len(exp) and out[:n].tolist() == exp
    assert ctypes.sizeof(_lib.StepParams) == 4 * _lib.STEP_PARAMS_WORDS == 32
