"""The packed-kernel physics (mbd_b200/csrc/xpbd_pk.cuh), compiled for the host, against the CPU oracle — bit for bit.

The sm_90a kernel k_rollout_pk instantiates the same templated phase functions with T = f2 (two samples per thread, every
operation issued on both).  Here they are built with g++ for T = float and for the {float, float} emulation of f2 and driven link
by link, phase by phase (tests/host_pk/pk_harness.cpp).  What this pins without a GPU: the translation of every physics
expression into the scalar layer, the phase split, the two-sample data flow."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import mbd_b200
from oracle import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_f32p = ctypes.POINTER(ctypes.c_float)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pk") / "libpk_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-mfma", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "include"),
                    "-I" + os.path.join(ROOT, "mbd_b200", "csrc"), os.path.join(ROOT, "tests", "host_pk", "pk_harness.cpp"), "-o", so],
                   check=True, env={**os.environ, "CC": "", "CXX": ""})
    return ctypes.CDLL(so)


def _run(lib, blob, state, Y0s, packed, nsub=0):
    blob = np.ascontiguousarray(blob, dtype=np.uint32)
    L = int(blob.view(np.int32)[1])
    state = np.ascontiguousarray(state, dtype=np.float32).reshape(L, 13)
    Y0s = np.ascontiguousarray(Y0s, dtype=np.float32)
    n, H, _ = Y0s.shape
    rews = np.zeros(n, np.float32)
    final = np.zeros((n, L, 13), np.float32)
    rc = lib.pk_host_rollout(blob.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), state.ctypes.data_as(_f32p), Y0s.ctypes.data_as(_f32p),
                             n, H, packed, nsub, rews.ctypes.data_as(_f32p), final.ctypes.data_as(_f32p))
    assert rc == 0
    return rews, final


def _case(env_name, n, H, seed, scale=0.88):
    env = mbd_b200.envs.get_env(env_name)
    rng = np.random.default_rng(seed)
    state = env.reset(mbd_b200.prng.PRNGKey(seed)).pipeline_state.raw
    Y0s = np.clip(rng.normal(size=(n, H, env.action_size)) * scale, -1, 1).astype(np.float32)
    return env, state, Y0s


@pytest.mark.parametrize("env_name,n,H", [("humanoidrun", 7, 12), ("humanoidstandup", 5, 8), ("humanoidtrack", 4, 10)])
@pytest.mark.parametrize("packed", [0, 1], ids=["float", "f2"])
def test_phases_match_oracle_bit_exact(harness, env_name, n, H, packed):
    env, state, Y0s = _case(env_name, n, H, seed=3)
    ref = orc.xpbd_rollout(env.blob, state, Y0s, want_final=True)
    rews, final = _run(harness, env.blob, state, Y0s, packed)
    assert np.array_equal(final.view(np.uint32), ref["final"].view(np.uint32))
    if env_name != "humanoidtrack":  # its reward is taken before the step; the harness only implements post-step rewards
        assert np.array_equal(rews.view(np.uint32), ref["rews"].view(np.uint32))


def test_two_sample_type_with_contacts_and_saturated_actions(harness):
    env, state, Y0s = _case("humanoidrun", 6, 40, seed=11, scale=3.0)   # long enough for falls and foot contacts
    Y0s[1] = 0.0
    ref = orc.xpbd_rollout(env.blob, state, Y0s, want_final=True)
    for packed in (0, 1):
        rews, final = _run(harness, env.blob, state, Y0s, packed)
        assert np.array_equal(final.view(np.uint32), ref["final"].view(np.uint32))
        assert np.array_equal(rews.view(np.uint32), ref["rews"].view(np.uint32))


def test_no_packed_contraction(tmp_path):
    """a multiply that ptxas fused into a following add would change rounding where the arithmetic contract has a
    separate multiply and add.  The physics routes every such sum through add_nf / sub_nf (pk_scalar.cuh) and is built
    with -fmad=false; here every multiply of the PTX of the two-sample phases must survive into the SASS as an FMUL,
    and the SASS may hold no FFMA the PTX did not ask for."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not (os.path.exists(nvcc) and os.path.exists(cuobjdump)):
        pytest.skip("CUDA toolkit not available")
    src = os.path.join(ROOT, "tests", "host_pk", "pk_device_probe.cu")
    flags = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false", "-I" + os.path.join(ROOT, "include"),
             "-I" + os.path.join(ROOT, "mbd_b200", "csrc")]
    ptx, cubin = str(tmp_path / "probe.ptx"), str(tmp_path / "probe.cubin")
    subprocess.run([nvcc] + flags + ["-ptx", src, "-o", ptx], check=True, capture_output=True)
    subprocess.run([nvcc] + flags + ["-cubin", src, "-o", cubin], check=True, capture_output=True)
    text = open(ptx).read()
    n_mul = text.count("mul.rn.f32 ")
    n_fma = text.count("fma.rn.f32 ")
    sass = subprocess.run([cuobjdump, "-sass", cubin], check=True, capture_output=True, text=True).stdout
    n_fmul, n_ffma = len(re.findall(r"\bFMUL\b", sass)), len(re.findall(r"\bFFMA\b", sass))
    assert n_mul > 1000 and n_fma > 1000
    assert n_fmul == n_mul, f"{n_mul - n_fmul} products were contracted into FFMA"
    assert n_ffma <= n_fma


def test_algorithmic_operation_count(harness):
    """SURVEY 8d: the flops of one XPBD substep, counted by running the physics with an operation-counting scalar type
    (DESIGN.md section 4 quotes these numbers; the SASS-level count of the kernel is ~15 % higher because division,
    reciprocal and square root expand into a MUFU seed plus Newton FMAs on the device)."""
    env, state, Y0s = _case("humanoidrun", 1, 50, seed=1)
    blob = np.ascontiguousarray(env.blob, dtype=np.uint32)
    st = np.ascontiguousarray(state, dtype=np.float32).reshape(11, 13)
    ops = (ctypes.c_ulonglong * 9)()
    rews = np.zeros(1, np.float32)
    harness.pk_host_count_ops(blob.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), st.ctypes.data_as(_f32p), Y0s.ctypes.data_as(_f32p),
                              50, 0, ops, rews.ctypes.data_as(_f32p))
    ref = orc.xpbd_rollout(env.blob, state, Y0s)
    assert rews[0] == ref["rews"][0]                      # the counting type computes the same rollout
    mul, add, fma, div, rcp, sqrt = [ops[i] / (50 * 7) for i in range(6)]
    flop = mul + add + 2 * fma + div + rcp + sqrt
    assert 9000 < flop < 9700                             # 9.34 kFLOP per sample and substep (2296 mul, 799 add, 3024 fma)
    assert 190 <= div + rcp + sqrt <= 200                 # 64 div + 62 rcp + 68 sqrt: the contact-free part is data independent


def test_simd_cpu_arm_matches_the_scalar_oracle():
    """oracle/mbd_oracle_simd.cpp (bench.py's timed CPU arm: the same templated physics on a 16-lane host type, OpenMP over lane
    groups) gives the scalar C oracle's returns and final states bit for bit, ragged tail group included"""
    if orc.use_simd() is None:
        pytest.skip("the SIMD arm does not build on this host")
    for env_name, n, H in (("humanoidrun", 37, 9), ("humanoidstandup", 19, 6)):
        env, state, Y0s = _case(env_name, n, H, seed=5)
        ref = orc.xpbd_rollout(env.blob, state, Y0s, want_final=True)
        out = orc.simd_rollout(env.blob, state, Y0s, want_final=True, nthreads=3)
        assert out is not None
        assert np.array_equal(out["rews"].view(np.uint32), ref["rews"].view(np.uint32))
        assert np.array_equal(out["final"].view(np.uint32), ref["final"].view(np.uint32))
    hop = mbd_b200.envs.get_env("hopper")   # slide dofs / other rewards are not covered: the caller falls back to the scalar oracle
    assert orc.simd_rollout(hop.blob, hop.pipeline_init(hop.sys.init_q, np.zeros(6)).raw, np.zeros((4, 2, 3), np.float32)) is None


def test_no_packed_contraction_in_the_product_kernels():
    """the same check on the product kernels themselves (scripts/check_pk_contraction.py compiles csrc/mbd_b200.cu to PTX and SASS):
    no multiply of any k_rollout_pk instantiation disappears into an FFMA."""
    import shutil, sys
    if not shutil.which("nvcc"):
        pytest.skip("CUDA toolkit not available")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "check_pk_contraction.py")], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert r.stdout.count(" ok") >= 3   # fused, non-fused and batched instantiations
