"""The C-ABI library loads on a CPU-only box, exports every symbol include/mbd_b200.h declares and fails loudly (no CPU
fallback) without a GPU; the ctypes and integer mirrors of the C headers agree with them (compiled with g++, no library)."""
import ctypes
import os
import re
import subprocess

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


# ---- the ctypes and integer mirrors against the C headers, at compile time ---------------------------------------------------
HEADERS = ("mbd_b200.h", "mbd_model.h", "mbd_kin64.h", "mbd_sac_learn.h")   # mbd_sac_learn.h includes mbd_sac.h
# the structs of mbd_b200.h that Python does not mirror
UNMIRRORED = {"mbd_model": "opaque: Python holds a pointer to it",
              "mbd_step_ctl": "the engines allocate it as STEP_CTL_WORDS int32 words"}
# the constants whose C counterpart is not MBD_<NAME>
C_NAME = {"MAGIC": "MBD_MODEL_MAGIC",
          "STEP_PARAMS_WORDS": "sizeof(mbd_step_params) / 4",   # the engines allocate parameter rows as int32 words
          "STEP_CTL_WORDS": "sizeof(mbd_step_ctl) / 4"}         # and the control block
UNCHECKED = {"PI_TOPK": "kCemTop, which lives in the device-only csrc/step_tail.cuh"}
# the dicts of _lib, each entry checked against MBD_<prefix><KEY>
DICTS = {"VEC_OBS": "VEC_OBS_", "VEC_RESET": "VEC_RESET_", "BBO_FNS": "BBO_", "PI_METHODS": "PI_"}
KINDS = ("FLOAT", "SIGNED", "UNSIGNED", "POINTER")
_KIND = {**dict.fromkeys("fd", "FLOAT"), **dict.fromkeys("bhilq", "SIGNED"), **dict.fromkeys("BHILQ", "UNSIGNED")}


def mirrors():
    return [v for v in vars(_lib).values() if isinstance(v, type) and issubclass(v, ctypes.Structure)]


def constants():
    """[(item, C expression, value)] for every public int constant of _lib and blob and every entry of the dicts"""
    out = []
    for mod, tag in ((_lib, "_lib"), (blob, "blob")):
        for name, v in vars(mod).items():
            if not name.startswith("_") and type(v) is int and name not in UNCHECKED:
                out.append((f"{tag}.{name}", C_NAME.get(name, "MBD_" + name), v))
    for d, prefix in DICTS.items():
        out += [(f"_lib.{d}['{k}']", "MBD_" + prefix + k.upper().replace("-", ""), v) for k, v in getattr(_lib, d).items()]
    return out


def _kind(t):
    """the kind of a field's ctypes type (an array's by its element): FLOAT, SIGNED, UNSIGNED, POINTER or a mirror's C name"""
    while issubclass(t, ctypes.Array):
        t = t._type_
    if issubclass(t, ctypes.Structure):
        return t._c_name_
    return "POINTER" if issubclass(t, (ctypes._Pointer, ctypes.c_void_p)) else _KIND[t._type_]


def abi_source(structs, consts):
    """C++17 that compiles only if every struct and constant agrees with the headers; each line names the item it checks"""
    lines = ["#include <cstddef>", "#include <type_traits>"] + [f'#include "{h}"' for h in HEADERS] + [
        "enum kind { FLOAT, SIGNED, UNSIGNED, POINTER, STRUCT };",
        "template <class M> constexpr kind kind_of() {",
        "  using E = std::remove_cv_t<std::remove_all_extents_t<M>>;",
        "  return std::is_floating_point_v<E> ? FLOAT : std::is_pointer_v<E> ? POINTER : std::is_class_v<E> ? STRUCT",
        "       : std::is_signed_v<E> ? SIGNED : UNSIGNED;",
        "}",
        'static_assert(offsetof(mbd_step_ctl, ticket) == 16, "mbd_step_ctl.ticket: offset");']
    for cls in structs:
        S = cls._c_name_
        for name, t in cls._fields_:
            f, k, m = getattr(cls, name), _kind(t), f"decltype({S}::{name})"
            kind = f"kind_of<{m}>() == {k}" if k in KINDS else f"std::is_same_v<std::remove_all_extents_t<{m}>, {k}>"
            lines += [f'static_assert(offsetof({S}, {name}) == {f.offset}, "{S}.{name}: offset");',
                      f'static_assert(sizeof({S}::{name}) == {f.size}, "{S}.{name}: size");',
                      f'static_assert({kind}, "{S}.{name}: kind");']
        lines += [f'static_assert(sizeof({S}) == {ctypes.sizeof(cls)}, "{S}: size");',
                  # a structured binding needs one name per member: a mirror that misses one, even into padding, fails here
                  f"[[maybe_unused]] static void {S}_members({S}& s) {{ [[maybe_unused]] auto& [{', '.join(n for n, _ in cls._fields_)}] = s; }}"]
    lines += [f'static_assert({c} == {v}, "{item}");' for item, c, v in consts]
    return "\n".join(lines) + "\n"


def compile_abi(src, tmp_path):
    path = tmp_path / "abi_check.cpp"
    path.write_text(src)
    return subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(path)],
                          capture_output=True, text=True)


def test_mirrors_match_the_c_headers(tmp_path):
    """every field of every ctypes mirror in _lib (offset, size, kind), every mirror's size and member count, and every int constant
    of _lib and blob agree with the C headers; the library is not loaded"""
    structs = mirrors()
    unnamed = [c.__name__ for c in structs if not hasattr(c, "_c_name_")]
    assert not unnamed, f"ctypes mirrors without a C name (_c_name_): {unnamed}"
    src = open(os.path.join(ROOT, "include", "mbd_b200.h")).read()
    declared = set(re.findall(r"typedef struct (mbd_\w+)", src))
    assert declared == {c._c_name_ for c in structs} | set(UNMIRRORED)
    consts = constants()
    res = compile_abi(abi_source(structs, consts), tmp_path)
    assert res.returncode == 0, res.stderr
    ndict = sum(len(getattr(_lib, d)) for d in DICTS)
    print(f"{len(structs)} structs, {sum(len(c._fields_) for c in structs)} fields, {len(consts) - ndict} integer constants and "
          f"{ndict} dict values agree; not checked: {', '.join(UNCHECKED)}")


def _edit(cls, edit):
    """a copy of mirror cls with edit applied to its field list"""
    fields = list(cls._fields_)
    edit(fields, [n for n, _ in fields])
    return type(cls.__name__, (ctypes.Structure,), {"_c_name_": cls._c_name_, "_fields_": fields})


def _swap(a, b):
    def edit(f, names):
        i, j = names.index(a), names.index(b)
        f[i], f[j] = f[j], f[i]
    return edit


def _retype(a, t):
    return lambda f, names: f.__setitem__(names.index(a), (a, t))


def _rename(a, new):
    return lambda f, names: f.__setitem__(names.index(a), (new, f[names.index(a)][1]))


@pytest.mark.parametrize("item, cls, edit", [
    ("mbd_vec_plan.nq", _lib.VecPlan, _swap("nq", "nqd")),                                        # two int32 swapped
    ("mbd_ppo_plan.reward_scaling", _lib.PpoPlan, _retype("reward_scaling", ctypes.c_int32)),     # float as int32
    ("mbd_mnist_bufs.n_test", _lib.MnistBufs, _retype("n_test", ctypes.c_float)),                  # int32 as float
    ("mbd_vec_plan.factors", _lib.VecPlan, _rename("factors_dev", "factors")),                    # renamed
    ("mbd_step_plan", _lib.StepPlan, lambda f, names: f.pop()),                                   # last field missing, in padding
    ("mbd_vec_plan", _lib.VecPlan, lambda f, names: f.pop()),                                     # last field missing
    ("mbd_mpc_pi_plan.base", _lib.MpcPiPlan, _retype("base", _lib.EnsDrawPlan)),                  # another struct
    ("blob.D_GEAR", None, None),                                                                  # wrong constant
    ("_lib.VEC_RESET['pusht']", None, None),                                                      # wrong dict entry
])
def test_planted_mistakes_fail_to_compile(item, cls, edit, tmp_path):
    structs = [_edit(c, edit) if c is cls else c for c in mirrors()]
    consts = [(i, c, v + (i == item)) for i, c, v in constants()]   # a planted constant is one too large
    res = compile_abi(abi_source(structs, consts), tmp_path)
    assert res.returncode != 0 and item in res.stderr, res.stderr
