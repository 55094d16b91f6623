"""LoRA adapters on a resident base (kk_derive_adapter), CPU tier: the out-of-place launch of the merge kernel, replayed on the CPU through
the kernel's header (kk_lora_emul_launch_oop, tests/emul/kk_lora_emul_oop.cpp), over the cases of test_lora.py.  The targets of dst are
the C oracle's merge of src, src is left as it was, dst holds its poison everywhere else, and src == dst gives the bytes of the in-place
launch of kk_load_adapter (tests/emul/kk_lora_emul.cpp)."""
import ctypes as C
import os
import shutil

import numpy as np
import pytest

from kukeon_b200 import gpupool
from tests import lora_fixtures as lf
from tests.test_lora import CASES, _case


_oop_lib = []


def _oop_emul() -> C.CDLL:
    """tests/emul/kk_lora_emul_oop.cpp, built on first use as lora_fixtures builds the in-place replay."""
    if not _oop_lib:
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
        src = os.path.join(lf._EMUL, "kk_lora_emul_oop.cpp")
        deps = [src, os.path.join(lf._CSRC, "kk_lora.cuh"), os.path.join(lf._CSRC, "kk_ops.h")]
        L = C.CDLL(lf._build(src, "libkk_lora_emul_oop.so", cxx, deps, ["-std=c++17", "-x", "c++"]))
        L.kk_lora_emul_launch_oop.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.kk_lora_emul_launch_oop.restype = C.c_int
        _oop_lib.append(L)
    return _oop_lib[0]


def _oop(src: np.ndarray, dst: np.ndarray, targets) -> None:
    L = _oop_emul()
    tab, ad, tiles = lf.target_table(targets)
    assert L.kk_lora_emul_launch_oop(lf._ptr(tab), len(tab), tiles, lf._ptr(ad), lf._ptr(src), lf._ptr(dst)) == 0


def _inside(targets, n: int) -> np.ndarray:
    m = np.zeros(n, bool)
    for t in targets:
        m[t["w_off"]:t["w_off"] + t["rows"] * t["cols"] * (4 if t["out"] == "F32" else 2)] = True
    return m


@pytest.mark.parametrize("case", sorted(CASES))
def test_out_of_place_replay_equals_c_oracle_of_src(case):
    rng = np.random.default_rng(sorted(CASES).index(case) + 40)
    src, targets = _case(rng, CASES[case])
    poison = np.random.default_rng(1000 + sorted(CASES).index(case)).integers(0, 256, src.size, dtype=np.uint8)
    src0, dst = src.copy(), poison.copy()
    _oop(src, dst, targets)
    assert np.array_equal(src, src0), "the launch wrote into its source pool"
    exp = src0.copy()
    for t in targets:
        lf.oracle_merge(exp, t["w_off"], t["rows"], t["cols"], t["row0"], t["col0"], t["a"], t["b"], t["s"], t["out"])
    inside = _inside(targets, src.size)
    diff = np.flatnonzero(dst[inside] != exp[inside])
    assert diff.size == 0, f"{diff.size} target bytes differ from the oracle's merge of src"
    assert np.array_equal(dst[~inside], poison[~inside]), "the launch wrote outside the targets of dst"


@pytest.mark.parametrize("case", sorted(CASES))
def test_out_of_place_with_src_equal_dst_is_the_in_place_launch(case):
    rng = np.random.default_rng(sorted(CASES).index(case) + 40)
    pool, targets = _case(rng, CASES[case])
    in_place, same = pool.copy(), pool.copy()
    lf.emul_merge(in_place, targets)
    _oop(same, same, targets)
    assert np.array_equal(same, in_place)
    assert not np.array_equal(same, pool)


def test_derive_refuses_null_arguments_without_a_device(native):
    h = C.c_void_p()
    assert native.kk_derive_adapter(None, b"/nonexistent", C.byref(h)) == -1  # KK_EINVAL
    assert native.kk_derive_adapter(None, None, C.byref(h)) == -1
    assert h.value is None
    assert "kk_derive_adapter" in gpupool.ABI_SYMBOLS
