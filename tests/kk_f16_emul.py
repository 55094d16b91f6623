"""The CPU replay of the fp16 convert kernel (tests/emul/kk_f16_emul.cpp) as the fp16 tests drive it.

`load()` builds the library next to the bf16 replay's (same compiler and flags as tests/emul/Makefile) when a source is newer than it,
and returns a handle whose `kk_emul_launch` is the fp16 launch walk (kk_emul_launch_f16, same arguments), so that tests/kk_emul.launch
and tests/test_launch_emul.play_part play fp16 launches unchanged; `kk_emul_pack` and `kk_emul_block_geom` are bound as well."""
import ctypes as C
import os
import shutil
import subprocess

from tests import kk_emul

_EMUL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
_CSRC = os.path.join(os.path.dirname(_EMUL), "..", "kukeon_b200", "csrc")
LIB = os.path.join(_EMUL, "_build", "libkk_f16_emul.so")
LAUNCH_F16 = 0x4  # ConvertLaunch::flags (csrc/kk_ops.h KK_LAUNCH_F16)


def _sources():
    return [os.path.join(_EMUL, f) for f in ("kk_f16_emul.cpp", "kk_dequant_emul.cpp")] + \
        [os.path.join(_CSRC, f) for f in os.listdir(_CSRC) if f.endswith((".cuh", ".h"))]


def build() -> str:
    if os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in _sources()):
        return LIB
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    tmp = LIB + f".{os.getpid()}.tmp"
    subprocess.run([cxx, "-O1", "-std=c++17", "-march=x86-64-v2", "-mf16c", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall",
                    "-Wextra", "-Wno-unknown-pragmas", "-x", "c++", "-o", tmp, os.path.join(_EMUL, "kk_f16_emul.cpp")], check=True)
    os.replace(tmp, LIB)
    return LIB


class Replay:
    """The fp16 replay library: kk_emul_launch plays kk_convert_f16_kernel's launch walk."""
    def __init__(self, lib):
        self.lib = lib
        lib.kk_emul_launch_f16.argtypes = kk_emul.load().kk_emul_launch.argtypes
        lib.kk_emul_launch_f16.restype = C.c_int
        lib.kk_emul_pack.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint64]
        lib.kk_emul_pack.restype = C.c_int
        lib.kk_emul_block_geom.argtypes = [C.c_uint32] + [C.POINTER(C.c_uint32)] * 3
        lib.kk_emul_block_geom.restype = None
        self.kk_emul_launch = lib.kk_emul_launch_f16
        self.kk_emul_pack = lib.kk_emul_pack
        self.kk_emul_block_geom = lib.kk_emul_block_geom


def load() -> Replay:
    return Replay(C.CDLL(build()))
