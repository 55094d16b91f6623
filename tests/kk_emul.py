"""The CPU replay of kk_convert_kernel (tests/emul/kk_dequant_emul.cpp, kk_emul_launch) as the emulator tests drive it: the library, the
segment table entry it takes, its failure codes, destination pools with their hit counters and store masks, and `launch` — one staged
chunk played with a few segments."""
import ctypes as C
import os
import subprocess

import numpy as np

from tests import helpers

_HERE = os.path.dirname(os.path.abspath(__file__))
LAUNCH_MULTIMEM = 0x2  # ConvertLaunch::flags (csrc/kk_ops.h): NVLS stores, so aligned copies take the consumers' register path
ERR = {1: "shared load outside the staged payload", 2: "misaligned shared load", 3: "store outside the pool / misaligned", 4: "pool bytes stored twice",
       6: "stage store misaligned or outside the stage", 7: "too many shuffles / votes per lane", 8: "codebook index out of range",
       9: "tile_begin[] not monotone", 10: "bulk copy violates 16-byte alignment / size / stage capacity", 11: "bulk copy reads outside the staged chunk",
       12: "bytes issued != bytes announced to the mbarrier", 13: "bulk store misaligned or outside the pool",
       14: "row-split bulk piece: destination, stage offset or length not 16-byte aligned", 15: "row-split store outside the destination pool",
       16: "row-split store reads outside the staged bytes", 17: "row-split store to a rank without a pool", 18: "row-split tile with zero row or slice bytes",
       19: "tile payload runs past the staged chunk", -1: "bad destination pool count"}


class KKSeg(C.Structure):
    _fields_ = [("src_off", C.c_uint64), ("dst_off", C.c_uint64), ("units", C.c_uint64), ("op", C.c_uint32), ("tile_begin", C.c_uint32),
                ("p0", C.c_uint32), ("p1", C.c_uint32), ("p2", C.c_uint32), ("p3", C.c_uint32)]


NO_EXCHANGE = (None, 0, None, None, None)


def load():
    """Build (make -C tests/emul) and load the replay library; KK_EMUL_LIB points at another build of it (A/B variants)."""
    subprocess.run(["make", "-C", os.path.join(_HERE, "emul"), "-s"], check=True)
    L = C.CDLL(os.environ.get("KK_EMUL_LIB") or os.path.join(_HERE, "emul", "_build", "libkk_dequant_emul.so"))
    L.kk_emul_launch.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(KKSeg), C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p), C.c_uint32, C.c_uint64,
                                 C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.POINTER(C.c_void_p), C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                 C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.kk_emul_launch.restype = C.c_int
    L.kk_emul_block_geom.argtypes = [C.c_uint32] + [C.POINTER(C.c_uint32)] * 3
    L.kk_emul_block_geom.restype = None
    assert C.sizeof(KKSeg) == 48
    return L


class Pools:
    """n destination pools of nbytes, filled with 0xCD, and pool 0's 16-byte hit counters and 2-byte / 1-byte store masks."""
    def __init__(self, n, nbytes):
        self.bufs = [np.full(nbytes, 0xCD, np.uint8) for _ in range(n)]
        self.hits = np.zeros((nbytes + 15) // 16, np.uint8)
        self.m2 = np.zeros(nbytes // 2 + 1, np.uint8)
        self.m1 = np.zeros(nbytes + 1, np.uint8)
        self.ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in self.bufs])


def seg_tiles(seg):
    """Tiles of one segment (csrc/kk_ops.h kk_seg_tiles)."""
    if seg.op in helpers.BLOCK_GEOM:
        return -(-seg.units // helpers.BLOCK_GEOM[seg.op][2])
    if helpers.OP_T_F32_BF16 <= seg.op <= helpers.OP_T_B32:
        es = 4 if seg.op in (helpers.OP_T_F32_BF16, helpers.OP_T_B32) else 2
        return -(-seg.units // 8) * -(-seg.p0 // helpers.t_width(seg.p0, es))
    return -(-seg.units // {helpers.OP_F32: 8192, helpers.OP_F16: 16384}.get(seg.op, 32768))


def launch(L, chunk, segs, pool_bytes, flags=0, src_bytes=None):
    """One launch over the staged chunk `chunk` (uint8; the launch sees its first src_bytes, all of it by default) with the segments `segs`
    (KKSeg; tile_begin is filled in here, each segment's tiles following the previous one's) into one pool of pool_bytes.
    Returns (failure code, Pools, stats: shared-memory wavefronts, their ideal, 16-byte store instructions, lines, sectors)."""
    begin = 0
    for s in segs:
        s.tile_begin = begin
        begin += seg_tiles(s)
    pools = Pools(1, pool_bytes)
    stats = (C.c_uint64 * 5)()
    rc = L.kk_emul_launch(chunk.ctypes.data, chunk.size if src_bytes is None else src_bytes, (KKSeg * len(segs))(*segs), len(segs), begin, flags,
                          pools.ptrs, 1, pool_bytes, pools.hits.ctypes.data, pools.m2.ctypes.data, pools.m1.ctypes.data, *NO_EXCHANGE, None, stats)
    return rc, pools, list(stats)
