"""Independent restatement of the fp16 output format (KK_LOAD_F16, include/kukeon_gpuload.h) over the oracle.  It shares no code with
the library: the pool layout is oracle.plan_pool of the same load without the flag with the float dtype replaced, and the values are
the oracle's fp32 dequantisers and the cast inputs as fp32, rounded once by numpy's astype(float16) (round to nearest even, overflow to
infinity, fp16 subnormals kept), with every NaN a conversion produces set to the canonical 0x7FFF.  F16 sources stay verbatim.  It sits
here, next to the tests that use it, because oracle/ is the suite's fixed reference and a new feature's rule is added beside it."""
from __future__ import annotations

from typing import List, Tuple

import numpy as np

from oracle import oracle

LOAD_F16 = 0x80
NAN16 = 0x7FFF  # the NaN every conversion stores (cvt.rn.f16x2.f32 and the FP8 pair conversions on an H100)


def f32_bits_to_f16(u32: np.ndarray) -> np.ndarray:
    """fp32 bit patterns -> fp16 bit patterns, RNE; any NaN -> 0x7FFF."""
    x = np.ascontiguousarray(u32, dtype=np.uint32).view(np.float32)
    with np.errstate(all="ignore"):
        h = x.astype(np.float16).view(np.uint16).copy()
    h[np.isnan(x)] = NAN16
    return h


def f32_to_f16(x: np.ndarray) -> np.ndarray:
    return f32_bits_to_f16(np.ascontiguousarray(x, dtype=np.float32).view(np.uint32))


def bf16_bits_to_f16(u16: np.ndarray) -> np.ndarray:
    """bf16 -> fp32 is exact (the bits shifted up), then RNE to fp16: the bf16 range overflows fp16 and bf16's small values become
    fp16 subnormals or zero."""
    return f32_bits_to_f16(np.ascontiguousarray(u16, dtype=np.uint16).astype(np.uint32) << np.uint32(16))


def f8e4m3_bits_to_f16(u8: np.ndarray) -> np.ndarray:
    """OCP E4M3 -> fp16, exact (every E4M3 value, subnormals included, is an fp16 normal); NaN -> 0x7FFF."""
    return bf16_bits_to_f16(oracle.f8e4m3_bits_to_bf16(u8))


def f8e5m2_bits_to_f16(u8: np.ndarray) -> np.ndarray:
    """E5M2 is the top byte of an fp16: the byte shifted up, +-inf kept; NaN -> 0x7FFF."""
    h = np.ascontiguousarray(u8, dtype=np.uint8).astype(np.uint16) << np.uint16(8)
    h[(h & 0x7FFF) > 0x7C00] = NAN16
    return h


def pool_dtype(dt: str, flags: int = 0) -> str:
    d = oracle.pool_dtype(dt, flags & ~LOAD_F16)
    return "F16" if flags & LOAD_F16 and d == "BF16" else d


def plan_pool(recs: List[dict], mode: int = oracle.MODE_SINGLE, flags: int = 0, n_parts: int = 1, part: int = 0) -> Tuple[List[dict], int]:
    """The layout of the same load without KK_LOAD_F16, every bf16 slot an fp16 one."""
    plan, total = oracle.plan_pool(recs, mode, flags & ~LOAD_F16, n_parts, part)
    if flags & LOAD_F16:
        for p in plan:
            if p["dtype"] == "BF16":
                p["dtype"] = "F16"
    return plan, total


def dequant_f16(dtype: str, blocks: np.ndarray) -> np.ndarray:
    """Block-quantised bytes of `dtype` -> fp16 bit patterns [n_blocks, weights per block]: the oracle's fp32, one RNE rounding."""
    nel, nb, fn = oracle.BLOCK_QUANTS[dtype]
    return f32_to_f16(fn(np.ascontiguousarray(blocks, dtype=np.uint8).reshape(-1, nb))).reshape(-1, nel)


def convert_tensor(rec: dict, raw: bytes, flags: int = 0) -> np.ndarray:
    """File bytes of one tensor -> pool bytes under `flags` (before any slicing / transposition)."""
    if not flags & LOAD_F16:
        return oracle.convert_tensor(rec, raw, flags)
    dt = rec["dtype"]
    a = np.frombuffer(raw, dtype=np.uint8)
    if dt == "F32" and not flags & oracle.LOAD_KEEP_F32:
        return f32_bits_to_f16(a.view("<u4")).view(np.uint8)
    if dt == "F16":
        return a.copy()
    if dt == "BF16":
        return bf16_bits_to_f16(a.view("<u2")).view(np.uint8)
    if dt == "F8_E4M3" and flags & oracle.LOAD_F8_TO_BF16:
        return f8e4m3_bits_to_f16(a).view(np.uint8)
    if dt == "F8_E5M2" and flags & oracle.LOAD_F8_TO_BF16:
        return f8e5m2_bits_to_f16(a).view(np.uint8)
    if dt in oracle.BLOCK_QUANTS:
        return dequant_f16(dt, a).reshape(-1).view(np.uint8)
    return oracle.convert_tensor(rec, raw, flags & ~LOAD_F16)


def expected_pool(shards: List[str], recs: List[dict], mode: int = oracle.MODE_SINGLE, flags: int = 0,
                  n_parts: int = 1, part: int = 0) -> Tuple[np.ndarray, List[dict]]:
    """Whole expected pool of one device (gaps zero), as oracle.expected_pool with this module's values."""
    plan, total = plan_pool(recs, mode, flags, n_parts, part)
    pool = np.zeros(total, np.uint8)
    fhs = [open(s, "rb") for s in shards]
    try:
        for r, p in zip(recs, plan):
            fh = fhs[r["shard"]]
            fh.seek(r["file_offset"])
            out = convert_tensor(r, fh.read(r["nbytes"]), flags)
            nel = int(np.prod(r["shape"]))
            es = out.size // nel if nel else 1
            if p["transposed"]:
                R, C = r["shape"]
                out = np.ascontiguousarray(out.reshape(R, C, es).transpose(1, 0, 2)).reshape(-1)
            elif p["slice_dim"] is not None:
                R, C = r["shape"]
                k, b = p["shape"][p["slice_dim"]], p["slice_begin"]
                v = out.reshape(R, C, es)
                out = np.ascontiguousarray(v[b:b + k] if p["slice_dim"] == 0 else v[:, b:b + k]).reshape(-1)
            assert out.size == p["nbytes"], (r["name"], out.size, p["nbytes"])
            pool[p["pool_offset"]: p["pool_offset"] + out.size] = out
    finally:
        for fh in fhs:
            fh.close()
    return pool, plan
