"""Test helpers: small checkpoint builders and a CPU emulator of kk_plan_describe output."""
from __future__ import annotations

import json
import os
import struct
from typing import Dict, List, Sequence, Tuple

import numpy as np

from oracle import oracle

OP_COPY, OP_F32, OP_F16, OP_Q4K, OP_T_F32_BF16, OP_T_F16_BF16, OP_T_B16, OP_T_B32, OP_Q8_0, OP_Q6K, OP_ROWSPLIT = range(11)
OP_Q4_0, OP_Q4_1, OP_Q5_0, OP_Q5_1, OP_Q2K, OP_Q3K, OP_Q5K, OP_F8E4M3, OP_F8E5M2 = range(11, 20)
OP_IQ4NL, OP_IQ4XS, OP_MXFP4 = 23, 24, 25  # 20..22 and 26..28: round 1's candidate transpose geometries (retired, numbers not reused)
OP_IQ2XXS, OP_IQ2XS, OP_IQ2S, OP_IQ3XXS, OP_IQ3S, OP_IQ1S, OP_IQ1M, OP_TQ1_0, OP_TQ2_0, OP_NVFP4 = range(29, 39)
# block-dequantising ops: op -> (source bytes per block, bf16 bytes per block, blocks per tile)   (csrc/kk_ops.h kk_block_geom)
BLOCK_GEOM = {OP_Q4K: (144, 512, 224), OP_Q8_0: (34, 64, 960), OP_Q6K: (210, 512, 152), OP_Q4_0: (18, 64, 1816), OP_Q4_1: (20, 64, 1632),
              OP_Q5_0: (22, 64, 1488), OP_Q5_1: (24, 64, 1360), OP_Q2K: (84, 512, 388), OP_Q3K: (110, 512, 296), OP_Q5K: (176, 512, 186),
              OP_IQ4NL: (18, 64, 1816), OP_IQ4XS: (136, 512, 240), OP_MXFP4: (17, 64, 1920), OP_IQ2XXS: (66, 512, 496), OP_IQ2XS: (74, 512, 440),
              OP_IQ2S: (82, 512, 392), OP_IQ3XXS: (98, 512, 328), OP_IQ3S: (110, 512, 296), OP_IQ1S: (50, 512, 648), OP_IQ1M: (56, 512, 584),
              OP_TQ1_0: (54, 512, 600), OP_TQ2_0: (66, 512, 496), OP_NVFP4: (36, 128, 908)}
BLOCK_DTYPE = {OP_Q4K: "Q4_K", OP_Q8_0: "Q8_0", OP_Q6K: "Q6_K", OP_Q4_0: "Q4_0", OP_Q4_1: "Q4_1", OP_Q5_0: "Q5_0", OP_Q5_1: "Q5_1",
               OP_Q2K: "Q2_K", OP_Q3K: "Q3_K", OP_Q5K: "Q5_K", OP_IQ4NL: "IQ4_NL", OP_IQ4XS: "IQ4_XS", OP_MXFP4: "MXFP4",
               OP_IQ2XXS: "IQ2_XXS", OP_IQ2XS: "IQ2_XS", OP_IQ2S: "IQ2_S", OP_IQ3XXS: "IQ3_XXS", OP_IQ3S: "IQ3_S", OP_IQ1S: "IQ1_S", OP_IQ1M: "IQ1_M",
               OP_TQ1_0: "TQ1_0", OP_TQ2_0: "TQ2_0", OP_NVFP4: "NVFP4"}


def t_width(C: int, es: int) -> int:
    """Columns per transpose tile (csrc/kk_ops.h kk_t_width)."""
    wmax = 4096 // es
    if C > wmax:
        n = -(-C // wmax)
        return min((-(-C // n) + 7) & ~7, wmax)
    return wmax


def emulate_part(plan: dict, part: int, pool_bytes: int, exchange: dict | None = None) -> Tuple[np.ndarray, np.ndarray]:
    """Execute one part of a kk_plan_describe plan on the CPU with the oracle's arithmetic.
    Returns (pool, written-mask).  This checks the planner (reads, segments, offsets), not the kernels.
    `exchange` (rank -> (pool, mask)) receives what KK_OP_ROWSPLIT segments deal to the other ranks' pools."""
    pool = np.zeros(pool_bytes, np.uint8)
    mask = np.zeros(pool_bytes, bool)
    fhs = [open(s, "rb") for s in plan["shards"]]
    try:
        for ch in plan["parts"][part]["chunks"]:
            buf = np.zeros(ch["buf_bytes"] + 64, np.uint8)
            fh = fhs[ch["shard"]]
            covered = np.zeros(ch["buf_bytes"], bool)
            for fo, ln, bo in ch["reads"]:
                assert bo + ln <= ch["buf_bytes"], "read lands outside the chunk buffer"
                assert not covered[bo:bo + ln].any(), "two reads overlap in the chunk buffer"
                covered[bo:bo + ln] = True
                fh.seek(fo)
                raw = fh.read(ln)
                assert len(raw) == ln, "read runs past the end of the shard"
                buf[bo:bo + ln] = np.frombuffer(raw, np.uint8)
            tiles = 0
            for sg in ch["segs"]:
                assert sg["tile_begin"] == tiles, "tile_begin must be the running tile count of the chunk"
                op, so, do, u = sg["op"], sg["src_off"], sg["dst_off"], sg["units"]
                assert do % 16 == 0
                if op in BLOCK_GEOM:
                    src_bytes = BLOCK_GEOM[op][0] * u
                else:
                    src_bytes = {OP_COPY: u, OP_F32: 4 * u, OP_F16: 2 * u, OP_ROWSPLIT: u, OP_F8E4M3: u, OP_F8E5M2: u,
                                 OP_T_F32_BF16: 4 * u * sg["p0"], OP_T_B32: 4 * u * sg["p0"],
                                 OP_T_F16_BF16: 2 * u * sg["p0"], OP_T_B16: 2 * u * sg["p0"]}[op]
                assert so + src_bytes <= ch["buf_bytes"], "segment reads past the bytes staged for its chunk"
                assert covered[so:so + src_bytes].all(), "segment consumes bytes no read put there"
                if op == OP_ROWSPLIT:
                    row_bytes, w, r0, done = sg["p0"], sg["p1"], sg["p2"], sg["p3"]
                    assert exchange is not None and row_bytes % w == 0
                    pos = done + np.arange(u, dtype=np.int64)
                    row, col = pos // row_bytes, pos % row_bytes
                    j, within = col // w, col % w
                    dsto = do + (r0 + row) * w + within
                    src = buf[so:so + u]
                    for rk in np.unique(j):
                        sel = j == rk
                        pj, mj = exchange[int(rk)]
                        assert not mj[dsto[sel]].any(), "exchange pieces overlap"
                        pj[dsto[sel]] = src[sel]
                        mj[dsto[sel]] = True
                    tiles += -(-u // 32768)
                    continue
                if op == OP_COPY:
                    out = buf[so:so + u]
                    tiles += -(-u // 32768)
                elif op == OP_F32:
                    out = oracle.f32_bits_to_bf16(buf[so:so + 4 * u].copy().view("<u4")).view(np.uint8)
                    tiles += -(-u // 8192)
                elif op == OP_F16:
                    out = oracle.f16_bits_to_bf16(buf[so:so + 2 * u].copy().view("<u2")).view(np.uint8)
                    tiles += -(-u // 16384)
                elif op in (OP_F8E4M3, OP_F8E5M2):
                    fn = oracle.f8e4m3_bits_to_bf16 if op == OP_F8E4M3 else oracle.f8e5m2_bits_to_bf16
                    out = fn(buf[so:so + u]).view(np.uint8)
                    tiles += -(-u // 32768)
                elif op in BLOCK_GEOM:
                    bb, _, tb = BLOCK_GEOM[op]
                    out = oracle.dequant_bf16(BLOCK_DTYPE[op], buf[so:so + bb * u].reshape(-1, bb)).reshape(-1).view(np.uint8)
                    tiles += -(-u // tb)
                else:
                    C, R, r0 = sg["p0"], sg["p1"], sg["p2"]
                    es = 4 if op in (OP_T_F32_BF16, OP_T_B32) else 2
                    src = buf[so:so + u * C * es].reshape(u, C, es)
                    if op == OP_T_F32_BF16:
                        v = oracle.f32_bits_to_bf16(src.reshape(-1).copy().view("<u4")).view(np.uint8).reshape(u, C, 2)
                    elif op == OP_T_F16_BF16:
                        v = oracle.f16_bits_to_bf16(src.reshape(-1).copy().view("<u2")).view(np.uint8).reshape(u, C, 2)
                    else:
                        v = src
                    oes = v.shape[2]
                    dst = pool[do:do + C * R * oes].reshape(C, R, oes)
                    dst[:, r0:r0 + u, :] = v.transpose(1, 0, 2)
                    mask[do:do + C * R * oes].reshape(C, R, oes)[:, r0:r0 + u, :] = True
                    tiles += -(-u // 8) * -(-C // t_width(C, es))  # 8-row tiles, rows wider than a stage row cut into equal pieces (kk_t_width)
                    continue
                assert do + out.size <= pool_bytes, "segment writes past the end of the pool"
                assert not mask[do:do + out.size].any(), "segment overlaps an earlier one"
                pool[do:do + out.size] = out
                mask[do:do + out.size] = True
            assert tiles == ch["n_tiles"]
    finally:
        for fh in fhs:
            fh.close()
    return pool, mask


def rowsplit_tile_classes(plan: dict) -> Tuple[int, int]:
    """(bulk-store tiles, byte-granular tiles) of every KK_OP_ROWSPLIT segment of every part: kk_make_tile's condition for bulk == 3,
    with the chunk's base 16-byte aligned as the staging buffers and the resident image are."""
    T = 32768
    bulk = fallback = 0
    for part in plan["parts"]:
        for ch in part["chunks"]:
            for sg in ch["segs"]:
                if sg["op"] != OP_ROWSPLIT:
                    continue
                for o in range(0, sg["units"], T):
                    n = min(T, sg["units"] - o)
                    if (sg["src_off"] + o) % 16 == 0 and sg["p0"] % 16 == 0 and sg["p1"] % 16 == 0 and n % 16 == 0 and sg["dst_off"] % 16 == 0:
                        bulk += 1
                    else:
                        fallback += 1
    return bulk, fallback


# Row-parallel tensors whose row-split exchange leaves the aligned bulk path: a 7-element norm first (14 bytes, so everything after it sits off
# 16 in an unpadded file), slices that are no multiple of 16 bytes, verbatim U8 / FP8, rows longer than a tile (57 KB) and a tensor with
# fewer rows (5) than there are ranks at n = 8.
ROWSPLIT_ODD_TENSORS = [("model.layers.0.input_layernorm.weight", "BF16", [7]),
                        ("model.layers.0.self_attn.o_proj.weight", "BF16", [100, 120]),
                        ("model.layers.0.mlp.down_proj.weight", "BF16", [67, 3000]),
                        ("model.layers.1.mlp.down_proj.weight", "U8", [33, 840]),
                        ("model.layers.1.self_attn.o_proj.weight", "F8_E4M3", [129, 360]),
                        ("model.layers.2.mlp.down_proj.weight", "BF16", [40, 28672]),
                        ("model.layers.2.self_attn.o_proj.weight", "BF16", [5, 16])]


def expected_mask(plan_pool: List[dict], total: int) -> np.ndarray:
    m = np.zeros(total, bool)
    for p in plan_pool:
        m[p["pool_offset"]:p["pool_offset"] + p["nbytes"]] = True
    return m


def write_raw_safetensors(path: str, header: dict | bytes, data: bytes, n_override: int | None = None) -> None:
    raw = header if isinstance(header, bytes) else json.dumps(header, separators=(",", ":")).encode()
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(raw) if n_override is None else n_override))
        f.write(raw)
        f.write(data)


def mixed_safetensors(path: str, seed: int = 11, pad_header: bool = True) -> List[Tuple[str, str, List[int]]]:
    """A small file that exercises every op: bf16 copy, f32/f16 casts, verbatim ints, ragged tails,
    zero-size and scalar tensors."""
    from tools import synth
    tensors = [
        ("a.bf16", "BF16", [33, 77]), ("b.f32", "F32", [129, 65]), ("c.f16", "F16", [7, 1001]), ("d.i64", "I64", [5, 3]),
        ("e.u8", "U8", [1021]), ("f.empty", "F32", [0]), ("g.scalar", "F32", []), ("h.bf16.big", "BF16", [700, 1024]),
        ("i.f32.odd", "F32", [3]), ("j.f16.one", "F16", [1]), ("k.bool", "BOOL", [13]),
    ]
    synth.write_safetensors(path, tensors, seed, pad_header=pad_header)
    return tensors
