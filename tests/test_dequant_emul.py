"""CPU tier: the device dequantisers (kukeon_b200/csrc/kk_dequant.cuh), compiled for the host by tests/emul and played lane by lane
inside launches of one or a few segments (tests/kk_emul.py), against the oracle (which tests/test_oracle_values.py pins to gguf-py bit for
bit).  Every tile is the one the kernel's producer builds for the segment (kk_make_tile), staged by its copies; the consumers may read its
payload only.

Covers every block op that lives in that header: Q8_0 and Q6_K (proven on the GPU in round 1 — they validate the
harness) and the §8(f4) additions Q4_0, Q4_1, Q5_0, Q5_1, Q2_K, Q3_K, Q5_K.  Cases: a full tile (KK_*_TILE_BLOCKS), ragged
block counts around the warp-iteration sizes, and every source alignment class a tile can start at (pay_off 0..15)."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle
from tests import helpers, kk_emul
from tests.kk_emul import ERR, KKSeg
from tools import synth

OPS = {"Q4_K": helpers.OP_Q4K, "Q8_0": helpers.OP_Q8_0, "Q6_K": helpers.OP_Q6K, "Q4_0": helpers.OP_Q4_0, "Q4_1": helpers.OP_Q4_1, "Q5_0": helpers.OP_Q5_0,
       "Q5_1": helpers.OP_Q5_1, "Q2_K": helpers.OP_Q2K, "Q3_K": helpers.OP_Q3K, "Q5_K": helpers.OP_Q5K, "IQ4_NL": helpers.OP_IQ4NL,
       "IQ4_XS": helpers.OP_IQ4XS, "MXFP4": helpers.OP_MXFP4, "IQ2_XXS": helpers.OP_IQ2XXS, "IQ2_XS": helpers.OP_IQ2XS, "IQ2_S": helpers.OP_IQ2S,
       "IQ3_XXS": helpers.OP_IQ3XXS, "IQ3_S": helpers.OP_IQ3S, "IQ1_S": helpers.OP_IQ1S, "IQ1_M": helpers.OP_IQ1M, "TQ1_0": helpers.OP_TQ1_0,
       "TQ2_0": helpers.OP_TQ2_0, "NVFP4": helpers.OP_NVFP4}


@pytest.fixture(scope="module")
def emul():
    return kk_emul.load()


def geom(L, op):
    a, b, c = C.c_uint32(), C.c_uint32(), C.c_uint32()
    L.kk_emul_block_geom(op, C.byref(a), C.byref(b), C.byref(c))
    return a.value, b.value, c.value


def run_blocks(L, dtype, blocks, pay_off):
    """The blocks as one segment that starts pay_off bytes into its chunk (so its first tile's payload sits at stage offset pay_off) and
    ends at the chunk's end.  Returns the bf16 output per block."""
    nel, nb, _ = oracle.BLOCK_QUANTS[dtype]
    n = blocks.shape[0]
    chunk = np.full(pay_off + n * nb, 0xA5, np.uint8)
    chunk[pay_off:] = blocks.reshape(-1)
    rc, pools, _ = kk_emul.launch(L, chunk, [KKSeg(src_off=pay_off, units=n, op=OPS[dtype])], n * nel * 2)
    assert rc == 0, f"{dtype}: {ERR.get(rc, rc)}"
    assert (pools.hits == 16).all(), f"{dtype}: {int((pools.hits != 16).sum())} output vectors not stored exactly once"
    return pools.bufs[0].view(np.uint16).reshape(n, nel)


@pytest.mark.parametrize("dtype", sorted(OPS))
def test_geometry_tables_agree(emul, dtype):
    nel, nb, _ = oracle.BLOCK_QUANTS[dtype]
    bb, ob, tb = geom(emul, OPS[dtype])
    assert (bb, ob) == (nb, 2 * nel)
    assert helpers.BLOCK_GEOM[OPS[dtype]] == (bb, ob, tb)
    assert bb * tb <= 32768 and (bb * tb) % 16 == 0


@pytest.mark.parametrize("dtype", sorted(OPS))
def test_full_tile_finite_scales(emul, dtype):
    nel, nb, _ = oracle.BLOCK_QUANTS[dtype]
    tb = geom(emul, OPS[dtype])[2]
    blocks = synth.gen_bytes(dtype, nb * tb, 11, 3).reshape(tb, nb)
    assert (run_blocks(emul, dtype, blocks, 0) == oracle.dequant_bf16(dtype, blocks)).all()


@pytest.mark.parametrize("dtype", sorted(OPS))
def test_ragged_counts_and_every_alignment_random_bytes(emul, dtype):
    """Fully random bytes (Inf/NaN scales included: NaN -> 0x7FFF on both sides) at every start alignment a tile can have."""
    nel, nb, _ = oracle.BLOCK_QUANTS[dtype]
    per_iter = 8 if nel == 32 else 4 if dtype in ("Q4_K", "Q5_K", "NVFP4") else 1  # blocks one warp iteration covers
    rng = np.random.default_rng(5)
    counts = [1, 2, per_iter - 1 or 1, per_iter, per_iter + 1, 16 * per_iter - 1, 16 * per_iter, 16 * per_iter + 1, 16 * per_iter + 5, 37 * per_iter + 3]
    for k, n in enumerate(counts):
        blocks = rng.integers(0, 256, (n, nb), dtype=np.uint8)
        for pay_off in ([0, 2, 4, 8, 10] if k else range(16)):
            got = run_blocks(emul, dtype, blocks, pay_off)
            assert (got == oracle.dequant_bf16(dtype, blocks)).all(), (dtype, n, pay_off)


@pytest.mark.parametrize("dtype", sorted(OPS))
def test_multi_tile_segments_walked_like_the_producer(emul, dtype):
    """2.4 tiles of every type, starting 16-byte aligned and not: the per-tile split (kk_block_tile, shared with the kernel)
    hands every block to exactly one tile and every output vector is stored exactly once at the right pool offset."""
    nel, nb, _ = oracle.BLOCK_QUANTS[dtype]
    tb = geom(emul, OPS[dtype])[2]
    n = 2 * tb + tb * 2 // 5 + 3
    blocks = synth.gen_bytes(dtype, nb * n, 13, 5).reshape(n, nb)
    want = oracle.dequant_bf16(dtype, blocks)
    for mis in (0, 8, 6):
        assert (run_blocks(emul, dtype, blocks, mis) == want).all(), (dtype, mis)


def run_elementwise(L, op, src, n_units, pay_off, out_bytes, flags=0):
    """src as one segment of n_units that starts pay_off bytes into its chunk; every output byte must be stored exactly once."""
    chunk = np.full(pay_off + src.size, 0x5A, np.uint8)
    chunk[pay_off:] = src
    rc, pools, _ = kk_emul.launch(L, chunk, [KKSeg(src_off=pay_off, units=n_units, op=op)], out_bytes, flags=flags)
    assert rc == 0, ERR.get(rc, rc)
    want_hits = np.full(pools.hits.size, 16, np.uint8)
    if out_bytes % 16:
        want_hits[-1] = out_bytes % 16
    assert (pools.hits == want_hits).all(), "every output byte stored exactly once"
    return pools.bufs[0]


@pytest.mark.parametrize("dtype,op,fn", [("F8_E4M3", helpers.OP_F8E4M3, oracle.f8e4m3_bits_to_bf16), ("F8_E5M2", helpers.OP_F8E5M2, oracle.f8e5m2_bits_to_bf16)])
def test_fp8_widening_every_byte_value_every_alignment_and_tail(emul, dtype, op, fn):
    """Elementwise FP8 -> bf16: all 256 byte values, counts that end inside a 16-element group, aligned and byte-assembled loads."""
    rng = np.random.default_rng(8)
    for n in (1, 15, 16, 17, 256, 511 * 16 + 3, 512 * 16, 512 * 16 + 9, 32768):
        src = np.concatenate([np.arange(256, dtype=np.uint8), rng.integers(0, 256, max(0, n - 256), dtype=np.uint8)])[:n]
        for pay_off in (0, 1, 2, 4, 8, 13):
            out = run_elementwise(emul, op, src, n, pay_off, 2 * n)
            assert (out.view(np.uint16) == fn(src)).all(), (dtype, n, pay_off)


T8 = {"F32": (helpers.OP_T_F32_BF16, 4), "F16": (helpers.OP_T_F16_BF16, 2), "BF16": (helpers.OP_T_B16, 2), "B32": (helpers.OP_T_B32, 4)}  # B32: 4-byte verbatim


def t8_expected(dtype, src_rc):
    """[nr, nc] source elements (as raw uint of the element width) -> bf16 bits [nc, nr] (the transposed, converted tile)."""
    if dtype == "F32":
        v = oracle.f32_bits_to_bf16(src_rc.reshape(-1)).reshape(src_rc.shape)
    elif dtype == "F16":
        v = oracle.f16_bits_to_bf16(src_rc.reshape(-1)).reshape(src_rc.shape)
    else:
        v = src_rc
    return np.ascontiguousarray(v.T)


def run_transpose_segment(emul, dtype, nr, C_src, R, row0, staged, seed=21):
    """nr source rows of C_src columns as one transpose segment whose first row is row0 of a tensor with R rows, so that its tiles are
    nr x kk_t_width(C_src) at destination column row0.  The source starts 16-byte aligned (staged: the producer's bulk copies bring the
    tiles in when their rows are whole 16-byte units) or 2 / 4 bytes off (the consumers gather every tile).  The destination tensor sits
    between 8 rows and 3 rows of margin: values vs the oracle, every destination element written exactly once and nothing else touched.
    Returns the launch's statistics."""
    op, es = T8[dtype]
    rng = np.random.default_rng(seed)
    udt = np.uint32 if es == 4 else np.uint16
    odt, oes, fill = (np.uint32, 4, 0xCDCDCDCD) if dtype == "B32" else (np.uint16, 2, 0xCDCD)
    if dtype in ("BF16", "B32"):
        src = rng.integers(0, 1 << (8 * es), (nr, C_src), dtype=np.uint64).astype(udt)
    else:
        src = synth.gen_bytes(dtype, nr * C_src * es, 3, nr + C_src).view(udt).reshape(nr, C_src)
    pad = 0 if staged else es
    chunk = np.zeros(pad + src.nbytes, np.uint8)
    chunk[pad:] = src.view(np.uint8).reshape(-1)
    rows = 8 + C_src + 3
    seg = KKSeg(src_off=pad, dst_off=8 * R * oes, units=nr, op=op, p0=C_src, p1=R, p2=row0)
    rc, pools, st = kk_emul.launch(emul, chunk, [seg], rows * R * oes)
    assert rc == 0, f"{dtype} {nr}x{C_src}: {ERR.get(rc, rc)}"
    want = np.full((rows, R), fill, odt)
    want[8:8 + C_src, row0:row0 + nr] = t8_expected(dtype, src)
    assert (pools.bufs[0].view(odt).reshape(rows, R) == want).all(), (dtype, nr, C_src, R, row0)
    m = np.zeros((rows, R), bool)
    m[8:8 + C_src, row0:row0 + nr] = True
    per16 = np.add.reduceat(np.repeat(m.reshape(-1), oes).astype(np.uint8), np.arange(0, rows * R * oes, 16))
    assert (pools.hits == per16).all(), "bytes stored per 16-byte unit differ from the tile's footprint"
    return st


@pytest.mark.parametrize("dtype", sorted(T8))
@pytest.mark.parametrize("staged", [1, 0])
def test_t8_transpose_tiles_values_write_once_and_bank_conflicts(emul, dtype, staged):
    """8-row transpose tiles: full width (one tile spanning whole rows — one bulk copy — and two tiles per row group — one bulk copy per row),
    ragged width, fewer than 8 rows, destination rows that defeat the 16-byte store (R % 8 != 0), 4-byte verbatim elements.  Staged full
    tiles must read shared memory conflict-free."""
    _, es = T8[dtype]
    W = 4096 // es
    # (rows, tile columns, R, row0, source columns)
    cases = [(8, W, 768, 0, W), (8, W, 768, 16, 2 * W), (8, 768, 3072, 8, 768), (8, 40, 24, 0, 40), (5, 72, 64, 8, 72),
             (8, 129 if not staged else 136, 20, 0, 129 if not staged else 136), (8, 16, 36, 4, 16), (1, 8, 8, 0, 8)]
    for nr, nc, R, row0, C_src in cases:
        if staged and (nc * es) % 16:
            continue
        st = run_transpose_segment(emul, dtype, nr, C_src, R, row0, staged)
        if staged and nr == 8 and nc % 32 == 0:
            assert st[0] == st[1], f"{dtype} {nr}x{nc}: {st[0]} shared-memory wavefronts for {st[1]} warp loads"


def test_copy_and_casts_register_paths_every_alignment_and_tail(emul):
    """The non-TMA consumer paths of the headline ops: COPY (misaligned / ragged tiles, and aligned ones under NVLS stores, which turn the
    bulk store off), F32 -> bf16 and F16 -> bf16 — aligned vector loads and byte-assembled ones, counts that end inside a 16-byte group, a
    full 32 KiB tile."""
    rng = np.random.default_rng(4)
    for n in (1, 15, 16, 17, 255, 8191 * 4 + 3, 32768):
        src = rng.integers(0, 256, n, dtype=np.uint8)
        for pay_off in (0, 1, 4, 8, 15):
            flags = kk_emul.LAUNCH_MULTIMEM if pay_off == 0 and n % 16 == 0 else 0
            assert (run_elementwise(emul, helpers.OP_COPY, src, n, pay_off, n, flags) == src).all(), ("COPY", n, pay_off)
    for n in (1, 7, 8, 9, 513, 8192):
        f32 = synth.gen_bytes("F32", 4 * n, 6, n)
        f32[:4 * min(n, 4)] = np.array([0x7F800000, 0xFF800001, 0x3F808000, 0x00000001], "<u4").view(np.uint8)[:4 * min(n, 4)]  # inf, NaN, tie, subnormal
        f16 = synth.gen_bytes("F16", 2 * n, 7, n)
        for pay_off in (0, 2, 4, 6, 8, 12) + ((1, 3) if n < 600 else ()):
            got = run_elementwise(emul, helpers.OP_F32, f32, n, pay_off, 2 * n).view(np.uint16)
            assert (got == oracle.f32_bits_to_bf16(f32.view("<u4"))).all(), ("F32", n, pay_off)
            got = run_elementwise(emul, helpers.OP_F16, f16, n, pay_off, 2 * n).view(np.uint16)
            assert (got == oracle.f16_bits_to_bf16(f16.view("<u2"))).all(), ("F16", n, pay_off)


def test_q4k_shuffle_emulation_is_live(emul):
    """Q4_K is the one consumer whose lanes trade values (__shfl_sync, emulated by record/replay): swapping two sub-block scale bytes
    of one block must change exactly that block's output."""
    blocks = synth.gen_bytes("Q4_K", 144 * 9, 2, 1).reshape(9, 144)
    base = run_blocks(emul, "Q4_K", blocks, 0)
    mut = blocks.copy()
    mut[5, 4], mut[5, 5] = blocks[5, 5] ^ 0x15, blocks[5, 4] ^ 0x2A
    got = run_blocks(emul, "Q4_K", mut, 0)
    assert (got == oracle.dequant_bf16("Q4_K", mut)).all()
    assert (got[5] != base[5]).any() and (np.delete(got, 5, 0) == np.delete(base, 5, 0)).all()


def test_super_block_dequantisers_read_shared_memory_conflict_free(emul):
    """Bank-conflict accounting from the recorded addresses of the 16/32-bit shared loads: every 256-weight type (one block per warp
    iteration, lanes side by side inside the block) needs exactly one wavefront per warp load; the 32-weight legacy blocks straddle
    more than 128 bytes per warp iteration and stay below 2.5."""
    for dt, op in sorted(OPS.items()):
        nel, nb, _ = oracle.BLOCK_QUANTS[dt]
        if dt in ("Q4_K", "Q5_K"):
            continue  # vector loads (lds128 / lds64), not traced
        per_sweep = 16 * (8 if nel == 32 else 4 if dt == "NVFP4" else 1)
        n = geom(emul, op)[2] // per_sweep * per_sweep  # whole sweeps: every lane of every warp executes the same loads
        blocks = synth.gen_bytes(dt, nb * n, 1, 1)
        rc, _, st = kk_emul.launch(emul, blocks, [KKSeg(units=n, op=op)], n * nel * 2)
        assert rc == 0, (dt, ERR.get(rc, rc))
        ratio = st[0] / st[1]
        assert (ratio == 1.0) if nel >= 64 else (ratio < 2.5), (dt, st[0], st[1])


def test_harness_sees_wrong_answers(emul):
    """The checker is live: feeding Q5_0 blocks to the Q4_0 function must not reproduce the Q5_0 oracle."""
    blocks = synth.gen_bytes("Q5_0", 22 * 9 * 8, 2, 1).reshape(-1, 22)
    chunk = blocks.reshape(-1)
    n = chunk.size // 18
    rc, pools, _ = kk_emul.launch(emul, chunk, [KKSeg(units=n, op=helpers.OP_Q4_0)], n * 64)
    assert rc == 0
    assert not (pools.bufs[0].view(np.uint16)[: 32 * 8] == oracle.dequant_bf16("Q5_0", blocks)[:8].reshape(-1)).all()
    # and a chunk one byte shorter than the blocks its segment says it holds is refused, not read past
    assert kk_emul.launch(emul, chunk, [KKSeg(units=n, op=helpers.OP_Q4_0)], n * 64, src_bytes=n * 18 - 1)[0] == 19
