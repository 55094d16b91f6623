"""CPU tier: the fp16 instantiation of the convert kernel's consumer bodies (KK_LAUNCH_F16), played through the CPU replay
(tests/emul/kk_f16_emul.cpp, kk_emul_launch_f16) against the fp16 oracle (tests/f16_oracle.py): every block type at every start alignment with ragged counts,
the casts with misaligned payloads and tails, FP8, staged and gathered transposes, and whole-plan launches of KK_LOAD_F16 loads — single,
broadcast and scatter with the row exchange.  Every output byte must be stored exactly once and nothing else touched."""
import os

import numpy as np
import pytest

from kukeon_b200 import gpupool
from oracle import oracle
from tests import f16_oracle as fo
from tests import helpers, kk_emul, kk_f16_emul
from tests.kk_emul import ERR, KKSeg, Pools
from tests.test_dequant_emul import OPS
from tests.test_launch_emul import Exchange, check, play_part
from tools import synth

LAUNCH_F16 = kk_f16_emul.LAUNCH_F16
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MB = 1 << 20
F16 = gpupool.LOAD_F16


@pytest.fixture(scope="module")
def emul():
    return kk_f16_emul.load()


@pytest.fixture(scope="module")
def emul_bf16():
    return kk_emul.load()


def test_launch_flag_matches_the_header():
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "kukeon_b200", "csrc", "kk_ops.h")).read()
    assert "#define KK_LAUNCH_F16 0x4u" in src


def run_elementwise(L, op, src, n_units, pay_off, out_bytes, flags=LAUNCH_F16):
    chunk = np.full(pay_off + src.size, 0x5A, np.uint8)
    chunk[pay_off:] = src
    rc, pools, _ = kk_emul.launch(L, chunk, [KKSeg(src_off=pay_off, units=n_units, op=op)], out_bytes, flags=flags)
    assert rc == 0, ERR.get(rc, rc)
    want = np.full(pools.hits.size, 16, np.uint8)
    if out_bytes % 16:
        want[-1] = out_bytes % 16
    assert (pools.hits == want).all(), "every output byte stored exactly once"
    return pools.bufs[0]


def run_blocks(L, dtype, blocks, pay_off):
    nel, nb, _ = oracle.BLOCK_QUANTS[dtype]
    n = blocks.shape[0]
    chunk = np.full(pay_off + n * nb, 0xA5, np.uint8)
    chunk[pay_off:] = blocks.reshape(-1)
    rc, pools, _ = kk_emul.launch(L, chunk, [KKSeg(src_off=pay_off, units=n, op=OPS[dtype])], n * nel * 2, flags=LAUNCH_F16)
    assert rc == 0, f"{dtype}: {ERR.get(rc, rc)}"
    assert (pools.hits == 16).all(), f"{dtype}: output vectors not stored exactly once"
    return pools.bufs[0].view(np.uint16).reshape(n, nel)


@pytest.mark.parametrize("dtype", sorted(OPS))
def test_block_types_every_alignment_ragged_counts(emul, dtype):
    """Random bytes (Inf / NaN / negative scales: NaN -> 0x7FFF on both sides), a full tile, counts around the warp-iteration sizes, and
    every start alignment a tile can have."""
    nel, nb, _ = oracle.BLOCK_QUANTS[dtype]
    per_iter = 8 if nel == 32 else 4 if dtype in ("Q4_K", "Q5_K", "NVFP4") else 1
    tb = helpers.BLOCK_GEOM[OPS[dtype]][2]
    full = synth.gen_bytes(dtype, nb * tb, 11, 3).reshape(tb, nb)
    assert (run_blocks(emul, dtype, full, 0) == fo.dequant_f16(dtype, full)).all()
    rng = np.random.default_rng(6)
    for k, n in enumerate([1, per_iter + 1, 16 * per_iter - 1, 16 * per_iter + 5, 37 * per_iter + 3]):
        blocks = rng.integers(0, 256, (n, nb), dtype=np.uint8)
        for pay_off in (range(16) if k == 0 else (0, 2, 8, 10)):
            assert (run_blocks(emul, dtype, blocks, pay_off) == fo.dequant_f16(dtype, blocks)).all(), (dtype, n, pay_off)


def test_f32_and_bf16_casts_misaligned_payloads_and_tails(emul):
    """F32 -> f16 (KK_OP_F32_BF16) and BF16 -> f16 (KK_OP_F16_BF16 in an f16 launch): aligned vector loads and byte-assembled ones, counts
    that end inside a group, a full tile, and the specials (inf, NaN, ties, values that overflow fp16 or land in its subnormals)."""
    specials = np.array([0x7F800000, 0xFF800001, 0x3F801000, 0x00000001, 0x477FF000, 0x47800000, 0x33800000, 0x387FC000], "<u4")
    bspecials = np.array([0x7F80, 0xFFC1, 0x4780, 0x477F, 0x3380, 0x3300, 0x8001, 0x3F81], "<u2")
    for n in (1, 3, 7, 8, 9, 513, 8192):
        f32 = synth.gen_bytes("F32", 4 * n, 6, n).copy()
        f32[:4 * min(n, 8)] = specials.view(np.uint8)[:4 * min(n, 8)]
        bf = np.random.default_rng(n).integers(0, 1 << 16, n, dtype=np.uint32).astype("<u2")
        bf[:min(n, 8)] = bspecials[:min(n, 8)]
        bf = bf.view(np.uint8)
        for pay_off in (0, 2, 4, 6, 8, 12) + ((1, 3) if n < 600 else ()):
            got = run_elementwise(emul, helpers.OP_F32, f32, n, pay_off, 2 * n).view(np.uint16)
            assert (got == fo.f32_bits_to_f16(f32.view("<u4"))).all(), ("F32", n, pay_off)
            got = run_elementwise(emul, helpers.OP_F16, bf, n, pay_off, 2 * n).view(np.uint16)
            assert (got == fo.bf16_bits_to_f16(bf.view("<u2"))).all(), ("BF16", n, pay_off)


def test_bf16_cast_every_bit_pattern(emul):
    u = np.arange(65536, dtype=np.uint32).astype("<u2")
    for n, pay_off in ((16384, 0), (16384, 6), (16381, 1)):
        got = run_elementwise(emul, helpers.OP_F16, u[:n].view(np.uint8), n, pay_off, 2 * n).view(np.uint16)
        assert (got == fo.bf16_bits_to_f16(u[:n])).all()
        u = np.roll(u, -n)


@pytest.mark.parametrize("op,fn", [(helpers.OP_F8E4M3, fo.f8e4m3_bits_to_f16), (helpers.OP_F8E5M2, fo.f8e5m2_bits_to_f16)])
def test_fp8_every_byte_value_every_alignment_and_tail(emul, op, fn):
    rng = np.random.default_rng(8)
    for n in (1, 15, 16, 17, 256, 511 * 16 + 3, 32768):
        src = np.concatenate([np.arange(256, dtype=np.uint8), rng.integers(0, 256, max(0, n - 256), dtype=np.uint8)])[:n]
        for pay_off in (0, 1, 2, 4, 8, 13):
            assert (run_elementwise(emul, op, src, n, pay_off, 2 * n).view(np.uint16) == fn(src)).all(), (op, n, pay_off)


# source dtype -> (op in an f16 launch, element bytes, value map to fp16 bits)
T8 = {"F32": (helpers.OP_T_F32_BF16, 4, fo.f32_bits_to_f16), "BF16": (helpers.OP_T_F16_BF16, 2, fo.bf16_bits_to_f16),
      "F16": (helpers.OP_T_B16, 2, lambda u: u)}


@pytest.mark.parametrize("dtype", sorted(T8))
@pytest.mark.parametrize("staged", [1, 0])
def test_transpose_tiles_staged_and_gathered(emul, dtype, staged):
    op, es, fn = T8[dtype]
    udt = np.uint32 if es == 4 else np.uint16
    W = 4096 // es
    for nr, nc, R, row0 in ((8, W, 768, 0), (8, 768, 3072, 8), (5, 72, 64, 8), (8, 16, 36, 4), (1, 8, 8, 0), (8, 40, 24, 0)):
        if staged and (nc * es) % 16:
            continue
        rng = np.random.default_rng(nr * nc)
        src = rng.integers(0, 1 << (8 * es), (nr, nc), dtype=np.uint64).astype(udt)
        src.reshape(-1)[:4] = np.array([0x7F800000, 0x7FC00001, 0x00000001, 0x477FF000] if es == 4 else [0x7F80, 0xFFC1, 0x4780, 0x0001], udt)
        pad = 0 if staged else es
        chunk = np.zeros(pad + src.nbytes, np.uint8)
        chunk[pad:] = src.view(np.uint8).reshape(-1)
        rows = 8 + nc + 3
        seg = KKSeg(src_off=pad, dst_off=8 * R * 2, units=nr, op=op, p0=nc, p1=R, p2=row0)
        rc, pools, _ = kk_emul.launch(emul, chunk, [seg], rows * R * 2, flags=LAUNCH_F16)
        assert rc == 0, f"{dtype} {nr}x{nc}: {ERR.get(rc, rc)}"
        want = np.full((rows, R), 0xCDCD, np.uint16)
        want[8:8 + nc, row0:row0 + nr] = np.ascontiguousarray(fn(src.reshape(-1)).reshape(nr, nc).T)
        assert (pools.bufs[0].view(np.uint16).reshape(rows, R) == want).all(), (dtype, nr, nc, R, row0)
        m = np.zeros((rows, R), bool)
        m[8:8 + nc, row0:row0 + nr] = True
        assert (pools.hits == np.add.reduceat(np.repeat(m.reshape(-1), 2).astype(np.uint8), np.arange(0, rows * R * 2, 16))).all()


def replay(L, path, mode=gpupool.MODE_SINGLE, flags=F16, n_parts=1, chunk=1 * MB):
    """Every part of the library's plan of an f16 load, played with KK_LAUNCH_F16 as the loader launches it, against the fp16 oracle."""
    shards, recs = oracle.index_path(path)
    plan = gpupool.plan_describe(path, mode=mode, flags=flags, n_parts=n_parts, chunk_bytes=chunk)
    oflags = flags & (1 | 2 | 16 | F16)
    x = None
    if mode == gpupool.MODE_SCATTER:
        exps = [fo.expected_pool(shards, recs, mode, oflags, n_parts, g) for g in range(n_parts)]
        ranks = [Pools(1, len(exp)) for exp, _ in exps]
        x = Exchange(ranks)
        for g in range(n_parts):
            play_part(L, plan, g, ranks[g], flags=LAUNCH_F16, x=x)
        for g in range(n_parts):
            check(ranks[g], *exps[g])
    else:
        exp, pl = fo.expected_pool(shards, recs, mode, oflags)
        pools = Pools(n_parts, len(exp))
        for g in range(n_parts):
            play_part(L, plan, g, pools, flags=LAUNCH_F16)
        check(pools, exp, pl)
    return plan, (tuple(x.tiles) if x else (0, 0))


def test_whole_launches_single_broadcast_scatter_with_the_exchange(emul, tmp_path):
    X = gpupool.LOAD_SCATTER_EXCHANGE
    for dt in ("F16", "BF16"):
        d = str(tmp_path / f"llama_{dt}")
        synth.make_llama(d, dict(hidden=256, ffn=704, layers=2, kv_dim=64, vocab=1000), max_shard_bytes=2_500_000, dtype=dt)
        replay(emul, d)
        replay(emul, d, mode=gpupool.MODE_BROADCAST, n_parts=3)
        plan, tiles = replay(emul, d, mode=gpupool.MODE_SCATTER, flags=F16 | X, n_parts=4)
        # the exchange deals the row-parallel tensors the pool holds verbatim: an F16 file's under the flag, none of a BF16 file's
        assert (tiles[0] + tiles[1] > 0) == (dt == "F16"), (dt, tiles)
        replay(emul, d, mode=gpupool.MODE_SCATTER, n_parts=2)


def test_mixed_safetensors_fixtures_and_flags(emul, tmp_path):
    p = str(tmp_path / "m.safetensors")
    synth.write_safetensors(p, [("a", "BF16", [7]), ("b", "BF16", [33, 77]), ("c", "F32", [129, 65]), ("d", "F16", [7, 1001]), ("e", "U8", [3]),
                                ("f", "BF16", [4099]), ("g", "F32", [5]), ("h", "F16", [2, 3]), ("k", "F8_E4M3", [300, 70]), ("l", "F8_E5M2", [37])], 5, pad_header=False)
    for fl in (F16, F16 | gpupool.LOAD_KEEP_F32 | gpupool.LOAD_F8_TO_BF16):
        replay(emul, p, flags=fl)
    helpers.mixed_safetensors(str(tmp_path / "mixed.safetensors"))
    replay(emul, str(tmp_path / "mixed.safetensors"), mode=gpupool.MODE_BROADCAST, n_parts=2)
    replay(emul, os.path.join(G, "st_mixed.safetensors"))
    replay(emul, os.path.join(G, "sharded"), flags=F16 | gpupool.LOAD_KEEP_F32)


def test_golden_gguf_fixtures_and_alignment_8(emul, tmp_path):
    from tests.test_plan import f4_tensors
    for g in ("q4k.gguf", "q4km_mix.gguf", "quants_f4.gguf", "quants_cb.gguf", "quants_iq.gguf"):
        replay(emul, os.path.join(G, g))
    p = str(tmp_path / "a8.gguf")
    synth.write_gguf(p, [("pad.weight", "F32", [4])] + f4_tensors(hidden=256, ffn=512, layers=1, vocab=256), 21, alignment=8)
    replay(emul, p, mode=gpupool.MODE_SCATTER, n_parts=2)


def test_gpt2_transposes_every_dtype(emul, tmp_path):
    T = gpupool.LOAD_GPT2_CONV1D_T
    for dt, d, pad in (("F32", 96, True), ("F16", 40, True), ("BF16", 40, True), ("BF16", 72, False), ("F32", 41, True), ("BF16", 43, True)):
        p = str(tmp_path / f"gpt2_{dt}_{d}_{int(pad)}.safetensors")
        synth.write_safetensors(p, [("x", "U8", [3])] + synth.gpt2_tensors(n_layer=1, d=d, vocab=50, n_pos=8, dtype=dt), 3, pad_header=pad)
        plan, _ = replay(emul, p, flags=F16 | T)
        ops = {sg["op"] for ch in plan["parts"][0]["chunks"] for sg in ch["segs"]}
        want = {"F32": helpers.OP_T_F32_BF16, "BF16": helpers.OP_T_F16_BF16, "F16": helpers.OP_T_B16}[dt]
        assert want in ops, (dt, ops)


def test_the_replay_tells_the_two_formats_apart(emul_bf16):
    """Liveness: the same F32 tile played by the bf16 replay gives bf16, which the fp16 oracle must reject."""
    f32 = synth.gen_bytes("F32", 4 * 4096, 2, 1)
    b = run_elementwise(emul_bf16, helpers.OP_F32, f32, 4096, 0, 8192, flags=0).view(np.uint16)
    assert (b == oracle.f32_bits_to_bf16(f32.view("<u4"))).all()
    assert (b != fo.f32_bits_to_f16(f32.view("<u4"))).mean() > 0.9
