"""CPU tier: whole launches of kk_convert_kernel replayed through the device source (tests/emul kk_emul_launch).

For every staged chunk the planner produces (kk_plan_describe), the chunk buffer is filled as the reader threads would fill it and the
launch is played tile by tile: segment lookup from tile_begin[], `kk_make_tile` (csrc/kk_tile.h — the function the kernel's producer warp
calls), the bulk copies it asks for with the TMA constraints checked, then the consumer code of csrc/kk_consume_core.cuh / kk_dequant.cuh
for all 16 x 32 lanes, storing into every destination pool of the launch.  The scatter row exchange (KK_OP_ROWSPLIT) is played through the
kernel's own row-split addressing (kk_rowsplit_* in kk_tile.h): every rank's launch stores into all ranks' pools, its bulk-store pieces with
their 16-byte alignment checked.  The pools must equal the oracle's, every pool byte a tensor owns must have been stored exactly once across
all launches, and nothing else may have been touched.

Not covered here (GPU tests only): the mbarrier / proxy-fence protocol and anything about timing."""
import ctypes as C
import os

import numpy as np
import pytest

from kukeon_b200 import gpupool
from oracle import oracle
from tests import helpers, kk_emul
from tests.kk_emul import ERR, NO_EXCHANGE, KKSeg, Pools
from tools import synth

_HERE = os.path.dirname(os.path.abspath(__file__))
G = os.path.join(_HERE, "golden")
MB = 1 << 20


@pytest.fixture(scope="module")
def emul():
    return kk_emul.load()


class Exchange:
    """The pools of all ranks as a row-split launch sees them (ConvertLaunch::xdst), with each pool's hit counters and byte mask, and the
    row-split tiles played so far: tiles[0] by bulk stores, tiles[1] by the byte-granular consumer."""
    def __init__(self, ranks):
        n = len(ranks)
        self.args = ((C.c_void_p * n)(*[r.bufs[0].ctypes.data for r in ranks]), n, (C.c_uint64 * n)(*[r.bufs[0].size for r in ranks]),
                     (C.c_void_p * n)(*[r.hits.ctypes.data for r in ranks]), (C.c_void_p * n)(*[r.m1.ctypes.data for r in ranks]))
        self.tiles = (C.c_uint64 * 2)()


def play_part(L, plan, part, pools, flags=0, x=None):
    fhs = [open(s, "rb") for s in plan["shards"]]
    try:
        for ch in plan["parts"][part]["chunks"]:
            buf = np.zeros(ch["buf_bytes"], np.uint8)
            for fo, ln, bo in ch["reads"]:
                fhs[ch["shard"]].seek(fo)
                buf[bo:bo + ln] = np.frombuffer(fhs[ch["shard"]].read(ln), np.uint8)
            segs = (KKSeg * len(ch["segs"]))(*[KKSeg(s["src_off"], s["dst_off"], s["units"], s["op"], s["tile_begin"], s["p0"], s["p1"], s["p2"], s["p3"])
                                              for s in ch["segs"]])
            rc = L.kk_emul_launch(buf.ctypes.data, buf.size, segs, len(ch["segs"]), ch["n_tiles"], flags, pools.ptrs, len(pools.bufs), pools.bufs[0].size,
                                  pools.hits.ctypes.data, pools.m2.ctypes.data, pools.m1.ctypes.data, *(x.args if x else NO_EXCHANGE), x.tiles if x else None, None)
            assert rc == 0, f"part {part}: {ERR.get(rc, rc)}"
    finally:
        for fh in fhs:
            fh.close()


def check(pools, exp, pl):
    mask = helpers.expected_mask(pl, len(exp))
    per16 = np.add.reduceat(mask.astype(np.uint8), np.arange(0, len(exp), 16))
    assert (pools.hits[:len(per16)] == per16).all(), "a pool byte owned by a tensor was not stored exactly once (or padding was written)"
    for k, b in enumerate(pools.bufs):
        assert (b[mask] == exp[mask]).all(), f"pool {k} differs from the oracle"
        assert (b[~mask] == 0xCD).all(), f"pool {k}: bytes outside every tensor were written"


def replay(L, path, mode=gpupool.MODE_SINGLE, flags=0, n_parts=1, chunk=1 * MB, plan=None):
    """Replay every part of the plan (or of `plan`, when given) and check the pools.  Returns the plan and the row-split tiles played
    (bulk-store, byte-granular)."""
    shards, recs = oracle.index_path(path)
    plan = plan or gpupool.plan_describe(path, mode=mode, flags=flags, n_parts=n_parts, chunk_bytes=chunk)
    oflags = flags & (1 | 2 | 16)
    x = None
    if mode == gpupool.MODE_SCATTER:
        exps = [oracle.expected_pool(shards, recs, mode, oflags, n_parts, g) for g in range(n_parts)]
        ranks = [Pools(1, len(exp)) for exp, _ in exps]
        x = Exchange(ranks)  # every rank's launch may store into every rank's pool: the row exchange
        for g in range(n_parts):
            play_part(L, plan, g, ranks[g], x=x)
        for g in range(n_parts):
            check(ranks[g], *exps[g])
    else:
        exp, pl = oracle.expected_pool(shards, recs, mode, oflags)
        pools = Pools(n_parts, len(exp))  # every rank's launch stores into all N pools (the fused fan-out)
        for g in range(n_parts):
            play_part(L, plan, g, pools)
        check(pools, exp, pl)
    return plan, (tuple(x.tiles) if x else (0, 0))


def test_llama_bf16_bulk_store_path_single_broadcast_scatter(emul, tmp_path):
    d = str(tmp_path / "llama")
    synth.make_llama(d, dict(hidden=256, ffn=704, layers=2, kv_dim=64, vocab=1000), max_shard_bytes=2_500_000)
    replay(emul, d)
    replay(emul, d, mode=gpupool.MODE_BROADCAST, n_parts=4)
    replay(emul, d, mode=gpupool.MODE_SCATTER, n_parts=4)  # column slices: thousands of short runs per chunk


def test_mixed_safetensors_casts_tails_and_misaligned_payloads(emul, tmp_path):
    for pad in (True, False):
        p = str(tmp_path / f"m{int(pad)}.safetensors")
        tensors = [("a", "BF16", [7]), ("b", "BF16", [33, 77]), ("c", "F32", [129, 65]), ("d", "F16", [7, 1001]), ("e", "U8", [3]), ("f", "BF16", [4099]),
                   ("g", "F32", [5]), ("h", "F16", [2, 3]), ("i", "U8", [1021]), ("j", "BF16", [64, 512]), ("k", "F8_E4M3", [300, 70]), ("l", "F8_E5M2", [37])]
        synth.write_safetensors(p, tensors, 5, pad_header=pad)
        replay(emul, p)
        replay(emul, p, flags=gpupool.LOAD_KEEP_F32 | gpupool.LOAD_F8_TO_BF16, mode=gpupool.MODE_BROADCAST, n_parts=3)
    replay(emul, os.path.join(G, "st_mixed.safetensors"))
    replay(emul, os.path.join(G, "sharded"))


def test_every_gguf_block_type_through_whole_launches(emul, tmp_path):
    from tests.test_plan import f4_tensors, q4km_tensors
    p = str(tmp_path / "q4km.gguf")
    synth.write_gguf(p, q4km_tensors(), 9)
    replay(emul, p)
    replay(emul, p, mode=gpupool.MODE_BROADCAST, n_parts=2)
    p = str(tmp_path / "f4.gguf")
    synth.write_gguf(p, f4_tensors(hidden=256, ffn=768, layers=1, vocab=512), 11)
    replay(emul, p)
    replay(emul, p, mode=gpupool.MODE_SCATTER, n_parts=2)
    p = str(tmp_path / "a8.gguf")  # general.alignment = 8: block payloads 8 bytes off a 16-byte boundary in the stage
    synth.write_gguf(p, [("pad.weight", "F32", [4])] + f4_tensors(hidden=256, ffn=512, layers=1, vocab=256), 21, alignment=8)
    replay(emul, p)
    for g in ("q4k.gguf", "q4km_mix.gguf", "quants_f4.gguf", "quants_cb.gguf", "quants_iq.gguf"):
        replay(emul, os.path.join(G, g))


def test_transpose_tiles_through_whole_launches(emul, tmp_path):
    """GPT-2 Conv1D transposes replayed tile for tile: every dtype, rows wider than one tile (3096 / 4128 columns), destination rows that are not 16-byte
    multiples (d = 41, 43 -> scalar stores), an unpadded header (rows not 16-byte aligned -> the consumers' gather fallback), 4-byte outputs
    (KEEP_F32), and a three-way fan-out."""
    T = gpupool.LOAD_GPT2_CONV1D_T
    tr = {helpers.OP_T_F32_BF16, helpers.OP_T_F16_BF16, helpers.OP_T_B16, helpers.OP_T_B32}
    for dt, d, pad in (("F32", 96, True), ("F16", 40, True), ("BF16", 40, True), ("F32", 72, False), ("BF16", 264, True),
                       ("F32", 41, True), ("F16", 43, True)):
        p = str(tmp_path / f"gpt2_{dt}_{d}_{int(pad)}.safetensors")
        synth.write_safetensors(p, [("x", "U8", [3])] + synth.gpt2_tensors(n_layer=1, d=d, vocab=50, n_pos=8, dtype=dt), 3, pad_header=pad)
        plan, _ = replay(emul, p, flags=T)
        assert {sg["op"] for ch in plan["parts"][0]["chunks"] for sg in ch["segs"]} & tr
    # rows wider than one tile: 3096 and 4128 columns are cut into equal pieces (a whole d = 1032 layer is 50 MB of pools and hit maps; 72 rows of it do)
    p = str(tmp_path / "gpt2_wide.safetensors")
    synth.write_safetensors(p, [("h.0.attn.c_attn.weight", "F32", [72, 3096]), ("h.0.mlp.c_fc.weight", "F32", [72, 4128]), ("h.0.mlp.c_proj.weight", "F16", [4128, 72])], 3)
    plan, _ = replay(emul, p, flags=T)
    assert {sg["op"] for ch in plan["parts"][0]["chunks"] for sg in ch["segs"]} & tr
    p = str(tmp_path / "gpt2_b.safetensors")
    synth.make_gpt2(p, n_layer=2, d=96, vocab=301, n_pos=40)
    replay(emul, p, flags=T, mode=gpupool.MODE_BROADCAST, n_parts=3)
    replay(emul, p, flags=T | gpupool.LOAD_KEEP_F32)


def test_scatter_row_exchange_through_whole_launches(emul, tmp_path):
    """KK_LOAD_SCATTER_EXCHANGE, every rank replayed: the ROWSPLIT tiles of rank i deal every row's column slices to all n pools, through
    the bulk-store pieces (bulk == 3) where the geometry is 16-byte aligned and the byte-granular consumer elsewhere.  Llama shapes (all
    aligned), then a file of odd shapes padded and unpadded at n = 2..8, with 1 MB chunks and the smallest the planner accepts (64 KB), which
    split pieces mid-row.  The tiles of each class that ran must be those the plan calls for, and both classes must run where the shapes ask."""
    X = gpupool.LOAD_SCATTER_EXCHANGE
    d = str(tmp_path / "llama")
    synth.make_llama(d, dict(hidden=512, ffn=1408, layers=2, kv_dim=128, vocab=2048), max_shard_bytes=6_000_000)
    for n in (2, 4, 8):
        for chunk in (8 * MB, 64 * 1024):
            plan, tiles = replay(emul, d, mode=gpupool.MODE_SCATTER, flags=X, n_parts=n, chunk=chunk)
            assert tiles == helpers.rowsplit_tile_classes(plan) and tiles[0] > 0, (n, chunk, tiles)
    for pad in (True, False):
        p = str(tmp_path / f"odd{int(pad)}.safetensors")
        synth.write_safetensors(p, helpers.ROWSPLIT_ODD_TENSORS, 3, pad_header=pad)
        for n in (2, 3, 4, 5, 6, 8):
            for chunk in (1 * MB, 64 * 1024):
                plan, tiles = replay(emul, p, mode=gpupool.MODE_SCATTER, flags=X, n_parts=n, chunk=chunk)
                assert tiles == helpers.rowsplit_tile_classes(plan), (pad, n, chunk, tiles)
                assert tiles[1] > 0 and (tiles[0] > 0 or n == 6), (pad, n, chunk, tiles)  # n = 6: no slice is a multiple of 16 bytes
                if chunk < MB:
                    assert any(sg["op"] == helpers.OP_ROWSPLIT and sg["p3"] % sg["p0"] for part in plan["parts"] for ch in part["chunks"] for sg in ch["segs"])


def test_the_replay_notices_a_wrong_row_split_plan(emul, tmp_path):
    """Liveness of the exchange replay: a ROWSPLIT segment with a wrong slice width (p1) or first row (p2) must fail it."""
    p = str(tmp_path / "odd.safetensors")
    synth.write_safetensors(p, helpers.ROWSPLIT_ODD_TENSORS, 3)
    X, n = gpupool.LOAD_SCATTER_EXCHANGE, 4
    for field, delta in (("p1", 16), ("p1", -16), ("p2", 1), ("p2", -1)):
        for bulk in (True, False):  # a segment with 16-byte slices (bulk-store pieces), and one without (the byte-granular consumer)
            plan = gpupool.plan_describe(p, mode=gpupool.MODE_SCATTER, flags=X, n_parts=n, chunk_bytes=1 * MB)
            segs = [sg for sg in plan["parts"][1]["chunks"][0]["segs"] if sg["op"] == helpers.OP_ROWSPLIT and (sg["p1"] % 16 == 0) == bulk and sg["p2"] > 0]
            segs[0][field] += delta
            with pytest.raises(AssertionError):
                replay(emul, p, mode=gpupool.MODE_SCATTER, flags=X, n_parts=n, plan=plan)


def test_the_replay_notices_a_wrong_plan(emul, tmp_path):
    """Liveness of the checker: a segment table whose tile_begin skips a tile, and a chunk that is shorter than its segments say."""
    p = str(tmp_path / "m.safetensors")
    synth.write_safetensors(p, [("a", "F32", [4096, 9])], 1)
    plan = gpupool.plan_describe(p, chunk_bytes=1 * MB)
    shards, recs = oracle.index_path(p)
    exp, pl = oracle.expected_pool(shards, recs)
    ch = plan["parts"][0]["chunks"][0]
    raw = np.fromfile(plan["shards"][0], np.uint8)
    buf = np.zeros(ch["buf_bytes"], np.uint8)
    for fo, ln, bo in ch["reads"]:
        buf[bo:bo + ln] = raw[fo:fo + ln]
    s = ch["segs"][0]
    seg = (KKSeg * 1)(KKSeg(s["src_off"], s["dst_off"], s["units"], s["op"], 1, 0, 0, 0, 0))  # first tile has no segment
    pools = Pools(1, len(exp))
    assert emul.kk_emul_launch(buf.ctypes.data, buf.size, seg, 1, ch["n_tiles"], 0, pools.ptrs, 1, len(exp), pools.hits.ctypes.data, pools.m2.ctypes.data, pools.m1.ctypes.data, *NO_EXCHANGE, None, None) == 9
    seg = (KKSeg * 1)(KKSeg(s["src_off"], s["dst_off"], s["units"], s["op"], 0, 0, 0, 0, 0))
    pools = Pools(1, len(exp))
    assert emul.kk_emul_launch(buf.ctypes.data, buf.size // 2, seg, 1, ch["n_tiles"], 0, pools.ptrs, 1, len(exp), pools.hits.ctypes.data, pools.m2.ctypes.data, pools.m1.ctypes.data, *NO_EXCHANGE, None, None) == 11


# ---- property tests: random inventories through whole launches of the device code ---------------------------------------------------------
from hypothesis import HealthCheck, given, settings, strategies as st  # noqa: E402

from tests.test_plan_property import gguf_inventories, inventories  # noqa: E402


@settings(max_examples=int(os.environ.get("KK_HYP_EXAMPLES", 120)), deadline=None, suppress_health_check=[HealthCheck.too_slow, HealthCheck.function_scoped_fixture])
@given(inv=inventories(), mode=st.sampled_from([0, 1, 2]), n_parts=st.integers(1, 6), pad=st.booleans(),
       flags=st.sampled_from([0, 2, 16, 18, 33, 35, 49, 65, 67, 81, 8, 10, 24, 26, 41, 43, 57, 73, 75, 89]))  # each set also with the row exchange (8)
def test_random_safetensors_inventories_replayed_through_the_device_code(emul, inv, mode, n_parts, pad, flags):
    import tempfile
    if mode == 0:
        n_parts = 1
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.safetensors")
        synth.write_safetensors(p, inv, seed=7, pad_header=pad)
        replay(emul, p, mode=mode, flags=flags, n_parts=n_parts)


@settings(max_examples=int(os.environ.get("KK_HYP_EXAMPLES", 120)), deadline=None, suppress_health_check=[HealthCheck.too_slow, HealthCheck.function_scoped_fixture])
@given(inv=gguf_inventories(), mode=st.sampled_from([0, 1, 2]), n_parts=st.integers(1, 6), alignment=st.sampled_from([8, 32, 64]))
def test_random_gguf_inventories_replayed_through_the_device_code(emul, inv, mode, n_parts, alignment):
    import tempfile
    if mode == 0:
        n_parts = 1
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.gguf")
        synth.write_gguf(p, inv, seed=8, alignment=alignment)
        replay(emul, p, mode=mode, n_parts=n_parts)
