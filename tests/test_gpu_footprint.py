"""Whole-pool footprints over poisoned pools: every byte a launch should write holds the oracle's value, every other byte still holds the
random poison written before it.  Covers what only the GPU runs: the fan-out's per-rank stores into peer pools, the scheduler counters
that back-to-back launches share, and the device bindings of every block dequantiser on fully random block bytes."""
import os

import numpy as np
import pytest

from kukeon_b200 import gpupool
from oracle import oracle
from tests import helpers
from tests.test_gpu_load import _virtual_ranks, expected_exact, load_and_check, poison_all
from tools import synth

MB = 1 << 20
SLOT = 2 * MB  # staging slots of the footprint pool: small chunks, so that the checkpoints below give every rank some of them


@pytest.fixture(scope="module")
def slot_pool(native):
    with gpupool.Pool([0], n_staging_buffers=4, staging_buffer_bytes=SLOT, n_reader_threads=2) as p:
        yield p


# ---- the checker itself (CPU) -----------------------------------------------------------------------------------------------------------
def test_checker_names_each_class_of_difference():
    rng = np.random.default_rng(5)
    placements = [("a", 0, 100), ("b", 256, 50)]
    exp = rng.integers(0, 256, 512, dtype=np.uint8)
    fill = (exp + rng.integers(1, 256, 512, dtype=np.uint8)).astype(np.uint8)  # differs from exp everywhere
    mask = helpers.expected_mask([{"pool_offset": a, "nbytes": n} for _, a, n in placements], 512)
    good = np.where(mask, exp, fill)
    helpers.check_pool_bytes(good, exp, mask, fill, placements, "clean")

    got = good.copy()
    got[150] ^= 1             # a store into the padding between a and b
    got[10] = fill[10]        # a byte of a nobody wrote
    got[260] = exp[260] ^ 0x80 if exp[260] ^ 0x80 != fill[260] else exp[260] ^ 0x40  # a wrong value in b
    got[400:403] ^= 0xFF      # stores past the last placement
    with pytest.raises(helpers.PoolMismatch) as e:
        helpers.check_pool_bytes(got, exp, mask, fill, placements, "fake")
    assert e.value.findings == [("unwritten", "a", 10, 1), ("stray store", "gap between a and b", 150, 1),
                                ("wrong value", "b", 260, 1), ("stray store", "tail after b", 400, 3)]
    assert "gap between a and b" in str(e.value) and str(e.value).startswith("fake:")

    allow = np.zeros(512, bool)
    allow[100:256] = True     # a rewrite the caller allows (PULL's gaps) is no finding; the others still are
    with pytest.raises(helpers.PoolMismatch) as e:
        helpers.check_pool_bytes(got, exp, mask, fill, placements, "fake", may_rewrite=allow)
    assert [f[0] for f in e.value.findings] == ["unwritten", "wrong value", "stray store"]

    only_b = mask.copy()
    only_b[:256] = False
    lead = np.where(only_b, exp, fill)
    lead[0] ^= 1
    with pytest.raises(helpers.PoolMismatch) as e:  # a store before the first placement
        helpers.check_pool_bytes(lead, exp, only_b, fill, [("b", 256, 50)], "lead")
    assert e.value.findings == [("stray store", "gap before b", 0, 1)]


@pytest.mark.gpu
def test_checker_reports_a_pool_nobody_converted(pool, tmp_path):
    p = str(tmp_path / "m.safetensors")
    helpers.mixed_safetensors(p)
    shards, recs = oracle.index_path(p)
    exp, mask = expected_exact(shards, recs)
    m = pool.load(p, flags=gpupool.LOAD_DEFER)
    try:
        assert m.pool_ptr(0)[1] == oracle.plan_pool(recs)[1] == len(exp)
        fill = helpers.poison(m, 0)
        with pytest.raises(helpers.PoolMismatch) as e:
            helpers.assert_pool_exact(m, 0, exp, mask, fill, "never converted")
        assert {f[0] for f in e.value.findings} == {"unwritten"}
        assert sum(f[3] for f in e.value.findings) > 0.99 * mask.sum()
    finally:
        m.release()


# ---- per-rank footprint of the fan-out (virtual ranks on one GPU) -----------------------------------------------------------------------
def _footprints(path, mode, flags, n):
    """foot[r][k]: (bytes, mask) rank r's launches store into rank k's pool, from helpers.emulate_part on the plan the pool runs."""
    plan = gpupool.plan_describe(path, mode=mode, flags=flags, n_parts=n, chunk_bytes=SLOT)
    size = [plan["layouts"][k if mode == gpupool.MODE_SCATTER else 0]["pool_bytes"] for k in range(n)]
    foot = []
    for r in range(n):
        if mode == gpupool.MODE_BROADCAST:
            foot.append([helpers.emulate_part(plan, r, size[0])] * n)
            continue
        ex = {k: (np.zeros(size[k], np.uint8), np.zeros(size[k], bool)) for k in range(n)}
        own, own_mask = helpers.emulate_part(plan, r, size[r], exchange=ex)
        ex[r][0][own_mask] = own[own_mask]
        ex[r][1][own_mask] = True
        foot.append([ex[k] for k in range(n)])
    return plan, foot


def _rank_by_rank(pool, path, mode, flags, n, oracle_flags=0):
    """Poison all n pools, run one rank at a time and check every pool after each: it holds exactly the footprints of the ranks run so
    far.  Once for the streaming load, once for the resident conversion."""
    name = os.path.basename(path)
    plan, foot = _footprints(path, mode, flags, n)
    shards, recs = oracle.index_path(path)
    ms = _virtual_ranks(pool, path, mode, n, flags)
    try:
        for phase in ("load_part", "convert_resident"):
            if phase == "convert_resident":
                for m in ms:
                    m.stage_resident()
            fills = poison_all(ms)
            exp = [np.zeros(len(f), np.uint8) for f in fills]
            mask = [np.zeros(len(f), bool) for f in fills]
            for r in range(n):
                getattr(ms[r], phase)()
                for k in range(n):
                    b, w = foot[r][k]
                    exp[k][w] = b[w]
                    mask[k] |= w
                for k in range(n):
                    helpers.assert_pool_exact(ms[k], 0, exp[k], mask[k], fills[k], f"{name}: {phase} of ranks 0..{r} of {n}, pool {k}")
            if phase == "load_part":
                ran = [next((q["chunks"], q["tiles"]) for q in m.stats()["parts"]) for m in ms]
                assert ran == [(len(q["chunks"]), sum(c["n_tiles"] for c in q["chunks"])) for q in plan["parts"]], "the load ran another plan"
            for k in range(n):  # all ranks together: the oracle's pool
                want, want_mask = expected_exact(shards, recs, mode, oracle_flags, n if mode == gpupool.MODE_SCATTER else 1, k)
                assert (mask[k] == want_mask).all() and (exp[k][want_mask] == want[want_mask]).all(), (name, phase, k)
    finally:
        for m in ms:
            m.release()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_broadcast_footprint_rank_by_rank(slot_pool, tmp_path, n):
    from tests.test_plan import q4km_tensors
    d = str(tmp_path / "llama")
    synth.make_llama(d, dict(hidden=256, ffn=704, layers=4, kv_dim=64, vocab=4000), max_shard_bytes=3_000_000)
    g = str(tmp_path / "q4km.gguf")
    synth.write_gguf(g, q4km_tensors(hidden=1024, ffn=2816, layers=2, vocab=2048), 9)
    f = str(tmp_path / "gpt2.safetensors")
    synth.make_gpt2(f, n_layer=2, d=256, vocab=2000, n_pos=64)
    mixed = str(tmp_path / "mixed.safetensors")
    helpers.mixed_safetensors(mixed, pad_header=False)
    T = gpupool.LOAD_GPT2_CONV1D_T
    for path, flags in ((d, 0), (g, 0), (f, T), (mixed, 0)):
        _rank_by_rank(slot_pool, path, gpupool.MODE_BROADCAST, flags, n, oracle_flags=flags)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_scatter_exchange_footprint_rank_by_rank(slot_pool, tmp_path, n):
    for pad in (True, False):
        p = str(tmp_path / f"odd{int(pad)}.safetensors")
        synth.write_safetensors(p, helpers.ROWSPLIT_ODD_TENSORS, 3, pad_header=pad)
        _rank_by_rank(slot_pool, p, gpupool.MODE_SCATTER, gpupool.LOAD_SCATTER_EXCHANGE, n)


# ---- back-to-back launches of different models on one stream ----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("other", ["q4k_gguf", "gpt2_transposed"])
def test_back_to_back_launches_across_models(native, tmp_path, other):
    """Every launch starts from the scheduler counters the previous launch on the device's stream left behind.  A: one bf16 shard of
    ~600 copy tiles; B: ~250 Q4_K tiles, or a GPT-2 of 69 tiles (cast and transpose), whose grid is smaller than the SM count of an H100
    (132).  A launch of more tiles than CTAs that started from stale counters would skip tiles."""
    a = str(tmp_path / "llama")
    synth.make_llama(a, dict(hidden=512, ffn=1408, layers=2, kv_dim=128, vocab=4096))
    if other == "q4k_gguf":
        b, bflags = str(tmp_path / "q4k.gguf"), 0
        synth.write_gguf(b, synth.mixtral_gguf_tensors(hidden=512, ffn=1024, layers=2, experts=4, vocab=2048, kv_dim=256), 17)
    else:
        b, bflags = str(tmp_path / "gpt2.safetensors"), gpupool.LOAD_GPT2_CONV1D_T
        synth.make_gpt2(b, n_layer=1, d=64, vocab=200, n_pos=32)
        import torch
        tiles = sum(c["n_tiles"] for c in gpupool.plan_describe(b, flags=bflags, chunk_bytes=8 * MB)["parts"][0]["chunks"])
        assert tiles < torch.cuda.get_device_properties(0).multi_processor_count, tiles
    # a context of its own: its counters start at zero, so the first launch is clean whatever ran before
    with gpupool.Pool([0], n_staging_buffers=2, staging_buffer_bytes=8 * MB, n_reader_threads=1) as pl:
        models = {}
        for key, path, flags in (("A", a, 0), ("B", b, bflags)):
            shards, recs = oracle.index_path(path)
            m = pl.load(path, flags=flags | gpupool.LOAD_DEFER)
            m.stage_resident()
            models[key] = (m, *expected_exact(shards, recs, flags=flags))
        try:
            for i, key in enumerate("ABAAAAA"):
                m, exp, mask = models[key]
                fill = helpers.poison(m, 0)
                m.convert_resident()
                helpers.assert_pool_exact(m, 0, exp, mask, fill, f"launch {i + 1} (model {key}, B = {other})")
        finally:
            for m, _, _ in models.values():
                m.release()


# ---- every block type on fully random bytes, through the device bindings ----------------------------------------------------------------
def _random_block_gguf(path, dtype, alignment, seed):
    """One tensor of 2 tiles + 37 blocks of `dtype` whose bytes are all Philox-random (scales NaN, Inf, subnormal or zero included),
    between an F32 pad tensor (sized so that at alignment 8 the blocks start 8 bytes off a 16-byte boundary) and an F16 tail."""
    op = next(o for o, t in helpers.BLOCK_DTYPE.items() if t == dtype)
    bb, _, per_tile = helpers.BLOCK_GEOM[op]
    nel = oracle.BLOCK_QUANTS[dtype][0]
    nblk = 2 * per_tile + 37
    for pad in (2, 4):
        synth.write_gguf(path, [("pad.weight", "F32", [pad]), ("blk.0.ffn_up.weight", dtype, [nblk, nel]), ("tail.weight", "F16", [3])],
                         seed, alignment=alignment)
        r = next(x for x in oracle.index_path(path)[1] if x["dtype"] == dtype)
        if alignment != 8 or r["file_offset"] % 16 == 8:
            break
    else:
        raise AssertionError("could not place the blocks 8 bytes off a 16-byte boundary")
    assert r["nbytes"] == nblk * bb
    raw = np.frombuffer(np.random.Generator(np.random.Philox(seed)).bytes(r["nbytes"]), np.uint8)
    with open(path, "r+b") as fh:
        fh.seek(r["file_offset"])
        fh.write(raw.tobytes())


@pytest.mark.gpu
@pytest.mark.parametrize("alignment", [32, 8])
@pytest.mark.parametrize("dtype", sorted(helpers.BLOCK_DTYPE.values()))
def test_every_block_type_on_random_bytes(pool, tmp_path, dtype, alignment):
    """The oracle (oracle.dequant_bf16, every NaN as 0x7FFF) against the kernel's real bindings (__half2float, cvt.rn.bf16x2.f32,
    __fmaf_rn, the FP8 pair conversion, __funnelshift_r, the __ldg codebooks), which the CPU replay replaces with its own."""
    p = str(tmp_path / f"{dtype}_a{alignment}.gguf")
    _random_block_gguf(p, dtype, alignment, seed=1000 + 7 * alignment + sorted(helpers.BLOCK_DTYPE.values()).index(dtype))
    load_and_check(pool, p)  # a plain load, then a poisoned streaming load and three poisoned resident conversions, byte for byte
