"""GPU parity for the §8(f4) quant types (Q4_0, Q4_1, Q5_0, Q5_1, Q2_K, Q3_K, Q5_K, the codebook and lattice i-quants, ternary types, MXFP4 / NVFP4,
FP8 widening), the transposing loads and KK_FANOUT_PULL / KK_FANOUT_NVLS, through the C ABI, bit for bit against the oracle and against the
committed gguf-py fixtures.  Error paths live in tests/test_zz_gpu_errors.py (sorted last); the Q4_K_M mixes (Q6_K / Q8_0) are at the
front of tests/test_gpu_load.py."""
import os

import numpy as np
import pytest

from kukeon_b200 import gpupool
from oracle import oracle
from tests import helpers
from tests.test_gpu_load import _virtual_ranks, assert_pool_matches, expected_exact, load_and_check, poison_all
from tests.test_plan import F4_MIX, f4_tensors
from tools import synth

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MB = 1 << 20


@pytest.mark.parametrize("fixture", ["quants_f4.gguf", "quants_cb.gguf", "quants_iq.gguf"])
def test_golden_fixture_values_vs_gguf_py(pool, fixture):
    g = os.path.join(G, fixture)
    load_and_check(pool, g)
    outs = np.load(g + ".bf16.npz")
    m = pool.load(g)
    try:
        for name in outs.files:
            pl = m.placements(name)[0]
            assert pl.dtype == "BF16" and np.array_equal(m.read(0, pl.pool_offset, pl.nbytes).view(np.uint16), outs[name]), name
    finally:
        m.release()


@pytest.mark.parametrize("dtype", F4_MIX)
def test_one_type_multi_tile_and_ragged(pool, tmp_path, dtype):
    """Per type: one tensor of 2.4 tiles, one of a single block row, one ragged count that ends mid warp-iteration."""
    nel = oracle.BLOCK_QUANTS[dtype][0]
    p = str(tmp_path / f"{dtype}.gguf")
    synth.write_gguf(p, [("blk.0.ffn_up.weight", dtype, [137, 16 * nel if nel == 256 else 137 * nel]), ("blk.0.attn_q.weight", dtype, [1, nel]),
                         ("blk.0.attn_k.weight", dtype, [3, 7 * nel]), ("blk.0.attn_norm.weight", "F32", [5])], 31)
    load_and_check(pool, p)


def test_llama_shaped_mix_of_every_type(pool, tmp_path):
    p = str(tmp_path / "f4.gguf")
    synth.write_gguf(p, f4_tensors(hidden=512, ffn=1536, layers=2, vocab=1024), 11)
    st = load_and_check(pool, p)
    assert st["n_tensors"] == 2 * 21 + 3


def a8_file(path):
    """general.alignment = 8 with a leading pad tensor sized so that every quantised tensor starts 8 bytes off a 16-byte boundary."""
    for pad_elems in (2, 4):
        tensors = [("pad.weight", "F32", [pad_elems])] + f4_tensors(hidden=256, ffn=512, layers=1, vocab=256) + [("tail.weight", "F16", [3])]
        synth.write_gguf(path, tensors, 21, alignment=8)
        recs = gpupool.index(path)
        if {r["dtype"] for r in recs if r["file_offset"] % 16 == 8} >= set(F4_MIX):
            return recs
    raise AssertionError("could not place the quantised tensors off a 16-byte boundary")


def test_alignment_8_feeds_the_byte_assembled_loads(pool, tmp_path):
    """Blocks that start 8 bytes off a 16-byte boundary: lds32_any's 16-bit and byte paths run for every type."""
    p = str(tmp_path / "a8.gguf")
    a8_file(p)
    load_and_check(pool, p)


def test_small_chunks_split_tensors_across_launches(native, tmp_path):
    p = str(tmp_path / "f4.gguf")
    synth.write_gguf(p, f4_tensors(hidden=512, ffn=1536, layers=2, vocab=1024), 12)
    with gpupool.Pool([0], n_staging_buffers=4, staging_buffer_bytes=1 * MB, n_reader_threads=2) as pl:
        st = load_and_check(pl, p)
        assert st["parts"][0]["chunks"] >= 2


def test_scatter_keeps_whole_rows_of_blocks(native, tmp_path):
    """Virtual ranks on one GPU: every rank's pool equals the oracle's slice pool (dim-0 slices of block-quantised tensors)."""
    p = str(tmp_path / "f4.gguf")
    synth.write_gguf(p, f4_tensors(hidden=256, ffn=768, layers=1, vocab=512), 13)
    shards, recs = oracle.index_path(p)
    with gpupool.Pool([0], n_staging_buffers=4, staging_buffer_bytes=2 * MB, n_reader_threads=2) as pl:
        for part in range(4):
            m = pl.load(p, mode=gpupool.MODE_SCATTER, part_index=part, part_count=4)
            try:
                assert_pool_matches(m, 0, shards, recs, mode=gpupool.MODE_SCATTER, n_parts=4, part=part)
            finally:
                m.release()


def test_fp8_safetensors_verbatim_by_default_and_widened_on_request(pool, tmp_path):
    """F8_E4M3 / F8_E5M2: bytes kept by default; KK_LOAD_F8_TO_BF16 widens exactly (cvt.rn.f16x2.e4m3x2 path), all 256 patterns present,
    sizes that end inside a 16-element group, a header that leaves the data off 16-byte alignment."""
    for pad in (True, False):
        p = str(tmp_path / f"fp8_{int(pad)}.safetensors")
        t = [("a.weight", "F8_E4M3", [300, 512]), ("a.weight_scale_inv", "F32", [3, 4]), ("b.weight", "F8_E5M2", [129, 65]), ("c.weight", "F8_E4M3", [7]),
             ("d.weight", "BF16", [33, 77]), ("e.weight", "F8_E4M3", [40000]), ("f.weight", "F8_E5M2", [3, 5, 7])]
        synth.write_safetensors(p, t, 23, pad_header=pad)
        raw = synth.gen_bytes("F8_E4M3", 300 * 512, 23, 0)
        assert len(set(raw.tolist())) == 256
        load_and_check(pool, p)
        load_and_check(pool, p, flags=gpupool.LOAD_F8_TO_BF16)
        m = pool.load(p, flags=gpupool.LOAD_F8_TO_BF16)
        try:
            assert m.placements("a.weight")[0].dtype == "BF16" and m.placements("a.weight")[0].nbytes == 300 * 512 * 2
        finally:
            m.release()


# ---- 2-D transposes (GPT-2 Conv1D; 8-row tiles) ----------------------------------------------------------------------------------------
T = gpupool.LOAD_GPT2_CONV1D_T


def test_gpt2_transposes_every_dtype_and_odd_shapes(pool, tmp_path):
    """Bit for bit vs the oracle: GPT-2 shaped (R = 96..384: staged path, whole-row tiles of one bulk copy), rows wider than one tile
    (d = 1032: 3096-column c_attn rows cut into equal pieces), 16-bit sources, shapes whose R is not a multiple of 8 (scalar stores),
    4-byte outputs (KEEP_F32), and an unpadded header (rows off 16-byte alignment -> gather fallback)."""
    p = str(tmp_path / "gpt2.safetensors")
    synth.make_gpt2(p, n_layer=2, d=96, vocab=301, n_pos=40)
    load_and_check(pool, p, flags=T)
    load_and_check(pool, p, flags=T | gpupool.LOAD_KEEP_F32)
    for dt, d in (("F16", 40), ("BF16", 40), ("F32", 41), ("F16", 43), ("F32", 1032), ("BF16", 1032)):
        q = str(tmp_path / f"gpt2_{dt}_{d}.safetensors")
        synth.write_safetensors(q, synth.gpt2_tensors(n_layer=1, d=d, vocab=50, n_pos=8, dtype=dt), 3)
        load_and_check(pool, q, flags=T)
    q = str(tmp_path / "gpt2_f32_1032_keep.safetensors")
    synth.write_safetensors(q, synth.gpt2_tensors(n_layer=1, d=1032, vocab=50, n_pos=8, dtype="F32"), 3)
    load_and_check(pool, q, flags=T | gpupool.LOAD_KEEP_F32)
    for pad in (False, True):
        q = str(tmp_path / f"unpadded_{int(pad)}.safetensors")
        synth.write_safetensors(q, [("x", "U8", [3])] + synth.gpt2_tensors(n_layer=1, d=72, vocab=20, n_pos=8, dtype="F32"), 4, pad_header=pad)
        load_and_check(pool, q, flags=T)


def test_full_size_gpt2_transposed_vs_numpy(pool, tmp_path):
    """GPT-2-small at full size (0.5 GB): every transposed tensor against a numpy transpose of the oracle's RNE cast, every other tensor
    against the oracle's checksum."""
    p = str(tmp_path / "gpt2_full.safetensors")
    synth.make_gpt2(p)
    shards, recs = oracle.index_path(p)
    m = pool.load(p, flags=T)
    try:
        for r in recs:
            pl = m.placements(r["name"])[0]
            raw = np.fromfile(shards[0], np.uint8, r["nbytes"], offset=r["file_offset"]).view("<u4")
            want = oracle.f32_bits_to_bf16(raw)
            if r["name"].endswith(("attn.c_attn.weight", "attn.c_proj.weight", "mlp.c_fc.weight", "mlp.c_proj.weight")):
                want = np.ascontiguousarray(want.reshape(r["shape"]).T)
                assert pl.shape == r["shape"][::-1], r["name"]
            assert m.checksum(0, pl.pool_offset, pl.nbytes) == oracle.checksum(want.reshape(-1).view(np.uint8)), r["name"]
    finally:
        m.release()


def test_transposes_virtual_rank_fan_out(pool, tmp_path):
    """The transposing tiles through the n-destination store ladder (broadcast to 4 virtual ranks on one GPU)."""
    from tests.test_gpu_load import _virtual_ranks
    f = str(tmp_path / "gpt2.safetensors")
    synth.make_gpt2(f, n_layer=2, d=96, vocab=301, n_pos=40)
    shards, recs = oracle.index_path(f)
    ms = _virtual_ranks(pool, f, gpupool.MODE_BROADCAST, 4, T)
    try:
        for m in ms:
            m.load_part()
        for m in ms:
            assert_pool_matches(m, 0, shards, recs, flags=gpupool.LOAD_GPT2_CONV1D_T)
    finally:
        for m in ms:
            m.release()


# ---- KK_FANOUT_PULL: one-process-per-GPU broadcast where peers map only 1/N slice buffers (first hardware run) --------------------------
def _pull_ranks(pool, path, n, flags=0):
    import ctypes as C
    ms = [pool.load(path, mode=gpupool.MODE_BROADCAST, fanout=gpupool.FANOUT_PULL, flags=flags | gpupool.LOAD_DEFER, part_index=i, part_count=n) for i in range(n)]
    ptrs = [m.export_buffer(0, gpupool.BUF_SLICE_PTR) for m in ms]  # raw device pointer in the first 8 bytes
    assert all(int.from_bytes(p[:8], "little") for p in ptrs)
    for i, m in enumerate(ms):
        for j in range(n):
            if j != i:
                m.peer_attach_buffer(j, gpupool.BUF_SLICE_PTR, ptrs[j])
    return ms


@pytest.mark.parametrize("n", [2, 4, 8])
def test_pull_fan_out_virtual_ranks_on_one_gpu(pool, tmp_path, n):
    """n ranks hosted by one process on one GPU (slice buffers attached by raw pointer): stage 1 on every rank, then stage 2 — every
    pool must equal the oracle's; stage 1 alone leaves a rank with only its own part and `loaded` false."""
    from tests.test_plan import q4km_tensors
    d = str(tmp_path / "llama")
    synth.make_llama(d, dict(hidden=256, ffn=704, layers=2, kv_dim=64, vocab=3000), max_shard_bytes=3_000_000)
    g = str(tmp_path / "q4km.gguf")
    synth.write_gguf(g, q4km_tensors(), 9)
    for path in (d, g):
        shards, recs = oracle.index_path(path)
        ms = _pull_ranks(pool, path, n)
        exp, mask = expected_exact(shards, recs)
        name = os.path.basename(path)

        def check(fills, what):
            # Stage 2 copies each peer's whole pool range [pool_lo, pool_hi) from its slice buffer, gaps between placements included, and
            # nothing ever writes a slice buffer's gap bytes: inside the peers' ranges (not the rank's own) the gaps may change.  That is
            # the only exception; every placement and every other gap byte is checked.
            ranges = [next((q["pool_lo"], q["pool_hi"]) for q in m.stats()["parts"]) for m in ms]
            for i, m in enumerate(ms):
                peer_range = np.zeros(len(exp), bool)
                for j, (lo, hi) in enumerate(ranges):
                    if j != i:
                        peer_range[lo:hi] = True
                helpers.assert_pool_exact(m, 0, exp, mask, fills[i], f"{name} PULL rank {i} of {n}, {what}", may_rewrite=peer_range & ~mask)

        try:
            fills = poison_all(ms)
            for m in ms:
                m.load_part()
                assert not m.info()["loaded"]
            for m in ms:
                assert m.convert_local() >= 0.0
                assert m.info()["loaded"]
            if ms[0].stats()["parts"] and ms[1].stats()["parts"][0]["out_bytes"] >= 4096:
                assert ms[0].probe_peer(1, gpupool.BUF_SLICE, 1 << 20) > 0.0  # copy-engine read of rank 1's attached slice buffer (here: the same GPU)
            check(fills, "streaming load")
            for m in ms:  # again through the resident image (what bench.py times)
                m.stage_resident()
            fills = poison_all(ms)
            for m in ms:
                m.convert_resident()
            for m in ms:
                m.convert_local()
            check(fills, "resident")
        finally:
            for m in ms:
                m.release()


def _pull_rank_main(rank, world, port, path, out_dir):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.cuda.set_device(rank)
        from kukeon_b200 import gpupool as gp
        from oracle import oracle as orc
        shards, recs = orc.index_path(path)
        with gp.Pool([rank], n_staging_buffers=2, staging_buffer_bytes=1 << 20, n_reader_threads=1) as pl:
            m = pl.load(path, mode=gp.MODE_BROADCAST, fanout=gp.FANOUT_PULL, flags=gp.LOAD_DEFER, part_index=rank, part_count=world)
            try:
                hs = [None] * world
                dist.all_gather_object(hs, m.export_buffer(rank, gp.BUF_SLICE))
                for r, hh in enumerate(hs):
                    if r != rank:
                        m.peer_attach_buffer(r, gp.BUF_SLICE, hh)
                dist.barrier()
                m.load_part()
                dist.barrier()
                m.convert_local()
                exp, plan = orc.expected_pool(shards, recs, 1, 0)
                got = m.read(rank, 0, len(exp))
                for p in plan:
                    a, b = p["pool_offset"], p["pool_offset"] + p["nbytes"]
                    assert np.array_equal(got[a:b], exp[a:b]), f"rank {rank} PULL: {p['name']} differs"
                dist.barrier()
                m.peer_detach_all()
            finally:
                m.release()
        open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
def test_pull_one_process_per_gpu_over_ipc(native, tmp_path):
    import torch
    import torch.multiprocessing as mp
    from tests.test_gpu_multi import _free_port
    ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if ngpu < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if ngpu < 4 else 4
    d = str(tmp_path / "llama")
    synth.make_llama(d, dict(hidden=256, ffn=704, layers=3, kv_dim=64, vocab=3000), max_shard_bytes=3_000_000)
    out = str(tmp_path / "out")
    os.makedirs(out)
    mp.spawn(_pull_rank_main, args=(world, _free_port(), d, out), nprocs=world, join=True)
    assert sorted(os.listdir(out)) == [f"ok{r}" for r in range(world)]


# ---- KK_FANOUT_NVLS: multimem.st through an NVSwitch multicast object (one process, >= 2 GPUs; skipped where the host has no NVLS) --------
@pytest.mark.multigpu
def test_nvls_broadcast_single_process(native, tmp_path):
    import torch
    ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if ngpu < 2:
        pytest.skip("needs >= 2 GPUs")
    n = min(ngpu, 8)
    d = str(tmp_path / "llama")
    synth.make_llama(d, dict(hidden=256, ffn=704, layers=3, kv_dim=64, vocab=3000), max_shard_bytes=3_000_000)
    g = str(tmp_path / "mix.gguf")
    synth.write_gguf(g, synth.mixtral_gguf_tensors(hidden=256, ffn=768, layers=2, experts=2, vocab=512, kv_dim=256), 7)
    odd = str(tmp_path / "odd.safetensors")
    synth.write_safetensors(odd, [("a", "BF16", [7])], 1)  # 14 bytes: not a whole 16-byte vector
    with gpupool.Pool(list(range(n)), n_staging_buffers=4, staging_buffer_bytes=1 * MB, n_reader_threads=2) as pl:
        try:
            m = pl.load(d, mode=gpupool.MODE_BROADCAST, fanout=gpupool.FANOUT_NVLS)
        except gpupool.ErrUnsupported as e:
            pytest.skip(f"host does not expose NVLS: {e}")
        try:
            shards, recs = oracle.index_path(d)
            for dev in range(n):
                assert_pool_matches(m, dev, shards, recs)
            assert len({m.checksum(dev, 0, m.info()["pool_bytes"] // 8 * 8) for dev in range(n)}) == 1
            with pytest.raises(gpupool.ErrUnsupported, match="cudaIpcMemHandle"):
                m.export(0)
            m.stage_resident()
            fills = [helpers.poison(m, dev) for dev in range(n)]
            m.convert_resident()
            exp, mask = expected_exact(shards, recs)
            for dev in range(n):
                helpers.assert_pool_exact(m, dev, exp, mask, fills[dev], f"NVLS device {dev}, resident")
        finally:
            m.release()
        m = pl.load(g, mode=gpupool.MODE_BROADCAST, fanout=gpupool.FANOUT_NVLS)
        try:
            shards, recs = oracle.index_path(g)
            for dev in range(n):
                assert_pool_matches(m, dev, shards, recs)
        finally:
            m.release()
        with pytest.raises(gpupool.ErrUnsupported, match="16-byte"):
            pl.load(odd, mode=gpupool.MODE_BROADCAST, fanout=gpupool.FANOUT_NVLS)
    with gpupool.Pool([0], n_staging_buffers=2, staging_buffer_bytes=1 * MB, n_reader_threads=1) as one:
        with pytest.raises(gpupool.ErrUnsupported, match="at least two devices"):
            one.load(d, mode=gpupool.MODE_BROADCAST, fanout=gpupool.FANOUT_NVLS)
