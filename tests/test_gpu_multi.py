"""Multi-GPU parity (skipped on a single-GPU box): the fused convert + P2P fan-out kernel, scatter slices,
and the one-process-per-GPU path with CUDA-IPC peer pools — every pool compared bit for bit with the oracle."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

from kukeon_b200 import gpupool
from oracle import oracle
from tests import helpers
from tools import synth

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MB = 1 << 20


def _ngpu():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


needs2 = pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")


def check_pool(m, device, shards, recs, mode=0, flags=0, n_parts=1, part=0):
    exp, plan = oracle.expected_pool(shards, recs, mode, flags, n_parts, part)
    got = m.read(device, 0, len(exp))
    for p in plan:
        a, b = p["pool_offset"], p["pool_offset"] + p["nbytes"]
        assert np.array_equal(got[a:b], exp[a:b]), f"device {device}: {p['name']} differs"


def make_mixed(tmp_path):
    d = str(tmp_path / "llama")
    synth.make_llama(d, dict(hidden=256, ffn=704, layers=3, kv_dim=64, vocab=3000), max_shard_bytes=3_000_000)
    g = str(tmp_path / "mix.gguf")
    synth.write_gguf(g, synth.mixtral_gguf_tensors(hidden=256, ffn=768, layers=2, experts=2, vocab=512, kv_dim=256), 7)
    f = str(tmp_path / "gpt2.safetensors")
    synth.make_gpt2(f, n_layer=2, d=96, vocab=301, n_pos=40)
    return d, g, f


@needs2
def test_single_process_broadcast_fused_p2p(native, tmp_path):
    n = min(_ngpu(), 8)
    d, g, f = make_mixed(tmp_path)
    with gpupool.Pool(list(range(n)), n_staging_buffers=4, staging_buffer_bytes=1 * MB, n_reader_threads=2) as pl:
        for path, flags in ((d, 0), (g, 0), (f, gpupool.LOAD_GPT2_CONV1D_T)):
            shards, recs = oracle.index_path(path)
            m = pl.load(path, mode=gpupool.MODE_BROADCAST, fanout=gpupool.FANOUT_P2P, flags=flags)
            try:
                st = m.stats()
                assert st["n_parts"] == n and len(st["parts"]) == n
                assert sum(p["src_bytes"] for p in st["parts"]) == st["file_bytes"], "each byte is ingested by exactly one GPU"
                for dev in range(n):
                    check_pool(m, dev, shards, recs, flags=flags)
                sums = {m.checksum(dev, 0, m.info()["pool_bytes"] // 8 * 8) for dev in range(n)}
                assert len(sums) == 1, "all pools bit-identical"
            finally:
                m.release()


@needs2
def test_single_process_raw_fanout(native, tmp_path):
    """Variant (ii) of SURVEY.md §8(d) config 4: all-gather the quantised file bytes, dequantise on every GPU."""
    n = min(_ngpu(), 8)
    d, g, f = make_mixed(tmp_path)
    with gpupool.Pool(list(range(n)), n_staging_buffers=4, staging_buffer_bytes=1 * MB, n_reader_threads=2) as pl:
        for path in (g, d):
            shards, recs = oracle.index_path(path)
            m = pl.load(path, mode=gpupool.MODE_BROADCAST, fanout=gpupool.FANOUT_RAW)
            try:
                for dev in range(n):
                    check_pool(m, dev, shards, recs)
            finally:
                m.release()


@needs2
def test_single_process_broadcast_without_fanout_is_replicas(native, tmp_path):
    d, _, _ = make_mixed(tmp_path)
    shards, recs = oracle.index_path(d)
    with gpupool.Pool([0, 1], n_staging_buffers=2, staging_buffer_bytes=1 * MB, n_reader_threads=1, flags=gpupool.CFG_NO_PEER_ACCESS) as pl:
        m = pl.load(d, mode=gpupool.MODE_BROADCAST, fanout=gpupool.FANOUT_P2P)
        try:
            for dev in (0, 1):
                check_pool(m, dev, shards, recs)
        finally:
            m.release()


@needs2
def test_single_process_scatter(native, tmp_path):
    n = 2 if _ngpu() < 4 else 4
    d = str(tmp_path / "llama")
    synth.make_llama(d, dict(hidden=256, ffn=704, layers=2, kv_dim=64, vocab=1024), max_shard_bytes=2_500_000)
    shards, recs = oracle.index_path(d)
    with gpupool.Pool(list(range(n)), n_staging_buffers=2, staging_buffer_bytes=1 * MB, n_reader_threads=1) as pl:
        m = pl.load(d, mode=gpupool.MODE_SCATTER)
        try:
            for dev in range(n):
                check_pool(m, dev, shards, recs, mode=gpupool.MODE_SCATTER, n_parts=n, part=dev)
            pls = m.placements("model.layers.0.mlp.down_proj.weight")
            assert [p.slice_begin for p in pls] == [704 // n * i for i in range(n)] and all(p.slice_dim == 1 for p in pls)
        finally:
            m.release()


@needs2
def test_single_process_scatter_exchange(native, tmp_path):
    """Llama shapes, then a file of odd shapes whose row-split tiles also take the byte-granular consumer."""
    n = min(_ngpu(), 8)
    d = str(tmp_path / "llama")
    synth.make_llama(d, dict(hidden=512, ffn=1408, layers=2, kv_dim=128, vocab=2048), max_shard_bytes=6_000_000)
    q = str(tmp_path / "odd.safetensors")
    synth.write_safetensors(q, helpers.ROWSPLIT_ODD_TENSORS, 3, pad_header=False)
    with gpupool.Pool(list(range(n)), n_staging_buffers=2, staging_buffer_bytes=1 * MB, n_reader_threads=1) as pl:
        for path in (d, q):
            shards, recs = oracle.index_path(path)
            m = pl.load(path, mode=gpupool.MODE_SCATTER, flags=gpupool.LOAD_SCATTER_EXCHANGE)
            try:
                for dev in range(n):
                    check_pool(m, dev, shards, recs, mode=gpupool.MODE_SCATTER, n_parts=n, part=dev)
            finally:
                m.release()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_main(rank, world, port, paths, out_dir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from kukeon_b200 import gpupool as gp
        from oracle import oracle as orc
        with gp.Pool([rank], n_staging_buffers=2, staging_buffer_bytes=1 << 20, n_reader_threads=1) as pl:
            for path, flags in paths:
                shards, recs = orc.index_path(path)
                m = pl.load(path, mode=gp.MODE_BROADCAST, fanout=gp.FANOUT_P2P, flags=flags | gp.LOAD_DEFER, part_index=rank, part_count=world)
                try:
                    h, man = m.export(rank)
                    hs = [None] * world
                    dist.all_gather_object(hs, h)
                    for r, hh in enumerate(hs):
                        if r != rank:
                            m.peer_attach(r, hh)
                    dist.barrier()
                    m.load_part()   # my 1/world of the bytes, stored into every pool by the fused kernel
                    dist.barrier()  # all ranks' kernels done => every pool complete
                    exp, plan = orc.expected_pool(shards, recs, 1, flags)
                    got = m.read(rank, 0, len(exp))
                    for p in plan:
                        a, b = p["pool_offset"], p["pool_offset"] + p["nbytes"]
                        assert np.array_equal(got[a:b], exp[a:b]), f"rank {rank}: {p['name']} differs"
                    # resident-image path (what bench.py times) must give the same pools
                    m.stage_resident()
                    fill = helpers.poison(m, rank)  # before the barrier: every rank's launch stores into this pool
                    dist.barrier()
                    m.convert_resident()
                    dist.barrier()
                    helpers.assert_pool_exact(m, rank, exp, helpers.expected_mask(plan, len(exp)), fill, f"rank {rank} after resident convert")
                    dist.barrier()
                    m.peer_detach_all()
                finally:
                    m.release()
            # RAW fan-out across processes: exchange the raw-image handles, stage 1, barrier, stage 2
            path = paths[1][0]
            shards, recs = orc.index_path(path)
            m = pl.load(path, mode=gp.MODE_BROADCAST, fanout=gp.FANOUT_RAW, flags=gp.LOAD_DEFER, part_index=rank, part_count=world)
            try:
                hs = [None] * world
                dist.all_gather_object(hs, m.export_buffer(rank, gp.BUF_RAW))
                for r, hh in enumerate(hs):
                    if r != rank:
                        m.peer_attach_buffer(r, gp.BUF_RAW, hh)
                dist.barrier()
                m.load_part()
                assert not m.info()["loaded"]
                dist.barrier()
                m.convert_local()
                assert m.info()["loaded"]
                exp, plan = orc.expected_pool(shards, recs, 1, 0)
                got = m.read(rank, 0, len(exp))
                for p in plan:
                    a, b = p["pool_offset"], p["pool_offset"] + p["nbytes"]
                    assert np.array_equal(got[a:b], exp[a:b]), f"rank {rank} RAW: {p['name']} differs"
                dist.barrier()
                m.peer_detach_all()
            finally:
                m.release()
        open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    finally:
        dist.destroy_process_group()


@needs2
def test_one_process_per_gpu_broadcast_over_ipc(native, tmp_path):
    import torch.multiprocessing as mp
    world = 2 if _ngpu() < 4 else 4
    d, g, f = make_mixed(tmp_path)
    out = str(tmp_path / "out")
    os.makedirs(out)
    mp.spawn(_rank_main, args=(world, _free_port(), [(d, 0), (g, 0), (f, gpupool.LOAD_GPT2_CONV1D_T)], out), nprocs=world, join=True)
    assert sorted(os.listdir(out)) == [f"ok{r}" for r in range(world)]
