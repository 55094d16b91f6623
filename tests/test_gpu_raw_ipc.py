"""KK_FANOUT_RAW across processes on one GPU: two processes, each a one-device context on cuda:0 as rank r of 2, exchange their raw
images over CUDA IPC (allowed between processes on the same device).  This runs the multi-process RAW path — peer raw-image attach, the
peer destinations of stage 1, and the resident fan-out with peers — on a single-GPU machine, where test_gpu_multi.py skips."""
import os
import socket
import sys

import numpy as np
import pytest

from tools import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORLD = 2


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _check(m, rank, exp, plan, what):
    got = m.read(0, 0, len(exp))
    for p in plan:
        a, b = p["pool_offset"], p["pool_offset"] + p["nbytes"]
        assert np.array_equal(got[a:b], exp[a:b]), f"rank {rank} {what}: {p['name']} differs"


def _rank_main(rank, port, path, out_dir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=WORLD)
    try:
        from kukeon_b200 import gpupool as gp
        from oracle import oracle as orc
        shards, recs = orc.index_path(path)
        exp, plan = orc.expected_pool(shards, recs, gp.MODE_BROADCAST, 0)
        # 1 MiB slots and two readers: every rank's part is several chunks, staged by both readers
        with gp.Pool([0], n_staging_buffers=4, staging_buffer_bytes=1 << 20, n_reader_threads=2) as pl:
            m = pl.load(path, mode=gp.MODE_BROADCAST, fanout=gp.FANOUT_RAW, flags=gp.LOAD_DEFER, part_index=rank, part_count=WORLD)
            try:
                hs = [None] * WORLD
                dist.all_gather_object(hs, m.export_buffer(0, gp.BUF_RAW))
                for r, h in enumerate(hs):
                    if r != rank:
                        m.peer_attach_buffer(r, gp.BUF_RAW, h)
                dist.barrier()
                m.load_part()  # stage 1: own part into the own raw image and, by the COPY fan-out, into the peer's
                assert not m.info()["loaded"]
                dist.barrier()
                m.convert_local()  # stage 2: the whole gathered image into the own pool
                assert m.info()["loaded"]
                _check(m, rank, exp, plan, "RAW")
                # resident measurement path: stage the own part again, time the fan-out alone, convert again
                m.stage_resident()
                dist.barrier()
                ms, per = m.convert_resident()
                assert len(per) == 1 and ms >= 0.0  # one fan-out launch over this rank's chunks
                dist.barrier()
                m.convert_local()
                _check(m, rank, exp, plan, "RAW after the resident fan-out")
                dist.barrier()
                m.peer_detach_all()
            finally:
                m.release()
        open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    finally:
        dist.destroy_process_group()


def test_raw_fan_out_between_two_processes_on_one_gpu(native, tmp_path):
    import torch.multiprocessing as mp
    g = str(tmp_path / "mixtral.gguf")
    synth.write_gguf(g, synth.mixtral_gguf_tensors(hidden=256, ffn=1024, layers=4, experts=4, vocab=512, kv_dim=256), 11)
    out = str(tmp_path / "out")
    os.makedirs(out)
    mp.spawn(_rank_main, args=(_free_port(), g, out), nprocs=WORLD, join=True)
    assert sorted(os.listdir(out)) == [f"ok{r}" for r in range(WORLD)]
