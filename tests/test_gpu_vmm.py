"""GPU tests of VMM pools (KK_CFG_VMM_POOLS): the pool is exported as a POSIX file descriptor over the staged Unix socket and mapped READ-ONLY by
another process — the isolation a cudaIpcMemHandle cannot give (round-1 review: any cell could overwrite the weights every other cell reads)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from kukeon_b200 import gpupool, modelhub
from oracle import oracle
from tests import helpers
from tests.test_gpu_load import assert_pool_matches

pytestmark = pytest.mark.gpu
MB = 1 << 20

# The consumer: receives the pool's fd over the staged socket and finds the exporter's GPU by its UUID.
_CHILD_SETUP = r'''
import json, os, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from kukeon_b200 import gpupool, modelhub
from cuda.bindings import runtime as cudart
sock, off, n, want_uuid = sys.argv[2], int(sys.argv[3]), int(sys.argv[4]), sys.argv[5]
fd, size = modelhub.receive_pool_fd(sock)
err, cnt = cudart.cudaGetDeviceCount(); assert err == 0, err
dev = None
for i in range(cnt):
    err, pr = cudart.cudaGetDeviceProperties(i); assert err == 0, err
    b = bytes(pr.uuid.bytes)
    if "GPU-%s-%s-%s-%s-%s" % (b[0:4].hex(), b[4:6].hex(), b[6:8].hex(), b[8:10].hex(), b[10:16].hex()) == want_uuid: dev = i
assert dev is not None
out = {}
'''

_CHILD = _CHILD_SETUP + r'''
im = gpupool.ImportedPool(fd, dev, size, readonly=True)
buf = np.empty(n, np.uint8)
err, = cudart.cudaMemcpy(buf.ctypes.data, im.ptr + off, n, cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost); assert err == 0, err
out["hex"] = buf.tobytes().hex()
# a store through the read-only mapping: must fail here (synchronously or at the next sync) and never reach the exporter's pool
e1, = cudart.cudaMemset(im.ptr + off, 0xFF, n)
e2, = cudart.cudaDeviceSynchronize()
out["write_errors"] = [int(e1), int(e2)]
print(json.dumps(out))
sys.stdout.flush()
os._exit(0)  # the context may be poisoned by the fault: do not run teardown through it
'''

# Reads only: maps the pool read-only twice, each time reading the bytes back and closing the import (kk_import_close unmaps and releases
# the mapping; the second import finds nothing of the first left over), then exits through the normal teardown.
_CHILD_READ = _CHILD_SETUP + r'''
out["hex"] = []
for _ in range(2):
    im = gpupool.ImportedPool(fd, dev, size, readonly=True)
    buf = np.empty(n, np.uint8)
    err, = cudart.cudaMemcpy(buf.ctypes.data, im.ptr + off, n, cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost); assert err == 0, err
    out["hex"].append(buf.tobytes().hex())
    im.close()
os.close(fd)
err, = cudart.cudaDeviceSynchronize(); assert err == 0, err
print(json.dumps(out))
'''


def test_vmm_pool_loads_like_any_other_and_has_no_ipc_handle(native, tmp_path):
    p = str(tmp_path / "m.safetensors")
    helpers.mixed_safetensors(p)
    shards, recs = oracle.index_path(p)
    with gpupool.Pool([0], n_staging_buffers=2, staging_buffer_bytes=4 * MB, n_reader_threads=1, flags=gpupool.CFG_VMM_POOLS) as pl:
        m = pl.load(p)
        try:
            assert_pool_matches(m, 0, shards, recs)
            with pytest.raises(gpupool.ErrUnsupported, match="kk_export_fd"):
                m.export(0)
            fd, size = m.export_fd(0)
            os.close(fd)
            assert size >= m.info()["pool_bytes"] and size % (2 * MB) == 0
        finally:
            m.release()
    # and a cudaMalloc pool has no fd to give
    with gpupool.Pool([0], n_staging_buffers=2, staging_buffer_bytes=4 * MB, n_reader_threads=1) as pl:
        m = pl.load(p)
        try:
            with pytest.raises(gpupool.ErrUnsupported, match="KK_CFG_VMM_POOLS"):
                m.export_fd(0)
        finally:
            m.release()


def test_another_process_maps_the_pool_read_only_through_the_staged_socket(native, tmp_path):
    p = str(tmp_path / "m.safetensors")
    helpers.mixed_safetensors(p)
    shards, recs = oracle.index_path(p)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with gpupool.Pool([0], n_staging_buffers=2, staging_buffer_bytes=4 * MB, n_reader_threads=1, flags=gpupool.CFG_VMM_POOLS) as pl:
        m = pl.load(p)
        spec = None
        try:
            spec = modelhub.Mount(m, 0, str(tmp_path / "cell" / "container"))
            env = dict(e.split("=", 1) for e in spec.env)
            assert "KUKEON_GPUPOOL_IPC_HANDLE" not in env and env["KUKEON_GPUPOOL_FD_SOCKET"] == "/run/kukeon/gpupool/pool.sock"
            assert not os.path.exists(os.path.join(spec.host_dir, "ipc.handle")) and os.path.exists(os.path.join(spec.host_dir, "pool.sock"))
            want, _ = oracle.plan_pool(recs)
            t = want[7]  # h.bf16.big
            exp, _ = oracle.expected_pool(shards, recs)
            before = m.checksum(0, 0, m.info()["pool_bytes"] // 8 * 8)
            r = subprocess.run([sys.executable, "-c", _CHILD, root, os.path.join(spec.host_dir, "pool.sock"), str(t["pool_offset"]), "4096", env["KUKEON_GPUPOOL_DEVICE_UUID"]],
                               capture_output=True, text=True, timeout=180)
            assert r.returncode == 0, r.stderr[-2000:]
            out = json.loads(r.stdout.strip().splitlines()[-1])
            assert bytes.fromhex(out["hex"]) == exp[t["pool_offset"]:t["pool_offset"] + 4096].tobytes()
            assert any(out["write_errors"]), "a store through the read-only mapping must fail in the consumer"
            assert m.checksum(0, 0, m.info()["pool_bytes"] // 8 * 8) == before, "the consumer's store reached the shared pool"
            assert_pool_matches(m, 0, shards, recs)
        finally:
            if spec is not None:
                modelhub.unmount(spec)
            m.release()


def test_ipc_mount_detects_a_pool_that_was_written_to(pool, tmp_path):
    """cudaMalloc pools are exported read-write (cudaIpcMemHandle): Mount records the pool checksum and refuses to hand a pool that changed
    since to one more cell."""
    import ctypes as C
    p = str(tmp_path / "m.safetensors")
    helpers.mixed_safetensors(p)
    m = pool.load(p)
    try:
        modelhub.Mount(m, 0, str(tmp_path / "cell" / "a"))
        modelhub.Mount(m, 0, str(tmp_path / "cell" / "b"))  # unchanged: fine
        ptr, n = m.pool_ptr(0)
        from cuda.bindings import runtime as cudart
        err, = cudart.cudaMemset(ptr + 4096, 0x5A, 64)  # what a misbehaving cell could do through its IPC mapping
        assert err == 0
        cudart.cudaDeviceSynchronize()
        with pytest.raises(RuntimeError, match="changed since it was first mounted"):
            modelhub.Mount(m, 0, str(tmp_path / "cell" / "c"))
    finally:
        modelhub.forget_pool(m)
        m.release()


def test_another_process_reads_the_pool_through_a_read_only_import_and_closes_it(native, tmp_path):
    p = str(tmp_path / "m.safetensors")
    helpers.mixed_safetensors(p)
    shards, recs = oracle.index_path(p)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with gpupool.Pool([0], n_staging_buffers=2, staging_buffer_bytes=4 * MB, n_reader_threads=1, flags=gpupool.CFG_VMM_POOLS) as pl:
        m = pl.load(p)
        spec = None
        try:
            spec = modelhub.Mount(m, 0, str(tmp_path / "cell" / "container"))
            env = dict(e.split("=", 1) for e in spec.env)
            want, _ = oracle.plan_pool(recs)
            t = want[7]  # h.bf16.big
            exp, _ = oracle.expected_pool(shards, recs)
            before = m.checksum(0, 0, m.info()["pool_bytes"] // 8 * 8)
            r = subprocess.run([sys.executable, "-c", _CHILD_READ, root, os.path.join(spec.host_dir, "pool.sock"), str(t["pool_offset"]), "4096",
                                env["KUKEON_GPUPOOL_DEVICE_UUID"]], capture_output=True, text=True, timeout=180)
            assert r.returncode == 0, r.stderr[-2000:]
            out = json.loads(r.stdout.strip().splitlines()[-1])
            assert [bytes.fromhex(h) for h in out["hex"]] == [exp[t["pool_offset"]:t["pool_offset"] + 4096].tobytes()] * 2
            assert m.checksum(0, 0, m.info()["pool_bytes"] // 8 * 8) == before
            assert_pool_matches(m, 0, shards, recs)
        finally:
            if spec is not None:
                modelhub.unmount(spec)
            m.release()
