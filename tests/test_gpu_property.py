"""Random checkpoints through the real loader and kernel, every pool byte checked against the oracle.

Each example draws a checkpoint: a safetensors inventory (test_plan_property.inventories) or a GGUF one (gguf_inventories, alignment 8, 32
or 64), plus at most one tensor of 2 to 6 MB whose chunk boundaries land wherever the staging size puts them.  Each tensor holds synth's
finite values or Philox-random bytes, which put NaN, Inf, subnormals and rounding ties into every op, the transposes included.  The
example also draws a load shape (SINGLE, BROADCAST over 1-4 virtual ranks, BROADCAST/RAW, SCATTER over 1-5 ranks with or without the
row exchange, PULL over 2-4 ranks), the transposing / F32-keeping / FP8-widening flags, one of three staging contexts and whether the
shards live on tmpfs.

On the GPU every rank's pool is poisoned, loaded (and converted by the second stage where the shape has one), checked whole against the
oracle, then staged resident, poisoned, converted again and checked again; the load must also have run the chunks and tiles that
kk_plan_describe reports.  On the CPU the same examples, drawn by the same derandomized test function, are replayed through the device
code at the same chunk size (test_launch_emul.replay).  An example that fails on the GPU while its CPU twin passes points at code only the
GPU runs: the staging ring and reader threads, the resident image, the RAW and PULL second stages, zero-copy staging and VMM pools, the
kernel's mbarrier ring, tile scheduler, TMA byte counts and its PTX conversions.

The last test reaches deterministically what random inventories rarely do: a shard with so many segments that the resident image splits it
into several launches of at most kMaxSegsPerLaunch (4096) segments each."""
import os
import shutil
import tempfile
from dataclasses import dataclass
from typing import List, Tuple

import numpy as np
import pytest
from hypothesis import HealthCheck, Phase, given, settings, strategies as st

from kukeon_b200 import gpupool
from oracle import oracle
from tests import helpers, kk_emul
from tests.test_gpu_load import _virtual_ranks, expected_exact, poison_all
from tests.test_gpu_quants import _pull_ranks
from tests.test_launch_emul import replay
from tests.test_plan_property import GG_NAMES, GG_TYPES, ST_DTYPES, SUFFIXES, gguf_inventories, inventories
from tools import synth

MB = 1 << 20
T, K, F8, X = gpupool.LOAD_GPT2_CONV1D_T, gpupool.LOAD_KEEP_F32, gpupool.LOAD_F8_TO_BF16, gpupool.LOAD_SCATTER_EXCHANGE
FILE_BUDGET = 24 * MB
# staging contexts: the session pool (8 MiB slots), two 2 MiB slots behind one reader (a slot is reused every other chunk), and zero-copy
# staging with VMM pools (three 2 MiB slots, three readers).  A context's slot size is the chunk size of its plans.
SLOT_BYTES = {"pool": 8 * MB, "ring2": 2 * MB, "zerocopy_vmm": 2 * MB}
CONV1D = oracle.GPT2_CONV1D


@dataclass(frozen=True)
class Example:
    fmt: str                                  # "safetensors" | "gguf"
    tensors: Tuple[Tuple[str, str, Tuple[int, ...]], ...]
    random: Tuple[bool, ...]                  # per tensor: Philox-random bytes over synth's content
    seed: int
    pad: bool                                 # safetensors: header padded to 8 bytes
    alignment: int                            # gguf: general.alignment
    flags: int
    shape: str                                # single | broadcast | raw | scatter | exchange | pull
    n: int                                    # ranks
    ctx: str                                  # key of SLOT_BYTES
    tmpfs: bool                               # shards under /dev/shm (the mapped read path) rather than the temporary directory

    @property
    def mode(self) -> int:
        return {"single": gpupool.MODE_SINGLE, "scatter": gpupool.MODE_SCATTER, "exchange": gpupool.MODE_SCATTER}.get(self.shape, gpupool.MODE_BROADCAST)

    @property
    def load_flags(self) -> int:
        return self.flags | (X if self.shape == "exchange" else 0)


def _nbytes(dt: str, shape) -> int:
    return synth._nbytes(dt, shape)


@st.composite
def _large_tensor(draw, name: str, dtypes):
    """One tensor of 2 to 6 MB: its chunk boundaries (2 or 8 MiB slots) fall inside it, for block types on the block boundaries the planner
    picks.  Row counts are multiples of 60 half the time, so that SCATTER at n = 1..5 slices it."""
    target = draw(st.integers(2 * MB, 6 * MB))
    dt = draw(st.sampled_from(dtypes))
    blk = synth.GGML[dt][1] if dt in synth.GGML else 1
    cols = blk * draw(st.sampled_from([8, 16, 24, 37])) if blk > 1 else draw(st.sampled_from([1032, 1920, 3000, 4099]))
    rows = max(1, target // _nbytes(dt, [1, cols]))
    if draw(st.booleans()) and rows >= 60:
        rows -= rows % 60
    return (name, dt, (rows, cols))


@st.composite
def examples(draw) -> Example:
    # The load shape and the context first: hypothesis varies the earliest choices most evenly across examples.  It also favours the first
    # entry of a list, so the flag sets start with the transposing ones.
    fmt = draw(st.sampled_from(["safetensors", "gguf"]))
    flags = draw(st.sampled_from([T | F8, T, K, T | K, F8, T | K | F8, K | F8, 0])) if fmt == "safetensors" else 0
    shapes = ["single", "broadcast", "raw", "scatter"] + (["exchange"] if fmt == "safetensors" else []) + ([] if flags & T else ["pull"])
    shape = draw(st.sampled_from(shapes))
    n = {"single": 1, "raw": 1, "broadcast": (1, 4), "scatter": (1, 5), "exchange": (2, 5), "pull": (2, 4)}[shape]
    if isinstance(n, tuple):
        n = draw(st.integers(*n))
    ctx, tmpfs = draw(st.sampled_from(sorted(SLOT_BYTES))), draw(st.booleans())
    if fmt == "safetensors":
        # with the transposing flag there is always a large tensor, a float Conv1D weight: rows wider than a tile, cut at chunk boundaries
        if flags & T:
            big = draw(_large_tensor(f"model.layers.7.{draw(st.sampled_from(CONV1D))}", ("F32", "F16", "BF16")))
        else:
            big = draw(st.none() | _large_tensor(f"model.layers.7.{draw(st.sampled_from(SUFFIXES))}", ST_DTYPES))
        inv = draw(inventories())
    else:
        big = draw(st.none() | _large_tensor(f"blk.6.{draw(st.sampled_from(GG_NAMES))}", GG_TYPES))
        inv = draw(gguf_inventories())
    tensors = [(name, dt, tuple(s)) for name, dt, s in inv]
    while sum(_nbytes(dt, s) for _, dt, s in tensors) + (_nbytes(big[1], big[2]) if big else 0) > FILE_BUDGET:
        tensors.remove(max(tensors, key=lambda t: _nbytes(t[1], t[2])))
    if big:
        tensors.insert(draw(st.integers(0, len(tensors))), big)
    rnd = tuple(draw(st.sampled_from([True, False])) for _ in tensors)  # random bytes first: hypothesis favours the first choice
    return Example(fmt, tuple(tensors), rnd, draw(st.integers(0, 1 << 16)), draw(st.booleans()), draw(st.sampled_from([8, 32, 64])), flags,
                   shape, n, ctx, tmpfs)


def write_example(d: str, ex: Example) -> str:
    """Write the example's checkpoint into `d` and return its path: synth's content, then Philox-random bytes over each tensor drawn so."""
    if ex.fmt == "safetensors":
        path = os.path.join(d, "m.safetensors")
        synth.write_safetensors(path, ex.tensors, ex.seed, pad_header=ex.pad)
    else:
        path = os.path.join(d, "m.gguf")
        synth.write_gguf(path, ex.tensors, ex.seed, alignment=ex.alignment)
    recs = {r["name"]: r for r in oracle.index_path(path)[1]}
    with open(path, "r+b") as fh:
        for k, ((name, _, _), rnd) in enumerate(zip(ex.tensors, ex.random)):
            r = recs[name]
            if rnd and r["nbytes"]:
                fh.seek(r["file_offset"])
                fh.write(np.random.Generator(np.random.Philox([ex.seed, k])).bytes(r["nbytes"]))
    return path


def _shard_dir(tmp_path, ex: Example) -> str:
    if ex.tmpfs and os.path.isdir("/dev/shm"):
        return tempfile.mkdtemp(prefix="kk_prop_", dir="/dev/shm")
    return tempfile.mkdtemp(dir=str(tmp_path))


_CUDA_FAULT: List[gpupool.ErrCUDA] = []  # a CUDA error ends the run: hypothesis's closing replay of the failing example raises it again without touching the GPU


def _load(ctx, path: str, ex: Example) -> list:
    if ex.shape == "single":
        return [ctx.load(path, flags=ex.flags | gpupool.LOAD_DEFER)]
    if ex.shape == "raw":
        return [ctx.load(path, mode=gpupool.MODE_BROADCAST, fanout=gpupool.FANOUT_RAW, flags=ex.flags | gpupool.LOAD_DEFER)]
    if ex.shape == "pull":
        return _pull_ranks(ctx, path, ex.n, ex.flags)
    return _virtual_ranks(ctx, path, ex.mode, ex.n, ex.load_flags)


def _run_on_gpu(ctx, path: str, ex: Example) -> None:
    shards, recs = oracle.index_path(path)
    want = [expected_exact(shards, recs, ex.mode, ex.flags & (T | K | F8), ex.n, i) for i in range(ex.n)]
    plan = gpupool.plan_describe(path, mode=ex.mode, flags=ex.load_flags, n_parts=ex.n, chunk_bytes=SLOT_BYTES[ex.ctx])
    second_stage = ex.shape in ("raw", "pull")
    ms = _load(ctx, path, ex)
    try:
        def check(fills, what):
            may_rewrite = None
            if ex.shape == "pull":  # stage 2 copies each peer's whole pool range, gaps included (test_pull_fan_out_virtual_ranks_on_one_gpu)
                ranges = [next((q["pool_lo"], q["pool_hi"]) for q in m.stats()["parts"]) for m in ms]
            for i, m in enumerate(ms):
                exp, mask = want[i]
                if ex.shape == "pull":
                    may_rewrite = np.zeros(len(exp), bool)
                    for j, (lo, hi) in enumerate(ranges):
                        if j != i:
                            may_rewrite[lo:hi] = True
                    may_rewrite &= ~mask
                helpers.assert_pool_exact(m, 0, exp, mask, fills[i], f"{ex.shape} rank {i} of {ex.n}, {what}", may_rewrite=may_rewrite)

        fills = poison_all(ms)
        for m in ms:
            m.load_part()
        if second_stage:
            for m in ms:
                m.convert_local()
        check(fills, "streaming load")
        ran = [next((q["chunks"], q["tiles"]) for q in m.stats()["parts"] if q["part"] == i) for i, m in enumerate(ms)]
        assert ran == [(len(q["chunks"]), sum(ch["n_tiles"] for ch in q["chunks"])) for q in plan["parts"]], "the load ran another plan"
        for m in ms:
            m.stage_resident()
        fills = poison_all(ms)
        for m in ms:
            m.convert_resident()
        if second_stage:
            for m in ms:
                m.convert_local()
        check(fills, "resident conversion")
    finally:
        for m in ms:
            m.release()


@pytest.fixture(scope="module")
def ring2(native):
    p = gpupool.Pool([0], n_staging_buffers=2, staging_buffer_bytes=2 * MB, n_reader_threads=1)
    yield p
    p.close()


@pytest.fixture(scope="module")
def zerocopy_vmm(native):
    p = gpupool.Pool([0], n_staging_buffers=3, staging_buffer_bytes=2 * MB, n_reader_threads=3, flags=gpupool.CFG_ZEROCOPY | gpupool.CFG_VMM_POOLS)
    yield p
    p.close()


@pytest.fixture(scope="module")
def emul():
    return kk_emul.load()


# Both parameters draw the same examples: derandomized, the seed follows from the test function, which they share.  No shrinking: a failing
# example is reported once, not re-run on a shared GPU dozens of times.
@pytest.mark.parametrize("where", [pytest.param("gpu", marks=pytest.mark.gpu), "cpu"])
@settings(max_examples=int(os.environ.get("KK_HYP_EXAMPLES", 200)), derandomize=True, database=None, deadline=None,
          phases=(Phase.explicit, Phase.generate), report_multiple_bugs=False,
          suppress_health_check=[HealthCheck.too_slow, HealthCheck.function_scoped_fixture, HealthCheck.data_too_large])
@given(ex=examples())
def test_random_checkpoints_through_the_loader(request, tmp_path, where, ex):
    """gpu: the real loader and kernel, every rank's whole pool after the streaming load and after a resident conversion, and the plan the
    load ran; cpu: the same example's plan replayed through the device code (test_launch_emul.replay)."""
    if where == "gpu" and _CUDA_FAULT:
        raise _CUDA_FAULT[0]
    d = _shard_dir(tmp_path, ex)
    try:
        path = write_example(d, ex)
        if where == "cpu":
            replay(request.getfixturevalue("emul"), path, mode=ex.mode, flags=ex.load_flags, n_parts=ex.n, chunk=SLOT_BYTES[ex.ctx])
            return
        try:
            _run_on_gpu(request.getfixturevalue(ex.ctx), path, ex)
        except gpupool.ErrCUDA as e:
            _CUDA_FAULT.append(e)
            raise
    finally:
        shutil.rmtree(d, ignore_errors=True)


@pytest.mark.gpu
def test_resident_image_splits_a_shard_into_launches_of_4096_segments(pool, tmp_path):
    """One shard of 10,000 tiny tensors (1-40 elements, five dtypes): the planner closes a chunk at 1024 segments, and the resident image
    merges a shard's chunks into one launch only up to kMaxSegsPerLaunch (4096) segments, so a rank's image runs several launches for its
    one shard.  At 2 virtual BROADCAST ranks each rank's half still holds more than 4096.  Every pool is checked whole after the streaming
    load and after each of two back-to-back resident conversions (the second starting from the scheduler counters the first left)."""
    rng = np.random.default_rng(3)
    dts = ["BF16", "F32", "F16", "U8", "I64"]
    p = str(tmp_path / "many.safetensors")
    synth.write_safetensors(p, [(f"t.{i:05d}", dts[i % len(dts)], [int(rng.integers(1, 41))]) for i in range(10_000)], 17, pad_header=False)
    shards, recs = oracle.index_path(p)
    exp, mask = expected_exact(shards, recs)
    assert len(shards) == 1
    for n in (1, 2):
        plan = gpupool.plan_describe(p, mode=gpupool.MODE_BROADCAST, n_parts=n, chunk_bytes=8 * MB)
        assert all(sum(len(ch["segs"]) for ch in q["chunks"]) > 4096 for q in plan["parts"]), "every rank's image must need a second launch"
        ms = _virtual_ranks(pool, p, gpupool.MODE_BROADCAST, n)
        try:
            fills = poison_all(ms)
            for m in ms:
                m.load_part()
            for i, m in enumerate(ms):
                assert m.stats()["parts"][0]["chunks"] >= 5
                helpers.assert_pool_exact(m, 0, exp, mask, fills[i], f"rank {i} of {n}, streaming load")
            for m in ms:
                m.stage_resident()
            for k in range(2):
                fills = poison_all(ms)
                launches = [len(m.convert_resident()[1]) for m in ms]
                for i, m in enumerate(ms):
                    helpers.assert_pool_exact(m, 0, exp, mask, fills[i], f"rank {i} of {n}, resident conversion {k + 1}")
                assert all(nl > len(shards) for nl in launches), f"{launches} launches for {len(shards)} shard"
        finally:
            for m in ms:
                m.release()
