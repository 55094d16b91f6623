"""GPU tier: KK_LOAD_F16 through the real loader and the fp16 convert kernel (kk_convert_f16_kernel).

Every pool is poisoned before the kernel writes it and checked whole (helpers.assert_pool_exact) against the fp16 oracle
(tests/f16_oracle.py): golden GGUF fixtures and random bytes of every block type, the safetensors fixtures under every flag the output
format composes with, special values through every cast (which settles the NaN rule on the hardware), the GPT-2 transposes, every load
shape on one GPU (each also after a resident conversion), a consumer in another process, and a short property over random checkpoints."""
import dataclasses
import json
import os
import subprocess
import sys

import numpy as np
import pytest
from hypothesis import HealthCheck, Phase, given, settings

from kukeon_b200 import gpupool, modelhub
from oracle import oracle
from tests import f16_oracle as fo
from tests import helpers, layer_oracle
from tests.test_gpu_property import _load, examples, ring2, write_example, zerocopy_vmm  # noqa: F401  (fixtures)
from tests.test_gpu_stage import ranks, run_checked
from tools import synth

pytestmark = pytest.mark.gpu
MB = 1 << 20
S, B, SC = gpupool.MODE_SINGLE, gpupool.MODE_BROADCAST, gpupool.MODE_SCATTER
F16, K, F8, T, X, DEFER = gpupool.LOAD_F16, gpupool.LOAD_KEEP_F32, gpupool.LOAD_F8_TO_BF16, gpupool.LOAD_GPT2_CONV1D_T, gpupool.LOAD_SCATTER_EXCHANGE, gpupool.LOAD_DEFER
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GGUF_FIXTURES = ("q4k.gguf", "q4km_mix.gguf", "quants_f4.gguf", "quants_cb.gguf", "quants_iq.gguf")


def exp16(path, mode=S, flags=F16, n=1, part=0, layers=None):
    """(expected pool, written mask) of one device holding `part` of an f16 load."""
    shards, recs = oracle.index_path(path)
    if layers:
        recs = layer_oracle.select_layers(recs, *layers)
    exp, pl = fo.expected_pool(shards, recs, mode, flags & (T | K | F8 | F16), n, part)
    return exp, helpers.expected_mask(pl, len(exp))


def single(pool, path, flags, label, resident_passes=1):
    m = pool.load(path, flags=flags | DEFER)
    try:
        run_checked([m], [exp16(path, flags=flags)], label, resident_passes=resident_passes)
    finally:
        m.release()


def randomise(path, seed):
    """Philox-random bytes over every tensor of the file: NaN / Inf / negative scales and every bit pattern reach the kernel."""
    _, recs = oracle.index_path(path)
    with open(path, "r+b") as fh:
        for k, r in enumerate(recs):
            if r["nbytes"]:
                fh.seek(r["file_offset"])
                fh.write(np.random.Generator(np.random.Philox([seed, k])).bytes(r["nbytes"]))


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("gpu_f16")
    out = {"mixtral": str(d / "mixtral.gguf"), "llama_f16": str(d / "llama_f16"), "llama_bf16": str(d / "llama_bf16")}
    synth.write_gguf(out["mixtral"], synth.mixtral_gguf_tensors(hidden=256, ffn=768, layers=4, experts=2, vocab=512, kv_dim=256), 9)
    for dt in ("F16", "BF16"):
        synth.make_llama(out[f"llama_{dt.lower()}"], dict(hidden=256, ffn=704, layers=4, kv_dim=64, vocab=1000), max_shard_bytes=1_500_000, dtype=dt)
    return out


def test_golden_gguf_fixtures_streaming_and_resident(pool):
    for g in GGUF_FIXTURES:
        single(pool, os.path.join(G, g), F16, f"{g} f16")


def test_random_bytes_every_block_type_at_alignments_32_and_8(pool, tmp_path):
    for alignment in (32, 8):
        p = str(tmp_path / f"rnd{alignment}.gguf")
        tensors = [("pad.weight", "F32", [3])] + [(f"blk.0.{dt.lower()}.weight", dt, [7, oracle.BLOCK_QUANTS[dt][0] * 5]) for dt in sorted(oracle.BLOCK_QUANTS)]
        synth.write_gguf(p, tensors, 4, alignment=alignment)
        randomise(p, alignment)
        single(pool, p, F16, f"random block bytes, alignment {alignment}")


def test_safetensors_fixtures_with_and_without_keep_f32_and_f8(pool, tmp_path):
    mixed = str(tmp_path / "mixed.safetensors")
    helpers.mixed_safetensors(mixed)
    f8 = str(tmp_path / "f8.safetensors")
    synth.write_safetensors(f8, [("a", "F8_E4M3", [300, 70]), ("b", "F8_E5M2", [37]), ("c", "BF16", [33, 77]), ("d", "F32", [129, 65])], 5, pad_header=False)
    for path in (os.path.join(G, "st_mixed.safetensors"), os.path.join(G, "sharded"), mixed, f8):
        for flags in (F16, F16 | K, F16 | F8, F16 | K | F8):
            single(pool, path, flags, f"{os.path.basename(path)} flags {flags:#x}")


def special_file(path, pad):
    """Every bf16 and every fp16 bit pattern, all 256 patterns of both FP8 types, and the fp32 specials (NaNs of both signs and payloads,
    +-inf, +-0, overflow past 65504, ties, values in and below the fp16 subnormal range), each tensor with a ragged tail; pad=False leaves
    the payloads 2 / 4 bytes off a 16-byte boundary (the byte-assembled cast paths)."""
    from tests.test_f16_oracle import f32_specials
    u16 = np.arange(65536, dtype=np.uint32).astype("<u2")
    blobs = [("bf", "BF16", u16.tobytes() + u16[:5].tobytes()), ("h", "F16", u16.tobytes() + u16[:3].tobytes()),
             ("e4", "F8_E4M3", np.arange(256, dtype=np.uint8).tobytes() * 3 + b"\x7f\xff\x80"), ("e5", "F8_E5M2", np.arange(256, dtype=np.uint8).tobytes() * 3 + b"\x7d\xfe"),
             ("f", "F32", f32_specials().tobytes())]
    if not pad:
        blobs.insert(0, ("x", "U8", b"\x01\x02"))
    hdr, data = {}, b""
    for n, dt, b in blobs:
        es = {"F8_E4M3": 1, "F8_E5M2": 1, "U8": 1, "F32": 4, "BF16": 2, "F16": 2}[dt]
        hdr[n] = {"dtype": dt, "shape": [len(b) // es], "data_offsets": [len(data), len(data) + len(b)]}
        data += b
    helpers.write_raw_safetensors(path, hdr, data)


def test_special_values_through_every_cast(pool, tmp_path):
    for pad in (True, False):
        p = str(tmp_path / f"special{int(pad)}.safetensors")
        special_file(p, pad)
        for flags in (F16 | F8, F16 | F8 | K):
            single(pool, p, flags, f"special values pad={pad} flags {flags:#x}")
    # the NaN rule on the hardware: every NaN a conversion produced is 0x7FFF
    m = pool.load(str(tmp_path / "special1.safetensors"), flags=F16 | F8)
    try:
        for name in ("bf", "e4", "e5", "f"):
            pl = m.placements(name)[0]
            got = m.read(0, pl.pool_offset, pl.nbytes).view(np.uint16)
            nan = (got & 0x7FFF) > 0x7C00
            assert nan.any() and (got[nan] == 0x7FFF).all(), name
    finally:
        m.release()


def test_gpt2_transposes_every_dtype_staged_and_gathered(pool, tmp_path):
    for dt in ("F32", "F16", "BF16"):
        for d, pad in ((96, True), (41, False)):  # whole 16-byte rows (staged by bulk copies) / neither (gathered by the consumers)
            p = str(tmp_path / f"gpt2_{dt}_{d}.safetensors")
            synth.write_safetensors(p, [("x", "U8", [3])] + synth.gpt2_tensors(n_layer=1, d=d, vocab=50, n_pos=8, dtype=dt), 3, pad_header=pad)
            randomise(p, d)
            for flags in ((F16 | T, F16 | T | K) if dt == "F32" else (F16 | T,)):
                single(pool, p, flags, f"gpt2 {dt} d={d} flags {flags:#x}")


def test_load_shapes_on_one_gpu(pool, files):
    for key in ("llama_f16", "llama_bf16"):
        p = files[key]
        for n in (2, 3):
            ms = ranks(pool, p, None, B, n, F16)
            try:
                run_checked(ms, [exp16(p)] * n, f"{key} BROADCAST/P2P x{n}", resident_passes=1)
            finally:
                for m in ms:
                    m.release()
        ms = ranks(pool, p, None, B, 2, F16, fanout=gpupool.FANOUT_PULL)
        try:
            run_checked(ms, [exp16(p)] * 2, f"{key} BROADCAST/PULL", stage2=True, resident_passes=1)
        finally:
            for m in ms:
                m.release()
        for n in (2, 4):
            for flags in (F16 | X, F16):
                ms = ranks(pool, p, None, SC, n, flags)
                try:
                    run_checked(ms, [exp16(p, SC, flags, n, i) for i in range(n)], f"{key} SCATTER x{n} flags {flags:#x}", resident_passes=1)
                finally:
                    for m in ms:
                        m.release()
        layers = (1, 3)
        ms = ranks(pool, p, layers, B, 2, F16)
        try:
            run_checked(ms, [exp16(p, layers=layers)] * 2, f"{key} stage {layers} BROADCAST/P2P", resident_passes=1)
        finally:
            for m in ms:
                m.release()
    m = pool.load(files["mixtral"], mode=B, fanout=gpupool.FANOUT_RAW, flags=F16 | DEFER)
    try:
        run_checked([m], [exp16(files["mixtral"])], "mixtral BROADCAST/RAW", stage2=True)
    finally:
        m.release()


def test_vmm_pools_and_zero_copy_staging(zerocopy_vmm, files):  # noqa: F811
    single(zerocopy_vmm, files["mixtral"], F16, "mixtral, VMM pools + zero-copy staging")


def test_nvls_fan_out_where_the_host_has_it(native, files, gpu_count):
    if gpu_count < 2:
        pytest.skip("NVLS needs two GPUs")
    with gpupool.Pool(list(range(gpu_count)), n_staging_buffers=2, staging_buffer_bytes=8 * MB, n_reader_threads=1) as pl:
        try:
            m = pl.load(files["llama_f16"], mode=B, fanout=gpupool.FANOUT_NVLS, flags=F16)
        except gpupool.ErrUnsupported as e:
            pytest.skip(f"no NVLS on this host: {e}")
        try:
            exp, mask = exp16(files["llama_f16"])
            for dev in range(gpu_count):
                assert (m.read(dev, 0, len(exp))[mask] == exp[mask]).all()
        finally:
            m.release()


def test_f16_and_bf16_loads_of_one_file_are_two_models(pool, files):
    p = files["llama_bf16"]
    a, b = pool.load(p), pool.load(p, flags=F16)
    try:
        assert a.handle != b.handle and a.info()["refcount"] == b.info()["refcount"] == 1
        again = modelhub.Load(pool, p, flags=F16)
        assert again.handle == b.handle and b.info()["refcount"] == 2
        again.release()
        assert {t["dtype"] for t in b.manifest(0)["tensors"]} == {"F16"} and {t["dtype"] for t in a.manifest(0)["tensors"]} == {"BF16"}
        assert {pl.dtype for t in b.tensors() for pl in b.placements(t["name"])} == {"F16"}
        assert (a.info()["pool_bytes"], [pl.pool_offset for t in a.tensors() for pl in a.placements(t["name"])]) == \
            (b.info()["pool_bytes"], [pl.pool_offset for t in b.tensors() for pl in b.placements(t["name"])])
        exp, mask = exp16(p)
        assert (b.read(0, 0, len(exp))[mask] == exp[mask]).all()
        exp, _ = oracle.expected_pool(*oracle.index_path(p))
        assert (a.read(0, 0, len(exp))[mask] == exp[mask]).all(), "the bf16 model is untouched by the f16 one"
    finally:
        a.release()
        b.release()


_CHILD = r'''
import sys, json, numpy as np, torch
from cuda.bindings import runtime as cudart
hpath, mpath, name = sys.argv[1], sys.argv[2], sys.argv[3]
man = json.load(open(mpath))
t = next(x for x in man["tensors"] if x["name"] == name)
assert t["dtype"] == "F16", t["dtype"]
h = cudart.cudaIpcMemHandle_t(); h.reserved = open(hpath, "rb").read()
err, = cudart.cudaSetDevice(0); assert err == 0, err
err, ptr = cudart.cudaIpcOpenMemHandle(h, cudart.cudaIpcMemLazyEnablePeerAccess); assert err == 0, err
buf = np.empty(t["nbytes"], np.uint8)
err, = cudart.cudaMemcpy(buf.ctypes.data, ptr + t["offset"], t["nbytes"], cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost); assert err == 0, err
x = torch.frombuffer(bytearray(buf.tobytes()), dtype={"F16": torch.float16}[t["dtype"]]).reshape(t["shape"])
sys.stdout.write(x.view(torch.int16).numpy().tobytes().hex())
cudart.cudaIpcCloseMemHandle(ptr)
'''


def test_a_consumer_process_views_the_exported_pool_as_float16(pool, files, tmp_path):
    p = files["llama_bf16"]
    m = pool.load(p, flags=F16)
    try:
        spec = modelhub.Mount(m, 0, str(tmp_path / "cell" / "container"))
        name = "model.layers.0.self_attn.q_proj.weight"
        r = subprocess.run([sys.executable, "-c", _CHILD, os.path.join(spec.host_dir, "ipc.handle"), os.path.join(spec.host_dir, "manifest.json"), name],
                           capture_output=True, text=True, timeout=120)
        assert r.returncode == 0, r.stderr[-2000:]
        exp, plan = fo.expected_pool(*oracle.index_path(p), flags=F16)
        t = next(x for x in plan if x["name"] == name)
        assert bytes.fromhex(r.stdout) == exp[t["pool_offset"]:t["pool_offset"] + t["nbytes"]].tobytes()
        assert json.load(open(os.path.join(spec.host_dir, "manifest.json")))["tensors"][0]["dtype"] == "F16"
    finally:
        m.release()


@settings(max_examples=int(os.environ.get("KK_HYP_EXAMPLES_GPU_F16", 25)), derandomize=True, database=None, deadline=None,
          phases=(Phase.explicit, Phase.generate), report_multiple_bugs=False,
          suppress_health_check=[HealthCheck.too_slow, HealthCheck.function_scoped_fixture, HealthCheck.data_too_large])
@given(ex=examples())
def test_random_checkpoints_property(request, tmp_path, ex):
    """test_gpu_property's examples (random inventories and bytes, every load shape, three staging contexts) loaded with KK_LOAD_F16."""
    ex = dataclasses.replace(ex, flags=ex.flags | F16)
    d = str(tmp_path / f"ex{abs(hash(ex)) % 10 ** 9}")
    os.makedirs(d, exist_ok=True)
    path = write_example(d, ex)
    ms = _load(request.getfixturevalue(ex.ctx), path, ex)
    try:
        want = [exp16(path, ex.mode, ex.flags, ex.n, i) for i in range(ex.n)]
        run_checked(ms, want, f"{ex.shape} x{ex.n} flags {ex.load_flags:#x}", stage2=ex.shape in ("raw", "pull"), resident_passes=1)
    finally:
        for m in ms:
            m.release()
