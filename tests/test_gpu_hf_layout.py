"""GPU tier: KK_LOAD_HF_LAYOUT through the real loader and convert kernel.

A synthetic HF checkpoint written as safetensors and as the GGUF llama.cpp's converter makes of it (names, permuted Q/K rows, stacked
experts) loads to the same bytes under the same names; the committed fixture loads to the expected tensors computed with transformers and
gguf-py; every load shape on one GPU is pool-exact against tests/hf_oracle.py with pools poisoned first and checked whole (each also after
a resident conversion); and a consumer in another process finds an HF name in the manifest and reads the un-permuted rows."""
import json
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from kukeon_b200 import gpupool, modelhub
from oracle import oracle
from tests import helpers, hf_oracle, layer_oracle
from tests.test_gpu_property import zerocopy_vmm  # noqa: F401  (fixture)
from tests.test_gpu_stage import ranks, run_checked
from tools import synth

pytestmark = pytest.mark.gpu
MB = 1 << 20
S, B, SC = gpupool.MODE_SINGLE, gpupool.MODE_BROADCAST, gpupool.MODE_SCATTER
HF, F16, K, X, DEFER = gpupool.LOAD_HF_LAYOUT, gpupool.LOAD_F16, gpupool.LOAD_KEEP_F32, gpupool.LOAD_SCATTER_EXCHANGE, gpupool.LOAD_DEFER
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def gguf_file(path, n_head, n_head_kv, experts=0, qtype="Q4_K", **cfg):
    c = dict(hidden=256, ffn=512, layers=4, vocab=512, n_head=n_head, n_head_kv=n_head_kv, qtype=qtype, experts=experts)
    c.update(cfg)
    synth.write_gguf(path, synth.llama_gguf_tensors(**c), 17, extra_kv=synth.gguf_head_kv("llama", n_head, n_head_kv, experts))
    return path


def exp_hf(path, n_head, n_head_kv, mode=S, flags=0, n=1, part=0, layers=None):
    """(expected pool, written mask) of one device holding `part` of an HF-layout load."""
    shards, recs = oracle.index_path(path)
    hf = hf_oracle.hf_view(recs, "llama", n_head, n_head_kv)
    if layers:
        hf = layer_oracle.select_layers(hf, *layers)
    exp, pl = hf_oracle.expected_pool(shards, hf, mode, flags & (K | F16), n, part)
    return exp, helpers.expected_mask(pl, len(exp))


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("gpu_hf")
    # 6 query heads over 2 key/value heads: scatter at N = 4 cuts (head, half) groups; Mixtral with 4 experts; a bf16 llama with biases
    return {"mixtral": (gguf_file(str(d / "mixtral.gguf"), 6, 2, experts=4, hidden=768, ffn=256), 6, 2),
            "llama": (gguf_file(str(d / "llama.gguf"), 4, 2, qtype="BF16", bias=True, ffn=384, vocab=100), 4, 2),
            "nemo": (gguf_file(str(d / "nemo.gguf"), 4, 2, qtype="Q8_0", head_dim=96, hidden=256), 4, 2)}


def test_every_load_shape(pool, files):
    for key, (p, nh, nkv) in files.items():
        m = pool.load(p, flags=HF | DEFER)
        try:
            run_checked([m], [exp_hf(p, nh, nkv)], f"{key} SINGLE", resident_passes=1)
        finally:
            m.release()
        m = pool.load(p, flags=HF | F16 | DEFER)
        try:
            run_checked([m], [exp_hf(p, nh, nkv, flags=F16)], f"{key} SINGLE f16", resident_passes=1)
        finally:
            m.release()
        for fanout, stage2 in ((gpupool.FANOUT_P2P, False), (gpupool.FANOUT_PULL, True)):
            ms = ranks(pool, p, None, B, 2, HF, fanout=fanout)
            try:
                run_checked(ms, [exp_hf(p, nh, nkv)] * 2, f"{key} BROADCAST fan-out {fanout}", stage2=stage2, resident_passes=1)
            finally:
                for m in ms:
                    m.release()
        for n in (2, 4):
            for flags in (HF | X, HF):
                ms = ranks(pool, p, None, SC, n, flags)
                try:
                    run_checked(ms, [exp_hf(p, nh, nkv, SC, flags, n, i) for i in range(n)], f"{key} SCATTER x{n} flags {flags:#x}", resident_passes=1)
                finally:
                    for m in ms:
                        m.release()
        layers = (1, 3)
        ms = ranks(pool, p, layers, B, 2, HF)
        try:
            run_checked(ms, [exp_hf(p, nh, nkv, layers=layers)] * 2, f"{key} stage {layers} BROADCAST/P2P", resident_passes=1)
        finally:
            for m in ms:
                m.release()
        m = pool.load(p, mode=B, fanout=gpupool.FANOUT_RAW, flags=HF | DEFER)
        try:
            run_checked([m], [exp_hf(p, nh, nkv)], f"{key} BROADCAST/RAW", stage2=True, resident_passes=1)
        finally:
            m.release()


def test_vmm_pools_and_zero_copy_staging(zerocopy_vmm, files):  # noqa: F811
    p, nh, nkv = files["mixtral"]
    m = zerocopy_vmm.load(p, flags=HF | DEFER)
    try:
        run_checked([m], [exp_hf(p, nh, nkv)], "mixtral, VMM pools + zero-copy staging", resident_passes=1)
    finally:
        m.release()


def test_committed_fixture_equals_transformers(pool):
    p = os.path.join(G, "hf_llama_moe.gguf")
    want = np.load(p + ".hf.npz")
    m = pool.load(p, flags=HF)
    try:
        names = [t["name"] for t in m.tensors()]
        assert sorted(names) == sorted(want.files)
        for n in names:
            pl = m.placements(n)[0]
            assert list(pl.shape) == list(want[n].shape), n
            assert np.array_equal(m.read(0, pl.pool_offset, pl.nbytes), want[n].view(np.uint8).reshape(-1)), n
        with pytest.raises(gpupool.ErrNotFound):
            m.placements("blk.0.attn_q.weight")
        man = m.manifest(0)
        assert man["layout"] == "hf" and man["architecture"] == "llama"
        assert m.info()["n_tensors"] == len(want.files)
    finally:
        m.release()


# ---- round trip: HF safetensors against the GGUF llama.cpp makes of it -------------------------------------------------------------
def _write_gguf(path, tensors, kv):
    """Minimal GGUF v3 writer: tensors = (name, ggml type, shape outermost-first, bytes); kv = (key, value type, payload)."""
    s = lambda x: struct.pack("<Q", len(x.encode())) + x.encode()
    head = struct.pack("<IIQQ", 0x46554747, 3, len(tensors), len(kv) + 1) + s("general.architecture") + struct.pack("<I", 8) + s("llama")
    for k, vt, payload in kv:
        head += s(k) + struct.pack("<I", vt) + payload
    rel, offs = 0, []
    for name, gt, shape, data in tensors:
        ne = list(reversed(shape))
        head += s(name) + struct.pack("<I", len(ne)) + struct.pack(f"<{len(ne)}Q", *ne) + struct.pack("<IQ", gt, rel)
        offs.append(rel)
        rel += (len(data) + 31) // 32 * 32
    head += b"\0" * ((-len(head)) % 32)
    with open(path, "wb") as f:
        f.write(head)
        for (_, _, _, data), o in zip(tensors, offs):
            f.seek(len(head) + o)
            f.write(data)
        f.truncate(len(head) + rel)


def _round_trip_files(d, dt, n_head=4, n_kv=2, hd=64, hidden=256, ffn=128, layers=2, experts=4, vocab=64):
    rng = np.random.default_rng(5)
    bits = lambda *shape: rng.integers(0, 0x7F00, size=shape, dtype=np.uint16) ^ (rng.integers(0, 2, size=shape, dtype=np.uint16) << 15)
    hf = {"model.embed_tokens.weight": bits(vocab, hidden)}
    for i in range(layers):
        p = f"model.layers.{i}."
        hf.update({p + "input_layernorm.weight": bits(hidden), p + "self_attn.q_proj.weight": bits(n_head * hd, hidden),
                   p + "self_attn.k_proj.weight": bits(n_kv * hd, hidden), p + "self_attn.v_proj.weight": bits(n_kv * hd, hidden),
                   p + "self_attn.o_proj.weight": bits(hidden, n_head * hd), p + "post_attention_layernorm.weight": bits(hidden),
                   p + "block_sparse_moe.gate.weight": bits(experts, hidden)})
        for e in range(experts):
            q = f"{p}block_sparse_moe.experts.{e}."
            hf.update({q + "w1.weight": bits(ffn, hidden), q + "w2.weight": bits(hidden, ffn), q + "w3.weight": bits(ffn, hidden)})
    hf.update({"model.norm.weight": bits(hidden), "lm_head.weight": bits(vocab, hidden)})
    # safetensors
    hdr, data = {}, b""
    for n, a in hf.items():
        b = a.tobytes()
        hdr[n] = {"dtype": dt, "shape": list(a.shape), "data_offsets": [len(data), len(data) + len(b)]}
        data += b
    st_path = os.path.join(d, f"hf_{dt}.safetensors")
    helpers.write_raw_safetensors(st_path, hdr, data)
    # GGUF as llama.cpp's converter writes it: llama.cpp names, Q/K rows permuted, experts stacked
    gt = {"BF16": 30, "F16": 1}[dt]
    ten = [("token_embd.weight", gt, [vocab, hidden], hf["model.embed_tokens.weight"].tobytes())]
    for i in range(layers):
        p = f"model.layers.{i}."
        g = f"blk.{i}."
        ten += [(g + "attn_norm.weight", gt, [hidden], hf[p + "input_layernorm.weight"].tobytes()),
                (g + "attn_q.weight", gt, [n_head * hd, hidden], hf_oracle.permute(hf[p + "self_attn.q_proj.weight"], n_head).tobytes()),
                (g + "attn_k.weight", gt, [n_kv * hd, hidden], hf_oracle.permute(hf[p + "self_attn.k_proj.weight"], n_kv).tobytes()),
                (g + "attn_v.weight", gt, [n_kv * hd, hidden], hf[p + "self_attn.v_proj.weight"].tobytes()),
                (g + "attn_output.weight", gt, [hidden, n_head * hd], hf[p + "self_attn.o_proj.weight"].tobytes()),
                (g + "ffn_norm.weight", gt, [hidden], hf[p + "post_attention_layernorm.weight"].tobytes()),
                (g + "ffn_gate_inp.weight", gt, [experts, hidden], hf[p + "block_sparse_moe.gate.weight"].tobytes())]
        for base, w, shape in (("ffn_gate_exps", "w1", [ffn, hidden]), ("ffn_up_exps", "w3", [ffn, hidden]), ("ffn_down_exps", "w2", [hidden, ffn])):
            stack = np.stack([hf[f"{p}block_sparse_moe.experts.{e}.{w}.weight"] for e in range(experts)])
            ten.append((g + base + ".weight", gt, [experts] + shape, stack.tobytes()))
    ten += [("output_norm.weight", gt, [hidden], hf["model.norm.weight"].tobytes()), ("output.weight", gt, [vocab, hidden], hf["lm_head.weight"].tobytes())]
    gg_path = os.path.join(d, f"hf_{dt}.gguf")
    _write_gguf(gg_path, ten, [(k, 4, struct.pack("<I", v)) for k, v in (("llama.attention.head_count", n_head), ("llama.attention.head_count_kv", n_kv),
                                                                           ("llama.expert_count", experts))])
    return st_path, gg_path


@pytest.mark.parametrize("dt", ["BF16", "F16"])
def test_round_trip_against_the_hf_checkpoint_bit_exact(pool, tmp_path, dt):
    st_path, gg_path = _round_trip_files(str(tmp_path), dt)
    for flags in (0, F16):
        a, b = pool.load(st_path, flags=flags), pool.load(gg_path, flags=flags | HF)
        try:
            ta, tb = {t["name"]: t for t in a.manifest(0)["tensors"]}, {t["name"]: t for t in b.manifest(0)["tensors"]}
            assert sorted(ta) == sorted(tb)
            for n in ta:
                assert (ta[n]["dtype"], ta[n]["shape"], ta[n]["nbytes"]) == (tb[n]["dtype"], tb[n]["shape"], tb[n]["nbytes"]), n
                assert np.array_equal(a.read(0, ta[n]["offset"], ta[n]["nbytes"]), b.read(0, tb[n]["offset"], tb[n]["nbytes"])), (dt, flags, n)
        finally:
            a.release()
            b.release()


def test_refusal_comes_before_the_pool_is_used(pool, tmp_path):
    """A GGUF without head counts is refused by the flag, and the same file still loads without it."""
    p = str(tmp_path / "nokv.gguf")
    synth.write_gguf(p, synth.llama_gguf_tensors(256, 256, 1, 4, 2, 64), 3)
    with pytest.raises(gpupool.ErrFormat, match="head_count"):
        pool.load(p, flags=HF)
    m = pool.load(p)
    try:
        assert m.tensors()[0]["name"] == "token_embd.weight"
    finally:
        m.release()


_CHILD = r'''
import sys, json, numpy as np
from cuda.bindings import runtime as cudart
hpath, mpath, name = sys.argv[1], sys.argv[2], sys.argv[3]
man = json.load(open(mpath))
assert man["layout"] == "hf", man.get("layout")
t = next(x for x in man["tensors"] if x["name"] == name)
h = cudart.cudaIpcMemHandle_t(); h.reserved = open(hpath, "rb").read()
err, = cudart.cudaSetDevice(0); assert err == 0, err
err, ptr = cudart.cudaIpcOpenMemHandle(h, cudart.cudaIpcMemLazyEnablePeerAccess); assert err == 0, err
buf = np.empty(t["nbytes"], np.uint8)
err, = cudart.cudaMemcpy(buf.ctypes.data, ptr + t["offset"], t["nbytes"], cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost); assert err == 0, err
sys.stdout.write(json.dumps({"shape": t["shape"], "dtype": t["dtype"], "hex": buf.tobytes().hex()}))
cudart.cudaIpcCloseMemHandle(ptr)
'''


def test_a_consumer_process_finds_hf_names_through_the_manifest(pool, tmp_path):
    p = os.path.join(G, "hf_llama_moe.gguf")
    want = np.load(p + ".hf.npz")
    m = pool.load(p, flags=HF)
    try:
        spec = modelhub.Mount(m, 0, str(tmp_path / "cell" / "container"))
        name = "model.layers.0.self_attn.q_proj.weight"
        r = subprocess.run([sys.executable, "-c", _CHILD, os.path.join(spec.host_dir, "ipc.handle"), os.path.join(spec.host_dir, "manifest.json"), name],
                           capture_output=True, text=True, timeout=120)
        assert r.returncode == 0, r.stderr[-2000:]
        got = json.loads(r.stdout)
        assert got["dtype"] == "BF16" and got["shape"] == list(want[name].shape)
        assert bytes.fromhex(got["hex"]) == want[name].tobytes()
    finally:
        m.release()
