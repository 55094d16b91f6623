"""Synthetic checkpoint writers for the configs in BASELINE.json / SURVEY.md §8(d).

There is no network and no real checkpoint in this environment, so tests and bench.py build files of
the named architectures' exact tensor inventories with seeded counter-based random content
(counter-based splitmix64 keyed by (seed, tensor index, position) in tools/synth_fill.c, so any
piece of any tensor can be regenerated without keeping a copy).
The writers emit the container formats directly (safetensors: u64 header length | JSON | data;
GGUF v3) and are themselves checked against the format owners' readers (safetensors.safe_open,
gguf.GGUFReader) in tests/test_index.py.
Neither the product nor the oracle is used here.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import struct
import subprocess
from typing import Dict, List, Sequence, Tuple

import numpy as np

ST_ITEMSIZE = {"F32": 4, "F16": 2, "BF16": 2, "I64": 8, "I32": 4, "U8": 1, "I8": 1, "BOOL": 1, "F64": 8, "I16": 2, "U16": 2, "U32": 4,
               "F8_E4M3": 1, "F8_E5M2": 1}
GGML = {"F32": (0, 1, 4), "F16": (1, 1, 2), "Q4_K": (12, 256, 144), "BF16": (30, 1, 2), "Q8_0": (8, 32, 34), "Q6_K": (14, 256, 210),
        "Q4_0": (2, 32, 18), "Q4_1": (3, 32, 20), "Q5_0": (6, 32, 22), "Q5_1": (7, 32, 24), "Q2_K": (10, 256, 84), "Q3_K": (11, 256, 110),
        "Q5_K": (13, 256, 176), "IQ4_NL": (20, 32, 18), "IQ4_XS": (23, 256, 136), "MXFP4": (39, 32, 17),
        "IQ2_XXS": (16, 256, 66), "IQ2_XS": (17, 256, 74), "IQ2_S": (22, 256, 82), "IQ3_XXS": (18, 256, 98), "IQ3_S": (21, 256, 110), "IQ1_S": (19, 256, 50), "IQ1_M": (29, 256, 56), "TQ1_0": (34, 256, 54), "TQ2_0": (35, 256, 66), "NVFP4": (40, 64, 36)}
_KIND = {"BF16": 1, "F16": 2, "F32": 3, "Q4_K": 4, "Q8_0": 5, "Q6_K": 6, "Q4_0": 7, "Q4_1": 8, "Q5_0": 9, "Q5_1": 10, "Q2_K": 11, "Q3_K": 12,
         "Q5_K": 13, "IQ4_NL": 14, "IQ4_XS": 15, "MXFP4": 16,
         "IQ2_XXS": 17, "IQ2_XS": 18, "IQ2_S": 19, "IQ3_XXS": 20, "IQ3_S": 21, "IQ1_S": 22, "IQ1_M": 23, "TQ1_0": 24, "TQ2_0": 25, "NVFP4": 26}
_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libkk_synth.so")
_lib = None


def _c():
    """tools/synth_fill.c (OpenMP): content of (seed, tensor index, position) generated and pwritten in C."""
    global _lib
    if _lib is None:
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(os.path.join(_HERE, "synth_fill.c")):
            subprocess.run(["make", "-C", _HERE, "-s"], check=True)
        L = C.CDLL(_SO)
        L.synth_write.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_int, C.c_uint64, C.c_uint64]
        L.synth_write.restype = C.c_int
        L.synth_fill.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_uint64, C.c_uint64]
        L.synth_fill.restype = None
        L.synth_set_threads.argtypes = [C.c_int]
        L.synth_set_threads(int(os.environ.get("KK_SYNTH_THREADS", "0")) or (os.cpu_count() or 1))
        _lib = L
    return _lib


def gen_bytes(dtype: str, nbytes: int, seed: int, idx: int) -> np.ndarray:
    """Content of a whole tensor of file dtype `dtype` (BF16/F16: finite patterns; F32: U(-0.04,0.04);
    block-quantised types: random blocks whose fp16 scales are finite, magnitude in [2^-10, 2^-4]; anything else: random bytes)."""
    a = np.empty(nbytes, np.uint8)
    _c().synth_fill(a.ctypes.data_as(C.c_void_p), nbytes, _KIND.get(dtype, 0), seed, idx)
    return a


def _nbytes(dtype: str, shape: Sequence[int]) -> int:
    n = 1
    for s in shape:
        n *= s
    if dtype in GGML and GGML[dtype][1] > 1:
        return n // GGML[dtype][1] * GGML[dtype][2]
    return n * ST_ITEMSIZE[dtype]


def _write_at(fd: int, at: int, dtype: str, nbytes: int, seed: int, idx: int) -> None:
    if nbytes:
        rc = _c().synth_write(fd, at, nbytes, _KIND.get(dtype, 0), seed, idx)
        if rc != 0:
            raise OSError(-rc, os.strerror(-rc))


def write_safetensors(path: str, tensors: Sequence[Tuple[str, str, Sequence[int]]], seed: int, first_idx: int = 0,
                      metadata: Dict[str, str] | None = None, pad_header: bool = True) -> int:
    """tensors: (name, dtype, shape) in file order; tensor k gets content index first_idx + k. Returns bytes written."""
    hdr: Dict[str, object] = {}
    if metadata:
        hdr["__metadata__"] = metadata
    off = 0
    offs = []
    for name, dt, shape in tensors:
        nb = _nbytes(dt, shape)
        hdr[name] = {"dtype": dt, "shape": list(shape), "data_offsets": [off, off + nb]}
        offs.append(off)
        off += nb
    raw = json.dumps(hdr, separators=(",", ":")).encode("utf-8")
    if pad_header:
        raw += b" " * ((-(8 + len(raw))) % 8)
    base = 8 + len(raw)
    fd = os.open(path, os.O_WRONLY | os.O_CREAT | os.O_TRUNC, 0o644)
    try:
        os.pwrite(fd, struct.pack("<Q", len(raw)) + raw, 0)
        for k, (name, dt, shape) in enumerate(tensors):
            _write_at(fd, base + offs[k], dt, _nbytes(dt, shape), seed, first_idx + k)
    finally:
        os.close(fd)
    return base + off


def write_sharded(dirpath: str, tensors: Sequence[Tuple[str, str, Sequence[int]]], seed: int, max_shard_bytes: int,
                  threads: int = 8) -> List[str]:
    """HF layout: model-0000i-of-0000N.safetensors + model.safetensors.index.json (weight_map, total_size)."""
    os.makedirs(dirpath, exist_ok=True)
    groups: List[List[int]] = [[]]
    cur = 0
    for i, (_, dt, shape) in enumerate(tensors):
        nb = _nbytes(dt, shape)
        if groups[-1] and cur + nb > max_shard_bytes:
            groups.append([])
            cur = 0
        groups[-1].append(i)
        cur += nb
    n = len(groups)
    names = [f"model-{k + 1:05d}-of-{n:05d}.safetensors" for k in range(n)] if n > 1 else ["model.safetensors"]
    wm = {}
    for k, g in enumerate(groups):
        for i in g:
            wm[tensors[i][0]] = names[k]

    for k, g in enumerate(groups):
        write_safetensors(os.path.join(dirpath, names[k]), [tensors[i] for i in g], seed, first_idx=g[0])
    if n > 1:
        total = sum(_nbytes(dt, sh) for _, dt, sh in tensors)
        with open(os.path.join(dirpath, "model.safetensors.index.json"), "w") as f:
            json.dump({"metadata": {"total_size": total}, "weight_map": dict(sorted(wm.items()))}, f)
    return [os.path.join(dirpath, x) for x in names]


# ---- architectures ---------------------------------------------------------------------------
def llama_tensors(hidden: int, ffn: int, layers: int, kv_dim: int, vocab: int, dtype: str = "BF16"):
    """HF LlamaForCausalLM state_dict inventory (untied): 9*layers + 3 tensors (SURVEY.md Appendix C.1)."""
    t = [("model.embed_tokens.weight", dtype, [vocab, hidden])]
    for i in range(layers):
        p = f"model.layers.{i}."
        t += [(p + "self_attn.q_proj.weight", dtype, [hidden, hidden]), (p + "self_attn.k_proj.weight", dtype, [kv_dim, hidden]),
              (p + "self_attn.v_proj.weight", dtype, [kv_dim, hidden]), (p + "self_attn.o_proj.weight", dtype, [hidden, hidden]),
              (p + "mlp.gate_proj.weight", dtype, [ffn, hidden]), (p + "mlp.up_proj.weight", dtype, [ffn, hidden]),
              (p + "mlp.down_proj.weight", dtype, [hidden, ffn]), (p + "input_layernorm.weight", dtype, [hidden]),
              (p + "post_attention_layernorm.weight", dtype, [hidden])]
    t += [("model.norm.weight", dtype, [hidden]), ("lm_head.weight", dtype, [vocab, hidden])]
    return t


LLAMA3_8B = dict(hidden=4096, ffn=14336, layers=32, kv_dim=1024, vocab=128256)     # 291 tensors, 16,060,522,496 B
LLAMA3_70B = dict(hidden=8192, ffn=28672, layers=80, kv_dim=1024, vocab=128256)    # 723 tensors, 141,107,412,992 B


def gpt2_tensors(n_layer: int = 12, d: int = 768, vocab: int = 50257, n_pos: int = 1024, dtype: str = "F32"):
    """HF GPT-2 inventory without the tied lm_head: 12*n_layer + 4 tensors; Conv1D weights are [in, out]."""
    t = [("wte.weight", dtype, [vocab, d]), ("wpe.weight", dtype, [n_pos, d])]
    for i in range(n_layer):
        p = f"h.{i}."
        t += [(p + "ln_1.weight", dtype, [d]), (p + "ln_1.bias", dtype, [d]),
              (p + "attn.c_attn.weight", dtype, [d, 3 * d]), (p + "attn.c_attn.bias", dtype, [3 * d]),
              (p + "attn.c_proj.weight", dtype, [d, d]), (p + "attn.c_proj.bias", dtype, [d]),
              (p + "ln_2.weight", dtype, [d]), (p + "ln_2.bias", dtype, [d]),
              (p + "mlp.c_fc.weight", dtype, [d, 4 * d]), (p + "mlp.c_fc.bias", dtype, [4 * d]),
              (p + "mlp.c_proj.weight", dtype, [4 * d, d]), (p + "mlp.c_proj.bias", dtype, [d])]
    t += [("ln_f.weight", dtype, [d]), ("ln_f.bias", dtype, [d])]
    return t


def mixtral_gguf_tensors(hidden: int = 4096, ffn: int = 14336, layers: int = 32, experts: int = 8, vocab: int = 32000, kv_dim: int = 1024,
                         qtype: str = "Q4_K"):
    """llama.cpp naming, merged experts: 10*layers + 3 tensors (SURVEY.md §8(d) config 4). Shapes outermost-first.
    qtype: block type of the 2-D weights (Q4_K is the BASELINE config; the others measure the remaining dequantisers at the same shapes)."""
    t = [("token_embd.weight", qtype, [vocab, hidden])]
    for i in range(layers):
        p = f"blk.{i}."
        t += [(p + "attn_norm.weight", "F32", [hidden]), (p + "attn_q.weight", qtype, [hidden, hidden]),
              (p + "attn_k.weight", qtype, [kv_dim, hidden]), (p + "attn_v.weight", qtype, [kv_dim, hidden]),
              (p + "attn_output.weight", qtype, [hidden, hidden]), (p + "ffn_norm.weight", "F32", [hidden]),
              (p + "ffn_gate_inp.weight", "F32", [experts, hidden]),
              (p + "ffn_gate_exps.weight", qtype, [experts, ffn, hidden]), (p + "ffn_up_exps.weight", qtype, [experts, ffn, hidden]),
              (p + "ffn_down_exps.weight", qtype, [experts, hidden, ffn])]
    t += [("output_norm.weight", "F32", [hidden]), ("output.weight", qtype, [vocab, hidden])]
    return t


def llama_gguf_tensors(hidden: int, ffn: int, layers: int, n_head: int, n_head_kv: int, vocab: int, head_dim: int = 0, qtype: str = "BF16",
                       arch: str = "llama", experts: int = 0, bias: bool = False, bias_types: Sequence[str] = ("F32", "F32", "F32")):
    """llama.cpp naming of a llama / qwen2 / qwen3 model (Mixtral with experts > 0) with explicit head counts; head_dim defaults to
    hidden / n_head (Mistral-Nemo has another).  Norms and the router are F32, the q / k / v biases bias_types, every other weight qtype."""
    hd = head_dim or hidden // n_head
    t = [("token_embd.weight", qtype, [vocab, hidden])]
    for i in range(layers):
        p = f"blk.{i}."
        t += [(p + "attn_norm.weight", "F32", [hidden]), (p + "attn_q.weight", qtype, [n_head * hd, hidden]),
              (p + "attn_k.weight", qtype, [n_head_kv * hd, hidden]), (p + "attn_v.weight", qtype, [n_head_kv * hd, hidden])]
        if bias:
            t += [(p + "attn_q.bias", bias_types[0], [n_head * hd]), (p + "attn_k.bias", bias_types[1], [n_head_kv * hd]),
                  (p + "attn_v.bias", bias_types[2], [n_head_kv * hd])]
        if arch == "qwen3":
            t += [(p + "attn_q_norm.weight", "F32", [hd]), (p + "attn_k_norm.weight", "F32", [hd])]
        t += [(p + "attn_output.weight", qtype, [hidden, n_head * hd]), (p + "ffn_norm.weight", "F32", [hidden])]
        if experts:
            t += [(p + "ffn_gate_inp.weight", "F32", [experts, hidden]), (p + "ffn_gate_exps.weight", qtype, [experts, ffn, hidden]),
                  (p + "ffn_up_exps.weight", qtype, [experts, ffn, hidden]), (p + "ffn_down_exps.weight", qtype, [experts, hidden, ffn])]
        else:
            t += [(p + "ffn_gate.weight", qtype, [ffn, hidden]), (p + "ffn_up.weight", qtype, [ffn, hidden]), (p + "ffn_down.weight", qtype, [hidden, ffn])]
    t += [("output_norm.weight", "F32", [hidden]), ("output.weight", qtype, [vocab, hidden])]
    return t


def gguf_head_kv(arch: str, n_head: int, n_head_kv: int = 0, experts: int = 0):
    """extra_kv entries for write_gguf: <arch>.attention.head_count(_kv) and <arch>.expert_count as UINT32."""
    kv = [(f"{arch}.attention.head_count", 4, struct.pack("<I", n_head))]
    if n_head_kv:
        kv.append((f"{arch}.attention.head_count_kv", 4, struct.pack("<I", n_head_kv)))
    if experts:
        kv.append((f"{arch}.expert_count", 4, struct.pack("<I", experts)))
    return kv


def _gguf_str(s: str) -> bytes:
    b = s.encode("utf-8")
    return struct.pack("<Q", len(b)) + b


def write_gguf(path: str, tensors: Sequence[Tuple[str, str, Sequence[int]]], seed: int, alignment: int = 32, arch: str = "llama",
               extra_kv: Sequence[Tuple[str, int, bytes]] = ()) -> int:
    """GGUF v3 writer (header per gguf-py gguf_reader.py: `<IIQQ`, KVs, tensor infos, aligned data)."""
    kvs = [("general.architecture", 8, _gguf_str(arch)), ("general.alignment", 4, struct.pack("<I", alignment))] + list(extra_kv)
    head = struct.pack("<IIQQ", 0x46554747, 3, len(tensors), len(kvs))
    for k, vt, payload in kvs:
        head += _gguf_str(k) + struct.pack("<I", vt) + payload
    rel = 0
    infos = b""
    offs = []
    for name, dt, shape in tensors:
        ne = list(reversed(shape))
        infos += _gguf_str(name) + struct.pack("<I", len(ne)) + struct.pack(f"<{len(ne)}Q", *ne) + struct.pack("<IQ", GGML[dt][0], rel)
        offs.append(rel)
        rel += (_nbytes(dt, shape) + alignment - 1) // alignment * alignment
    head += infos
    pad = (-len(head)) % alignment
    fd = os.open(path, os.O_WRONLY | os.O_CREAT | os.O_TRUNC, 0o644)
    try:
        os.pwrite(fd, head + b"\0" * pad, 0)
        base = len(head) + pad
        for k, (name, dt, shape) in enumerate(tensors):
            _write_at(fd, base + offs[k], dt, _nbytes(dt, shape), seed, k)
        os.ftruncate(fd, base + rel)  # zero padding after the last tensor
    finally:
        os.close(fd)
    return len(head) + pad + rel


# ---- convenience builders ---------------------------------------------------------------------
def make_llama(dirpath: str, cfg: dict, seed: int = 8001, max_shard_bytes: int = 5_000_000_000, dtype: str = "BF16", threads: int = 8):
    return write_sharded(dirpath, llama_tensors(dtype=dtype, **cfg), seed, max_shard_bytes, threads)


def make_gpt2(path: str, seed: int = 1234, **kw) -> int:
    return write_safetensors(path, gpt2_tensors(**kw), seed)


def make_mixtral_gguf(path: str, seed: int = 8007, **kw) -> int:
    return write_gguf(path, mixtral_gguf_tensors(**kw), seed)


def total_bytes(tensors) -> int:
    return sum(_nbytes(dt, sh) for _, dt, sh in tensors)
