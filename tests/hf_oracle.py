"""Independent restatement of the Hugging Face view of a GGUF load (KK_LOAD_HF_LAYOUT, include/kukeon_gpuload.h) over the oracle.  It
shares no code with the library: the rename table and the expert split are restated from gguf-py's tensor_mapping and HF's Mixtral
files, the Q/K rows are un-permuted with numpy's reshape / swapaxes (llama.cpp's `permute` run backwards), the layout is the oracle's
plan_pool over the HF-view records, and the values are the oracle's (or, under KK_LOAD_F16, tests/f16_oracle.py's) conversions.  It sits
here, next to the tests that use it, because oracle/ is the suite's fixed reference and a new feature's rule is added beside it."""
from __future__ import annotations

import re
from typing import List, Optional, Tuple

import numpy as np

from oracle import oracle
from tests import f16_oracle

LOAD_HF_LAYOUT = 0x100
ARCHS = ("llama", "qwen2", "qwen3")

TOP = {"token_embd.weight": "model.embed_tokens.weight", "output_norm.weight": "model.norm.weight", "output.weight": "lm_head.weight",
       "rope_freqs.weight": "rope_freqs.weight"}
# per-layer base name -> (HF name under model.layers.N., architectures that carry it)
LAYER = {"attn_norm": ("input_layernorm", ARCHS), "ffn_norm": ("post_attention_layernorm", ARCHS),
         "attn_q": ("self_attn.q_proj", ARCHS), "attn_k": ("self_attn.k_proj", ARCHS), "attn_v": ("self_attn.v_proj", ARCHS),
         "attn_output": ("self_attn.o_proj", ARCHS), "attn_q_norm": ("self_attn.q_norm", ("qwen3",)), "attn_k_norm": ("self_attn.k_norm", ("qwen3",)),
         "ffn_gate": ("mlp.gate_proj", ARCHS), "ffn_up": ("mlp.up_proj", ARCHS), "ffn_down": ("mlp.down_proj", ARCHS),
         "ffn_gate_inp": ("block_sparse_moe.gate", ("llama",))}
EXPERTS = {"ffn_gate_exps": "w1", "ffn_up_exps": "w3", "ffn_down_exps": "w2"}  # llama (Mixtral) only


class Unmapped(ValueError):
    pass


def hf_view(recs: List[dict], arch: str, n_head: int = 0, n_head_kv: Optional[int] = None) -> List[dict]:
    """The oracle's GGUF records -> HF-view records, in the same (shard, offset) order.  Each keeps the GGUF name it came from as
    "gguf_name"; Q/K records of llama get "rope_heads"."""
    if arch not in ARCHS:
        raise Unmapped(arch)
    n_head_kv = n_head_kv or n_head
    out = []
    for r in recs:
        n = r["name"]
        if n in TOP:
            out.append(dict(r, name=TOP[n], gguf_name=n))
            continue
        m = re.fullmatch(r"blk\.(\d+)\.(\w+)\.(weight|bias)", n)
        if not m:
            raise Unmapped(n)
        layer, base, sfx = m.groups()
        pre = f"model.layers.{layer}."
        if base in EXPERTS and arch == "llama" and sfx == "weight":
            E = r["shape"][0]
            nb = r["nbytes"] // E
            for e in range(E):
                out.append(dict(r, name=f"{pre}block_sparse_moe.experts.{e}.{EXPERTS[base]}.weight", shape=list(r["shape"][1:]), nbytes=nb,
                                file_offset=r["file_offset"] + e * nb, gguf_name=n))
            continue
        if base not in LAYER or arch not in LAYER[base][1]:
            raise Unmapped(n)
        h = dict(r, name=f"{pre}{LAYER[base][0]}.{sfx}", gguf_name=n)
        if arch == "llama" and base in ("attn_q", "attn_k"):
            h["rope_heads"] = n_head if base == "attn_q" else n_head_kv
        out.append(h)
    return out


def permute(w: np.ndarray, heads: int) -> np.ndarray:
    """llama.cpp's converter (convert_hf_to_gguf.py LlamaModel.permute): HF rows -> GGUF rows."""
    return w.reshape(heads, 2, w.shape[0] // heads // 2, *w.shape[1:]).swapaxes(1, 2).reshape(w.shape)


def unpermute(w: np.ndarray, heads: int) -> np.ndarray:
    """GGUF rows -> HF rows: HF row h*hd + k*hd/2 + i is GGUF row h*hd + 2i + k."""
    return w.reshape(heads, w.shape[0] // heads // 2, 2, *w.shape[1:]).swapaxes(1, 2).reshape(w.shape)


def plan_pool(hf_recs: List[dict], mode: int = oracle.MODE_SINGLE, flags: int = 0, n_parts: int = 1, part: int = 0) -> Tuple[List[dict], int]:
    """The slot layout: the oracle's placement of the HF-view records (index order, 256-byte slots, scatter slices in HF rows)."""
    return f16_oracle.plan_pool(hf_recs, mode, flags & ~LOAD_HF_LAYOUT, n_parts, part)


def expected_pool(shards: List[str], hf_recs: List[dict], mode: int = oracle.MODE_SINGLE, flags: int = 0,
                  n_parts: int = 1, part: int = 0) -> Tuple[np.ndarray, List[dict]]:
    """Whole expected pool of one device (gaps zero): each tensor converted, its Q/K rows un-permuted, then sliced."""
    flags &= ~LOAD_HF_LAYOUT
    plan, total = plan_pool(hf_recs, mode, flags, n_parts, part)
    pool = np.zeros(total, np.uint8)
    fhs = [open(s, "rb") for s in shards]
    try:
        for r, p in zip(hf_recs, plan):
            fh = fhs[r["shard"]]
            fh.seek(r["file_offset"])
            out = f16_oracle.convert_tensor(r, fh.read(r["nbytes"]), flags)
            rows = r["shape"][0] if r["shape"] else 1
            if r.get("rope_heads"):
                out = unpermute(out.reshape(rows, -1), r["rope_heads"]).reshape(-1)
            if p["slice_dim"] is not None:
                R, C = r["shape"]
                es = out.size // (R * C)
                k, b = p["shape"][p["slice_dim"]], p["slice_begin"]
                v = out.reshape(R, C, es)
                out = np.ascontiguousarray(v[b:b + k] if p["slice_dim"] == 0 else v[:, b:b + k]).reshape(-1)
            assert out.size == p["nbytes"], (r["name"], out.size, p["nbytes"])
            pool[p["pool_offset"]: p["pool_offset"] + out.size] = out
    finally:
        for fh in fhs:
            fh.close()
    return pool, plan


def tensors(shards: List[str], hf_recs: List[dict], flags: int = 0) -> dict:
    """{HF name: pool bytes of the whole tensor} (no slicing)."""
    exp, plan = expected_pool(shards, hf_recs, oracle.MODE_SINGLE, flags)
    return {p["name"]: exp[p["pool_offset"]:p["pool_offset"] + p["nbytes"]] for p in plan}
