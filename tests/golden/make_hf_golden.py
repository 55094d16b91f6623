"""Generates the committed HF-layout fixture with the format owners' libraries:

    python tests/golden/make_hf_golden.py

A small Hugging Face style Mixtral checkpoint (llama architecture: 2 layers, 4 experts, GQA with 4 query and 2 key/value heads of
32, biases on q/k/v) is converted to GGUF the way llama.cpp's convert_hf_to_gguf.py does it: gguf-py's tensor_mapping names, the
q_proj / k_proj rows (weights and biases) permuted by llama.cpp's `permute`, experts stacked per projection, written with gguf-py's
GGUFWriter as F32 / F16 / BF16 / Q8_0 / Q4_0 / Q4_1 / Q5_0 (gguf-py's quantize).  The expected HF tensors are what transformers' GGUF
loader would give: gguf-py's dequantize of each GGUF tensor, LlamaTensorProcessor._reverse_permute_weights on q / k, the experts
split, rounded to bf16 by torch (RNE), F32 norms and biases rounded likewise.

Outputs: hf_llama_moe.gguf, hf_llama_moe.gguf.hf.npz (HF name -> bf16 bits) and hf_llama_moe.gguf.expected.json.
"""
import hashlib
import json
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
N_HEAD, N_KV, HD, HIDDEN, FFN, VOCAB, LAYERS, EXPERTS = 4, 2, 32, 128, 64, 32, 2, 4


def permute(w, n_head, n_head_kv):
    """llama.cpp convert_hf_to_gguf.py LlamaModel.permute."""
    if n_head_kv is not None and n_head != n_head_kv:
        n_head = n_head_kv
    return w.reshape(n_head, 2, w.shape[0] // n_head // 2, *w.shape[1:]).swapaxes(1, 2).reshape(w.shape)


def hf_checkpoint():
    g = np.random.default_rng(20261018)
    r = lambda *s: (g.standard_normal(s) * 0.05).astype(np.float32)
    t = {"model.embed_tokens.weight": r(VOCAB, HIDDEN)}
    for i in range(LAYERS):
        p = f"model.layers.{i}."
        t.update({p + "input_layernorm.weight": 1 + r(HIDDEN), p + "post_attention_layernorm.weight": 1 + r(HIDDEN),
                  p + "self_attn.q_proj.weight": r(N_HEAD * HD, HIDDEN), p + "self_attn.q_proj.bias": r(N_HEAD * HD),
                  p + "self_attn.k_proj.weight": r(N_KV * HD, HIDDEN), p + "self_attn.k_proj.bias": r(N_KV * HD),
                  p + "self_attn.v_proj.weight": r(N_KV * HD, HIDDEN), p + "self_attn.v_proj.bias": r(N_KV * HD),
                  p + "self_attn.o_proj.weight": r(HIDDEN, N_HEAD * HD), p + "block_sparse_moe.gate.weight": r(EXPERTS, HIDDEN)})
        for e in range(EXPERTS):
            q = f"{p}block_sparse_moe.experts.{e}."
            t.update({q + "w1.weight": r(FFN, HIDDEN), q + "w3.weight": r(FFN, HIDDEN), q + "w2.weight": r(HIDDEN, FFN)})
    t.update({"model.norm.weight": 1 + r(HIDDEN), "lm_head.weight": r(VOCAB, HIDDEN)})
    return t


def main():
    import gguf
    from gguf import quants
    from transformers.modeling_gguf_pytorch_utils import LlamaTensorProcessor

    Q = gguf.GGMLQuantizationType
    hf = hf_checkpoint()
    tmap = gguf.get_tensor_name_map(gguf.MODEL_ARCH.LLAMA, LAYERS)
    # the file's tensors in llama.cpp's order, with their type
    kinds = {"q_proj": Q.Q8_0, "k_proj": Q.Q4_0, "v_proj": Q.F16, "o_proj": Q.BF16, "w1": Q.Q4_1, "w3": Q.Q5_0, "w2": Q.Q8_0}
    out = []  # (gguf name, fp32 array in GGUF row order, type)
    done = set()
    for name, w in hf.items():
        base, sfx = name.rsplit(".", 1)
        if ".experts." in name:
            layer, rest = name.split(".block_sparse_moe.experts.")
            e, proj = rest.split(".")[:2]
            key = (layer, proj)
            if key in done:
                continue
            done.add(key)
            stack = np.stack([hf[f"{layer}.block_sparse_moe.experts.{x}.{proj}.weight"] for x in range(EXPERTS)])
            out.append((tmap.get_name(f"{layer}.block_sparse_moe.experts.{proj}") + ".weight", stack, kinds[proj]))
            continue
        if base.endswith(("q_proj", "k_proj")):
            w = permute(w, N_HEAD, N_HEAD if base.endswith("q_proj") else N_KV)
        proj = base.rsplit(".", 1)[-1]
        if w.ndim == 1 or "norm" in base or base.endswith("gate"):
            ty = Q.F32
        elif base.endswith(("embed_tokens", "lm_head")):
            ty = Q.F16
        else:
            ty = kinds[proj]
        out.append((tmap.get_name(base) + "." + sfx, w, ty))

    path = os.path.join(HERE, "hf_llama_moe.gguf")
    wr = gguf.GGUFWriter(path, "llama")
    wr.add_block_count(LAYERS)
    wr.add_head_count(N_HEAD)
    wr.add_head_count_kv(N_KV)
    wr.add_expert_count(EXPERTS)
    wr.add_embedding_length(HIDDEN)
    for n, w, ty in out:
        data = w if ty == Q.F32 else w.astype(np.float16) if ty == Q.F16 else quants.quantize(w, ty)
        wr.add_tensor(n, data, raw_dtype=ty)
    wr.write_header_to_file()
    wr.write_kv_data_to_file()
    wr.write_tensors_to_file()
    wr.close()

    # expected HF tensors, the way transformers' GGUF loader reads the file
    rd = gguf.GGUFReader(path)
    proc = LlamaTensorProcessor(config={"num_attention_heads": N_HEAD, "num_key_value_heads": N_KV})
    inv = {tmap.get_name(n.rsplit(".", 1)[0]) + "." + n.rsplit(".", 1)[1]: n for n in hf if ".experts." not in n}
    exp = {}
    for t in rd.tensors:
        w = quants.dequantize(t.data, t.tensor_type).astype(np.float32)
        w = w.reshape([int(x) for x in reversed(t.shape)]) if w.ndim == 1 and len(t.shape) > 1 else w
        if "_exps" in t.name:
            layer = t.name.split(".")[1]
            proj = {"ffn_gate_exps": "w1", "ffn_up_exps": "w3", "ffn_down_exps": "w2"}[t.name.split(".")[2]]
            for x in range(EXPERTS):
                exp[f"model.layers.{layer}.block_sparse_moe.experts.{x}.{proj}.weight"] = w[x]
            continue
        w = proc.process(w, t.name).weights
        exp[inv[t.name]] = w
    for n, w in exp.items():
        assert np.allclose(w, hf[n], atol=0.02), n  # the round trip is the HF checkpoint up to quantisation error
    bits = {n: torch.from_numpy(np.ascontiguousarray(w)).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16) for n, w in exp.items()}
    np.savez(path + ".hf.npz", **bits)
    with open(path, "rb") as f:
        digest = hashlib.sha256(f.read()).hexdigest()
    json.dump({"architecture": "llama", "n_head": N_HEAD, "n_head_kv": N_KV, "sha256": digest,
               "tensors": {n: list(b.shape) for n, b in bits.items()}}, open(path + ".expected.json", "w"), indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
