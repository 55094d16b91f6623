"""Writes plan_digests.json: digests of the plans (kk_plan_describe) of a fixed corpus of checkpoints, load shapes, flag sets, layer
ranges and staging-chunk sizes, made by the library of the commit before the planner was folded into one placement function and one
chunk-filling loop.  tests/test_plan_digests.py recomputes every digest with the current library, so a change to where chunks are cut, how
reads are laid out or how tiles are counted fails even when the pools it produces stay right.

    python tests/golden/make_plan_digests.py <root of a checkout of that commit, its library built>

The corpus is every golden checkpoint plus synthetic ones written from fixed seeds with tools/synth.py (see synthetic()).  Each plan
contributes the sha256 of its JSON text, shard paths made relative to the checkpoint's directory, or the refusal's status and message.
The plans of one (checkpoint, shape, flag set) are hashed together into one group digest, so the file stays small and a mismatch names
the group.
"""
import hashlib
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = ["q4k.gguf", "q4km_mix.gguf", "quants_cb.gguf", "quants_f4.gguf", "quants_iq.gguf", "hf_llama_moe.gguf", "st_mixed.safetensors", "sharded"]
SHAPES = [(0, 1), (1, 2), (1, 3), (2, 2), (2, 3), (2, 8)]  # (mode, n_parts): SINGLE, BROADCAST x2 / x3, SCATTER x2 / x3 / x8
# 0, GPT2_CONV1D_T, KEEP_F32, SCATTER_EXCHANGE, F8_TO_BF16, F16, HF_LAYOUT, F16|HF_LAYOUT, HF_LAYOUT|SCATTER_EXCHANGE and mixed sets
FLAGS = [0x0, 0x1, 0x2, 0x8, 0x10, 0x80, 0x100, 0x180, 0x108, 0x3, 0x81, 0x92, 0x8A, 0x112, 0x19B]
LAYERS = [None, (0, 1), (1, 2)]
CHUNKS = [1 << 20, 4 << 20, 64 << 20]
GPT2_DTYPES = ["F32", "F16", "BF16", "I32", "I16"]  # with GPT2_CONV1D_T, KEEP_F32 and F16 these reach all four transpose ops


def synthetic(d: str) -> list:
    """Writes the synthetic checkpoints into d and returns their names (paths relative to d)."""
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from tools import synth
    # sharded llama whose dims divide by 2, 4 and 8: dim-0 slices, dim-1 gathered rows (split on 16 rows at 1 MiB) and the row exchange
    synth.write_sharded(os.path.join(d, "llama_st"), synth.llama_tensors(hidden=512, ffn=2048, layers=3, kv_dim=256, vocab=4096), 11,
                        max_shard_bytes=12 << 20)
    names = ["llama_st"]
    for dt in GPT2_DTYPES:  # c_fc is 1 MiB at F32: transposes split on KK_T_ROWS rows
        synth.write_safetensors(os.path.join(d, f"gpt2_{dt}.safetensors"), synth.gpt2_tensors(n_layer=2, d=256, vocab=1024, n_pos=256, dtype=dt), 12)
        names.append(f"gpt2_{dt}.safetensors")
    mx = dict(hidden=256, ffn=512, layers=3, n_head=4, n_head_kv=2, vocab=512, qtype="Q4_K", experts=4)
    synth.write_gguf(os.path.join(d, "mixtral.gguf"), synth.llama_gguf_tensors(**mx), 13, extra_kv=synth.gguf_head_kv("llama", 4, 2, 4))
    # 4 query heads of 48: a scatter over 3 ranks cuts the (head, half) row groups of Q and K
    ll = dict(hidden=256, ffn=384, layers=3, n_head=4, n_head_kv=2, vocab=384, head_dim=48, qtype="BF16", bias=True)
    synth.write_gguf(os.path.join(d, "llama_h4.gguf"), synth.llama_gguf_tensors(**ll), 14, extra_kv=synth.gguf_head_kv("llama", 4, 2))
    # one dtype per role: fp8 weights (cast under F8_TO_BF16) and f32 / f16 ones, sliced along both dims by a scatter
    mixed = []
    for i, (a, b, c) in enumerate([("F8_E4M3", "F8_E5M2", "F32"), ("F8_E5M2", "F16", "F8_E4M3")]):
        p = f"model.layers.{i}."
        mixed += [(p + "self_attn.q_proj.weight", a, [256, 512]), (p + "self_attn.o_proj.weight", b, [512, 256]),
                  (p + "mlp.down_proj.weight", c, [512, 1024]), (p + "input_layernorm.weight", "F32", [512])]
    synth.write_safetensors(os.path.join(d, "f8_mixed.safetensors"), mixed, 15)
    names += ["mixtral.gguf", "llama_h4.gguf", "f8_mixed.safetensors"]
    return names


class Describer:
    """kk_plan_describe through ctypes, one call per plan while the buffer is large enough."""

    def __init__(self, gpupool):
        import ctypes as C
        self.C, self.gp, self.L = C, gpupool, gpupool.lib()
        self.buf = C.create_string_buffer(1 << 22)

    def plan(self, path: str, root: str, mode: int, n_parts: int, flags: int, layers, chunk: int) -> dict:
        """{"json": text} or {"refused": status, "error": message}, paths under root made relative."""
        C = self.C
        o = self.gp.KKLoadOpts()
        o.mode, o.flags = mode, flags
        if layers:
            o.layer_begin, o.layer_end = layers
        need = C.c_size_t()
        while True:
            rc = self.L.kk_plan_describe(None, os.fsencode(path), C.byref(o), n_parts, chunk, self.buf, len(self.buf), C.byref(need))
            if rc == -9 and need.value > len(self.buf):  # KK_ERANGE
                self.buf = C.create_string_buffer(need.value)
                continue
            break
        strip = lambda s: s.replace(os.path.realpath(root) + "/", "").replace(root + "/", "")
        if rc != 0:
            return {"refused": rc, "error": strip(self.L.kk_last_error().decode("utf-8", "replace"))}
        return {"json": strip(self.buf.value.decode("utf-8"))}


def token(res: dict) -> str:
    if "json" in res:
        return hashlib.sha256(res["json"].encode("utf-8")).hexdigest()
    return f"refused {res['refused']}: {res['error']}"


def group_key(mode: int, n_parts: int, flags: int) -> str:
    return f"{mode}x{n_parts} {flags:#x}"


def corpus(d: str):
    """(checkpoint name, path, root for relative shard paths) of every checkpoint; writes the synthetic ones into d."""
    out = [(g, os.path.join(HERE, g), HERE) for g in GOLDEN]
    out += [(s, os.path.join(d, s), d) for s in synthetic(d)]
    return out


def plans(desc: Describer, path: str, root: str):
    """Yields ((mode, n_parts, flags), [(layers, chunk, result) ...]) per group."""
    for mode, n in SHAPES:
        for fl in FLAGS:
            yield (mode, n, fl), [(ly, ch, desc.plan(path, root, mode, n, fl, ly, ch)) for ly in LAYERS for ch in CHUNKS]


def digest(results) -> str:
    return hashlib.sha256("\n".join(token(r) for _, _, r in results).encode("utf-8")).hexdigest()[:32]


def main(lib_root: str) -> None:
    sys.path.insert(0, lib_root)
    from kukeon_b200 import gpupool
    assert os.path.realpath(gpupool.__file__).startswith(os.path.realpath(lib_root)), gpupool.__file__
    desc = Describer(gpupool)
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for name, path, root in corpus(d):
            out[name] = {group_key(*k): digest(rs) for k, rs in plans(desc, path, root)}
    with open(os.path.join(HERE, "plan_digests.json"), "w") as fh:
        json.dump(out, fh, sort_keys=True, indent=0, separators=(",", ":"))
        fh.write("\n")


if __name__ == "__main__":
    main(sys.argv[1])
