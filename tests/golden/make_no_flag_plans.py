"""Writes no_flag_plans.json: the index and the plan JSON (kk_plan_describe, single / broadcast x2 / scatter x2) of every golden checkpoint,
made by the library of the commit before KK_LOAD_HF_LAYOUT existed.  tests/test_hf_layout.py compares the current library's output with
it byte for byte, so a load without the flag is shown to index and plan exactly as before.

    python tests/golden/make_no_flag_plans.py <root of a checkout of that commit, its library built>

Shard paths are written relative to tests/golden/, so the file does not depend on where the checkout lives.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
FILES = ["q4k.gguf", "q4km_mix.gguf", "quants_cb.gguf", "quants_f4.gguf", "quants_iq.gguf", "hf_llama_moe.gguf", "st_mixed.safetensors", "sharded"]
SHAPES = [(0, 1), (1, 2), (2, 2)]  # (mode, n_parts)


def raw_plan(gpupool, path: str, mode: int, n_parts: int) -> str:
    """kk_plan_describe's JSON text as the library writes it, shard paths made relative to tests/golden/."""
    import ctypes as C
    L = gpupool.lib()
    o = gpupool.KKLoadOpts()
    o.mode = mode
    need = C.c_size_t()
    assert L.kk_plan_describe(None, os.fsencode(path), C.byref(o), n_parts, 0, None, 0, C.byref(need)) == 0
    buf = C.create_string_buffer(need.value)
    assert L.kk_plan_describe(None, os.fsencode(path), C.byref(o), n_parts, 0, buf, need.value, None) == 0
    return buf.value.decode("utf-8").replace(os.path.realpath(HERE) + "/", "")


def describe(gpupool, path: str) -> dict:
    return {"index": gpupool.index(path), "plans": {f"{m}x{n}": raw_plan(gpupool, path, m, n) for m, n in SHAPES}}


def main(lib_root: str) -> None:
    sys.path.insert(0, lib_root)
    from kukeon_b200 import gpupool
    assert os.path.realpath(gpupool.__file__).startswith(os.path.realpath(lib_root)), gpupool.__file__
    out = {f: describe(gpupool, os.path.join(HERE, f)) for f in FILES}
    with open(os.path.join(HERE, "no_flag_plans.json"), "w") as fh:
        json.dump(out, fh, sort_keys=True, separators=(",", ":"))


if __name__ == "__main__":
    main(sys.argv[1])
