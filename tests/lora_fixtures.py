"""LoRA adapters for the tests (kk_load_adapter): PEFT's saved format written with numpy + safetensors, the C oracle of the merge
(tests/emul/kk_lora_oracle.c) and the CPU replay of the merge kernel (tests/emul/kk_lora_emul.cpp), both built on first use.

peft is not installed here, so the format is restated from its documentation: `save_pretrained` writes `adapter_config.json`
(`r`, `lora_alpha`, `use_rslora`, `target_modules`, `bias`, ...) and `adapter_model.safetensors` with keys
`base_model.model.<module>.lora_A.weight` ([r, in_features]) and `base_model.model.<module>.lora_B.weight` ([out_features, r]), the adapter
name left out of the keys.  PEFT merges as W + (B @ A) * scaling with scaling = lora_alpha / r (lora_alpha / sqrt(r) under use_rslora)."""
from __future__ import annotations

import ctypes as C
import json
import os
import shutil
import subprocess
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import ml_dtypes
import numpy as np

_EMUL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
_CSRC = os.path.join(os.path.dirname(_EMUL), "..", "kukeon_b200", "csrc")
_BUILD = os.path.join(_EMUL, "_build")
PREFIX = "base_model.model."
OUT = {"BF16": 0, "F16": 1, "F32": 2}
TILE_R, TILE_C = 64, 128

# KKLoraTarget (kukeon_b200/csrc/kk_lora.cuh)
TARGET_DTYPE = np.dtype([("w_off", "<u8"), ("a_off", "<u8"), ("b_off", "<u8"), ("rows", "<u4"), ("cols", "<u4"), ("row0", "<u4"),
                         ("col0", "<u4"), ("a_ld", "<u4"), ("r", "<u4"), ("s", "<f4"), ("out", "<u4"), ("tile_begin", "<u4"),
                         ("tiles_c", "<u4")])
assert TARGET_DTYPE.itemsize == 64


def _build(src: str, lib: str, compiler: str, deps: Sequence[str], extra: Sequence[str]) -> str:
    out = os.path.join(_BUILD, lib)
    if os.path.exists(out) and all(os.path.getmtime(d) <= os.path.getmtime(out) for d in deps):
        return out
    os.makedirs(_BUILD, exist_ok=True)
    tmp = out + f".{os.getpid()}.tmp"
    subprocess.run([compiler, "-O2", "-march=x86-64-v2", "-mf16c", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall", "-Wextra",
                    *extra, "-o", tmp, src, "-lm"], check=True)
    os.replace(tmp, out)
    return out


_libs: Dict[str, C.CDLL] = {}


def oracle_lib() -> C.CDLL:
    if "oracle" not in _libs:
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
        src = os.path.join(_EMUL, "kk_lora_oracle.c")
        L = C.CDLL(_build(src, "libkk_lora_oracle.so", cc, [src], ["-std=c11"]))
        L.kk_lora_oracle_merge.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32,
                                           C.c_void_p, C.c_uint32, C.c_float, C.c_uint32]
        L.kk_lora_oracle_merge.restype = None
        _libs["oracle"] = L
    return _libs["oracle"]


def emul_lib() -> C.CDLL:
    if "emul" not in _libs:
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
        src = os.path.join(_EMUL, "kk_lora_emul.cpp")
        deps = [src, os.path.join(_CSRC, "kk_lora.cuh"), os.path.join(_CSRC, "kk_ops.h")]
        L = C.CDLL(_build(src, "libkk_lora_emul.so", cxx, deps, ["-std=c++17", "-x", "c++"]))
        L.kk_lora_emul_launch.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
        L.kk_lora_emul_launch.restype = C.c_int
        _libs["emul"] = L
    return _libs["emul"]


def _ptr(a: np.ndarray) -> int:
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data


# ---- adapters -------------------------------------------------------------------------------------------------------------------------
def rand_lora(rng: np.random.Generator, r: int, R: int, C_: int, dtype: str = "F32", scale: float = 0.05) -> Tuple[np.ndarray, np.ndarray]:
    """Seeded lora_A [r, C] and lora_B [R, r] in `dtype` (numpy arrays of that dtype)."""
    npdt = {"F32": np.float32, "BF16": ml_dtypes.bfloat16, "F16": np.float16}[dtype]
    a = (rng.standard_normal((r, C_)) * scale).astype(np.float32).astype(npdt)
    b = (rng.standard_normal((R, r)) * scale).astype(np.float32).astype(npdt)
    return a, b


def write_adapter(d: str, pairs: Dict[str, Tuple[np.ndarray, np.ndarray]], lora_alpha=16, config: Optional[dict] = None,
                  extra_tensors: Optional[Dict[str, np.ndarray]] = None) -> str:
    """PEFT's save_pretrained layout in directory d: pairs maps module name <M> -> (lora_A, lora_B).  config entries override the
    defaults (None removes a key).  Returns d."""
    from safetensors.numpy import save_file
    os.makedirs(d, exist_ok=True)
    ranks = {m: int(a.shape[0]) for m, (a, b) in pairs.items()}
    r0 = next(iter(ranks.values())) if ranks else 8
    cfg = {"peft_type": "LORA", "task_type": "CAUSAL_LM", "r": r0, "lora_alpha": lora_alpha, "lora_dropout": 0.0, "bias": "none",
           "use_rslora": False, "use_dora": False, "fan_in_fan_out": False, "alpha_pattern": {},
           "rank_pattern": {m: r for m, r in ranks.items() if r != r0}, "target_modules": sorted({m.split(".")[-1] for m in pairs}),
           "modules_to_save": None, "base_model_name_or_path": "synthetic"}
    for k, v in (config or {}).items():
        if v is None:
            cfg.pop(k, None)
        else:
            cfg[k] = v
    tensors = {}
    for m, (a, b) in pairs.items():
        tensors[f"{PREFIX}{m}.lora_A.weight"] = np.ascontiguousarray(a)
        tensors[f"{PREFIX}{m}.lora_B.weight"] = np.ascontiguousarray(b)
    tensors.update(extra_tensors or {})
    save_file(tensors, os.path.join(d, "adapter_model.safetensors"))
    with open(os.path.join(d, "adapter_config.json"), "w") as f:
        json.dump(cfg, f)
    return d


def seeded_adapter(d: str, targets: Iterable[Tuple[str, Sequence[int]]], r, seed: int, dtype: str = "F32", lora_alpha=16,
                   config: Optional[dict] = None) -> Dict[str, Tuple[np.ndarray, np.ndarray]]:
    """An adapter over (<M>.weight name, [R, C]) targets; r is an int or a callable of the target index.  Returns the pairs."""
    rng = np.random.default_rng(seed)
    pairs = {}
    for i, (name, shape) in enumerate(targets):
        assert name.endswith(".weight")
        rk = r(i) if callable(r) else r
        pairs[name[: -len(".weight")]] = rand_lora(rng, rk, int(shape[0]), int(shape[1]), dtype)
    write_adapter(d, pairs, lora_alpha, config)
    return pairs


def scaling(lora_alpha, r: int, rslora: bool = False) -> float:
    return float(np.float32(lora_alpha / (np.sqrt(r) if rslora else r)))


# ---- the merge on the host ------------------------------------------------------------------------------------------------------------
def f32(x: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(x.astype(np.float32))


def oracle_merge(pool: np.ndarray, w_off: int, rows: int, cols: int, row0: int, col0: int, a: np.ndarray, b: np.ndarray, s: float,
                 out: str) -> None:
    """The C oracle's merge of one target into the pool bytes (uint8 array, in place)."""
    A, B = f32(a), f32(b)
    assert pool.dtype == np.uint8 and pool.flags["C_CONTIGUOUS"]
    es = 4 if out == "F32" else 2
    assert w_off + rows * cols * es <= pool.size
    oracle_lib().kk_lora_oracle_merge(_ptr(pool), w_off, rows, cols, row0, col0, _ptr(A), A.shape[1], _ptr(B), A.shape[0], C.c_float(s), OUT[out])


def target_table(targets: Sequence[dict]) -> Tuple[np.ndarray, np.ndarray, int]:
    """(KKLoraTarget table, fp32 adapter buffer, tiles) for targets given as dicts w_off, rows, cols, row0, col0, a, b, s, out — the
    table the loader builds for one pool."""
    chunks, off = [], 0
    tab = np.zeros(len(targets), TARGET_DTYPE)
    tiles = 0
    for i, t in enumerate(targets):
        A, B = f32(t["a"]), f32(t["b"])
        tab[i]["w_off"], tab[i]["rows"], tab[i]["cols"] = t["w_off"], t["rows"], t["cols"]
        tab[i]["row0"], tab[i]["col0"], tab[i]["a_ld"], tab[i]["r"] = t["row0"], t["col0"], A.shape[1], A.shape[0]
        tab[i]["s"], tab[i]["out"] = t["s"], OUT[t["out"]]
        tab[i]["a_off"] = off
        chunks.append(A.ravel())
        off += A.size
        tab[i]["b_off"] = off
        chunks.append(B.ravel())
        off += B.size
        tab[i]["tile_begin"] = tiles
        tab[i]["tiles_c"] = -(-t["cols"] // TILE_C)
        tiles += -(-t["rows"] // TILE_R) * -(-t["cols"] // TILE_C)
    ad = np.ascontiguousarray(np.concatenate(chunks) if chunks else np.zeros(1, np.float32))
    return tab, ad, tiles


def emul_merge(pool: np.ndarray, targets: Sequence[dict]) -> None:
    """The CPU replay of one merge launch over the pool bytes (in place)."""
    tab, ad, tiles = target_table(targets)
    rc = emul_lib().kk_lora_emul_launch(_ptr(tab), len(tab), tiles, _ptr(ad), _ptr(pool))
    assert rc == 0


def expected_pool(base: np.ndarray, desc: dict, pairs: Dict[str, Tuple[np.ndarray, np.ndarray]], placements) -> np.ndarray:
    """The base pool with the C-oracle merge of every described target applied.  placements(name) -> (offset, shape, slice_dim, slice_begin)
    of that tensor in this pool."""
    exp = base.copy()
    for t in desc["targets"]:
        a, b = pairs[t["name"][: -len(".weight")]]
        off, shape, sd, sb = placements(t["name"])
        oracle_merge(exp, off, shape[0], shape[1], sb if sd == 0 else 0, sb if sd == 1 else 0, a, b, t["scaling"], t["dtype"])
    return exp
