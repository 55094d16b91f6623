"""LoRA adapters on load (kk_load_adapter / kk_adapter_describe), CPU tier: matching and scaling, every refusal with ctx = NULL, the C oracle
of the merge against a float64 restatement of PEFT's formula, the CPU replay of the merge kernel against the C oracle bit for bit, the
surfaces above the ABI and the kernel's compile.

Adapters are written by the tests in PEFT's saved format (adapter_config.json + adapter_model.safetensors, keys
base_model.model.<M>.lora_{A,B}.weight), seeded numpy + safetensors + json.  peft is not installed here, so the format is restated from
its documentation (tests/lora_fixtures.py)."""
import io
import json
import os
import re
import subprocess

import ml_dtypes
import numpy as np
import pytest

from kukeon_b200 import cli, gpupool, registry, schema
from tests import lora_fixtures as lf
from tools import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_GGUF = os.path.join(ROOT, "tests", "golden", "hf_llama_moe.gguf")
CFG = dict(hidden=256, ffn=704, layers=3, kv_dim=64, vocab=300)


@pytest.fixture(scope="module")
def llama(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("lora") / "llama")
    synth.make_llama(d, CFG)
    return d


def proj_targets(path, flags=0):
    recs = gpupool.index(path) if not flags else None
    if recs is None:
        plan = gpupool.plan_describe(path, flags=flags)
        recs = [dict(name=t["name"], shape=t["shape"]) for t in plan["layouts"][0]["tensors"]]
    return [(t["name"], t["shape"]) for t in recs if re.search(r"_proj\.weight$", t["name"]) and len(t["shape"]) == 2]


# ---- 1. describe: matching and scaling ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alpha,rslora", [(16, False), (16, True), (12.5, False), (7.25, True)])
def test_describe_matches_every_target_with_its_scaling(native, llama, tmp_path, alpha, rslora):
    tg = proj_targets(llama)
    ranks = [1, 7, 16, 64]  # a rank_pattern adapter: every pair's own rank
    pairs = lf.seeded_adapter(str(tmp_path / "ad"), tg, lambda i: ranks[i % 4], 5, "BF16", alpha, {"use_rslora": rslora})
    d = gpupool.adapter_describe(llama, str(tmp_path / "ad"))
    assert d["n_targets"] == len(tg) == len(pairs) and d["skipped"] == []
    assert d["use_rslora"] is rslora and d["lora_alpha"] == alpha
    by = {t["name"]: t for t in d["targets"]}
    for i, (name, shape) in enumerate(tg):
        t = by[name]
        r = ranks[i % 4]
        assert t["shape"] == shape and t["r"] == r and t["dtype"] == "BF16"
        assert t["lora_A"] == f"base_model.model.{name[:-7]}.lora_A.weight" and t["lora_B_dtype"] == "BF16"
        want = np.float32(alpha / (np.sqrt(np.float64(r)) if rslora else np.float64(r)))
        assert np.float32(t["scaling"]) == want, (name, t["scaling"], want)
    # the adapter file itself is an accepted spelling of the adapter
    assert gpupool.adapter_describe(llama, str(tmp_path / "ad" / "adapter_model.safetensors"))["targets"] == d["targets"]


def test_describe_follows_the_pool_dtype(native, llama, tmp_path):
    lf.seeded_adapter(str(tmp_path / "ad"), proj_targets(llama)[:3], 4, 1)
    assert {t["dtype"] for t in gpupool.adapter_describe(llama, str(tmp_path / "ad"), flags=gpupool.LOAD_F16)["targets"]} == {"F16"}
    f32 = str(tmp_path / "f32.safetensors")
    synth.write_safetensors(f32, [("model.layers.0.mlp.up_proj.weight", "F32", [96, 80]), ("model.norm.weight", "F32", [80])], 3)
    lf.seeded_adapter(str(tmp_path / "ad32"), [("model.layers.0.mlp.up_proj.weight", [96, 80])], 8, 2)
    assert gpupool.adapter_describe(f32, str(tmp_path / "ad32"), flags=gpupool.LOAD_KEEP_F32)["targets"][0]["dtype"] == "F32"
    assert gpupool.adapter_describe(f32, str(tmp_path / "ad32"))["targets"][0]["dtype"] == "BF16"


def test_describe_layer_stage_skips_targets_outside_it(native, llama, tmp_path):
    tg = proj_targets(llama)
    lf.seeded_adapter(str(tmp_path / "ad"), tg, 8, 3)
    d = gpupool.adapter_describe(llama, str(tmp_path / "ad"), layers=(1, 2))
    assert {t["name"] for t in d["targets"]} == {n for n, _ in tg if ".layers.1." in n}
    assert set(d["skipped"]) == {n for n, _ in tg if ".layers.1." not in n}


def test_describe_gguf_under_hf_layout(native, tmp_path):
    tg = proj_targets(GOLDEN_GGUF, gpupool.LOAD_HF_LAYOUT)
    assert any(".self_attn.q_proj." in n for n, _ in tg)
    lf.seeded_adapter(str(tmp_path / "ad"), tg, 4, 9)
    d = gpupool.adapter_describe(GOLDEN_GGUF, str(tmp_path / "ad"), flags=gpupool.LOAD_HF_LAYOUT)
    assert {t["name"] for t in d["targets"]} == {n for n, _ in tg}
    # the GGUF's own names are not the view a plain load plans over: the HF names do not exist there
    with pytest.raises(gpupool.ErrNotFound):
        gpupool.adapter_describe(GOLDEN_GGUF, str(tmp_path / "ad"))


def test_describe_scatter_parts(native, llama, tmp_path):
    lf.seeded_adapter(str(tmp_path / "ad"), proj_targets(llama), 8, 3)
    d = gpupool.adapter_describe(llama, str(tmp_path / "ad"), mode=gpupool.MODE_SCATTER, part_index=1, part_count=2)
    assert d["n_targets"] == len(proj_targets(llama))


# ---- 2. describe: refusals ------------------------------------------------------------------------------------------------------------
def _one(llama, d, **kw):
    name, shape = proj_targets(llama)[0]
    rng = np.random.default_rng(1)
    a, b = lf.rand_lora(rng, kw.pop("r", 4), shape[0], shape[1], kw.pop("dtype", "F32"))
    pairs = {name[:-7]: (a, b)}
    pairs.update(kw.pop("more", {}))
    lf.write_adapter(d, pairs, config=kw.pop("config", None), extra_tensors=kw.pop("extra", None))
    return d


def _refusals(llama, tmp):
    name, shape = proj_targets(llama)[0]
    m = name[:-7]
    rng = np.random.default_rng(2)
    a, b = lf.rand_lora(rng, 4, shape[0], shape[1])
    P = "base_model.model."
    cases = {
        "alpha_pattern": (gpupool.ErrUnsupported, dict(config={"alpha_pattern": {"q_proj": 8}})),
        "use_dora": (gpupool.ErrUnsupported, dict(config={"use_dora": True})),
        "magnitude": (gpupool.ErrUnsupported, dict(extra={f"{P}{m}.lora_magnitude_vector": np.ones(shape[0], np.float32)})),
        "fan_in_fan_out": (gpupool.ErrUnsupported, dict(config={"fan_in_fan_out": True})),
        "embedding": (gpupool.ErrUnsupported, dict(extra={f"{P}model.embed_tokens.lora_embedding_A": np.ones((4, 300), np.float32)})),
        "modules_to_save": (gpupool.ErrUnsupported, dict(extra={f"{P}lm_head.modules_to_save.default.weight": np.ones((4, 4), np.float32)})),
        "bias_tensor": (gpupool.ErrUnsupported, dict(extra={f"{P}{m}.lora_B.bias": np.ones(shape[0], np.float32)})),
        "bias_config": (gpupool.ErrUnsupported, dict(config={"bias": "lora_only"})),
        "dtype_f64": (gpupool.ErrUnsupported, dict(more={"model.layers.0.self_attn.k_proj": (np.ones((2, 256)), np.ones((64, 2)))})),
        "r_too_large": (gpupool.ErrUnsupported, dict(r=257)),
        "unpaired": (gpupool.ErrFormat, dict(extra={f"{P}model.layers.0.self_attn.k_proj.lora_A.weight": np.ones((4, 256), np.float32)})),
        "shape": (gpupool.ErrFormat, dict(more={"model.layers.0.self_attn.k_proj": (np.ones((4, 255), np.float32), np.ones((64, 4), np.float32))})),
        "rank_mismatch": (gpupool.ErrFormat, dict(more={"model.layers.0.self_attn.k_proj": (np.ones((4, 256), np.float32), np.ones((64, 3), np.float32))})),
        "alpha_missing": (gpupool.ErrFormat, dict(config={"lora_alpha": None})),
        "alpha_string": (gpupool.ErrFormat, dict(config={"lora_alpha": "16"})),
        "rslora_string": (gpupool.ErrFormat, dict(config={"use_rslora": "yes"})),
        "not_lora_key": (gpupool.ErrFormat, dict(extra={f"{P}{m}.ia3_l": np.ones(4, np.float32)})),
        "no_target": (gpupool.ErrNotFound, dict(more={"model.layers.9.self_attn.q_proj": (a, b)})),
        "not_2d": (gpupool.ErrUnsupported, dict(more={"model.layers.0.input_layernorm": (np.ones((4, 256), np.float32), np.ones((256, 4), np.float32))})),
    }
    return cases


def test_every_refusal_with_ctx_null(native, llama, tmp_path):
    for k, (err, kw) in _refusals(llama, tmp_path).items():
        d = _one(llama, str(tmp_path / k), **kw)
        with pytest.raises(err):
            gpupool.adapter_describe(llama, d)
        assert native.kk_adapter_describe(None, llama.encode(), None, d.encode(), None, 0, None) == -1  # NULL opts: KK_EINVAL


def test_refusals_of_files_and_load_shapes(native, llama, tmp_path):
    good = _one(llama, str(tmp_path / "good"))
    gpupool.adapter_describe(llama, good)
    with pytest.raises(gpupool.ErrNotFound):
        gpupool.adapter_describe(llama, str(tmp_path / "missing"))
    os.makedirs(tmp_path / "bin")
    open(tmp_path / "bin" / "adapter_model.bin", "wb").write(b"\x80\x02")
    json.dump({"lora_alpha": 8}, open(tmp_path / "bin" / "adapter_config.json", "w"))
    with pytest.raises(gpupool.ErrUnsupported):
        gpupool.adapter_describe(llama, str(tmp_path / "bin"))
    with pytest.raises(gpupool.ErrUnsupported):
        gpupool.adapter_describe(llama, str(tmp_path / "bin" / "adapter_model.bin"))
    os.remove(os.path.join(good, "adapter_config.json"))
    with pytest.raises(gpupool.ErrNotFound):
        gpupool.adapter_describe(llama, good)
    good = _one(llama, str(tmp_path / "good2"))
    with pytest.raises(gpupool.ErrUnsupported):
        gpupool.adapter_describe(llama, good, mode=gpupool.MODE_BROADCAST, fanout=gpupool.FANOUT_NVLS)
    for fanout in (gpupool.FANOUT_P2P, gpupool.FANOUT_RAW, gpupool.FANOUT_PULL):
        with pytest.raises(gpupool.ErrUnsupported):
            gpupool.adapter_describe(llama, good, mode=gpupool.MODE_BROADCAST, fanout=fanout, part_index=0, part_count=2)
    with pytest.raises(gpupool.ErrUnsupported):
        gpupool.adapter_describe(llama, good, mode=gpupool.MODE_SCATTER, flags=gpupool.LOAD_SCATTER_EXCHANGE, part_index=0, part_count=2)
    gpupool.adapter_describe(llama, good, mode=gpupool.MODE_SCATTER, part_index=0, part_count=2)


def test_refusals_of_pool_dtypes(native, tmp_path):
    p = str(tmp_path / "mixed.safetensors")
    synth.write_safetensors(p, [("model.layers.0.mlp.up_proj.weight", "F8_E4M3", [64, 64]), ("model.layers.0.mlp.down_proj.weight", "I32", [64, 64])], 4)
    for mod in ("model.layers.0.mlp.up_proj", "model.layers.0.mlp.down_proj"):
        d = str(tmp_path / mod)
        lf.write_adapter(d, {mod: lf.rand_lora(np.random.default_rng(0), 4, 64, 64)})
        with pytest.raises(gpupool.ErrUnsupported):
            gpupool.adapter_describe(p, d)
    gpupool.adapter_describe(p, str(tmp_path / "model.layers.0.mlp.up_proj"), flags=gpupool.LOAD_F8_TO_BF16)  # widened FP8 is bf16
    g = str(tmp_path / "gpt2.safetensors")
    synth.make_gpt2(g, n_layer=1, d=64, vocab=100, n_pos=16)
    d = str(tmp_path / "gpt2ad")
    lf.write_adapter(d, {"h.0.attn.c_proj": lf.rand_lora(np.random.default_rng(0), 4, 64, 64)})
    names = {t["name"] for t in gpupool.index(g)}
    if "h.0.attn.c_proj.weight" in names:
        with pytest.raises(gpupool.ErrUnsupported):
            gpupool.adapter_describe(g, d, flags=gpupool.LOAD_GPT2_CONV1D_T)


# ---- 3. the C oracle against PEFT's formula in float64 --------------------------------------------------------------------------------
def _ulp(x, dt):
    x = np.abs(x)
    mant, emin = {"BF16": (7, -126), "F16": (10, -14), "F32": (23, -126)}[dt]
    e = np.floor(np.log2(np.maximum(x, np.finfo(np.float64).tiny)))
    return np.exp2(np.maximum(e, emin) - mant)


@pytest.mark.parametrize("dt", ["BF16", "F16", "F32"])
@pytest.mark.parametrize("r", [1, 16, 256])
def test_c_oracle_against_peft_formula_in_float64(dt, r):
    import torch
    rng = np.random.default_rng(r * 7 + len(dt))
    R, Cc = 67, 131
    npdt = {"BF16": ml_dtypes.bfloat16, "F16": np.float16, "F32": np.float32}[dt]
    w = (rng.standard_normal((R, Cc)) * 0.5).astype(np.float32).astype(npdt)
    a, b = lf.rand_lora(rng, r, R, Cc, "BF16", scale=0.2)
    s = lf.scaling(32, r, rslora=r > 16)
    pool = np.ascontiguousarray(w).view(np.uint8).ravel().copy()
    lf.oracle_merge(pool, 0, R, Cc, 0, 0, a, b, s, dt)
    got = pool.view(npdt).reshape(R, Cc).astype(np.float64)
    W, A, B = (torch.from_numpy(np.asarray(x, np.float64)) for x in (w.astype(np.float32), a.astype(np.float32), b.astype(np.float32)))
    ref = (W + (B @ A) * s).numpy()  # PEFT: W + (B @ A) * scaling
    absba = (B.abs() @ A.abs()).numpy()
    eps = 2.0 ** -24
    bound = _ulp(ref, dt) + abs(s) * (r + 1) * eps * absba + eps * np.abs(ref)
    assert np.all(np.abs(got - ref) <= bound), np.max(np.abs(got - ref) / bound)


# ---- 4. the CPU replay of the kernel against the C oracle, bit for bit ----------------------------------------------------------------
def _specials(rng, n, dt):
    """Random pool elements with inf, NaN and subnormal patterns mixed in."""
    if dt == "F32":
        v = (rng.standard_normal(n) * 2).astype(np.float32).view(np.uint32)
        sp = np.array([0x7F800000, 0xFF800000, 0x7FC00001, 0xFFFFFFFF, 0x00000001, 0x807FFFFF, 0x7F7FFFFF, 0], np.uint32)
    else:
        npdt = ml_dtypes.bfloat16 if dt == "BF16" else np.float16
        v = (rng.standard_normal(n) * 2).astype(np.float32).astype(npdt).view(np.uint16)
        sp = np.array([0x7F80, 0xFF80, 0x7FC1, 0xFFFF, 0x0001, 0x807F, 0x7F7F] if dt == "BF16" else [0x7C00, 0xFC00, 0x7E01, 0xFFFF, 0x0001, 0x83FF, 0x7BFF],
                      np.uint16)
    k = rng.integers(0, n, n // 20)
    v[k] = sp[rng.integers(0, len(sp), len(k))]
    return v.view(np.uint8)


def _case(rng, specs):
    """A pool of random bytes holding one target per spec (R, C, r, dtype, slice_dim, n_slices, slice_index) at 256-byte boundaries."""
    targets, off, parts = [], 256, []
    for (R, Cc, r, dt, sd, n, k) in specs:
        a, b = lf.rand_lora(rng, r, R, Cc, ["F32", "BF16", "F16"][r % 3], scale=0.3)
        if r % 5 == 0:
            a = a.astype(np.float32)
            a.ravel()[rng.integers(0, a.size, 3)] = [np.inf, np.nan, 1e-40]
        rows, cols, row0, col0 = R, Cc, 0, 0
        if sd == 0:
            rows, row0 = R // n, R // n * k
        elif sd == 1:
            cols, col0 = Cc // n, Cc // n * k
        es = 4 if dt == "F32" else 2
        targets.append(dict(w_off=off, rows=rows, cols=cols, row0=row0, col0=col0, a=a, b=b, s=lf.scaling(16, r, r > 60), out=dt))
        parts.append((off, dt, rows * cols))
        off += (rows * cols * es + 255) // 256 * 256 + 256 * int(rng.integers(0, 3))
    pool = rng.integers(0, 256, off + 512, dtype=np.uint8)
    for o, dt, ne in parts:
        pool[o:o + ne * (4 if dt == "F32" else 2)] = _specials(rng, ne, dt)
    return pool, targets


CASES = {
    "ranks": [(130, 200, r, "BF16", None, 1, 0) for r in (1, 7, 16, 64, 256)],
    "edges": [(64, 128, 8, "BF16", None, 1, 0), (65, 129, 8, "F16", None, 1, 0), (1, 1, 3, "F32", None, 1, 0), (127, 255, 33, "BF16", None, 1, 0),
              (70, 12, 5, "F16", None, 1, 0), (9, 300, 2, "F32", None, 1, 0)],
    "slices": [(128, 192, 16, "BF16", 0, 2, 1), (96, 256, 7, "F16", 1, 4, 3), (200, 136, 64, "F32", 1, 2, 1), (150, 100, 16, "BF16", 0, 3, 2)],
    "dtypes": [(100, 300, 16, dt, None, 1, 0) for dt in ("BF16", "F16", "F32")],
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_cpu_replay_equals_c_oracle(case):
    rng = np.random.default_rng(sorted(CASES).index(case) + 40)
    pool, targets = _case(rng, CASES[case])
    got, exp = pool.copy(), pool.copy()
    lf.emul_merge(got, targets)
    for t in targets:
        lf.oracle_merge(exp, t["w_off"], t["rows"], t["cols"], t["row0"], t["col0"], t["a"], t["b"], t["s"], t["out"])
    diff = np.flatnonzero(got != exp)
    assert diff.size == 0, f"{diff.size} bytes differ, first at {diff[:8]}"
    inside = np.zeros(pool.size, bool)
    for t in targets:
        inside[t["w_off"]:t["w_off"] + t["rows"] * t["cols"] * (4 if t["out"] == "F32" else 2)] = True
    assert np.array_equal(got[~inside], pool[~inside]), "a byte outside the targets changed"
    assert (got[inside] != pool[inside]).any()


def test_replay_nan_is_canonical():
    rng = np.random.default_rng(5)
    for dt, nan in (("BF16", 0x7FFF), ("F16", 0x7FFF), ("F32", 0x7FFFFFFF)):
        es = 4 if dt == "F32" else 2
        w = np.full(64 * 128, 0xFFC00001 if es == 4 else 0xFFC1 if dt == "BF16" else 0xFE01, np.uint32 if es == 4 else np.uint16)
        pool = w.view(np.uint8).copy()
        a, b = lf.rand_lora(rng, 4, 64, 128)
        lf.emul_merge(pool, [dict(w_off=0, rows=64, cols=128, row0=0, col0=0, a=a, b=b, s=1.0, out=dt)])
        assert (pool.view(w.dtype) == nan).all()


# ---- 5. surfaces ----------------------------------------------------------------------------------------------------------------------
def test_abi_symbols_listed():
    assert {"kk_load_adapter", "kk_adapter_describe"} <= set(gpupool.ABI_SYMBOLS)


def test_schema_adapter(tmp_path):
    src = str(tmp_path)
    ok = schema.validate_models([dict(name="m", source=src, adapter=src)])
    assert ok[0].adapter == src
    assert schema.validate_models([dict(name="m", source=src)])[0].adapter is None
    for bad, sentinel in (("rel/ad", schema.Err.ModelAdapterRegistryNotSupported), ("hf://org/ad", schema.Err.ModelAdapterRegistryNotSupported),
                          ("ad", schema.Err.ModelAdapterNotAbsolute), (src + "/missing", schema.Err.ModelAdapterNotFound)):
        with pytest.raises(schema.SchemaError) as e:
            schema.validate_models([dict(name="m", source=src, adapter=bad)])
        assert e.value.sentinel == sentinel


def test_registry_round_trips_the_adapter(tmp_path):
    reg = registry.PoolRegistry(str(tmp_path), epoch="a")
    reg.reconcile()
    reg.record("k1", "/m", 0, 10, 20, [0], [], adapter="/ad")
    reg.record("k2", "/m", 0, 10, 20, [0], [])
    stale = {e.key: e for e in registry.PoolRegistry(str(tmp_path), epoch="b").reconcile()}
    assert stale["k1"].adapter == "/ad" and stale["k2"].adapter is None
    assert "adapter" not in stale["k2"].to_json()


def test_cli_plan_adapter(native, llama, tmp_path):
    tg = proj_targets(llama)
    lf.seeded_adapter(str(tmp_path / "ad"), tg, 8, 3)
    out = io.StringIO()
    assert cli.main(["model", "plan", llama, "--adapter", str(tmp_path / "ad")], out) == 0
    text = out.getvalue()
    assert "TARGET" in text and f"{len(tg)} tensors merged" in text and tg[0][0] in text
    out = io.StringIO()
    assert cli.main(["model", "plan", llama, "--adapter", str(tmp_path / "ad"), "--layers", "0:1", "-o", "json"], out) == 0
    doc = json.loads(out.getvalue())
    assert len(doc["adapter"]["targets"]) == len([n for n, _ in tg if ".layers.0." in n]) and doc["adapter"]["skipped"]
    out = io.StringIO()
    assert cli.main(["model", "plan", llama, "--adapter", str(tmp_path / "ad"), "-o", "yaml"], out) == 0
    assert "adapter:" in out.getvalue()
    out = io.StringIO()
    assert cli.main(["model", "plan", llama, "-o", "json"], out) == 0
    assert "adapter" not in json.loads(out.getvalue())


# ---- 6. compile check -----------------------------------------------------------------------------------------------------------------
def test_merge_kernel_compiles_without_spills(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc is not installed")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c",
                        os.path.join(ROOT, "kukeon_b200", "csrc", "kk_lora.cu"), "-o", str(tmp_path / "kk_lora.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    info = [ln for ln in r.stderr.splitlines() if "spill" in ln]
    assert info and all("0 bytes spill stores, 0 bytes spill loads" in ln for ln in info), r.stderr
    assert "kk_lora_merge_kernel" in r.stderr
    assert "0 bytes stack frame" in r.stderr
