"""CPU tier: KK_LOAD_F16 in the planner (through kk_plan_describe) and on the public surfaces.

For every file dtype and every combination of the flags it composes with, the plan must pick the ops and pool dtypes of the table in
include/kukeon_gpuload.h and lay the pool out byte for byte as the same load without the flag, only the float dtype differing; the scatter
row exchange must apply to what the pool holds verbatim (an F16 file's row-parallel tensors, not a BF16 file's); a pipeline stage must
compose.  Then the flag's value against the header, the manifest option, `kuke model plan --option f16`, and the library's environment
knobs, which the flag does not add to."""
import io
import itertools
import json
import os
import re

import pytest

from kukeon_b200 import cli, gpupool, schema
from oracle import oracle
from tests import f16_oracle as fo
from tests import helpers
from tools import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F16, KEEP, F8, T, X = gpupool.LOAD_F16, gpupool.LOAD_KEEP_F32, gpupool.LOAD_F8_TO_BF16, gpupool.LOAD_GPT2_CONV1D_T, gpupool.LOAD_SCATTER_EXCHANGE
FLAG_SETS = [sum(c) for n in range(4) for c in itertools.combinations((KEEP, F8, T, X), n)]


def test_flag_value_against_the_header_and_the_retired_numbers_stay_unused():
    h = open(os.path.join(ROOT, "include", "kukeon_gpuload.h")).read()
    assert int(re.search(r"#define KK_LOAD_F16 (0x[0-9a-f]+)u", h).group(1), 16) == F16 == 0x80 == fo.LOAD_F16
    used = {int(v, 16) for v in re.findall(r"#define KK_LOAD_\w+ (0x[0-9a-f]+)u", h)}
    assert not used & {0x20, 0x40}


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("f16plan")
    st = str(d / "all.safetensors")
    synth.write_safetensors(st, [("model.layers.0.self_attn.o_proj.weight", "BF16", [64, 96]), ("model.layers.0.mlp.down_proj.weight", "F16", [32, 128]),
                                 ("model.layers.0.self_attn.q_proj.weight", "F32", [64, 64]), ("h.0.attn.c_attn.weight", "BF16", [24, 72]),
                                 ("h.0.mlp.c_fc.weight", "F16", [24, 96]), ("h.0.mlp.c_proj.weight", "F32", [96, 24]), ("model.layers.1.e4", "F8_E4M3", [33, 16]),
                                 ("model.layers.1.e5", "F8_E5M2", [17]), ("model.layers.1.ids", "I64", [5]), ("model.layers.1.b", "BOOL", [7]),
                                 ("model.layers.1.d", "F64", [3]), ("model.layers.1.i16", "I16", [8, 24])], 4)
    gg = str(d / "q.gguf")
    from tests.test_plan import f4_tensors
    synth.write_gguf(gg, f4_tensors(hidden=256, ffn=512, layers=2, vocab=256), 3)
    return st, gg


def describe(path, flags, mode=gpupool.MODE_SINGLE, n=1, layers=None):
    return gpupool.plan_describe(path, mode=mode, flags=flags, n_parts=n, layers=layers)


def ops_by_tensor(plan):
    """{pool offset of the segment's tensor: set of ops}, from the segments of every part."""
    out = {}
    for part in plan["parts"]:
        for ch in part["chunks"]:
            for s in ch["segs"]:
                out.setdefault(s["dst_off"], set()).add(s["op"])
    return out


def table_op(dt, flags, transposed):
    """The op of a file dtype under `flags` as include/kukeon_gpuload.h's table gives it (KK_OP_* numbers; the launch format is F16)."""
    if transposed:
        return {"F32": helpers.OP_T_B32 if flags & KEEP else helpers.OP_T_F32_BF16, "BF16": helpers.OP_T_F16_BF16, "F16": helpers.OP_T_B16,
                "I16": helpers.OP_T_B16}[dt]
    if dt == "F32":
        return helpers.OP_COPY if flags & KEEP else helpers.OP_F32
    if dt == "BF16":
        return helpers.OP_F16
    if dt in ("F8_E4M3", "F8_E5M2") and flags & F8:
        return helpers.OP_F8E4M3 if dt == "F8_E4M3" else helpers.OP_F8E5M2
    return helpers.OP_COPY


@pytest.mark.parametrize("flags", FLAG_SETS)
@pytest.mark.parametrize("which", ["safetensors", "gguf"])
def test_ops_pool_dtypes_and_layout_against_the_unflagged_plan(files, flags, which):
    path = files[0] if which == "safetensors" else files[1]
    shards, recs = oracle.index_path(path)
    for mode, n in ((gpupool.MODE_SINGLE, 1), (gpupool.MODE_BROADCAST, 2), (gpupool.MODE_SCATTER, 2)):
        a, b = describe(path, flags, mode, n), describe(path, flags | F16, mode, n)
        assert len(a["layouts"]) == len(b["layouts"])
        for g, (la, lb) in enumerate(zip(a["layouts"], b["layouts"])):
            assert la["pool_bytes"] == lb["pool_bytes"]
            exp, _ = fo.plan_pool(recs, mode, flags | F16, n, g)
            for ta, tb, e in zip(la["tensors"], lb["tensors"], exp):
                want = "F16" if ta["dtype"] == "BF16" else ta["dtype"]
                assert tb == dict(ta, dtype=want), (flags, mode, ta["name"])
                assert (tb["dtype"], tb["pool_offset"], tb["nbytes"], tb["shape"]) == (e["dtype"], e["pool_offset"], e["nbytes"], e["shape"])
        ops, ops_a = ops_by_tensor(b), ops_by_tensor(a)
        rec = {r["name"]: r for r in recs}
        for tb, e in zip(b["layouts"][0]["tensors"], exp if mode != gpupool.MODE_SCATTER else fo.plan_pool(recs, mode, flags | F16, n, 0)[0]):
            if not tb["nbytes"] or tb["pool_offset"] not in ops:
                continue
            dt = rec[tb["name"]]["dtype"]
            got = ops[tb["pool_offset"]]
            if helpers.OP_ROWSPLIT in got:
                assert dt not in ("BF16", "F32") or (dt == "F32" and flags & KEEP), "the exchange moves only what the pool holds verbatim"
                continue
            if dt in oracle.BLOCK_QUANTS:
                assert got == ops_a[tb["pool_offset"]] and len(got) == 1, "block types keep their op: the launch's format decides the output"
                continue
            assert got == {table_op(dt, flags, e["transposed"])}, (tb["name"], dt, flags, mode, got)


def test_block_types_keep_their_ops_and_become_f16(files):
    _, gg = files
    a, b = describe(gg, 0), describe(gg, F16)
    assert ops_by_tensor(a) == ops_by_tensor(b), "the op codes do not change: the launch's format decides the output"
    assert {t["dtype"] for t in b["layouts"][0]["tensors"]} <= {"F16", "F32", "I32"}
    assert "F16" in {t["dtype"] for t in b["layouts"][0]["tensors"]}


def test_the_exchange_applies_to_an_f16_file_and_not_to_a_bf16_one(tmp_path):
    for dt in ("F16", "BF16"):
        d = str(tmp_path / dt)
        synth.make_llama(d, dict(hidden=256, ffn=512, layers=2, kv_dim=64, vocab=512), dtype=dt)
        for flags, want in ((X, dt == "BF16"), (X | F16, dt == "F16")):
            plan = describe(d, flags, gpupool.MODE_SCATTER, 4)
            has = any(s["op"] == helpers.OP_ROWSPLIT for p in plan["parts"] for ch in p["chunks"] for s in ch["segs"])
            assert has == want, (dt, flags)


def test_a_pipeline_stage_composes(tmp_path):
    d = str(tmp_path / "llama")
    synth.make_llama(d, dict(hidden=256, ffn=512, layers=4, kv_dim=64, vocab=512), dtype="BF16")
    for layers in ((0, 2), (2, 4)):
        a, b = describe(d, 0, layers=layers), describe(d, F16, layers=layers)
        assert b["layers"] == list(layers) and b["n_layers"] == 4
        assert [dict(t, dtype="F16" if t["dtype"] == "BF16" else t["dtype"]) for t in a["layouts"][0]["tensors"]] == b["layouts"][0]["tensors"]
        assert {t["dtype"] for t in b["layouts"][0]["tensors"]} == {"F16"}


def test_manifest_option_and_cli(files):
    specs = schema.validate_models([{"name": "a", "source": "/m", "options": {"f16": True}}, {"name": "b", "source": "/m", "options": {"f16": False}},
                                    {"name": "c", "source": "/m", "options": {"f16": True, "keepF32": True}}], stat=lambda p: None)
    assert [s.flags for s in specs] == [F16, 0, F16 | KEEP]
    st, _ = files
    out = io.StringIO()
    assert cli.main(["model", "plan", st, "--option", "f16", "-o", "json", "--full"], out) == 0
    doc = json.loads(out.getvalue())
    assert doc["flags"] == F16
    dts = {t["name"]: t["dtype"] for t in doc["layouts"][0]["tensors"]}
    assert dts["model.layers.0.self_attn.o_proj.weight"] == dts["model.layers.0.mlp.down_proj.weight"] == "F16"
    out = io.StringIO()
    assert cli.main(["model", "plan", st, "-o", "json", "--full"], out) == 0
    assert json.loads(out.getvalue())["layouts"][0]["tensors"][0]["dtype"] == "BF16"


def test_environment_knobs_are_unchanged():
    """The output format is a load flag, not an environment knob: the library reads the same two variables as before."""
    names = set()
    for f in os.listdir(os.path.join(ROOT, "kukeon_b200", "csrc")):
        if f.endswith((".cpp", ".cu", ".cuh", ".hpp", ".h")):
            names |= set(re.findall(r'getenv\("([A-Z0-9_]+)"\)', open(os.path.join(ROOT, "kukeon_b200", "csrc", f)).read()))
    assert names == {"KUKEON_GPULOAD_READ", "KUKEON_GPULOAD_TEST_NDST"}
