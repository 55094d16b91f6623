"""CPU tier: KK_LOAD_HF_LAYOUT (GGUF loads in Hugging Face layout) through kk_plan_describe and the CPU replay of the convert kernel.

The rename table is pinned to gguf-py's tensor_mapping and the un-permutation to transformers' GGUF loader and to llama.cpp's forward
permutation; the planner's output is checked for its invariants (every pool byte written once, reads inside the tensor, destination
offsets non-decreasing per part, PULL ranges disjoint and covering) and played through the device code against tests/hf_oracle.py, in
every mode, for every block type and float type, bf16 and fp16 output; refusals come with their status before any device is used; and a
load without the flag is what it was."""
import importlib.util
import io
import json
import os
import re
import struct

import numpy as np
import pytest
from hypothesis import HealthCheck, assume, given, settings, strategies as st

from kukeon_b200 import cli, gpupool, schema
from oracle import oracle
from tests import helpers, hf_oracle, kk_emul, kk_f16_emul, layer_oracle
from tests.kk_emul import Pools
from tests.test_launch_emul import Exchange, check, play_part
from tools import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")
HF, F16, KEEP, X, DEFER = gpupool.LOAD_HF_LAYOUT, gpupool.LOAD_F16, gpupool.LOAD_KEEP_F32, gpupool.LOAD_SCATTER_EXCHANGE, gpupool.LOAD_DEFER
MB = 1 << 20


def make(path, arch="llama", n_head=4, n_head_kv=2, seed=3, kv=None, **cfg):
    """A GGUF of llama.cpp's inventory with head counts; returns (shards, HF-view oracle records)."""
    c = dict(hidden=256, ffn=512, layers=2, vocab=256, n_head=n_head, n_head_kv=n_head_kv, arch=arch)
    c.update(cfg)
    experts = c.get("experts", 0)
    synth.write_gguf(path, synth.llama_gguf_tensors(**c), seed, arch=arch,
                     extra_kv=synth.gguf_head_kv(arch, n_head, n_head_kv, experts) if kv is None else kv)
    shards, recs = oracle.index_path(path)
    return shards, hf_oracle.hf_view(recs, arch, n_head, n_head_kv)


def test_flag_value_against_the_header_and_the_surfaces():
    h = open(os.path.join(ROOT, "include", "kukeon_gpuload.h")).read()
    assert int(re.search(r"#define KK_LOAD_HF_LAYOUT (0x[0-9a-f]+)u", h).group(1), 16) == HF == 0x100 == hf_oracle.LOAD_HF_LAYOUT
    assert "kFlagHFLayout = KK_LOAD_HF_LAYOUT" in open(os.path.join(ROOT, "host", "modelhub.hpp")).read()
    go = open(os.path.join(ROOT, "host", "go", "internal", "controller", "validate_models.go")).read()
    assert re.search(r'"hfLayout":\s+gpupool.FlagHFLayout', go)
    assert schema.OPTION_FLAGS["hfLayout"] == HF


# ---- the rename table and the permutation, pinned to their owners -------------------------------------------------------------------
@pytest.mark.parametrize("arch", hf_oracle.ARCHS)
def test_names_pinned_to_gguf_py(arch, tmp_path):
    gguf = pytest.importorskip("gguf")
    experts = 4 if arch == "llama" else 0
    p = str(tmp_path / "m.gguf")
    make(p, arch=arch, experts=experts, bias=True)
    plan = gpupool.plan_describe(p, flags=HF)
    assert plan["layout"] == "hf" and plan["architecture"] == arch
    names = [t["name"] for t in plan["layouts"][0]["tensors"]]
    _, recs = oracle.index_path(p)
    assert names == [r["name"] for r in hf_oracle.hf_view(recs, arch, 4, 2)]
    tmap = gguf.get_tensor_name_map({"llama": gguf.MODEL_ARCH.LLAMA, "qwen2": gguf.MODEL_ARCH.QWEN2, "qwen3": gguf.MODEL_ARCH.QWEN3}[arch], 2)
    # pair each of the plan's tensors with the file's tensor at the same place in (shard, offset) order: gguf-py must map the HF name to
    # exactly that GGUF name (a swap of w1 / w3 or q / k in the library and the restated table alike fails here)
    by_offset = [r["name"] for r in recs for _ in range(r["shape"][0] if r["name"].endswith("_exps.weight") else 1)]
    assert len(by_offset) == len(names)
    for n, src in zip(names, by_offset):
        base, sfx = n.rsplit(".", 1)
        m = re.fullmatch(r"(model\.layers\.\d+\.block_sparse_moe\.experts)\.\d+\.(w[123])", base)
        want = tmap.get_name(f"{m.group(1)}.{m.group(2)}" if m else base)  # per-expert names against the merged HF name
        assert want is not None and f"{want}.{sfx}" == src, (n, want, src)
    # and the expert index follows the byte order inside the stack
    for r in hf_oracle.hf_view(recs, arch, 4, 2):
        m = re.search(r"experts\.(\d+)\.", r["name"])
        if m:
            stack = next(x for x in recs if x["name"] == r["gguf_name"])
            assert r["file_offset"] == stack["file_offset"] + int(m.group(1)) * r["nbytes"]


def _permute_llama_cpp(w, n_head, n_head_kv=None):
    """llama.cpp convert_hf_to_gguf.py LlamaModel.permute, restated."""
    if n_head_kv is not None and n_head != n_head_kv:
        n_head = n_head_kv
    return w.reshape(n_head, 2, w.shape[0] // n_head // 2, *w.shape[1:]).swapaxes(1, 2).reshape(w.shape)


@pytest.mark.parametrize("n_head,n_head_kv,hd,cols", [(4, 4, 16, 24), (8, 2, 32, 40), (32, 8, 128, 5), (6, 3, 64, 0)])
def test_unpermutation_pinned_to_transformers_and_inverts_llama_cpp(n_head, n_head_kv, hd, cols):
    from transformers.modeling_gguf_pytorch_utils import LlamaTensorProcessor
    proc = LlamaTensorProcessor(config={"num_attention_heads": n_head, "num_key_value_heads": n_head_kv})
    rng = np.random.default_rng(n_head * 1000 + hd)
    for heads, kind in ((n_head, "q"), (n_head_kv, "k")):
        shape = (heads * hd, cols) if cols else (heads * hd,)  # cols == 0: a bias
        hfw = rng.standard_normal(shape).astype(np.float32)
        gg = _permute_llama_cpp(hfw, n_head, n_head_kv if kind == "k" else n_head)
        assert np.array_equal(hf_oracle.permute(gg * 0 + hfw, heads), gg)
        want = proc._reverse_permute_weights(gg, n_head, n_head_kv if kind == "k" else n_head)
        assert np.array_equal(hf_oracle.unpermute(gg, heads), want)
        assert np.array_equal(want, hfw)
        # the planner's row rule: HF row h*hd + k*hd/2 + i is file row h*hd + 2i + k
        rows = np.array([h * hd + 2 * i + k for h in range(heads) for k in range(2) for i in range(hd // 2)])
        assert np.array_equal(gg[rows], hfw)


# ---- plan invariants --------------------------------------------------------------------------------------------------------------
def _segs(plan, part):
    for ch in plan["parts"][part]["chunks"]:
        for s in ch["segs"]:
            yield ch, s


def check_plan(plan, shards, hf_recs, mode, flags, n):
    """Every pool byte written exactly once with the oracle's value (helpers.emulate_part asserts reads, segments and overlaps), reads
    inside their tensor, destination offsets non-decreasing per part, and (BROADCAST) part ranges disjoint and covering."""
    oflags = flags & (KEEP | F16)
    spans = []  # the tensors' file bytes, back-to-back tensors joined (the planner merges their reads)
    for s, a, b in sorted((r["shard"], r["file_offset"], r["file_offset"] + r["nbytes"]) for r in hf_recs):
        if spans and spans[-1][0] == s and spans[-1][2] == a:
            spans[-1][2] = b
        else:
            spans.append([s, a, b])
    for g in range(n):
        for ch in plan["parts"][g]["chunks"]:
            for fo, ln, _ in ch["reads"]:
                assert any(s == ch["shard"] and a <= fo and fo + ln <= b for s, a, b in spans), "a read leaves the tensors' bytes"
        dst = [s["dst_off"] for _, s in _segs(plan, g) if s["op"] != helpers.OP_ROWSPLIT]
        assert dst == sorted(dst), "destination offsets decrease inside a part"
    if mode == gpupool.MODE_SCATTER:
        for g in range(n):
            exp, pl = hf_oracle.expected_pool(shards, hf_recs, mode, oflags, n, g)
            assert plan["layouts"][g]["pool_bytes"] == len(exp)
            if not any(s["op"] == helpers.OP_ROWSPLIT for _, s in _segs(plan, g)):
                pool, mask = helpers.emulate_part(plan, g, len(exp))
                assert np.array_equal(mask, helpers.expected_mask(pl, len(exp)))
                if not oflags & F16:
                    assert np.array_equal(pool, exp)
        return
    exp, pl = hf_oracle.expected_pool(shards, hf_recs, mode, oflags)
    total = np.zeros(len(exp), np.uint8)
    ranges = []
    for g in range(n):
        pool, mask = helpers.emulate_part(plan, g, len(exp))
        assert not (total.astype(bool) & mask).any(), "two parts write one byte"
        total |= mask.astype(np.uint8)
        if mask.any():
            idx = np.flatnonzero(mask)
            ranges.append((idx[0], idx[-1] + 1))
        if not oflags & F16:
            assert np.array_equal(pool[mask], exp[mask])
    assert np.array_equal(total.astype(bool), helpers.expected_mask(pl, len(exp)))
    ranges.sort()
    assert all(a[1] <= b[0] for a, b in zip(ranges, ranges[1:])), "part pool ranges overlap"


@settings(max_examples=25, deadline=None, suppress_health_check=list(HealthCheck))
@given(n_head=st.sampled_from([2, 3, 4, 6]), kv_div=st.sampled_from([1, 2, 3]), hd=st.sampled_from([16, 32, 64, 128]),
       qtype=st.sampled_from(["BF16", "F16", "F32", "Q8_0", "Q4_0", "Q6_K", "Q4_K"]), experts=st.sampled_from([0, 2, 4]),
       bias=st.booleans(), mode_n=st.sampled_from([(0, 1), (1, 2), (1, 3), (2, 2), (2, 4)]), flags=st.sampled_from([0, F16, KEEP, DEFER]),
       chunk=st.sampled_from([1, 2]), stage=st.sampled_from([None, (0, 1), (1, 2)]))
def test_plan_properties(tmp_path_factory, n_head, kv_div, hd, qtype, experts, bias, mode_n, flags, chunk, stage):
    n_head_kv = n_head // kv_div if n_head % kv_div == 0 else n_head
    block = {"Q8_0": 32, "Q4_0": 32, "Q6_K": 256, "Q4_K": 256}.get(qtype, 1)
    assume((n_head * hd) % block == 0)  # o_proj's rows are n_head * hd long
    p = str(tmp_path_factory.mktemp("hfprop") / "m.gguf")
    shards, hf = make(p, n_head=n_head, n_head_kv=n_head_kv, head_dim=hd, hidden=256, ffn=256, qtype=qtype, experts=experts, bias=bias,
                      vocab=64, seed=n_head + hd)
    mode, n = mode_n
    plan = gpupool.plan_describe(p, mode=mode, flags=HF | flags, n_parts=n, chunk_bytes=chunk * MB, layers=stage)
    if stage:
        hf = layer_oracle.select_layers(hf, *stage)
    assert [t["name"] for t in plan["layouts"][0]["tensors"]] == [r["name"] for r in hf]
    check_plan(plan, shards, hf, mode, flags, n)


def test_scatter_slices_cut_head_groups(tmp_path):
    """N = 4 over 6 heads of 32 rows (q: 192 rows, 48 per rank): slice boundaries fall inside (head, half) groups."""
    p = str(tmp_path / "m.gguf")
    shards, hf = make(p, n_head=6, n_head_kv=2, head_dim=64, hidden=384, ffn=512, vocab=64)
    for n in (2, 4):
        plan = gpupool.plan_describe(p, mode=gpupool.MODE_SCATTER, flags=HF, n_parts=n)
        q = [t for t in plan["layouts"][1]["tensors"] if t["name"].endswith("q_proj.weight")][0]
        assert q["slice_dim"] == 0 and q["slice_begin"] == 384 // n
        check_plan(plan, shards, hf, gpupool.MODE_SCATTER, 0, n)


def test_plan_shape_counts(tmp_path):
    """The costs the header names: Q/K rows are read one row per read and each (head, half) group is its own segment."""
    p = str(tmp_path / "m.gguf")
    make(p, n_head=4, n_head_kv=2, qtype="Q4_K", layers=1)
    a, b = gpupool.plan_describe(p), gpupool.plan_describe(p, flags=HF)
    reads = lambda pl: sum(len(ch["reads"]) for part in pl["parts"] for ch in part["chunks"])
    segs = lambda pl: sum(len(ch["segs"]) for part in pl["parts"] for ch in part["chunks"])
    # q: 256 rows, k: 128 rows.  Without the flag the whole file is one read; with it every Q/K row is a read of its own (the bytes
    # before q and after k stay merged) and each tensor is 2 * heads segments
    assert reads(a) == 1 and reads(b) == 1 + 256 + 128
    assert segs(b) - segs(a) == (8 + 4) - 2


# ---- whole launches through the device code --------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul():
    return kk_emul.load()


@pytest.fixture(scope="module")
def emul_f16():
    return kk_f16_emul.load()


def replay(L, path, hf, mode=gpupool.MODE_SINGLE, flags=0, n=1, chunk=1 * MB, launch=0):
    shards = [path]
    plan = gpupool.plan_describe(path, mode=mode, flags=HF | flags, n_parts=n, chunk_bytes=chunk)
    oflags = flags & (KEEP | F16)
    if mode == gpupool.MODE_SCATTER:
        exps = [hf_oracle.expected_pool(shards, hf, mode, oflags, n, g) for g in range(n)]
        ranks = [Pools(1, len(e)) for e, _ in exps]
        x = Exchange(ranks)
        for g in range(n):
            play_part(L, plan, g, ranks[g], flags=launch, x=x)
        for g in range(n):
            check(ranks[g], *exps[g])
    else:
        exp, pl = hf_oracle.expected_pool(shards, hf, mode, oflags)
        pools = Pools(n, len(exp))
        for g in range(n):
            play_part(L, plan, g, pools, flags=launch)
        check(pools, exp, pl)


BLOCK_TYPES = ["Q4_0", "Q4_1", "Q5_0", "Q5_1", "Q8_0", "Q2_K", "Q3_K", "Q4_K", "Q5_K", "Q6_K", "IQ4_NL", "IQ4_XS", "MXFP4", "IQ2_XXS",
               "IQ2_XS", "IQ2_S", "IQ3_XXS", "IQ3_S", "IQ1_S", "IQ1_M", "TQ1_0", "TQ2_0", "NVFP4"]


@pytest.mark.parametrize("qtype", ["BF16", "F16", "F32"] + BLOCK_TYPES)
def test_whole_launches_every_type(emul, emul_f16, tmp_path, qtype):
    p = str(tmp_path / "m.gguf")
    _, hf = make(p, n_head=4, n_head_kv=2, hidden=256, ffn=256, vocab=32, layers=1, qtype=qtype, experts=2, bias=True)
    replay(emul, p, hf)
    replay(emul_f16, p, hf, flags=F16, launch=kk_f16_emul.LAUNCH_F16)


def test_whole_launches_broadcast_scatter_keep_f32(emul, emul_f16, tmp_path):
    for qtype in ("BF16", "F16", "Q4_K", "Q8_0"):
        p = str(tmp_path / f"{qtype}.gguf")
        _, hf = make(p, n_head=6, n_head_kv=2, head_dim=64 if qtype != "Q4_K" else 0, hidden=768 if qtype == "Q4_K" else 384, ffn=512,
                     vocab=64, layers=2, qtype=qtype, experts=4, bias=True)
        replay(emul, p, hf, gpupool.MODE_BROADCAST, n=3)
        replay(emul, p, hf, gpupool.MODE_SCATTER, n=2)
        replay(emul, p, hf, gpupool.MODE_SCATTER, flags=X, n=4)
        replay(emul, p, hf, flags=KEEP)
        replay(emul_f16, p, hf, gpupool.MODE_SCATTER, flags=F16, n=4, launch=kk_f16_emul.LAUNCH_F16)
        replay(emul, p, hf, chunk=2 * MB)


# ---- refusals -------------------------------------------------------------------------------------------------------------------
def _refused(path, exc, pattern, **kw):
    with pytest.raises(exc, match=pattern):
        gpupool.plan_describe(path, flags=HF, **kw)


def test_refusals(tmp_path):
    st_path = str(tmp_path / "a.safetensors")
    synth.write_safetensors(st_path, [("model.layers.0.self_attn.q_proj.weight", "BF16", [64, 64])], 1)
    _refused(st_path, gpupool.ErrInvalid, "GGUF checkpoints only")
    p = str(tmp_path / "nokv.gguf")
    make(p, kv=[])
    _refused(p, gpupool.ErrFormat, "head_count")
    p = str(tmp_path / "badkv.gguf")
    make(p, kv=[("llama.attention.head_count", 8, synth._gguf_str("four"))])
    _refused(p, gpupool.ErrFormat, "value type 8")
    p = str(tmp_path / "arr.gguf")
    make(p, kv=[("llama.attention.head_count", 9, struct.pack("<IQ", 4, 2) + struct.pack("<2I", 4, 4))])
    _refused(p, gpupool.ErrUnsupported, "per-layer array")
    p = str(tmp_path / "zero.gguf")
    make(p, kv=[("llama.attention.head_count", 4, struct.pack("<I", 0))])
    _refused(p, gpupool.ErrFormat, "out of range")
    p = str(tmp_path / "rows.gguf")
    make(p, n_head=3, n_head_kv=3, kv=synth.gguf_head_kv("llama", 5))
    _refused(p, gpupool.ErrFormat, "not a multiple of 2")
    p = str(tmp_path / "gpt2.gguf")
    synth.write_gguf(p, [("blk.0.attn_q.weight", "F32", [8, 8])], 1, arch="gpt2")
    _refused(p, gpupool.ErrUnsupported, "architecture \"gpt2\"")
    p = str(tmp_path / "extra.gguf")
    synth.write_gguf(p, [("blk.0.attn_q.weight", "F32", [8, 8]), ("blk.0.ffn_gate_shexp.weight", "F32", [8, 8])], 1, arch="qwen2")
    _refused(p, gpupool.ErrUnsupported, "ffn_gate_shexp")
    # every integer type is accepted, and a missing head_count_kv means MHA
    for vt, fmt in ((0, "<B"), (1, "<b"), (2, "<H"), (3, "<h"), (4, "<I"), (5, "<i"), (10, "<Q"), (11, "<q")):
        p = str(tmp_path / f"vt{vt}.gguf")
        _, hf = make(p, n_head=4, n_head_kv=4, kv=[("llama.attention.head_count", vt, struct.pack(fmt, 4))])
        assert [t["name"] for t in gpupool.plan_describe(p, flags=HF)["layouts"][0]["tensors"]] == [r["name"] for r in hf]


def test_block_quantised_qk_bias_is_refused_and_an_unmarked_one_loads(tmp_path):
    """A 1-D block-quantised q / k bias has rows of single elements, less than one block: its rows cannot be moved one by one, so the
    load refuses it rather than leave its slot unwritten.  A block-quantised v bias is not un-permuted and loads whole."""
    for i, bt in enumerate((("Q8_0", "F32", "F32"), ("F32", "Q4_0", "F32"))):
        p = str(tmp_path / f"qk{i}.gguf")
        make(p, hidden=128, ffn=128, layers=1, vocab=32, head_dim=32, bias=True, bias_types=bt)
        _refused(p, gpupool.ErrUnsupported, "cannot be un-permuted")
        assert gpupool.plan_describe(p)["layouts"][0]["tensors"], "the same file loads without the flag"
    p = str(tmp_path / "v.gguf")
    shards, hf = make(p, hidden=128, ffn=128, layers=2, vocab=32, head_dim=32, bias=True, bias_types=("F32", "F32", "Q8_0"), qtype="Q8_0")
    for mode, n in ((gpupool.MODE_SINGLE, 1), (gpupool.MODE_BROADCAST, 2), (gpupool.MODE_SCATTER, 2)):
        check_plan(gpupool.plan_describe(p, mode=mode, flags=HF, n_parts=n), shards, hf, mode, 0, n)


def test_split_gguf_takes_the_first_shards_keys(tmp_path):
    """A split GGUF (a directory of shards): the keys are the first shard's; a later shard that repeats one must agree, one that adds a
    key the first lacks is not a repeat."""
    t = synth.llama_gguf_tensors(hidden=256, ffn=256, layers=2, n_head=4, n_head_kv=2, vocab=64)
    half = len(t) // 2
    kv = synth.gguf_head_kv("llama", 4, 2)

    def split(name, kv1, kv2):
        d = tmp_path / name
        d.mkdir()
        synth.write_gguf(str(d / "m-00001-of-00002.gguf"), t[:half], 5, extra_kv=kv1)
        synth.write_gguf(str(d / "m-00002-of-00002.gguf"), t[half:], 6, extra_kv=kv2)
        return str(d)

    for d in (split("same", kv, kv), split("first_only", kv, []), split("later_adds", kv, synth.gguf_head_kv("llama", 4, 2, experts=8))):
        plan = gpupool.plan_describe(d, flags=HF)
        assert plan["layout"] == "hf" and len(plan["shards"]) == 2
    _refused(split("disagree", kv, synth.gguf_head_kv("llama", 8, 2)), gpupool.ErrFormat, "disagrees")
    _refused(split("later_only", [], kv), gpupool.ErrFormat, "head_count")


# ---- no flag, no change -------------------------------------------------------------------------------------------------------------
def _no_flag_plans():
    spec = importlib.util.spec_from_file_location("make_no_flag_plans", os.path.join(G, "make_no_flag_plans.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod, json.load(open(os.path.join(G, "no_flag_plans.json")))


@pytest.mark.parametrize("g", ["q4k.gguf", "q4km_mix.gguf", "quants_cb.gguf", "quants_f4.gguf", "quants_iq.gguf", "hf_llama_moe.gguf",
                               "st_mixed.safetensors", "sharded"])
def test_no_flag_identity(g):
    """Without the flag every golden checkpoint indexes and plans byte for byte as the library did before the flag existed
    (tests/golden/no_flag_plans.json, written by that library)."""
    mod, want = _no_flag_plans()
    got = mod.describe(gpupool, os.path.join(G, g))
    assert got["index"] == want[g]["index"]
    for shape, text in want[g]["plans"].items():
        assert got["plans"][shape] == text, (g, shape)
        assert '"layout"' not in text and '"architecture"' not in text


def test_manifest_option_and_cli(tmp_path):
    specs = schema.validate_models([{"name": "a", "source": "/m", "options": {"hfLayout": True, "f16": True}}], stat=lambda p: None)
    assert specs[0].flags == HF | F16
    p = str(tmp_path / "m.gguf")
    make(p)
    out = io.StringIO()
    assert cli.main(["model", "plan", p, "--option", "hfLayout", "-o", "json", "--full"], out) == 0
    doc = json.loads(out.getvalue())
    assert doc["flags"] == HF and doc["layout"] == "hf"
    assert doc["layouts"][0]["tensors"][0]["name"] == "model.embed_tokens.weight"


# ---- the committed fixture -----------------------------------------------------------------------------------------------------------
def test_golden_fixture_against_transformers_and_gguf_py(emul):
    """tests/golden/hf_llama_moe.gguf: the oracle's HF view equals the expected tensors the generator computed with gguf-py and
    transformers, and the plan replays to them."""
    p = os.path.join(G, "hf_llama_moe.gguf")
    meta = json.load(open(p + ".expected.json"))
    want = np.load(p + ".hf.npz")
    shards, recs = oracle.index_path(p)
    hf = hf_oracle.hf_view(recs, meta["architecture"], meta["n_head"], meta["n_head_kv"])
    got = hf_oracle.tensors(shards, hf)
    assert sorted(got) == sorted(want.files) == sorted(meta["tensors"])
    for n in want.files:
        assert np.array_equal(got[n], want[n].view(np.uint8).reshape(-1)), n
    replay(emul, p, hf)
    replay(emul, p, hf, gpupool.MODE_SCATTER, n=2)
