"""CPU tier: pipeline stages (kk_load_opts.layer_begin / layer_end) through kk_plan_describe.

The library's selection is compared with an independent restatement of the rule (tests/layer_oracle.py) and with a table of what each
stage of each architecture must hold; each stage's placements must equal the oracle's layout of the selected tensors, and no byte outside
the selected tensors may be read.  Stage plans are then replayed through the device code (kk_emul_launch) against the oracle's pools."""
import os

import numpy as np
import pytest
from hypothesis import HealthCheck, Phase, given, settings, strategies as st

from kukeon_b200 import gpupool
from oracle import oracle
from tests import kk_emul, layer_oracle
from tests.kk_emul import Pools
from tests.test_launch_emul import Exchange, check, play_part
from tools import synth

MB = 1 << 20
S, B, SC = gpupool.MODE_SINGLE, gpupool.MODE_BROADCAST, gpupool.MODE_SCATTER
X, T = gpupool.LOAD_SCATTER_EXCHANGE, gpupool.LOAD_GPT2_CONV1D_T


def names(plan, layout=0):
    return [t["name"] for t in plan["layouts"][layout]["tensors"]]


def check_stage(path, b, e, mode=S, n=1, flags=0, chunk=0):
    """One stage's plan against the oracle: selection, placements and pool size of every layout, and the bytes it reads."""
    shards, recs = oracle.index_path(path)
    want = layer_oracle.select_layers(recs, b, e)
    plan = gpupool.plan_describe(path, mode=mode, flags=flags, n_parts=n, chunk_bytes=chunk, layers=(b, e))
    assert plan["layers"] == [b, e] and plan["n_layers"] == layer_oracle.n_layers(recs)
    assert plan["shards"] == shards, "a stage keeps the checkpoint's shard list"
    assert plan["file_bytes"] == sum(r["nbytes"] for r in want)
    for L, lay in enumerate(plan["layouts"]):
        assert names(plan, L) == [r["name"] for r in want]
        exp, total = oracle.plan_pool(want, mode, flags & (1 | 2 | 16), n, L)
        assert lay["pool_bytes"] == total
        for got, p in zip(lay["tensors"], exp):
            assert (got["pool_offset"], got["nbytes"], got["shape"], got["slice_dim"], got["slice_begin"], got["dtype"]) == \
                (p["pool_offset"], p["nbytes"], p["shape"], p["slice_dim"], p["slice_begin"], p["dtype"]), got["name"]
    # every read lies inside a selected tensor of its shard, or a run of back-to-back selected tensors (the planner merges such reads)
    extents = {}
    for r in sorted(want, key=lambda r: (r["shard"], r["file_offset"])):
        ext = extents.setdefault(r["shard"], [])
        if ext and ext[-1][1] == r["file_offset"]:
            ext[-1] = (ext[-1][0], r["file_offset"] + r["nbytes"])
        else:
            ext.append((r["file_offset"], r["file_offset"] + r["nbytes"]))
    read = []
    for part in plan["parts"]:
        n_read = 0
        for ch in part["chunks"]:
            ext = extents[ch["shard"]]
            starts = [a for a, _ in ext]
            for fo, ln, _ in ch["reads"]:
                i = int(np.searchsorted(starts, fo, side="right")) - 1
                assert i >= 0 and fo + ln <= ext[i][1], f"read [{fo}, {fo + ln}) of shard {ch['shard']} is outside the stage's tensors"
                n_read += ln
        read.append(n_read)
    if mode != SC:
        assert sum(read) == plan["file_bytes"], "a stage reads exactly its tensors' bytes"
    elif not flags & X:
        for L in range(n):
            assert read[L] == sum(r["nbytes"] // n if oracle.slice_dim(r, n) is not None else r["nbytes"] for r in want)
    return plan, want


# ---- inventories ---------------------------------------------------------------------------------------------------------------------
LL = dict(hidden=128, ffn=320, layers=4, kv_dim=64, vocab=500)


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("stages")
    out = {}
    out["llama"] = str(d / "llama")
    synth.make_llama(out["llama"], LL, max_shard_bytes=400_000)  # several shards, a layer's tensors across a shard boundary
    out["tied"] = str(d / "tied.safetensors")
    synth.write_safetensors(out["tied"], [t for t in synth.llama_tensors(**LL) if t[0] != "lm_head.weight"], 3)
    out["gpt2"] = str(d / "gpt2.safetensors")
    synth.make_gpt2(out["gpt2"], n_layer=4, d=64, vocab=301, n_pos=40)
    out["mixtral"] = str(d / "mixtral.gguf")
    synth.write_gguf(out["mixtral"], synth.mixtral_gguf_tensors(hidden=256, ffn=512, layers=4, experts=2, vocab=320, kv_dim=128), 5)
    out["rope"] = str(d / "rope.gguf")
    synth.write_gguf(out["rope"], [("rope_freqs.weight", "F32", [32])] + synth.mixtral_gguf_tensors(hidden=256, ffn=256, layers=3, experts=2,
                                                                                                     vocab=256, kv_dim=256, qtype="Q8_0"), 6)
    return out


# (file, stage, tensors that must be in it, tensors that must not)
TABLE = [
    ("llama", (0, 2), ["model.embed_tokens.weight", "model.layers.0.self_attn.q_proj.weight", "model.layers.1.mlp.down_proj.weight"],
     ["model.layers.2.self_attn.q_proj.weight", "model.norm.weight", "lm_head.weight"]),
    ("llama", (2, 4), ["model.layers.2.input_layernorm.weight", "model.layers.3.mlp.up_proj.weight", "model.norm.weight", "lm_head.weight"],
     ["model.embed_tokens.weight", "model.layers.1.mlp.up_proj.weight"]),
    ("llama", (1, 3), ["model.layers.1.self_attn.o_proj.weight", "model.layers.2.self_attn.o_proj.weight"],
     ["model.embed_tokens.weight", "model.norm.weight", "lm_head.weight", "model.layers.3.self_attn.o_proj.weight"]),
    ("tied", (0, 2), ["model.embed_tokens.weight"], ["model.norm.weight"]),
    ("tied", (2, 4), ["model.embed_tokens.weight", "model.norm.weight"], ["model.layers.0.input_layernorm.weight"]),
    ("tied", (1, 3), [], ["model.embed_tokens.weight", "model.norm.weight"]),
    ("gpt2", (0, 2), ["wte.weight", "wpe.weight", "h.0.attn.c_attn.weight", "h.1.ln_2.bias"], ["ln_f.weight", "h.2.ln_1.weight"]),
    ("gpt2", (2, 4), ["wte.weight", "ln_f.weight", "ln_f.bias", "h.3.mlp.c_proj.weight"], ["wpe.weight", "h.1.ln_1.weight"]),
    ("mixtral", (0, 2), ["token_embd.weight", "blk.0.ffn_gate_exps.weight", "blk.1.attn_norm.weight"], ["output.weight", "output_norm.weight"]),
    ("mixtral", (2, 4), ["output.weight", "output_norm.weight", "blk.3.ffn_down_exps.weight"], ["token_embd.weight", "blk.1.attn_q.weight"]),
    ("rope", (0, 1), ["rope_freqs.weight", "token_embd.weight"], ["output.weight"]),
    ("rope", (1, 2), ["rope_freqs.weight", "blk.1.attn_q.weight"], ["token_embd.weight", "output.weight", "output_norm.weight"]),
    ("rope", (2, 3), ["rope_freqs.weight", "output.weight", "output_norm.weight"], ["token_embd.weight"]),
]


@pytest.mark.parametrize("name,stage,has,hasnt", TABLE, ids=[f"{t[0]}-{t[1][0]}-{t[1][1]}" for t in TABLE])
def test_rule_table(files, name, stage, has, hasnt):
    plan, _ = check_stage(files[name], *stage)
    got = set(names(plan))
    assert set(has) <= got, set(has) - got
    assert not set(hasnt) & got, set(hasnt) & got


SPLITS = {"llama": [[0, 4], [0, 2, 4], [0, 1, 3, 4], [0, 1, 2, 3, 4]], "tied": [[0, 2, 4], [0, 3, 4]], "gpt2": [[0, 2, 4], [0, 1, 2, 3, 4]],
          "mixtral": [[0, 2, 4], [0, 3, 4]], "rope": [[0, 1, 3], [0, 1, 2, 3]]}


@pytest.mark.parametrize("name", sorted(SPLITS))
def test_stages_cover_the_checkpoint(files, name):
    """k split points: every tensor is in exactly one stage, except the tied embedding (first and last) and the outer tensors that go to
    every stage."""
    _, recs = oracle.index_path(files[name])
    every = {"rope_freqs.weight"}
    tied = {"tied": "model.embed_tokens.weight", "gpt2": "wte.weight"}.get(name)
    for cuts in SPLITS[name]:
        count = {}
        for b, e in zip(cuts, cuts[1:]):
            plan, _ = check_stage(files[name], b, e)
            for t in names(plan):
                count[t] = count.get(t, 0) + 1
        k = len(cuts) - 1
        assert set(count) == {r["name"] for r in recs}
        for t, c in count.items():
            want = k if t in every else (2 if k > 1 else 1) if t == tied else 1
            assert c == want, (cuts, t, c, want)


def test_composition_with_broadcast_and_scatter(files):
    for b, e in ((0, 2), (2, 4), (1, 3), (0, 4)):
        for n in (1, 2, 3, 4):
            check_stage(files["llama"], b, e, B, n, chunk=1 * MB)
        for n in (2, 4):
            for flags in (0, X):
                check_stage(files["llama"], b, e, SC, n, flags, chunk=1 * MB)
    for b, e in ((0, 2), (2, 4)):
        check_stage(files["mixtral"], b, e, B, 3, chunk=1 * MB)
        check_stage(files["mixtral"], b, e, SC, 2)  # expert stacks and dim-1 q4_K weights stay whole, as without a stage
        check_stage(files["gpt2"], b, e, S, 1, T)
        check_stage(files["gpt2"], b, e, B, 2, T | gpupool.LOAD_KEEP_F32)


def test_whole_checkpoint_and_errors(files, tmp_path):
    p = files["llama"]
    whole = gpupool.plan_describe(p, mode=B, n_parts=2)
    assert "layers" not in whole and "n_layers" not in whole
    assert gpupool.plan_describe(p, mode=B, n_parts=2, layers=(0, 0)) == whole
    assert names(gpupool.plan_describe(p, layers=(0, 4))) == names(whole)
    for bad in ((3, 0), (2, 2), (3, 1)):
        with pytest.raises(gpupool.ErrInvalid):
            gpupool.plan_describe(p, layers=bad)
    with pytest.raises(gpupool.ErrInvalid, match=r"\b4 layers"):
        gpupool.plan_describe(p, layers=(2, 5))
    flat = str(tmp_path / "flat.safetensors")
    synth.write_safetensors(flat, [("embed.weight", "BF16", [8, 16]), ("head.weight", "BF16", [8, 16])], 1)
    with pytest.raises(gpupool.ErrUnsupported, match="no tensor with a layer index"):
        gpupool.plan_describe(flat, layers=(0, 1))
    assert "layers" not in gpupool.plan_describe(flat)
    two = str(tmp_path / "two.safetensors")
    synth.write_safetensors(two, [("model.layers.0.mlp.up_proj.weight", "BF16", [8, 16]),
                                  ("vision_tower.encoder.layers.0.mlp.fc1.weight", "BF16", [8, 16])], 1)
    with pytest.raises(gpupool.ErrUnsupported, match=r'"model\.layers\." and "vision_tower\.encoder\.layers\."'):
        gpupool.plan_describe(two, layers=(0, 1))
    # a range that does not fit kk_load_opts is refused before the call
    with pytest.raises(gpupool.ErrInvalid):
        gpupool.plan_describe(p, layers=(-1, 2))


def test_layer_index_is_the_first_whole_component_pair(tmp_path):
    """Only "<container>.<N>." with a whole container component and an all-digit N counts, and the first such pair wins."""
    p = str(tmp_path / "names.safetensors")
    inv = [("model.layers.3.block_sparse_moe.experts.7.w1.weight", "BF16", [4, 8]), ("transformer.h.0.attn.c_attn.weight", "BF16", [4, 8])]
    synth.write_safetensors(p, inv, 1)
    with pytest.raises(gpupool.ErrUnsupported, match="two numbered layer stacks"):
        gpupool.plan_describe(p, layers=(0, 1))
    q = str(tmp_path / "decoys.safetensors")
    inv = [("model.layers.3.block_sparse_moe.experts.7.w1.weight", "BF16", [4, 8]),   # layer 3, not expert 7
           ("model.xlayers.9.w.weight", "BF16", [4, 8]),                              # not a whole component: outer
           ("model.layers.x9.w.weight", "BF16", [4, 8]),                              # N not all digits: outer
           ("model.layers.0.mlp.up_proj.weight", "BF16", [4, 8])]
    synth.write_safetensors(q, inv, 1)
    assert gpupool.plan_describe(q, layers=(3, 4))["n_layers"] == 4
    assert set(names(gpupool.plan_describe(q, layers=(3, 4)))) == {"model.layers.3.block_sparse_moe.experts.7.w1.weight", "model.xlayers.9.w.weight",
                                                                   "model.layers.x9.w.weight"}
    for b, e in ((0, 1), (1, 3), (3, 4), (0, 4)):
        check_stage(q, b, e)


# ---- hypothesis: random layered inventories x random ranges x mode --------------------------------------------------------------------
PREFIXES = ["model.layers.", "transformer.h.", "blk.", "h."]
INNER = ["self_attn.q_proj.weight", "self_attn.o_proj.weight", "mlp.down_proj.weight", "input_layernorm.weight", "attn.c_attn.weight", "bias"]
OUTER = ["model.embed_tokens.weight", "lm_head.weight", "lm_head.bias", "model.norm.weight", "wte.weight", "wpe.weight", "ln_f.weight",
         "ln_f.bias", "output.weight", "output_norm.weight", "token_embd.weight", "rope_freqs.weight", "misc.weight"]


@st.composite
def stage_cases(draw):
    prefix = draw(st.sampled_from(PREFIXES))
    n_layers = draw(st.integers(1, 5))
    inv, seen = [], set()
    for _ in range(draw(st.integers(1, 9))):
        nm = f"{prefix}{draw(st.integers(0, n_layers - 1))}.{draw(st.sampled_from(INNER))}"
        if nm not in seen:
            seen.add(nm)
            inv.append((nm, draw(st.sampled_from(["BF16", "F32", "F16"])), [draw(st.sampled_from([1, 8, 16, 24])), draw(st.sampled_from([8, 40, 64]))]))
    for nm in draw(st.lists(st.sampled_from(OUTER), max_size=5, unique=True)):
        inv.append((nm, "BF16", [draw(st.sampled_from([8, 16])), 64]))
    if draw(st.integers(0, 7)) == 0:  # a second stack now and then: refused
        inv.append(("vision.layers.0.w.weight", "BF16", [8, 8]))
    n = 1 + max(int(nm[len(prefix):].split(".")[0]) for nm, _, _ in inv if nm.startswith(prefix))
    if draw(st.integers(0, 7)) == 0:  # any range, mostly refused
        b, e = draw(st.integers(0, n + 1)), draw(st.integers(0, n + 2))
    else:
        b = draw(st.integers(0, n - 1))
        e = draw(st.integers(b + 1, n))
    mode = draw(st.sampled_from([(S, 1, 0), (B, 2, 0), (B, 3, 0), (SC, 2, 0), (SC, 2, X), (SC, 4, X), (S, 1, T)]))
    return inv, draw(st.integers(0, 10**6)), b, e, mode


@settings(max_examples=int(os.environ.get("KK_HYP_EXAMPLES", 80)), deadline=None, derandomize=True,
          phases=[Phase.explicit, Phase.generate], suppress_health_check=[HealthCheck.too_slow, HealthCheck.function_scoped_fixture])
@given(stage_cases())
def test_random_inventories_and_ranges(tmp_path, case):
    inv, seed, b, e, (mode, n, flags) = case
    p = str(tmp_path / f"r{seed}.safetensors")
    synth.write_safetensors(p, inv, seed)
    _, recs = oracle.index_path(p)
    try:
        layer_oracle.select_layers(recs, b, e)
    except layer_oracle.StageError as err:
        with pytest.raises(gpupool.GPUPoolError) as got:
            gpupool.plan_describe(p, mode=mode, flags=flags, n_parts=n, layers=(b, e))
        assert got.value.code == err.code, (str(err), str(got.value))
        return
    if e == 0:
        return  # (0, 0): the whole checkpoint, covered by the parent's plan tests
    check_stage(p, b, e, mode, n, flags)


# ---- CPU replay of stage plans through the device code ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul():
    return kk_emul.load()


def replay_stage(L, path, b, e, mode=S, flags=0, n=1, chunk=1 * MB):
    shards, recs = oracle.index_path(path)
    want = layer_oracle.select_layers(recs, b, e)
    plan = gpupool.plan_describe(path, mode=mode, flags=flags, n_parts=n, chunk_bytes=chunk, layers=(b, e))
    oflags = flags & (1 | 2 | 16)
    if mode == SC:
        exps = [oracle.expected_pool(shards, want, mode, oflags, n, g) for g in range(n)]
        ranks = [Pools(1, len(exp)) for exp, _ in exps]
        x = Exchange(ranks)
        for g in range(n):
            play_part(L, plan, g, ranks[g], x=x)
        for g in range(n):
            check(ranks[g], *exps[g])
        return tuple(x.tiles)
    exp, pl = oracle.expected_pool(shards, want, mode, oflags)
    pools = Pools(n, len(exp))
    for g in range(n):
        play_part(L, plan, g, pools)
    check(pools, exp, pl)
    return None


def test_replay_mixtral_q4k_stages(emul, files):
    for b, e in ((0, 2), (2, 4)):
        replay_stage(emul, files["mixtral"], b, e)
        replay_stage(emul, files["mixtral"], b, e, B, n=2)


def test_replay_llama_scatter_exchange_stage(emul, files):
    for b, e in ((0, 2), (2, 4)):
        tiles = replay_stage(emul, files["llama"], b, e, SC, X, n=2)
        assert tiles[0] + tiles[1] > 0, "the stage's row-parallel tensors took the row exchange"
    replay_stage(emul, files["gpt2"], 2, 4, S, T)
