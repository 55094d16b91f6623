"""GPU tier: pipeline stages (kk_load_opts.layer_begin / layer_end) through the real loader and convert kernel.

Every pool is poisoned before the kernel writes it and checked whole against the oracle's pool of the tensors the stage keeps
(tests/layer_oracle.py selects them), so a tensor of another stage that leaks in, or a stage tensor that is skipped, fails."""
import os

import numpy as np
import pytest
from hypothesis import HealthCheck, Phase, given, settings

from kukeon_b200 import gpupool, modelhub
from oracle import oracle
from tests import helpers, layer_oracle
from tests.test_layer_stage import stage_cases
from tools import synth

pytestmark = pytest.mark.gpu
MB = 1 << 20
S, B, SC = gpupool.MODE_SINGLE, gpupool.MODE_BROADCAST, gpupool.MODE_SCATTER
X, T = gpupool.LOAD_SCATTER_EXCHANGE, gpupool.LOAD_GPT2_CONV1D_T
MANIFEST_KEYS = ["apiVersion", "kind", "device", "deviceUUID", "pciBusId", "poolBytes", "mode", "format", "align", "tensors"]


def stage_exp(path, layers, mode=S, flags=0, n=1, part=0):
    """(expected pool, written mask) of one device holding `part` of stage `layers`."""
    shards, recs = oracle.index_path(path)
    want = layer_oracle.select_layers(recs, *layers)
    exp, pl = oracle.expected_pool(shards, want, mode, flags & (1 | 2 | 16), n, part)
    return exp, helpers.expected_mask(pl, len(exp))


def ranks(pool, path, layers, mode, n, flags=0, fanout=gpupool.FANOUT_P2P):
    """n ranks of one stage group hosted by this process on device 0, each a deferred model of part i of n, attached to each other by raw
    device pointer (pools for P2P and the row exchange, slice buffers for PULL)."""
    ms = [pool.load(path, mode=mode, fanout=fanout, flags=flags | gpupool.LOAD_DEFER, part_index=i, part_count=n, layers=layers)
          for i in range(n)]
    assert len({m.handle for m in ms}) == n
    if fanout == gpupool.FANOUT_PULL:
        ptrs = [m.export_buffer(0, gpupool.BUF_SLICE_PTR) for m in ms]
        for i, m in enumerate(ms):
            for j in range(n):
                if j != i:
                    m.peer_attach_buffer(j, gpupool.BUF_SLICE_PTR, ptrs[j])
    elif mode == B or flags & X:
        ptrs = [m.pool_ptr(0)[0] for m in ms]
        for i, m in enumerate(ms):
            for j in range(n):
                if j != i:
                    m.peer_attach_local_pointer(j, ptrs[j])
    return ms


def run_checked(ms, want, label, stage2=False, resident_passes=2):
    """Poison, load, check every pool whole; then `resident_passes` back-to-back resident conversions, each checked whole."""
    def check(fills, what):
        for i, (m, fill) in enumerate(zip(ms, fills)):
            exp, mask = want[i]
            may = None
            if stage2 and len(ms) > 1:  # PULL copies each peer's whole pool range, gaps included (see test_pull_fan_out_virtual_ranks_on_one_gpu)
                may = np.zeros(len(exp), bool)
                for j, o in enumerate(ms):
                    if j != i:
                        q = o.stats()["parts"][0]
                        may[q["pool_lo"]:q["pool_hi"]] = True
                may &= ~mask
            helpers.assert_pool_exact(m, 0, exp, mask, fill, f"{label} rank {i} of {len(ms)}, {what}", may_rewrite=may)

    fills = [helpers.poison(m, 0) for m in ms]
    for m in ms:
        m.load_part()
    if stage2:
        for m in ms:
            m.convert_local()
    check(fills, "streaming load")
    if not resident_passes:
        return
    for m in ms:
        m.stage_resident()
    for k in range(resident_passes):
        fills = [helpers.poison(m, 0) for m in ms]
        for m in ms:
            m.convert_resident()
        if stage2:
            for m in ms:
                m.convert_local()
        check(fills, f"resident conversion {k + 1}")


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("gpu_stages")
    out = {"mixtral": str(d / "mixtral.gguf"), "llama": str(d / "llama"), "gpt2": str(d / "gpt2.safetensors")}
    synth.write_gguf(out["mixtral"], synth.mixtral_gguf_tensors(hidden=256, ffn=768, layers=4, experts=2, vocab=512, kv_dim=256), 9)
    synth.make_llama(out["llama"], dict(hidden=256, ffn=704, layers=4, kv_dim=64, vocab=1000), max_shard_bytes=1_500_000)
    synth.make_gpt2(out["gpt2"], n_layer=4, d=96, vocab=301, n_pos=40)
    return out


def test_two_mixtral_q4k_stages_resident_in_one_context(pool, files):
    p = files["mixtral"]
    stages = [(0, 2), (2, 4)]
    ms = [pool.load(p, flags=gpupool.LOAD_DEFER, layers=s) for s in stages]
    try:
        assert ms[0].handle != ms[1].handle, "two stages of one file are two models"
        _, recs = oracle.index_path(p)
        for m, s in zip(ms, stages):
            assert [t["name"] for t in m.tensors()] == [r["name"] for r in layer_oracle.select_layers(recs, *s)]
            assert m.info()["refcount"] == 1
        with pytest.raises(gpupool.ErrNotFound):
            ms[0].placements("output.weight")
        with pytest.raises(gpupool.ErrNotFound):
            ms[1].placements("token_embd.weight")
        # both stages resident at once: each load and conversion must leave the other stage's pool alone
        fills = [helpers.poison(m, 0) for m in ms]
        for m in ms:
            m.load_part()
        for m, s, fill in zip(ms, stages, fills):
            helpers.assert_pool_exact(m, 0, *stage_exp(p, s), fill, f"stage {s}: streaming load")
        for m in ms:
            m.stage_resident()
        for k in range(2):
            fills = [helpers.poison(m, 0) for m in ms]
            for m in ms:
                m.convert_resident()
            for m, s, fill in zip(ms, stages, fills):
                helpers.assert_pool_exact(m, 0, *stage_exp(p, s), fill, f"stage {s}: resident conversion {k + 1}")
        again = modelhub.Load(pool, p, flags=gpupool.LOAD_DEFER, layers=(0, 2))
        assert again.handle == ms[0].handle and ms[0].info()["refcount"] == 2
        again.release()
        assert ms[0].info()["refcount"] == 1
    finally:
        for m in ms:
            m.release()


def test_llama_stage_broadcast_p2p_and_pull_over_virtual_ranks(pool, files):
    p = files["llama"]
    for layers in ((0, 2), (1, 3), (2, 4)):
        for n in (2, 3):
            ms = ranks(pool, p, layers, B, n)
            try:
                run_checked(ms, [stage_exp(p, layers)] * n, f"llama {layers} BROADCAST/P2P")
            finally:
                for m in ms:
                    m.release()
        ms = ranks(pool, p, layers, B, 2, fanout=gpupool.FANOUT_PULL)
        try:
            run_checked(ms, [stage_exp(p, layers)] * 2, f"llama {layers} BROADCAST/PULL", stage2=True, resident_passes=1)
        finally:
            for m in ms:
                m.release()


@pytest.mark.parametrize("n", [2, 4])
def test_llama_stage_scatter_with_row_exchange_over_virtual_ranks(pool, files, n):
    p = files["llama"]
    for layers in ((0, 2), (2, 4)):
        for flags in (X, 0):
            ms = ranks(pool, p, layers, SC, n, flags)
            try:
                run_checked(ms, [stage_exp(p, layers, SC, flags, n, i) for i in range(n)], f"llama {layers} SCATTER flags {flags}",
                            resident_passes=1)
                st = ms[0].stats()
                assert st["file_bytes"] == sum(r["nbytes"] for r in layer_oracle.select_layers(oracle.index_path(p)[1], *layers))
            finally:
                for m in ms:
                    m.release()


def test_q4k_stage_raw_fan_out(pool, files):
    p = files["mixtral"]
    for layers in ((0, 2), (2, 4)):
        m = pool.load(p, mode=B, fanout=gpupool.FANOUT_RAW, flags=gpupool.LOAD_DEFER, layers=layers)
        try:
            run_checked([m], [stage_exp(p, layers)], f"mixtral {layers} BROADCAST/RAW", stage2=True)
        finally:
            m.release()


def test_gpt2_last_stage_keeps_the_tied_wte_and_transposes_exactly(pool, files):
    p = files["gpt2"]
    for layers in ((2, 4), (0, 2)):
        m = pool.load(p, flags=T | gpupool.LOAD_DEFER, layers=layers)
        try:
            names = {t["name"] for t in m.tensors()}
            assert "wte.weight" in names and ("ln_f.weight" in names) == (layers == (2, 4)) and ("wpe.weight" in names) == (layers == (0, 2))
            assert m.placements(f"h.{layers[0]}.attn.c_attn.weight")[0].shape == [3 * 96, 96], "Conv1D weight transposed"
            run_checked([m], [stage_exp(p, layers, flags=T)], f"gpt2 {layers} CONV1D_T")
        finally:
            m.release()


def test_two_contexts_on_one_device_one_stage_each(native, files):
    """The one-process deployment shape: one kk_ctx per stage group.  Here both groups are device 0, so both contexts hold their stage
    at the same time and each must be exact."""
    p = files["mixtral"]
    a = gpupool.Pool([0], n_staging_buffers=2, staging_buffer_bytes=2 * MB, n_reader_threads=1)
    try:
        b = gpupool.Pool([0], n_staging_buffers=2, staging_buffer_bytes=4 * MB, n_reader_threads=2)
        try:
            ms = [a.load(p, flags=gpupool.LOAD_DEFER, layers=(0, 2)), b.load(p, flags=gpupool.LOAD_DEFER, layers=(2, 4))]
            try:
                fills = [helpers.poison(m, 0) for m in ms]
                for m in ms:
                    m.load_part()
                for m, s, fill in zip(ms, ((0, 2), (2, 4)), fills):
                    helpers.assert_pool_exact(m, 0, *stage_exp(p, s), fill, f"context of stage {s}")
            finally:
                for m in ms:
                    m.release()
        finally:
            b.close()
    finally:
        a.close()


def test_mount_manifest_of_a_stage_and_of_the_whole_checkpoint(pool, files):
    p = files["llama"]
    _, recs = oracle.index_path(p)
    whole = pool.load(p)
    try:
        man = whole.manifest(0)
        assert list(man) == MANIFEST_KEYS, "the manifest of a whole-checkpoint load has no stage keys"
        assert [t["name"] for t in man["tensors"]] == [r["name"] for r in recs]
    finally:
        whole.release()
    m = pool.load(p, layers=(1, 3))
    try:
        man = m.manifest(0)
        assert list(man) == MANIFEST_KEYS[:-1] + ["layerBegin", "layerEnd", "nLayers", "tensors"]
        assert (man["layerBegin"], man["layerEnd"], man["nLayers"]) == (1, 3, 4)
        assert [t["name"] for t in man["tensors"]] == [r["name"] for r in layer_oracle.select_layers(recs, 1, 3)]
        for t in man["tensors"]:
            pl = m.placements(t["name"])[0]
            assert (t["offset"], t["nbytes"], t["shape"]) == (pl.pool_offset, pl.nbytes, pl.shape)
        info = m.info()
        assert info["n_tensors"] == len(man["tensors"]) and info["pool_bytes"] == man["poolBytes"]
    finally:
        m.release()


@settings(max_examples=int(os.environ.get("KK_HYP_EXAMPLES_GPU_STAGE", 30)), deadline=None, derandomize=True,
          phases=[Phase.explicit, Phase.generate], suppress_health_check=[HealthCheck.too_slow, HealthCheck.function_scoped_fixture])
@given(stage_cases())
def test_random_inventories_and_ranges_through_the_loader(pool, tmp_path, case):
    inv, seed, b, e, (mode, n, flags) = case
    p = str(tmp_path / f"r{seed}.safetensors")
    synth.write_safetensors(p, inv, seed)
    _, recs = oracle.index_path(p)
    try:
        layer_oracle.select_layers(recs, b, e)
    except layer_oracle.StageError as err:
        with pytest.raises(gpupool.GPUPoolError) as got:
            pool.load(p, mode=mode, flags=flags, part_index=0, part_count=n if n > 1 else 0, layers=(b, e))
        assert got.value.code == err.code
        return
    if e == 0:
        return
    ms = ranks(pool, p, (b, e), mode, n, flags) if n > 1 else [pool.load(p, mode=mode, flags=flags | gpupool.LOAD_DEFER, layers=(b, e))]
    try:
        want = [stage_exp(p, (b, e), mode, flags, n, i if mode == SC else 0) for i in range(len(ms))]
        run_checked(ms, want, f"random stage [{b}, {e}) mode {mode} x{n} flags {flags}", resident_passes=1)
    finally:
        for m in ms:
            m.release()
