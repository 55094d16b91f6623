"""LoRA adapters on a resident base (kk_derive_adapter), GPU tier.  The base's pools are poisoned before its kk_load_part, so their
padding holds random bytes; the derived pool must equal the base pool everywhere outside the targets, padding included, and the C oracle's
merge of the base's elements on the targets, over the whole pool.  Also: equality with a kk_load_adapter model of another context,
identity and refcount, the refusals, and concurrent callers."""
import ctypes as C
import os
import re
import threading

import numpy as np
import pytest

from kukeon_b200 import gpupool, registry
from tests import helpers
from tests import lora_fixtures as lf
from tools import synth

pytestmark = pytest.mark.gpu
CFG = dict(hidden=256, ffn=704, layers=3, kv_dim=64, vocab=300)
RANKS = [1, 7, 16, 64, 256]


def _targets(path, flags=0):
    plan = gpupool.plan_describe(path, flags=flags)
    return [(t["name"], t["shape"]) for t in plan["layouts"][0]["tensors"] if re.search(r"_proj\.weight$", t["name"]) and len(t["shape"]) == 2]


def _adapter(tmp_path, path, flags=0, seed=1, dtype="BF16", config=None):
    d = str(tmp_path / f"ad{seed}")
    pairs = lf.seeded_adapter(d, _targets(path, flags), lambda i: RANKS[i % len(RANKS)], seed, dtype, 16, config)
    return d, pairs


def _placements(m, device):
    return {t["name"]: p for t in m.tensors() for p in m.placements(t["name"]) if p.device == device}


def _poisoned_base(pool, path, **kw):
    """A DEFER load whose pools are poisoned on every device before kk_load_part writes the tensors."""
    flags = kw.pop("flags", 0)
    base = pool.load(path, flags=flags | gpupool.LOAD_DEFER, **kw)
    for dev in sorted({p.device for t in base.tensors() for p in base.placements(t["name"])}):
        helpers.poison(base, dev)
    base.load_part()
    return base


def _check_derived(base, m, device, pairs, desc, label):
    """Every byte of m's pool on `device`: the C oracle's merge of base's bytes on the described targets, base's byte everywhere else."""
    pb, pm = _placements(base, device), _placements(m, device)
    assert pb == pm, f"{label}: the derived layout differs from the base's"
    _, n = base.pool_ptr(device)
    assert m.pool_ptr(device)[1] == n
    src = base.read(device, 0, n)
    exp = lf.expected_pool(src, desc, pairs, lambda name: (pm[name].pool_offset, pm[name].shape, pm[name].slice_dim, pm[name].slice_begin))
    got = m.read(device, 0, n)
    inside = np.zeros(n, bool)
    for t in desc["targets"]:
        p = pm[t["name"]]
        inside[p.pool_offset:p.pool_offset + p.nbytes] = True
    bad_t = np.flatnonzero(inside & (got != exp))
    bad_o = np.flatnonzero(~inside & (got != src))
    assert bad_t.size == 0, f"{label}: {bad_t.size} target bytes differ from the oracle merge, first at {bad_t[:4]}"
    assert bad_o.size == 0, f"{label}: {bad_o.size} bytes outside the targets differ from the base pool, first at {bad_o[:4]}"
    assert desc["targets"] and (got[inside] != src[inside]).any(), f"{label}: the merge changed nothing"


def _derive_and_check(pool, path, ad, pairs, label, **kw):
    desc = gpupool.adapter_describe(path, ad, **kw)
    base = _poisoned_base(pool, path, **kw)
    try:
        m = base.derive(ad)
        try:
            _check_derived(base, m, 0, pairs, desc, label)
            st = m.stats()
            assert st["derive"]["base_key"] and st["derive"]["t_copy"] > 0 and st["derive"]["t_merge"] > 0 and st["derive"]["t_host"] > 0
            assert st["adapter"]["n_tensors"] == len(desc["targets"]) and st["adapter"]["t_merge"] == st["derive"]["t_merge"]
            assert "derive" not in base.stats() and "adapter" not in base.stats()
            return m.manifest(0)
        finally:
            m.release()
    finally:
        base.release()


@pytest.mark.parametrize("dtype,flags", [("BF16", 0), ("F16", 0), ("F32", gpupool.LOAD_KEEP_F32), ("BF16", gpupool.LOAD_F16)],
                         ids=["bf16", "f16", "f32_keep", "load_f16"])
def test_derived_pool_equals_base_plus_oracle_merge(pool, tmp_path, dtype, flags):
    d = str(tmp_path / "llama")
    synth.make_llama(d, CFG, dtype=dtype)
    ad, pairs = _adapter(tmp_path, d, dtype=["F32", "BF16", "F16"][len(dtype) % 3])
    _derive_and_check(pool, d, ad, pairs, f"{dtype}/{flags:#x}", flags=flags)


def test_q4k_gguf_under_hf_layout(pool, tmp_path):
    p = str(tmp_path / "llama_q4k.gguf")
    synth.write_gguf(p, synth.llama_gguf_tensors(256, 512, 2, 4, 2, 300, qtype="Q4_K"), 17, extra_kv=synth.gguf_head_kv("llama", 4, 2))
    ad, pairs = _adapter(tmp_path, p, gpupool.LOAD_HF_LAYOUT, seed=3)
    man = _derive_and_check(pool, p, ad, pairs, "q4_K hf", flags=gpupool.LOAD_HF_LAYOUT)
    assert man["layout"] == "hf"


def test_pipeline_stage_skips_targets_outside_it(pool, tmp_path):
    d = str(tmp_path / "llama")
    synth.make_llama(d, CFG)
    ad, pairs = _adapter(tmp_path, d, seed=4)
    assert gpupool.adapter_describe(d, ad, layers=(1, 2))["skipped"]
    _derive_and_check(pool, d, ad, pairs, "stage", layers=(1, 2))


def test_two_part_scatter_without_exchange_on_one_device(pool, tmp_path):
    d = str(tmp_path / "llama")
    synth.make_llama(d, CFG)
    ad, pairs = _adapter(tmp_path, d, seed=5)
    for k in range(2):
        _derive_and_check(pool, d, ad, pairs, f"scatter part {k}", mode=gpupool.MODE_SCATTER, part_index=k, part_count=2)
    base = pool.load(d, mode=gpupool.MODE_SCATTER, flags=gpupool.LOAD_SCATTER_EXCHANGE | gpupool.LOAD_DEFER, part_index=0, part_count=2)
    try:
        with pytest.raises(gpupool.ErrUnsupported):  # refused for the load shape, before the state is looked at
            base.derive(ad)
    finally:
        base.release()


@pytest.mark.multigpu
def test_broadcast_and_scatter_in_one_process(native, gpu_count, tmp_path):
    if gpu_count < 2:
        pytest.skip("needs 2 GPUs")
    d = str(tmp_path / "llama")
    synth.make_llama(d, CFG)
    ad, pairs = _adapter(tmp_path, d, seed=6)
    with gpupool.Pool([0, 1], n_staging_buffers=4, staging_buffer_bytes=8 << 20, n_reader_threads=2) as pl:
        for mode in (gpupool.MODE_BROADCAST, gpupool.MODE_SCATTER):
            base = _poisoned_base(pl, d, mode=mode)
            try:
                m = base.derive(ad)
                try:
                    for dev in (0, 1):
                        desc = gpupool.adapter_describe(d, ad, mode=mode, part_index=dev, part_count=2 if mode == gpupool.MODE_SCATTER else 0)
                        _check_derived(base, m, dev, pairs, desc, f"mode {mode} device {dev}")
                finally:
                    m.release()
            finally:
                base.release()


def _manifest_text(m, device):
    L = gpupool.lib()
    need = C.c_size_t()
    assert L.kk_export_size(m._h, device, C.byref(need)) == 0
    buf = C.create_string_buffer(need.value)
    assert L.kk_export(m._h, device, None, buf, need.value) == 0
    return buf.value


def test_equals_kk_load_adapter_of_another_context_and_a_restarted_daemon_reloads_it(pool, tmp_path):
    d = str(tmp_path / "llama")
    synth.make_llama(d, CFG)
    ad, _ = _adapter(tmp_path, d, seed=8)
    base = pool.load(d)
    try:
        m = base.derive(ad)
    finally:
        base.release()  # the derived model holds no reference on its base
    try:
        info = m.info()
        reg = registry.PoolRegistry(str(tmp_path / "run"), epoch="a")
        reg.reconcile()
        reg.record(m.stats()["derive"]["base_key"] + "|derived", d, info["mode"], info["file_bytes"], info["pool_bytes"], info["devices"], [],
                   adapter=ad)
        stale = registry.PoolRegistry(str(tmp_path / "run"), epoch="b").reconcile()  # a restarted daemon
        assert len(stale) == 1 and stale[0].adapter == ad
        with gpupool.Pool([0], n_staging_buffers=2, staging_buffer_bytes=4 << 20, n_reader_threads=1) as other:
            e = stale[0]
            loaded = other.load(e.path, mode=e.mode, adapter=e.adapter)
            try:
                assert _manifest_text(loaded, 0) == _manifest_text(m, 0)
                assert loaded.stats()["n_loads"] == 1 and "derive" not in loaded.stats()
                n = m.pool_ptr(0)[1]
                for name, p in _placements(m, 0).items():
                    a, b = p.pool_offset, p.pool_offset + p.nbytes
                    assert np.array_equal(m.read(0, a, b - a), loaded.read(0, a, b - a)), name
                assert loaded.pool_ptr(0)[1] == n
            finally:
                loaded.release()
    finally:
        m.release()


def test_identity_refcount_and_repeated_load_part(pool, tmp_path):
    d = str(tmp_path / "llama")
    synth.make_llama(d, CFG)
    ad, pairs = _adapter(tmp_path, d, seed=9)
    base = _poisoned_base(pool, d)
    m = base.derive(ad)
    try:
        m2 = base.derive(os.path.join(ad, "..", os.path.basename(ad)))  # the canonical path is the identity
        assert m2.handle == m.handle and m.info()["refcount"] == 2
        m2.release()
        n_loads = m.stats()["n_loads"]
        m3 = pool.load(d, adapter=ad)  # a load with the base's arguments finds the derived model
        assert m3.handle == m.handle and m.info()["refcount"] == 2 and m.stats()["n_loads"] == n_loads
        m3.release()
        assert m.info()["loaded"] and base.info()["refcount"] == 1
        desc = gpupool.adapter_describe(d, ad)
        _, n = base.pool_ptr(0)
        before = m.read(0, 0, n)
        _check_derived(base, m, 0, pairs, desc, "derived")
        base.release()
        base = None
        assert np.array_equal(m.read(0, 0, n), before), "the derived pool changed when its base was released"
    finally:
        m.release()
        if base is not None:
            base.release()
    # a model loaded with the adapter first is what a derive returns
    base = pool.load(d)
    try:
        la = pool.load(d, adapter=ad)
        try:
            dm = base.derive(ad)
            assert dm.handle == la.handle and la.info()["refcount"] == 2 and "derive" not in la.stats()
            dm.release()
        finally:
            la.release()
    finally:
        base.release()


def test_load_part_on_a_model_derived_from_a_deferred_base_merges_again(pool, tmp_path):
    d = str(tmp_path / "llama")
    synth.make_llama(d, CFG)
    ad, pairs = _adapter(tmp_path, d, seed=10)
    base = _poisoned_base(pool, d)
    try:
        m = base.derive(ad)
        try:
            _, n = m.pool_ptr(0)
            first = m.read(0, 0, n)
            m.load_part()  # streams the file into the derived pool and merges in place again
            again = m.read(0, 0, n)
            diff = np.flatnonzero(first != again)
            assert diff.size == 0, f"{diff.size} bytes differ after kk_load_part, first at {diff[:4]}"
            assert m.stats()["n_loads"] == 1
        finally:
            m.release()
    finally:
        base.release()


def test_refusals_leave_the_budget_and_the_registry_as_they_were(native, tmp_path):
    d = str(tmp_path / "llama")
    synth.make_llama(d, CFG)
    ad, _ = _adapter(tmp_path, d, seed=11)
    ad2, _ = _adapter(tmp_path, d, seed=12)
    dora, _ = _adapter(tmp_path, d, seed=13, config={"use_dora": True})
    missing = str(tmp_path / "missing")
    tg = _targets(d)
    lf.seeded_adapter(missing, tg[:1] + [("model.layers.0.self_attn.nope_proj.weight", tg[0][1])], 4, 14)
    pb = gpupool.plan_describe(d)["layouts"][0]["pool_bytes"]
    # room for the base and one derived model, not two
    pl = gpupool.Pool([0], pool_bytes_per_device=2 * pb + pb // 2, n_staging_buffers=2, staging_buffer_bytes=4 << 20, n_reader_threads=1)
    try:
        base = pl.load(d, flags=gpupool.LOAD_DEFER)
        with pytest.raises(gpupool.ErrState):
            base.derive(ad)
        base.load_part()
        for bad, err in ((dora, gpupool.ErrUnsupported), (missing, gpupool.ErrNotFound), (str(tmp_path / "nothing"), gpupool.ErrNotFound)):
            with pytest.raises(err):
                base.derive(bad)
        m = base.derive(ad)  # the refusals took no budget: the base and one derived model still fit
        with pytest.raises(gpupool.ErrInvalid):
            m.derive(ad2)  # adapters do not stack
        with pytest.raises(gpupool.ErrNoMemory):
            base.derive(ad2)
        assert m.info()["refcount"] == 1 and base.info()["refcount"] == 1
        m.release()
        m = base.derive(ad2)  # the refused derive took nothing, and the released one gave its budget back
        m.release()
        base.release()
    finally:
        pl.close()  # KK_EBUSY if a refused derive had left a model registered


def test_concurrent_derives_of_one_adapter_share_one_model(pool, tmp_path):
    d = str(tmp_path / "llama")
    synth.make_llama(d, CFG)
    ad, pairs = _adapter(tmp_path, d, seed=15)
    base = pool.load(d)
    got, errs = [], []

    def run():
        try:
            got.append(base.derive(ad))
        except Exception as e:  # reported below
            errs.append(e)

    th = [threading.Thread(target=run) for _ in range(8)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    try:
        assert not errs, errs
        assert len({m.handle for m in got}) == 1 and got[0].info()["refcount"] == 8
        _check_derived(base, got[0], 0, pairs, gpupool.adapter_describe(d, ad), "8 threads")
    finally:
        for m in got:
            m.release()
        base.release()
