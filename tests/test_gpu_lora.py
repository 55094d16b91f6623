"""LoRA adapters on load (kk_load_adapter), GPU tier: every pool of an adapter load equals the base load's pool with the C oracle's merge
applied to the targets, byte for byte over the whole pool (poisoned first, so a skipped tile or a stray store fails); the layout is the
base load's; identity, refcount, memory and the manifest.  Adapters are written in PEFT's saved format (tests/lora_fixtures.py)."""
import os
import re

import numpy as np
import pytest

from kukeon_b200 import gpupool
from tests import helpers
from tests import lora_fixtures as lf
from tools import synth

pytestmark = pytest.mark.gpu
CFG = dict(hidden=256, ffn=704, layers=3, kv_dim=64, vocab=300)
RANKS = [1, 7, 16, 64, 256]


def _targets(path, flags=0):
    plan = gpupool.plan_describe(path, flags=flags)
    return [(t["name"], t["shape"]) for t in plan["layouts"][0]["tensors"] if re.search(r"_proj\.weight$", t["name"]) and len(t["shape"]) == 2]


def _adapter(tmp_path, path, flags=0, seed=1, dtype="BF16", alpha=16):
    d = str(tmp_path / f"ad{seed}")
    pairs = lf.seeded_adapter(d, _targets(path, flags), lambda i: RANKS[i % len(RANKS)], seed, dtype, alpha)
    return d, pairs


def _placements(m, device):
    out = {}
    for t in m.tensors():
        for p in m.placements(t["name"]):
            if p.device == device:
                out[t["name"]] = p
    return out


def _check(base, m, device, adapter, pairs, desc, label, fill=None):
    """m's pool on `device` against base's pool there with every described target merged by the C oracle."""
    pb, pm = _placements(base, device), _placements(m, device)
    assert pb == pm, f"{label}: the adapter load's layout differs from the base load's"
    _, n = base.pool_ptr(device)
    exp = lf.expected_pool(base.read(device, 0, n), desc, pairs,
                           lambda name: (pm[name].pool_offset, pm[name].shape, pm[name].slice_dim, pm[name].slice_begin))
    mask = np.zeros(n, bool)
    for p in pm.values():
        mask[p.pool_offset:p.pool_offset + p.nbytes] = True
    if fill is None:
        got = m.read(device, 0, n)
        assert np.array_equal(got[mask], exp[mask]), f"{label}: {np.count_nonzero(got[mask] != exp[mask])} bytes differ"
    else:
        helpers.assert_pool_exact(m, device, exp, mask, fill, label)
    for t in desc["targets"]:  # the merge changed every target
        p = pm[t["name"]]
        a, b = p.pool_offset, p.pool_offset + p.nbytes
        assert not np.array_equal(exp[a:b], base.read(device, a, b - a)) or t["scaling"] == 0


def _deferred(pool, path, adapter, **kw):
    """Adapter load with DEFER, pool poisoned, then kk_load_part: returns (model, poison)."""
    flags = kw.pop("flags", 0)
    m = pool.load(path, flags=flags | gpupool.LOAD_DEFER, adapter=adapter, **kw)
    return m, helpers.poison(m, 0)


@pytest.mark.parametrize("dtype,flags", [("BF16", 0), ("F16", 0), ("F32", gpupool.LOAD_KEEP_F32), ("BF16", gpupool.LOAD_F16)],
                         ids=["bf16", "f16", "f32_keep", "load_f16"])
def test_single_pool_equals_base_plus_oracle_merge(pool, tmp_path, dtype, flags):
    d = str(tmp_path / "llama")
    synth.make_llama(d, CFG, dtype=dtype)
    ad, pairs = _adapter(tmp_path, d, dtype=["F32", "BF16", "F16"][len(dtype) % 3])
    desc = gpupool.adapter_describe(d, ad, flags=flags)
    base = pool.load(d, flags=flags)
    try:
        m, fill = _deferred(pool, d, ad, flags=flags)
        try:
            m.load_part()
            _check(base, m, 0, ad, pairs, desc, f"{dtype}/{flags:#x}", fill)
            st = m.stats()["adapter"]
            assert st["n_tensors"] == len(desc["targets"]) and st["bytes"] > 0 and st["t_merge"] > 0
        finally:
            m.release()
    finally:
        base.release()


def test_q4k_gguf_under_hf_layout(pool, tmp_path):
    p = str(tmp_path / "llama_q4k.gguf")
    synth.write_gguf(p, synth.llama_gguf_tensors(256, 512, 2, 4, 2, 300, qtype="Q4_K"), 17, extra_kv=synth.gguf_head_kv("llama", 4, 2))
    flags = gpupool.LOAD_HF_LAYOUT
    ad, pairs = _adapter(tmp_path, p, flags, seed=3)
    desc = gpupool.adapter_describe(p, ad, flags=flags)
    assert any(t["name"].endswith("self_attn.q_proj.weight") for t in desc["targets"])
    base = pool.load(p, flags=flags)
    try:
        m, fill = _deferred(pool, p, ad, flags=flags)
        try:
            m.load_part()
            _check(base, m, 0, ad, pairs, desc, "q4_K hf", fill)
        finally:
            m.release()
    finally:
        base.release()


def test_pipeline_stage_and_repeated_load_part(pool, tmp_path):
    d = str(tmp_path / "llama")
    synth.make_llama(d, CFG)
    ad, pairs = _adapter(tmp_path, d, seed=4)
    desc = gpupool.adapter_describe(d, ad, layers=(1, 2))
    assert desc["skipped"] and desc["targets"]
    base = pool.load(d, layers=(1, 2))
    try:
        m, fill = _deferred(pool, d, ad, layers=(1, 2))
        try:
            m.load_part()
            _check(base, m, 0, ad, pairs, desc, "stage", fill)
            m.load_part()  # rewrites the base bytes and merges again: identical
            _check(base, m, 0, ad, pairs, desc, "stage, second kk_load_part", fill)
            assert m.stats()["n_loads"] == 2
        finally:
            m.release()
    finally:
        base.release()


def test_two_rank_scatter_on_one_device(pool, tmp_path):
    d = str(tmp_path / "llama")
    synth.make_llama(d, CFG)
    ad, pairs = _adapter(tmp_path, d, seed=5)
    for k in range(2):
        desc = gpupool.adapter_describe(d, ad, mode=gpupool.MODE_SCATTER, part_index=k, part_count=2)
        base = pool.load(d, mode=gpupool.MODE_SCATTER, part_index=k, part_count=2)
        try:
            m, fill = _deferred(pool, d, ad, mode=gpupool.MODE_SCATTER, part_index=k, part_count=2)
            try:
                m.load_part()
                sliced = {p.slice_dim for p in _placements(m, 0).values()}
                assert {0, 1} <= sliced
                _check(base, m, 0, ad, pairs, desc, f"scatter rank {k}", fill)
            finally:
                m.release()
        finally:
            base.release()
    with pytest.raises(gpupool.ErrUnsupported):
        pool.load(d, mode=gpupool.MODE_SCATTER, flags=gpupool.LOAD_SCATTER_EXCHANGE | gpupool.LOAD_DEFER, part_index=0, part_count=2, adapter=ad)
    with pytest.raises(gpupool.ErrUnsupported):
        pool.load(d, mode=gpupool.MODE_BROADCAST, flags=gpupool.LOAD_DEFER, part_index=0, part_count=2, adapter=ad)


@pytest.mark.multigpu
def test_broadcast_p2p_and_scatter_in_one_process(native, gpu_count, tmp_path):
    if gpu_count < 2:
        pytest.skip("needs 2 GPUs")
    d = str(tmp_path / "llama")
    synth.make_llama(d, CFG)
    ad, pairs = _adapter(tmp_path, d, seed=6)
    with gpupool.Pool([0, 1], n_staging_buffers=4, staging_buffer_bytes=8 << 20, n_reader_threads=2) as pl:
        for mode in (gpupool.MODE_BROADCAST, gpupool.MODE_SCATTER):
            base = pl.load(d, mode=mode)
            m = pl.load(d, mode=mode, adapter=ad)
            try:
                for dev in (0, 1):
                    desc = gpupool.adapter_describe(d, ad, mode=mode, part_index=dev, part_count=2 if mode == gpupool.MODE_SCATTER else 0)
                    _check(base, m, dev, ad, pairs, desc, f"mode {mode} device {dev}")
            finally:
                m.release()
                base.release()


def test_identity_refcount_memory_and_manifest(pool, tmp_path):
    from cuda.bindings import runtime as cudart
    d = str(tmp_path / "llama")
    synth.make_llama(d, dict(hidden=1024, ffn=2816, layers=2, kv_dim=256, vocab=512))
    ad = str(tmp_path / "ad256")
    pairs = lf.seeded_adapter(ad, _targets(d), 256, 7, "F32")  # 36 MiB of A and B
    base = pool.load(d)
    try:
        def free():
            err, f, _ = cudart.cudaMemGetInfo()
            assert err == cudart.cudaError_t.cudaSuccess
            return f
        before = free()
        m = pool.load(d, adapter=ad)
        after = free()
        try:
            st = m.stats()
            assert st["adapter"]["bytes"] > 32 << 20
            pool_bytes = m.pool_ptr(0)[1]
            # the pool stays; the adapter's buffer (A and B as fp32, larger than the slack allowed here) is gone
            assert before - after <= (pool_bytes + (2 << 20) - 1) // (2 << 20) * (2 << 20) + (8 << 20), (before - after, pool_bytes)
            assert m.handle != base.handle and base.info()["refcount"] == 1
            m2 = pool.load(d, adapter=os.path.join(ad, "..", os.path.basename(ad)))  # the canonical path is the identity
            try:
                assert m2.handle == m.handle and m.info()["refcount"] == 2
            finally:
                m2.release()
            assert m.info()["refcount"] == 1
            man = m.manifest(0)
            assert man["adapter"] == {"path": os.path.realpath(ad), "nTensors": len(pairs)}
            assert "adapter" not in base.manifest(0) and "adapter" not in base.stats()
            desc = gpupool.adapter_describe(d, ad)
            _check(base, m, 0, ad, pairs, desc, "large")
        finally:
            m.release()
    finally:
        base.release()
