"""CPU tier: the pedigree of the fp16 oracle (tests/f16_oracle.py) and of the CPU replay's fp16 pack.

fp16 keeps three more mantissa bits of the dequantisers' fp32 than bf16 did, so the oracle's fp32 arithmetic is held to gguf-py at fp32, bit
for bit, on every block type of the golden GGUF fixtures and on random bytes with non-finite and negative scales.  The casts are held to
torch's .to(torch.float16) on every bf16 and fp16 bit pattern and on the fp32 specials; the replay's pack_f16x2 (F16C, checked against
the compiler's _Float16 conversion) to numpy on every fp32 special class."""
import os

import numpy as np
import pytest
import torch

from oracle import oracle
from tests import f16_oracle as fo
from tests import kk_emul, kk_f16_emul

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURES = ("q4k.gguf", "q4km_mix.gguf", "quants_f4.gguf", "quants_cb.gguf", "quants_iq.gguf")


def bits16(t):
    return t.contiguous().view(torch.int16).numpy().view(np.uint16)


def same_f32(a, b):
    return ((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all()


def fixture_types():
    seen = set()
    for f in FIXTURES:
        _, recs = oracle.index_path(os.path.join(G, f))
        seen |= {r["dtype"] for r in recs if r["dtype"] in oracle.BLOCK_QUANTS}
    return sorted(seen)


def test_the_fixtures_cover_every_block_type():
    assert set(fixture_types()) == set(oracle.BLOCK_QUANTS)


@pytest.mark.parametrize("fixture", FIXTURES)
def test_golden_fixture_dequantisers_equal_gguf_py_at_f32(fixture):
    from gguf import GGMLQuantizationType, quants
    p = os.path.join(G, fixture)
    _, recs = oracle.index_path(p)
    raw = open(p, "rb").read()
    n = 0
    for r in recs:
        if r["dtype"] not in oracle.BLOCK_QUANTS:
            continue
        nel, nb, fn = oracle.BLOCK_QUANTS[r["dtype"]]
        b = np.frombuffer(raw[r["file_offset"]:r["file_offset"] + r["nbytes"]], np.uint8).reshape(-1, nb)
        with np.errstate(all="ignore"):
            ref, got = quants.dequantize(b, getattr(GGMLQuantizationType, r["dtype"])).astype(np.float32), fn(b)
        assert same_f32(ref.reshape(got.shape), got), (fixture, r["name"])
        # and the fp16 the library stores is numpy's RNE of exactly that fp32
        assert (fo.dequant_f16(r["dtype"], b) == fo.f32_to_f16(ref.reshape(got.shape))).all()
        n += 1
    assert n


@pytest.mark.parametrize("dtype", sorted(oracle.BLOCK_QUANTS))
def test_random_bytes_with_non_finite_and_negative_scales_equal_gguf_py_at_f32(dtype):
    from gguf import GGMLQuantizationType, quants
    nel, nb, fn = oracle.BLOCK_QUANTS[dtype]
    rng = np.random.Generator(np.random.Philox(key=77))
    b = rng.integers(0, 256, size=(2048, nb), dtype=np.uint8)
    with np.errstate(all="ignore"):
        ref, got = quants.dequantize(b, getattr(GGMLQuantizationType, dtype)).astype(np.float32), fn(b)
    assert same_f32(ref.reshape(got.shape), got)
    assert (got < 0).any()
    h = fo.dequant_f16(dtype, b)
    nan = np.isnan(got)
    assert (h[nan] == fo.NAN16).all()
    with np.errstate(all="ignore"):
        assert (h[~nan] == got[~nan].astype(np.float16).view(np.uint16)).all()


def test_bf16_to_f16_every_pattern_vs_torch():
    u = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    ref = bits16(torch.from_numpy(u.view(np.int16).copy()).view(torch.bfloat16).to(torch.float16))
    got = fo.bf16_bits_to_f16(u)
    nan = (u & 0x7FFF) > 0x7F80
    assert (got[~nan] == ref[~nan]).all() and (got[nan] == 0x7FFF).all()
    assert (got == 0x7C00).any() and (got == 0x0001).any(), "overflow to inf and fp16 subnormals both occur"


def test_f16_to_f16_is_the_identity_and_f16_through_f32_round_trips():
    u = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    x = u.view(np.float16).astype(np.float32)
    got = fo.f32_to_f16(x)
    nan = (u & 0x7FFF) > 0x7C00
    assert (got[~nan] == u[~nan]).all() and (got[nan] == 0x7FFF).all()
    ref = bits16(torch.from_numpy(x.copy()).to(torch.float16))
    assert (got[~nan] == ref[~nan]).all()


def f32_specials():
    """Overflow, the largest finite half and its rounding boundary, the fp16 subnormal range and its underflow edge, ties to even in both
    directions (normal and subnormal), +-0, +-inf, NaNs of both signs and payloads, fp32 subnormals."""
    tie = 2.0 ** -11  # half an ulp of 1.0 in fp16
    v = [65504.0, 65519.0, 65519.996, 65520.0, 1e5, 3.4e38, 2.0 ** -14, 2.0 ** -15, 2.0 ** -24, 2.0 ** -25, 1.5 * 2.0 ** -25, 2.0 ** -26, 3 * 2.0 ** -25,
         1.0 + tie, 1.0 + 3 * tie, 1.0 + tie + 2.0 ** -20, 0.0, -0.0, np.inf, -np.inf, 1e-40, -1e-45, 2.0 ** -14 - 2.0 ** -25]
    v = np.array(v + [-x for x in v], np.float32)
    nans = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFFFFFFF, 0x7FBFFFFF], np.uint32).view(np.float32)
    rng = np.random.default_rng(12)
    rnd = rng.integers(0, 1 << 32, 20000, dtype=np.uint64).astype(np.uint32).view(np.float32)
    return np.concatenate([v, nans, rnd, (rng.standard_normal(4000) * 2.0 ** rng.integers(-30, 20, 4000)).astype(np.float32)])


def test_f32_to_f16_specials_vs_torch():
    x = f32_specials()
    ref = bits16(torch.from_numpy(x.copy()).to(torch.float16))
    got = fo.f32_to_f16(x)
    nan = np.isnan(x)
    assert (got[~nan] == ref[~nan]).all() and (got[nan] == 0x7FFF).all()
    assert {0x7C00, 0xFC00, 0x0001, 0x8000, 0x0000, 0x7BFF} <= set(got.tolist())


def test_fp8_to_f16_every_pattern_vs_torch():
    b = np.arange(256, dtype=np.uint8)
    for tdt, fn in ((torch.float8_e4m3fn, fo.f8e4m3_bits_to_f16), (torch.float8_e5m2, fo.f8e5m2_bits_to_f16)):
        ref = bits16(torch.from_numpy(b.copy()).view(tdt).to(torch.float16))
        got = fn(b)
        nan = (ref & 0x7FFF) > 0x7C00
        assert (got[~nan] == ref[~nan]).all() and (got[nan] == 0x7FFF).all()


@pytest.fixture(scope="module")
def emul():
    return kk_f16_emul.load()


def emul_pack(L, f16, x):
    x = np.ascontiguousarray(x, np.float32)
    if x.size % 2:
        x = np.concatenate([x, np.zeros(1, np.float32)])
    out = np.zeros(x.size, np.uint16)
    rc = L.kk_emul_pack(int(f16), x.ctypes.data, out.ctypes.data, x.size)
    assert rc == 0, kk_emul.ERR.get(rc, rc)
    return out


def test_replay_pack_f16x2_vs_numpy_on_every_f32_special_class(emul):
    x = f32_specials()
    got = emul_pack(emul, True, x)[:x.size]
    assert (got == fo.f32_to_f16(x)).all()
    # and the bf16 pack is still the oracle's
    assert (emul_pack(emul, False, x)[:x.size] == oracle.f32_to_bf16(x)).all()


def test_replay_pack_f16x2_on_every_f16_and_bf16_value(emul):
    h = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    assert (emul_pack(emul, True, h.view(np.float16).astype(np.float32)) == fo.f32_to_f16(h.view(np.float16).astype(np.float32))).all()
    bf = (h.astype(np.uint32) << 16).view(np.float32)
    assert (emul_pack(emul, True, bf) == fo.bf16_bits_to_f16(h)).all()
