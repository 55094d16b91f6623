"""CPU tier: the parts of bench.py that do not need a GPU — argument surface, workload inventories of the BASELINE configs, the CPU arm
(--impl reference) end to end on the small workload, and the one-JSON-line contract of that arm."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from tools import synth  # noqa: E402


def args_for(*argv):
    old = sys.argv
    sys.argv = ["bench.py", *argv]
    try:
        return bench.parse()
    finally:
        sys.argv = old


def test_defaults_follow_the_contract():
    a = args_for()
    assert (a.gpus, a.impl, a.workload, a.fanout) == (1, "ours", "llama3-8b", "p2p") and a.warmup >= 3 and a.steps >= 1  # fan-out only matters at N > 1
    assert not (a.nvls_compare or a.kernel_only or a.no_secondary) and a.qtype == "Q4_K"
    assert args_for("--workload", "gpt2").fanout == "p2p" and args_for("--fanout", "raw").fanout == "raw" and args_for("--fanout", "pull").fanout == "pull"


def test_workload_inventories_match_the_baseline_configs():
    """SURVEY.md §8(d): Llama-3-8B = 291 tensors / 16,060,522,496 B; Llama-3-70B = 723 tensors / 141,107,412,992 B; GPT-2-small = 148 tensors /
    497,759,232 B; Mixtral-8x7B merged experts = 10 x layers + 3 tensors, 16 of its 32 layers by default (the whole model in bf16 outgrows an
    80 GB H100)."""
    s = bench.workload_spec(args_for("--workload", "llama3-8b"))
    assert len(s["tensors"]) == 291 and synth.total_bytes(s["tensors"]) == 16_060_522_496 and s["mode"] == "broadcast"
    s = bench.workload_spec(args_for("--workload", "llama3-70b-scatter"))
    assert len(s["tensors"]) == 723 and synth.total_bytes(s["tensors"]) == 141_107_412_992 and s["mode"] == "scatter"
    s = bench.workload_spec(args_for("--workload", "gpt2"))
    assert len(s["tensors"]) == 148 and synth.total_bytes(s["tensors"]) == 497_759_232
    s = bench.workload_spec(args_for("--workload", "mixtral-q4k"))
    assert len(s["tensors"]) == 163 and "q4_k" in s["name"] and "layers 0-15 of 32" in s["name"]
    q = synth.total_bytes(s["tensors"])
    assert q == 13_211_156_480  # Q4_K blocks + F32 norms / routers of 16 layers
    assert len(synth.mixtral_gguf_tensors()) == 323  # the whole model: 32 layers
    s6 = bench.workload_spec(args_for("--workload", "mixtral-q4k", "--qtype", "Q6_K", "--layers", "2"))
    assert "q6_k" in s6["name"] and "REDUCED to 2 layers" in s6["name"] and {t[1] for t in s6["tensors"]} == {"Q6_K", "F32"}
    with pytest.raises(SystemExit):
        bench.workload_spec(args_for("--workload", "mixtral-q4k", "--qtype", "F32"))


def test_reference_arm_prints_one_json_line(tmp_path):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "gpt2", "--layers", "2", "--steps", "1", "--warmup", "1",
                        "--data-dir", str(tmp_path)], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, lines
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == bench.METRIC and d["unit"] == bench.UNIT and d["higher_is_better"] is True
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"] > 0
    assert d["e2e"] == {"value": d["value"], "unit": bench.UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0} and d["gpu_launches"] == 0
    assert d["config"]["workload"].startswith("GPT-2-small") and d["n_gpus"] == 1 and d["steps"] == 1
    assert d["config"]["same_config"] is True and "whole checkpoint" in d["cpu_baseline"]["sample"]


def test_page_cache_warm_up_stripes_every_byte_over_the_ranks(tmp_path):
    """bench.warm_page_cache: the ranks' stripes (32 MiB blocks dealt round-robin) cover every byte of every file exactly once; hidden files
    (the .complete marker) are not data."""
    d = tmp_path / "ck"
    d.mkdir()
    (d / "a.bin").write_bytes(b"x" * (70 << 20))
    (d / "b.bin").write_bytes(b"y" * (5 << 20))
    (d / ".complete").write_text("ok")
    per_rank = [bench.warm_page_cache(str(d), r, 3, passes=1, threads=2) for r in range(3)]
    assert sum(per_rank) == (70 << 20) + (5 << 20) and all(per_rank)
    assert bench.warm_page_cache(str(d), 0, 1, passes=1, threads=3) == (75 << 20)


def test_dump_outputs_writes_every_tensor_deterministically_within_the_budget(tmp_path):
    """bench.dump_outputs against a fake model: every tensor is written (bf16 and FP8 decoded exactly, integers as float64, other verbatim
    types as raw bytes), large tensors are sampled the same way every time, and the files stay under 64 MiB."""
    from types import SimpleNamespace

    from kukeon_b200.gpupool import Placement
    pool = np.random.default_rng(5).integers(0, 256, size=(40 << 20) + 4096, dtype=np.uint8)
    pool[40 << 20:(40 << 20) + 4] = [0x38, 0x40, 0xC8, 0x7F]  # F8_E4M3: 1.0, 2.0, -4.0, NaN
    base = 40 << 20
    pl = {"a.w": Placement(0, "BF16", 0, 40 << 20, [4096, 5120], None, 0), "f8": Placement(0, "F8_E4M3", base, 4, [4], None, 0),
          "i64": Placement(0, "I64", base + 64, 80, [10], None, 0), "q": Placement(0, "Q4_K", base + 256, 144, [256], None, 0)}
    m = SimpleNamespace(placements=lambda n: [pl[n]], read=lambda dev, off, n: pool[off:off + n].copy())
    ref = SimpleNamespace(tensors=[{"name": n} for n in pl])
    outs = []
    for k in range(2):
        d = tmp_path / f"d{k}"
        bench.dump_outputs(m, ref, 0, str(d))
        assert sorted(os.listdir(d)) == sorted(n + ".npy" for n in pl)
        assert sum(f.stat().st_size for f in d.iterdir()) <= bench.DUMP_MAX_BYTES
        outs.append({n: np.load(d / (n + ".npy")) for n in pl})
    assert all(np.array_equal(outs[0][n], outs[1][n], equal_nan=True) for n in pl)
    f8 = outs[0]["f8"]
    assert f8.dtype == np.float32 and list(f8[:3]) == [1.0, 2.0, -4.0] and np.isnan(f8[3])
    assert outs[0]["i64"].dtype == np.float64 and np.array_equal(outs[0]["i64"], pool[base + 64:base + 144].view("<i8").astype(np.float64))
    assert outs[0]["q"].dtype == np.float64 and outs[0]["q"].size == 144
    w = outs[0]["a.w"]
    assert w.dtype == np.float32 and 0 < w.size < 4096 * 5120 and w.size % 1024 == 0
