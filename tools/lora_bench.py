"""LoRA merge on load (kk_load_adapter) on a synthetic Llama-3-8B bf16 checkpoint: the merge kernel's time and rate, and kk_load_part with
and without the adapter.

Adapters: seeded bf16 at r = 8, 16 and 64 on q, k, v, o, gate, up and down of all 32 layers (PEFT's saved format, tests/lora_fixtures.py).
One DEFER model per adapter plus the base model are resident at once; after --warmup kk_load_part calls of each, --rounds rounds each run
kk_load_part once per model in turn, so drift in clocks or neighbours hits all alike.  Per load it records the merge kernel's CUDA-event time
(kk_stats adapter.t_merge) and the load's wall time (load_s).  The merge's rate is pool bytes read + written per second and FMAs per second;
its share of peak is the larger of the two roofline times (HBM 3.35 TB/s, FP32 67 TFLOP/s with an FMA as two FLOPs, the H100 SXM data
sheet) over the measured time, and the record names which bound applies.  Reads use KUKEON_GPULOAD_READ=pread unless it is set.  The record
carries the card's name and power limit.  --layers shrinks the model so the script can be rehearsed on a machine without a GPU.

    python tools/lora_bench.py [--warmup 1] [--rounds 3] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import shutil
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
os.environ.setdefault("KUKEON_GPULOAD_READ", "pread")

from kukeon_b200 import gpupool  # noqa: E402
from tests import lora_fixtures as lf  # noqa: E402
from tools import synth  # noqa: E402
from tools.stage_bench import card, data_dir  # noqa: E402

HBM_BPS, FP32_FLOPS = 3.35e12, 67e12
RANKS = (8, 16, 64)
TARGET_RE = re.compile(r"\.(self_attn\.[qkvo]_proj|mlp\.(gate|up|down)_proj)\.weight$")


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--layers", type=int, default=0, help="fewer layers (rehearsal)")
    ap.add_argument("--data-dir", default="")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    cfg = dict(synth.LLAMA3_8B, **({"layers": args.layers} if args.layers else {}))
    tmp = data_dir(synth.total_bytes(synth.llama_tensors(**cfg)) + (1 << 30), args.data_dir)
    try:
        ck = os.path.join(tmp, "llama")
        synth.make_llama(ck, cfg)
        targets = [(t["name"], t["shape"]) for t in gpupool.index(ck) if TARGET_RE.search(t["name"])]
        assert len(targets) == 7 * cfg["layers"]
        ads = {}
        for r in RANKS:
            ads[r] = os.path.join(tmp, f"lora_r{r}")
            lf.seeded_adapter(ads[r], targets, r, 100 + r, "BF16")
        pool_bytes = sum(2 * R * C for _, (R, C) in targets)  # bf16 pool bytes of the targets
        rec = {"card": None, "model": f"Llama-3-8B bf16{'' if not args.layers else f', {args.layers} layers'}", "targets": len(targets),
               "target_pool_bytes": pool_bytes, "read": os.environ["KUKEON_GPULOAD_READ"], "adapters": {}}
        with gpupool.Pool([0]) as pool:
            rec["card"] = card(0)
            models = {"base": pool.load(ck, flags=gpupool.LOAD_DEFER)}
            for r in RANKS:
                models[r] = pool.load(ck, flags=gpupool.LOAD_DEFER, adapter=ads[r])
            try:
                for _ in range(args.warmup):
                    for m in models.values():
                        m.load_part()
                merge = {r: [] for r in RANKS}
                load = {k: [] for k in models}
                for _ in range(args.rounds):
                    for k, m in models.items():
                        m.load_part()
                        st = m.stats()
                        load[k].append(st["load_s"])
                        if k != "base":
                            merge[k].append(st["adapter"]["t_merge"])
                rec["load_s_base"] = load["base"]
                for r in RANKS:
                    t = statistics.median(merge[r])
                    fmas = sum(R * C * r for _, (R, C) in targets)
                    t_hbm, t_fp32 = 2 * pool_bytes / HBM_BPS, 2 * fmas / FP32_FLOPS
                    rec["adapters"][r] = {
                        "merge_ms": [x * 1e3 for x in merge[r]], "merge_ms_median": t * 1e3,
                        "pool_gbps": 2 * pool_bytes / t / 1e9, "tflops_fp32": 2 * fmas / t / 1e12,
                        "bound": "HBM" if t_hbm >= t_fp32 else "FP32", "share_of_bound": max(t_hbm, t_fp32) / t,
                        "load_s": load[r], "load_overhead": statistics.median(load[r]) / statistics.median(load["base"]) - 1,
                        "adapter_bytes_on_device": models[r].stats()["adapter"]["bytes"]}
            finally:
                for m in models.values():
                    m.release()
        print(json.dumps(rec, indent=1))
        if args.out:
            with open(args.out, "w") as f:
                json.dump(rec, f, indent=1)
        return 0
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    sys.exit(main())
