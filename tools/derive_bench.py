"""LoRA adapters on a resident base: kk_derive_adapter against kk_load_adapter, on one GPU.

Checkpoints: synthetic Llama-3-8B bf16 with seeded bf16 adapters at r = 8, 16 and 64 on q, k, v, o, gate, up and down of all 32 layers (as
tools/lora_bench.py builds them), and the 4-layer Mixtral-8x7B q4_K GGUF loaded under KK_LOAD_HF_LAYOUT with an r = 16 adapter on q, k, v
and o.  The base of each checkpoint stays resident.  After --warmup rounds, --rounds rounds alternate per adapter:
  (a) kk_load_adapter of base + adapter from the file (KUKEON_GPULOAD_READ=pread unless set), wall time, then released;
  (b) kk_derive_adapter from the resident base, wall time and kk_stats derive.{t_copy, t_merge, t_host}, then released;
  (c) kk_probe_hbm's ld/st copy over the pool size: the rate a copy of the pool can reach on this card, the ceiling of (b)'s device work.
(b)'s device work moves 2 x pool bytes (every byte read once from the base pool and written once to the derived one).  Its copies are issued
before the adapter is read on the host and its merge after A and B are uploaded, so the two rarely overlap: device_s = t_copy + t_merge is
the time the device is busy, and device_gbps = 2 x pool bytes / device_s is compared with (c) and with the data sheet's 3.35 TB/s (H100 SXM
HBM3).  The record carries the card's name, power limit and SM clocks, read in the same run.  --layers shrinks the checkpoints so the
script can be rehearsed on a machine without a GPU as far as the first device call.

    python tools/derive_bench.py [--warmup 1] [--rounds 3] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import shutil
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
os.environ.setdefault("KUKEON_GPULOAD_READ", "pread")

from kukeon_b200 import gpupool  # noqa: E402
from tests import lora_fixtures as lf  # noqa: E402
from tools import synth  # noqa: E402
from tools.stage_bench import card, data_dir  # noqa: E402

HBM_BPS = 3.35e12
LLAMA_RE = re.compile(r"\.(self_attn\.[qkvo]_proj|mlp\.(gate|up|down)_proj)\.weight$")
ATTN_RE = re.compile(r"\.self_attn\.[qkvo]_proj\.weight$")


def sm_clocks(uuid: str) -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "-i", uuid, "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60, check=True).stdout.splitlines()[0]
        now, top = (s.strip() for s in out.split(","))
        return {"sm_clock": now, "sm_clock_max": top}
    except (OSError, subprocess.SubprocessError, IndexError, ValueError) as e:
        return {"sm_clock": None, "error": str(e)}


def timed(fn):
    t0 = time.perf_counter()
    m = fn()  # both calls return once every device has synchronised
    return m, time.perf_counter() - t0


def bench_adapter(pool, base, path, flags, ad, rounds, warmup) -> dict:
    pool_bytes = base.pool_ptr(0)[1]
    rows = []
    for i in range(warmup + rounds):
        m, t_load = timed(lambda: pool.load(path, flags=flags, adapter=ad))
        m.release()
        m, t_derive = timed(lambda: base.derive(ad))
        st = m.stats()["derive"]
        m.release()
        probe = pool.probe_hbm(0, gpupool.PROBE_COPY, pool_bytes)
        if i >= warmup:
            rows.append(dict(load_s=t_load, derive_s=t_derive, t_copy=st["t_copy"], t_merge=st["t_merge"], t_host=st["t_host"], probe_gbps=probe))
    med = {k: statistics.median(r[k] for r in rows) for k in rows[0]}
    device_s = med["t_copy"] + med["t_merge"]
    gbps = 2 * pool_bytes / device_s / 1e9
    return {"pool_bytes": pool_bytes, "rounds": rows, "median": med, "load_over_derive": med["load_s"] / med["derive_s"],
            "device_s": device_s, "device_gbps": gbps, "share_of_copy_probe": gbps / med["probe_gbps"], "share_of_hbm_datasheet": gbps * 1e9 / HBM_BPS,
            "host_share_of_derive": med["t_host"] / med["derive_s"]}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--layers", type=int, default=0, help="fewer layers (rehearsal)")
    ap.add_argument("--data-dir", default="")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    llama = dict(synth.LLAMA3_8B, **({"layers": args.layers} if args.layers else {}))
    mx = dict(hidden=4096, ffn=14336, layers=min(args.layers or 4, 4), n_head=32, n_head_kv=8, vocab=32000, qtype="Q4_K", experts=8)
    need = synth.total_bytes(synth.llama_tensors(**llama)) + synth.total_bytes(synth.llama_gguf_tensors(**mx)) + (1 << 30)
    tmp = data_dir(need, args.data_dir)
    rec = {"read": os.environ["KUKEON_GPULOAD_READ"], "warmup": args.warmup, "rounds": args.rounds, "checkpoints": []}
    try:
        ck = os.path.join(tmp, "llama")
        synth.make_llama(ck, llama)
        gg = os.path.join(tmp, "mixtral.gguf")
        synth.write_gguf(gg, synth.llama_gguf_tensors(**mx), 8007, extra_kv=synth.gguf_head_kv("llama", mx["n_head"], mx["n_head_kv"], mx["experts"]))
        HF = gpupool.LOAD_HF_LAYOUT
        cases = []
        tg = [(t["name"], t["shape"]) for t in gpupool.index(ck) if LLAMA_RE.search(t["name"])]
        assert len(tg) == 7 * llama["layers"]
        for r in (8, 16, 64):
            ad = os.path.join(tmp, f"llama_r{r}")
            lf.seeded_adapter(ad, tg, r, 100 + r, "BF16")
            cases.append((f"Llama-3-8B bf16, r = {r}, q/k/v/o/gate/up/down", ck, 0, ad))
        tg = [(t["name"], t["shape"]) for t in gpupool.plan_describe(gg, flags=HF)["layouts"][0]["tensors"] if ATTN_RE.search(t["name"])]
        assert len(tg) == 4 * mx["layers"]
        ad = os.path.join(tmp, "mixtral_r16")
        lf.seeded_adapter(ad, tg, 16, 216, "BF16")
        cases.append((f"Mixtral-8x7B q4_K {mx['layers']} layers, HF layout, r = 16, q/k/v/o", gg, HF, ad))
        with gpupool.Pool([0]) as pool:  # first device call
            rec["card"] = card(0)
            for path, flags in ((ck, 0), (gg, HF)):
                base = pool.load(path, flags=flags)
                try:
                    for name, p, f, ad in cases:
                        if p != path:
                            continue
                        res = dict(name=name, **bench_adapter(pool, base, path, flags, ad, args.rounds, args.warmup))
                        rec["checkpoints"].append(res)
                        print(json.dumps(res), flush=True)
                finally:
                    base.release()
            if rec["card"].get("uuid"):
                rec["card"].update(sm_clocks(rec["card"]["uuid"]))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)  # the directory data_dir created for this run, nothing else
    print(json.dumps(rec, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
