"""The cost of KK_LOAD_HF_LAYOUT on one GPU: the same GGUF loaded with and without the flag, in alternating rounds.

Files (synthetic content, real shapes and head counts, on tmpfs when it has room):

  * Llama-3-8B q4_K: 32 layers, 32 query / 8 key-value heads of 128, every 2-D weight Q4_K;
  * Mixtral-8x7B q4_K, 4 layers: 32 / 8 heads, 8 experts per layer.

For each file and each of --rounds rounds, first the flagged load and then the unflagged one:
  * the kernel stage from the resident image (kk_stage_resident / kk_convert_resident): --warmup conversions, then --steps timed ones,
    GB/s of algorithmic bytes (source read once + pool bytes written, DESIGN.md §6);
  * kk_load_part of a deferred load with KUKEON_GPULOAD_READ=pread: --steps loads of a fresh model each, wall time and GB/s of file bytes.
The plan's tiles, reads and segments of both loads are counted on the CPU, with the tiles of the Q/K segments the flag creates.  The
record carries the card's name and power limit.  --layers shrinks the models so the script can be rehearsed without a GPU: it runs up to
the first device call.

    python tools/hf_layout_bench.py [--steps 5] [--warmup 3] [--rounds 3] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

os.environ["KUKEON_GPULOAD_READ"] = "pread"  # the library reads it per load; set before any load
from kukeon_b200 import gpupool  # noqa: E402
from tools import synth  # noqa: E402
from tools.stage_bench import card, data_dir  # noqa: E402

HF = gpupool.LOAD_HF_LAYOUT


def plan_counts(path: str, flags: int) -> dict:
    """Tiles, reads and segments of the one-GPU plan, and the tiles of the segments that write q_proj / k_proj slots."""
    p = gpupool.plan_describe(path, flags=flags)
    qk = [(t["pool_offset"], t["pool_offset"] + t["nbytes"]) for t in p["layouts"][0]["tensors"] if t["name"].endswith(("q_proj.weight", "k_proj.weight", "attn_q.weight", "attn_k.weight"))]
    tiles = reads = segs = qk_tiles = qk_segs = 0
    for ch in p["parts"][0]["chunks"]:
        tiles += ch["n_tiles"]
        reads += len(ch["reads"])
        segs += len(ch["segs"])
        bounds = [s["tile_begin"] for s in ch["segs"]] + [ch["n_tiles"]]
        for k, s in enumerate(ch["segs"]):
            if any(a <= s["dst_off"] < b for a, b in qk):
                qk_tiles += bounds[k + 1] - bounds[k]
                qk_segs += 1
    return {"tiles": tiles, "reads": reads, "segs": segs, "chunks": len(p["parts"][0]["chunks"]), "qk_tiles": qk_tiles, "qk_segs": qk_segs}


def kernel_rate(m, steps: int) -> float:
    part = m.stats()["parts"][0]
    ms = sum(m.convert_resident()[0] for _ in range(steps)) / steps
    return (part["src_bytes"] + part["out_bytes"]) / (ms / 1e3) / 1e9


def e2e(pool, path: str, flags: int, steps: int) -> dict:
    walls, nbytes = [], 0
    for _ in range(steps):
        m = pool.load(path, flags=flags | gpupool.LOAD_DEFER)
        try:
            t0 = time.perf_counter()
            m.load_part()  # returns once the pool holds the model (the load synchronises its streams)
            walls.append(time.perf_counter() - t0)
            nbytes = m.stats()["local_src_bytes"]
        finally:
            m.release()
    w = sum(walls) / len(walls)
    return {"wall_s": w, "GBps": nbytes / w / 1e9}


def bench_file(pool, name: str, path: str, args) -> dict:
    out = {"file": name, "plan": {"hf": plan_counts(path, HF), "gguf": plan_counts(path, 0)}, "kernel_GBps": {"hf": [], "gguf": []},
           "e2e": {"hf": [], "gguf": []}}
    ms = {k: pool.load(path, flags=fl | gpupool.LOAD_DEFER) for k, fl in (("hf", HF), ("gguf", 0))}
    try:
        for m in ms.values():
            m.load_part()
            m.stage_resident()
            for _ in range(args.warmup):
                m.convert_resident()
        for _ in range(args.rounds):
            for k in ("hf", "gguf"):
                out["kernel_GBps"][k].append(kernel_rate(ms[k], args.steps))
    finally:
        for m in ms.values():
            m.release()
    for k, fl in (("hf", HF), ("gguf", 0)):  # warm-up loads
        e2e(pool, path, fl, args.warmup)
    for _ in range(args.rounds):
        for k, fl in (("hf", HF), ("gguf", 0)):
            out["e2e"][k].append(e2e(pool, path, fl, args.steps))
    mean = lambda v: sum(v) / len(v)
    out["kernel_hf_over_gguf"] = mean(out["kernel_GBps"]["hf"]) / mean(out["kernel_GBps"]["gguf"])
    out["e2e_wall_hf_over_gguf"] = mean([r["wall_s"] for r in out["e2e"]["hf"]]) / mean([r["wall_s"] for r in out["e2e"]["gguf"]])
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--layers", type=int, default=0, help="Llama layers (default: the full 32)")
    ap.add_argument("--data-dir", default="", help="parent of the run's own temporary directory (default: /dev/shm when it has room)")
    ap.add_argument("--out", default="")
    args = ap.parse_args(argv)
    L8 = dict(hidden=4096, ffn=14336, layers=args.layers or 32, n_head=32, n_head_kv=8, vocab=128256, qtype="Q4_K")
    MX = dict(hidden=4096, ffn=14336, layers=min(args.layers or 4, 4), n_head=32, n_head_kv=8, vocab=32000, qtype="Q4_K", experts=8)
    files = {"Llama-3-8B q4_K": (L8, 8001), "Mixtral-8x7B q4_K, 4 layers": (MX, 8007)}
    need = sum(synth.total_bytes(synth.llama_gguf_tensors(**c)) for c, _ in files.values())
    d = data_dir(need, args.data_dir)
    res = {"what": "KK_LOAD_HF_LAYOUT vs the same GGUF without it, alternating rounds; KUKEON_GPULOAD_READ=pread", "steps": args.steps,
           "warmup": args.warmup, "rounds": args.rounds, "files": []}
    try:
        paths = {}
        for name, (c, seed) in files.items():
            paths[name] = os.path.join(d, name.split()[0] + ".gguf")
            synth.write_gguf(paths[name], synth.llama_gguf_tensors(**c), seed,
                             extra_kv=synth.gguf_head_kv("llama", c["n_head"], c["n_head_kv"], c.get("experts", 0)))
        print(json.dumps({"planned": {n: {"hf": plan_counts(p, HF), "gguf": plan_counts(p, 0)} for n, p in paths.items()}}), flush=True)
        with gpupool.Pool([0]) as pool:  # first device call
            res["card"] = card(0)
            for name, p in paths.items():
                res["files"].append(bench_file(pool, name, p, args))
                print(json.dumps(res["files"][-1]), flush=True)
    finally:
        shutil.rmtree(d)  # the directory data_dir created for this run, nothing else
    text = json.dumps(res)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
