"""The kernel stage from the HBM-resident image, fp16 output (KK_LOAD_F16) against bf16 output on the same inputs, in alternating runs.

Pairs (each the f16 load first, then its bf16 counterpart):

  * Llama-3-8B, copy:  the F16 file loaded as f16 (verbatim)  vs  the BF16 file loaded as bf16 (verbatim);
  * Llama-3-8B, cast:  the BF16 file loaded as f16            vs  the F16 file loaded as bf16 (the 16-bit cast either way);
  * Mixtral-8x7B q4_K, 4 layers: the GGUF as f16 vs as bf16 (the same dequantiser, another pack);
  * GPT-2-small f32 with the Conv1D transposes: f16 vs bf16.

Both models of a pair are resident at once (kk_stage_resident); after --warmup conversions of each, --rounds rounds each time --steps
conversions of the f16 model and then --steps of the bf16 one, so drift in clocks or neighbours hits both alike.  Rates are GB/s of
algorithmic bytes (source read once + pool bytes written, DESIGN.md §6), per round; the record carries the card's name and power limit.
--layers / --gpt2-layers shrink the models so the script can be rehearsed on a machine without a GPU: it runs up to the first device call.

    python tools/f16_bench.py [--steps 5] [--warmup 3] [--rounds 3] [--out result.json]
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

from kukeon_b200 import gpupool  # noqa: E402
from tools import synth  # noqa: E402
from tools.stage_bench import card, data_dir  # noqa: E402

F16, T = gpupool.LOAD_F16, gpupool.LOAD_GPT2_CONV1D_T


def rates(m, steps: int) -> float:
    """Mean GB/s of algorithmic bytes over `steps` resident conversions of model m."""
    part = m.stats()["parts"][0]
    ms = sum(m.convert_resident()[0] for _ in range(steps)) / steps
    return (part["src_bytes"] + part["out_bytes"]) / (ms / 1e3) / 1e9


def pair(pool, name: str, a: tuple, b: tuple, args) -> dict:
    """a, b: (path, flags) of the f16 and the bf16 load.  Returns the per-round rates of both and their ratio."""
    ms = [pool.load(p, flags=fl | gpupool.LOAD_DEFER) for p, fl in (a, b)]
    try:
        for m in ms:
            m.load_part()
            m.stage_resident()
            for _ in range(args.warmup):
                m.convert_resident()
        r = {"f16": [], "bf16": []}
        for _ in range(args.rounds):
            r["f16"].append(rates(ms[0], args.steps))
            r["bf16"].append(rates(ms[1], args.steps))
        alg = [m.stats()["parts"][0] for m in ms]
    finally:
        for m in ms:
            m.release()
    mean = {k: sum(v) / len(v) for k, v in r.items()}
    return {"pair": name, "f16": {"load": os.path.basename(a[0]), "flags": a[1], "GBps_per_round": r["f16"], "GBps_mean": mean["f16"],
                                  "algorithmic_bytes": alg[0]["src_bytes"] + alg[0]["out_bytes"]},
            "bf16": {"load": os.path.basename(b[0]), "flags": b[1], "GBps_per_round": r["bf16"], "GBps_mean": mean["bf16"],
                     "algorithmic_bytes": alg[1]["src_bytes"] + alg[1]["out_bytes"]},
            "f16_over_bf16": mean["f16"] / mean["bf16"],
            "spread_bf16": (max(r["bf16"]) - min(r["bf16"])) / mean["bf16"], "spread_f16": (max(r["f16"]) - min(r["f16"])) / mean["f16"]}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--layers", type=int, default=0, help="Llama layers (default: the full 32)")
    ap.add_argument("--gpt2-layers", type=int, default=0, help="GPT-2 layers (default: the full 12)")
    ap.add_argument("--data-dir", default="", help="parent of the run's own temporary directory (default: /dev/shm when it has room)")
    ap.add_argument("--out", default="")
    args = ap.parse_args(argv)
    if args.steps < 5 or args.warmup < 3 or args.rounds < 2:
        raise SystemExit("--steps >= 5, --warmup >= 3, --rounds >= 2")
    cfg = dict(synth.LLAMA3_8B, **({"layers": args.layers} if args.layers else {}))
    mix = synth.mixtral_gguf_tensors(layers=4)
    g2 = synth.gpt2_tensors(n_layer=args.gpt2_layers, vocab=4096) if args.gpt2_layers else synth.gpt2_tensors()
    need = 2 * synth.total_bytes(synth.llama_tensors(**cfg)) + synth.total_bytes(mix) + synth.total_bytes(g2)
    d = data_dir(need, args.data_dir)
    res = {"what": "kernel stage from the resident image, f16 vs bf16 output, alternating rounds", "steps": args.steps, "warmup": args.warmup,
           "rounds": args.rounds}
    try:
        t0 = time.time()
        llama = {dt: os.path.join(d, f"llama_{dt.lower()}") for dt in ("F16", "BF16")}
        for dt, p in llama.items():
            synth.make_llama(p, cfg, dtype=dt)
        gg, gp = os.path.join(d, "mixtral_q4k_4l.gguf"), os.path.join(d, "gpt2.safetensors")
        synth.write_gguf(gg, mix, 8007)
        synth.write_safetensors(gp, g2, 1234)
        res["synth_s"] = time.time() - t0
        pairs = [("Llama-3-8B copy: F16 -> f16 vs BF16 -> bf16", (llama["F16"], F16), (llama["BF16"], 0)),
                 ("Llama-3-8B cast: BF16 -> f16 vs F16 -> bf16", (llama["BF16"], F16), (llama["F16"], 0)),
                 ("Mixtral-8x7B q4_K, 4 layers", (gg, F16), (gg, 0)),
                 ("GPT-2-small f32, Conv1D transposes", (gp, F16 | T), (gp, T))]
        for name, a, b in pairs:  # the plans, on the CPU: a rehearsal gets this far
            pa, pb = gpupool.plan_describe(a[0], flags=a[1]), gpupool.plan_describe(b[0], flags=b[1])
            assert pa["layouts"][0]["pool_bytes"] == pb["layouts"][0]["pool_bytes"] or a[0] != b[0], name
        print(json.dumps({"planned": [n for n, _, _ in pairs]}), flush=True)
        with gpupool.Pool([0]) as pool:  # first device call
            res["card"] = card(0)
            res["pairs"] = []
            for name, a, b in pairs:
                res["pairs"].append(pair(pool, name, a, b, args))
                print(json.dumps(res["pairs"][-1]), flush=True)
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
