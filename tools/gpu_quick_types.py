"""Torch-free roofline table of every dequantiser: one GGUF per block type with the same 2-D weight shapes, loaded once, then the
kernel stage timed from the HBM-resident image (CUDA events inside the library).  Writes gpurun_out/types_roofline.json:

    python tools/gpu_quick_types.py [--weights-m 1024] [--types Q4_K,Q6_K,...]

Algorithmic bytes = file bytes of the tensors + bf16 bytes written (2 per weight); peak = MEASURED_PEAKS.json hbm_gbs when present.
Not a bench.py replacement (no clocks sampling, no e2e leg): it is the quick A/B table that says which dequantiser to profile."""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kukeon_b200 import gpupool  # noqa: E402
from tools import synth  # noqa: E402

ALL = ["Q4_0", "Q4_1", "Q5_0", "Q5_1", "Q8_0", "Q2_K", "Q3_K", "Q4_K", "Q5_K", "Q6_K", "IQ4_NL", "IQ4_XS", "MXFP4", "IQ2_XXS", "IQ2_XS", "IQ2_S", "IQ3_XXS",
       "IQ3_S", "IQ1_S", "IQ1_M", "TQ1_0", "TQ2_0", "NVFP4", "BF16", "F16", "F32"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--weights-m", type=int, default=1024, help="millions of weights per file (bf16 output = 2x that in MB)")
    ap.add_argument("--types", default=",".join(ALL))
    ap.add_argument("--passes", type=int, default=10)
    args = ap.parse_args()
    peak = None
    pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peak = json.load(open(pk)).get("hbm_gbs")
    # static prediction (tools/sass_budget.py --json, when written next to this tool): hot-path instructions -> issue ceiling per op
    pred = {}
    pj = os.path.join(ROOT, "tools", "sass_budget.json")
    if os.path.exists(pj):
        pred = json.load(open(pj)).get("ops", {})
    opname = lambda dt: "KK_OP_" + dt.replace("_K", "K").replace("IQ4_NL", "IQ4NL").replace("IQ4_XS", "IQ4XS").replace("IQ2_XXS", "IQ2XXS").replace("IQ2_XS", "IQ2XS") \
        .replace("IQ2_S", "IQ2S").replace("IQ3_XXS", "IQ3XXS").replace("IQ3_S", "IQ3S").replace("IQ1_S", "IQ1S").replace("IQ1_M", "IQ1M") + "_BF16"  # noqa: E731
    rows = (args.weights_m << 20) // 8192 // 4 * 4
    out = {"weights": rows * 8192, "peak_GBps": peak, "types": {}}
    pool = gpupool.Pool([0])
    try:
        out["write_peak_GBps"] = max(pool.probe_hbm(0, gpupool.PROBE_WRITE, 4 << 30) for _ in range(3))
    except Exception as e:  # noqa: BLE001
        out["write_peak_GBps"] = f"error: {e}"
    with tempfile.TemporaryDirectory(dir="/dev/shm" if os.path.isdir("/dev/shm") else None) as d:
        for dt in args.types.split(","):
            p = os.path.join(d, f"{dt}.gguf")
            try:
                t0 = time.time()
                synth.write_gguf(p, [(f"blk.{i}.ffn_up.weight", dt, [rows // 4, 8192]) for i in range(4)], 40)
                m = pool.load(p, flags=gpupool.LOAD_DEFER)
                try:
                    m.stage_resident()
                    for _ in range(3):
                        m.convert_resident()
                    ms = sorted(m.convert_resident()[0] for _ in range(args.passes))
                    st = m.stats()["parts"][0]
                    alg = st["src_bytes"] + st["out_bytes"]
                    med = ms[len(ms) // 2]
                    row = {"ms_median": med, "ms_min": ms[0], "src_bytes": st["src_bytes"], "out_bytes": st["out_bytes"], "GBps": alg / (med / 1e3) / 1e9,
                           "write_GBps": st["out_bytes"] / (med / 1e3) / 1e9, "setup_s": time.time() - t0}
                    if peak:
                        row["frac_of_copy_peak"] = row["GBps"] / peak
                    pr = pred.get(opname(dt))
                    if pr:  # fraction of the issue slots the measured rate would need if only the hot path issued
                        row["predicted_issue_ceiling_GBps"] = pr["issue_ceiling_GBps"]
                        row["issue_fraction_at_measured_rate"] = row["GBps"] / pr["issue_ceiling_GBps"]
                    out["types"][dt] = row
                    print(dt, json.dumps(row), flush=True)
                finally:
                    m.release()
            except Exception as e:  # noqa: BLE001
                out["types"][dt] = {"error": str(e)}
                print(dt, "ERROR", e, flush=True)
            finally:
                if os.path.exists(p):
                    os.remove(p)
            os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
            json.dump(out, open(os.path.join(ROOT, "gpurun_out", os.environ.get("KK_QUICK_OUT", "types_roofline.json")), "w"), indent=1)
    pool.close()


if __name__ == "__main__":
    main()
