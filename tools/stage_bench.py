"""Two pipeline stages of the full 32-layer Mixtral-8x7B q4_K GGUF on one GPU, one after the other.

In bf16 the whole model is 93.4 GB, more than one H100's 80 GB, so it cannot load in one piece; as two stages, layers [0, 16) and
[16, 32), each fits.  This writes the real 32-layer file (synth.mixtral_gguf_tensors, seeded: 26.3 GB of blocks, on tmpfs when there is
room), loads stage 0, releases it and loads stage 1, and reports per stage:

  * the pool bytes and the file bytes the stage reads;
  * the kk_load_part wall time of a deferred load (the streaming load from the warm file);
  * the kernel stage from the HBM-resident image (kk_stage_resident / kk_convert_resident): >= 3 warm-ups, then --steps timed passes, GB/s of
    algorithmic bytes (source read once + pool bytes written, DESIGN.md §6) and of pool bytes made resident.

It records the card's name and power limit (nvidia-smi query) and, unless --no-bench, runs `bench.py --workload mixtral-q4k --gpus 1
--kernel-only` in the same call, whose synthetic 16-layer file is the comparison.  --layers / --hidden / --ffn / --vocab shrink the model
so the script can be rehearsed on a machine without a GPU: it runs up to the first device call, having written the file and planned both
stages.

    python tools/stage_bench.py [--steps 5] [--warmup 3] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from kukeon_b200 import gpupool  # noqa: E402
from tools import synth  # noqa: E402


def card(device: int) -> dict:
    """Name and power limit of CUDA device `device` of this process, queried by its UUID: nvidia-smi's own index order need not be
    CUDA's (CUDA_VISIBLE_DEVICES, CUDA_DEVICE_ORDER)."""
    try:
        uuid = gpupool.device_identity(device)["uuid"]
        out = subprocess.run(["nvidia-smi", "-i", uuid, "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60, check=True).stdout.splitlines()[0]
        name, limit = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": limit, "uuid": uuid}
    except (gpupool.GPUPoolError, OSError, subprocess.SubprocessError, IndexError, ValueError) as e:
        return {"name": None, "power_limit": None, "error": str(e)}


def data_dir(need: int, override: str) -> str:
    """A new directory of this run's own (under --data-dir when given), so that removing it afterwards removes only what this run wrote."""
    for base in ([override] if override else ["/dev/shm", tempfile.gettempdir()]):
        try:
            st = os.statvfs(base)
            if override or st.f_bavail * st.f_frsize > need * 1.1 + (2 << 30):
                return tempfile.mkdtemp(prefix="kk_stage_bench_", dir=base)
        except OSError:
            if override:
                raise
    raise SystemExit(f"no directory with {need / 1e9:.1f} GB free for the checkpoint")


def measure_stage(pool, path: str, layers, steps: int, warmup: int) -> dict:
    m = pool.load(path, flags=gpupool.LOAD_DEFER, layers=layers)
    try:
        t0 = time.perf_counter()
        m.load_part()  # returns once the pool holds the stage (the load synchronises its streams)
        wall = time.perf_counter() - t0
        st = m.stats()
        m.stage_resident()
        for _ in range(warmup):
            m.convert_resident()
        runs = [m.convert_resident() for _ in range(steps)]
        part = st["parts"][0]
        info = m.info()
    finally:
        m.release()
    ms = sum(t for t, _ in runs) / steps
    alg = part["src_bytes"] + part["out_bytes"]
    return {"layers": list(layers), "n_tensors": info["n_tensors"], "pool_bytes": info["pool_bytes"], "file_bytes_read": st["local_src_bytes"],
            "load_part_wall_s": wall, "load_s": st["load_s"], "load_GBps": st["local_src_bytes"] / wall / 1e9,
            "kernel_stage": {"steps": steps, "warmup": warmup, "ms_per_step": ms, "ms_min": min(t for t, _ in runs), "ms_max": max(t for t, _ in runs),
                             "launches_per_step": len(runs[0][1]), "algorithmic_bytes": alg, "algorithmic_GBps": alg / (ms / 1e3) / 1e9,
                             "pool_GBps": part["out_bytes"] / (ms / 1e3) / 1e9}}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--hidden", type=int, default=4096)
    ap.add_argument("--ffn", type=int, default=14336)
    ap.add_argument("--vocab", type=int, default=32000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--data-dir", default="", help="parent of the run's own temporary directory (default: /dev/shm when it has room)")
    ap.add_argument("--out", default="", help="also write the JSON result here")
    ap.add_argument("--no-bench", action="store_true", help="skip the bench.py comparison run")
    ap.add_argument("--keep-data", action="store_true")
    args = ap.parse_args(argv)
    if args.steps < 5 or args.warmup < 3:
        raise SystemExit("--steps >= 5 and --warmup >= 3")
    if args.layers < 2 or args.layers % 2:
        raise SystemExit("--layers must be even (two equal stages)")
    tensors = synth.mixtral_gguf_tensors(hidden=args.hidden, ffn=args.ffn, layers=args.layers, vocab=args.vocab)
    need = synth.total_bytes(tensors)
    d = data_dir(need, args.data_dir)
    path = os.path.join(d, "model.gguf")
    res = {"workload": f"Mixtral-8x7B GGUF q4_K -> bf16, {args.layers} layers (hidden {args.hidden}), two pipeline stages on one GPU in turn",
           "file": path, "file_bytes": need}
    try:
        t0 = time.time()
        synth.write_gguf(path, tensors, 8007)
        res["synth_s"] = time.time() - t0
        half = args.layers // 2
        stages = [(0, half), (half, args.layers)]
        whole = gpupool.plan_describe(path)
        res["whole_pool_bytes"] = whole["layouts"][0]["pool_bytes"]
        res["planned"] = [{"layers": list(s), "pool_bytes": p["layouts"][0]["pool_bytes"], "file_bytes": p["file_bytes"]}
                          for s, p in ((s, gpupool.plan_describe(path, layers=s)) for s in stages)]
        print(json.dumps({"planned": res["planned"], "whole_pool_bytes": res["whole_pool_bytes"]}), flush=True)
        with gpupool.Pool([0]) as pool:  # first device call
            res["card"] = card(0)
            res["stages"] = [measure_stage(pool, path, s, args.steps, args.warmup) for s in stages]
    finally:
        if not args.keep_data:
            shutil.rmtree(d)  # the directory data_dir created for this run, nothing else
    if not args.no_bench:
        cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--workload", "mixtral-q4k", "--gpus", "1", "--kernel-only",
               "--steps", str(args.steps), "--warmup", str(args.warmup)]
        out = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
        lines = [ln for ln in out.stdout.splitlines() if ln.startswith("{")]
        res["bench_16_layer_synthetic"] = json.loads(lines[-1]) if out.returncode == 0 and lines else {"returncode": out.returncode,
                                                                                                        "stderr_tail": out.stderr[-2000:]}
    text = json.dumps(res)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
