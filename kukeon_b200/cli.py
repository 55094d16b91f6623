"""`kuke model …` — Python model of the CLI verbs row f3 of SURVEY.md §8(f) proposes, patterned on `kuke image` (cmd/kuke/image/*.go):

    python -m kukeon_b200.cli model pull <path> [-o table|yaml|json]          index a local checkpoint ("pull" is local-path only)
    python -m kukeon_b200.cli model plan <path> [--mode M] [--gpus N] [--layers B:E] [--adapter DIR] [-o …]
                                                                              dry-run: pool layout and bytes per GPU, no device touched;
                                                                              --layers: only the pipeline stage of layers [B, E)
    python -m kukeon_b200.cli model validate <cell.yaml>                      check the `models:` entries of a Cell manifest

Like `kuke image`, these verbs run in-process (pkg/api/kukeonv1/client.go:93-98): they need no daemon and no GPU — `pull` is
`kk_index`, `plan` is `kk_plan_describe`.  The verbs that act on *resident* pools (`load`, `get`/`ls`, `rm`) belong to kukeond, whose
lifetime the pools share (internal/daemon/server.go:87,242); they are named here and refuse with that explanation.
Output conventions follow cmd/kuke/get/shared: table for lists by default, yaml/json on request, sizes like `formatSize`.
"""
from __future__ import annotations

import argparse
import json
import sys
from typing import List, Sequence

from . import gpupool, schema

MODES = {"single": gpupool.MODE_SINGLE, "broadcast": gpupool.MODE_BROADCAST, "scatter": gpupool.MODE_SCATTER}


def format_size(n: int) -> str:
    """cmd/kuke/image/get.go formatSize: 1024-based, one decimal, "-" for unknown."""
    if n < 0:
        return "-"
    if n < 1024:
        return f"{n} B"
    div, exp = 1024, 0
    m = n // 1024
    while m >= 1024:
        div *= 1024
        exp += 1
        m //= 1024
    return f"{n / div:.1f} {'KMGTPE'[exp]}iB"


def print_table(headers: Sequence[str], rows: List[Sequence[str]], out) -> None:
    widths = [max(len(str(h)), *(len(str(r[i])) for r in rows)) if rows else len(str(h)) for i, h in enumerate(headers)]
    for line in [headers] + rows:
        out.write("  ".join(str(c).ljust(w) for c, w in zip(line, widths)).rstrip() + "\n")


def emit(obj, fmt: str, out) -> None:
    if fmt == "json":
        out.write(json.dumps(obj, indent=2) + "\n")
    else:
        import yaml
        out.write(yaml.safe_dump(obj, sort_keys=False))


def parse_output(fmt: str) -> str:
    f = (fmt or "").strip().lower()
    if f not in ("", "yaml", "json", "table"):
        raise SystemExit(f"invalid output format: {fmt} (supported: yaml, json, table)")
    return f or "table"


def parse_layers(s: str) -> List[int]:
    """--layers B:E -> [B, E]; the library checks the range against the checkpoint."""
    b, sep, e = s.partition(":")
    if not (sep and b.isdigit() and e.isdigit() and int(b) < int(e)):
        raise argparse.ArgumentTypeError(f"invalid layer range {s!r}: expected B:E with integers 0 <= B < E")
    return [int(b), int(e)]


def cmd_pull(args, out) -> int:
    recs = gpupool.index(args.path)
    shards = gpupool.index_shards(args.path)
    fmt = parse_output(args.output)
    if fmt != "table":
        emit({"path": args.path, "shards": shards, "tensors": recs}, fmt, out)
        return 0
    if not recs:
        out.write(f"No tensors found in {args.path!r}.\n")
        return 0
    rows = [[r["name"], r["dtype"], "x".join(map(str, r["shape"])) or "scalar", str(r["shard"]), format_size(r["nbytes"])] for r in recs]
    print_table(["NAME", "DTYPE", "SHAPE", "SHARD", "SIZE"], rows, out)
    out.write(f"{len(recs)} tensors, {len(shards)} shard(s), {format_size(sum(r['nbytes'] for r in recs))}\n")
    return 0


def cmd_plan(args, out) -> int:
    flags = sum(schema.OPTION_FLAGS[o] for o in args.option or [])
    n = 1 if args.mode == "single" else args.gpus
    plan = gpupool.plan_describe(args.path, mode=MODES[args.mode], flags=flags, n_parts=n, layers=args.layers)
    summary = {"path": args.path, "mode": args.mode, "gpus": n, "fileBytes": plan["file_bytes"],
               "poolBytesPerGpu": [lay["pool_bytes"] for lay in plan["layouts"]] if args.mode == "scatter" else [plan["layouts"][0]["pool_bytes"]] * n,
               "ingestBytesPerGpu": [p["src_bytes"] for p in plan["parts"]],
               "tensors": len(plan["layouts"][0]["tensors"])}
    if args.layers:
        summary["layers"], summary["nLayers"] = plan["layers"], plan["n_layers"]
    adapter = None
    if args.adapter:
        # one process over n GPUs: a scatter pool is planned as n parts, a broadcast pool like a single one
        adapter = gpupool.adapter_describe(args.path, args.adapter, mode=MODES[args.mode], flags=flags, part_count=n if args.mode == "scatter" else 0,
                                           layers=args.layers)
        summary["adapter"] = {"path": adapter["adapter"], "targets": [{"name": t["name"], "shape": t["shape"], "r": t["r"], "scaling": t["scaling"]}
                                                                       for t in adapter["targets"]], "skipped": adapter["skipped"]}
    fmt = parse_output(args.output)
    if fmt != "table":
        emit(summary if not args.full else (plan if adapter is None else dict(plan, adapter=adapter)), fmt, out)
        return 0
    rows = [[str(g), format_size(summary["ingestBytesPerGpu"][g]), format_size(summary["poolBytesPerGpu"][g])] for g in range(n)]
    print_table(["GPU", "INGESTS", "POOL"], rows, out)
    stage = f", layers {plan['layers'][0]}-{plan['layers'][1] - 1} of {plan['n_layers']}" if args.layers else ""
    out.write(f"{summary['tensors']} tensors, {format_size(plan['file_bytes'])} in the files, mode {args.mode}{stage}\n")
    if adapter is not None:
        print_table(["TARGET", "SHAPE", "R", "SCALING"], [[t["name"], "x".join(map(str, t["shape"])), str(t["r"]), f"{t['scaling']:.9g}"]
                                                         for t in adapter["targets"]], out)
        skipped = f", {len(adapter['skipped'])} outside the stage" if adapter["skipped"] else ""
        out.write(f"adapter {adapter['adapter']}: {len(adapter['targets'])} tensors merged{skipped}\n")
    return 0


def cmd_validate(args, out) -> int:
    import yaml
    with open(args.manifest, "rb") as f:
        docs = [d for d in yaml.safe_load_all(f) if d]
    n = 0
    for doc in docs:
        if doc.get("kind") != "Cell":
            continue
        for cid, specs in schema.models_of_cell(doc).items():
            for s in specs:
                recs = gpupool.index(s.source)
                out.write(f"cell {doc.get('metadata', {}).get('name', '?')} container {cid}: model {s.name}: {len(recs)} tensors, "
                          f"{format_size(sum(r['nbytes'] for r in recs))}, mode {[k for k, v in MODES.items() if v == s.mode][0]}\n")
                n += 1
    out.write(f"{n} model(s) valid\n")
    return 0


def cmd_needs_daemon(args, out) -> int:
    sys.stderr.write(f"kuke model {args.verb}: resident pools live in kukeond (their lifetime is the daemon's: internal/daemon/server.go:87,242); "
                     f"this verb is served over its RPC, not in-process.  In-process verbs: pull, plan, validate.\n")
    return 2


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="kuke")
    sub = ap.add_subparsers(dest="noun", required=True)
    model = sub.add_parser("model", help="GPU-resident model weights").add_subparsers(dest="verb", required=True)
    p = model.add_parser("pull", help="Index a local checkpoint (safetensors / GGUF); no device is touched")
    p.add_argument("path")
    p.add_argument("-o", "--output", default="")
    p.set_defaults(fn=cmd_pull)
    p = model.add_parser("plan", help="Dry-run a load: pool layout and bytes per GPU")
    p.add_argument("path")
    p.add_argument("--mode", choices=sorted(MODES), default="single")
    p.add_argument("--gpus", type=int, default=1)
    p.add_argument("--option", action="append", choices=sorted(schema.OPTION_FLAGS))
    p.add_argument("--layers", type=parse_layers, metavar="B:E", help="pipeline stage: plan only layers [B, E) (half-open)")
    p.add_argument("--adapter", metavar="DIR", help="PEFT LoRA adapter (directory or adapter_model.safetensors): list the tensors its merge targets")
    p.add_argument("--full", action="store_true", help="yaml/json: the whole plan (chunks, reads, segments) instead of the summary")
    p.add_argument("-o", "--output", default="")
    p.set_defaults(fn=cmd_plan)
    p = model.add_parser("validate", help="Validate the models: entries of a Cell manifest")
    p.add_argument("manifest")
    p.set_defaults(fn=cmd_validate)
    for verb in ("load", "get", "ls", "rm"):
        p = model.add_parser(verb, help="(served by kukeond)")
        p.add_argument("rest", nargs="*")
        p.set_defaults(fn=cmd_needs_daemon)
    return ap


def main(argv=None, out=None) -> int:
    args = build_parser().parse_args(argv)
    out = out or sys.stdout
    try:
        return args.fn(args, out)
    except gpupool.GPUPoolError as e:
        sys.stderr.write(f"Error: {e}\n")
        return 1
    except schema.SchemaError as e:
        sys.stderr.write(f"Error: {e}\n")
        return 1


if __name__ == "__main__":
    sys.exit(main())
