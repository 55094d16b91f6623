"""Static instruction budget of kk_convert_kernel's consumer loops, read from the SASS (no GPU needed).

For every `case KK_OP_*:` of the consumer dispatch (kk_consume_tile in csrc/kk_consume_tile.cuh) this attributes the kernel's SASS
instructions to the op whose dispatch line they were inlined at (`nvdisasm -gi`, built with -lineinfo), finds the op's loops from the backward branches, and reports for
the op's main loop: warp instructions per iteration, the opcode mix, and — with the bytes one warp iteration reads and writes — warp
instructions per KiB of algorithmic HBM traffic.  Put against the issue rate of the machine (4 schedulers x 1 warp instruction per clock per
SM) this gives the traffic rate at which the loop would saturate instruction issue: a loop whose ceiling is below the HBM roofline is
issue-bound however well the memory side is arranged.

A static count is an upper estimate of what issues (predicated-off instructions count; code behind a forward branch that is not taken
counts) and knows nothing about stalls; it ranks the loops and says where the PRMT/FADD rewrites landed, it is not a measurement.

    python tools/sass_budget.py [--kernel kk_convert_f16_kernel] [--md sass_budget.md] [--json sass_budget.json]

--kernel names the kernel (a substring of its symbol): kk_convert_kernel, the bf16 kernel, by default; kk_convert_f16_kernel is the same
source instantiated for fp16 output (KK_LOAD_F16 models).
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kukeon_b200", "csrc")
KERNEL_CU = os.path.join(CSRC, "kk_kernels.cu")
DISPATCH = os.path.join(CSRC, "kk_consume_tile.cuh")

SM_COUNT, SM_GHZ, ISSUE_PER_CLK = 132, 1.98, 4  # H100 SXM: 132 SMs, 1980 MHz sampled during bench.py's timed steps (700 W limit), 4 warp schedulers per SM
HBM_PEAK_GBS = 3350.0                           # H100 SXM data sheet (HBM3); the store-only probe measured 3,165 GB/s on the same card

# bytes one WARP iteration of the op's main loop reads from the stage and writes to one pool: (in, out).  From the lane mappings in
# kk_consume_core.cuh / kk_dequant.cuh: the 256-weight types take one block per warp iteration, the 32-weight types eight, Q4_K four
# super-blocks; the per-thread loops (copy, casts) move one 16-byte output vector (fp8: two) per thread.  The block dequantisers other than
# Q4_K are unrolled twice (`#pragma unroll 2`: two independent load -> expand -> store chains per iteration), see UNROLL2 below.
_ITER_BYTES_1X = {
    "KK_OP_COPY": (512, 512), "KK_OP_F32_BF16": (1024, 512), "KK_OP_F16_BF16": (512, 512),
    "KK_OP_F8E4M3_BF16": (512, 1024), "KK_OP_F8E5M2_BF16": (512, 1024),
    "KK_OP_Q4K_BF16": (4 * 144, 2048), "KK_OP_Q6K_BF16": (210, 512), "KK_OP_Q8_0_BF16": (8 * 34, 512),
    "KK_OP_Q4_0_BF16": (8 * 18, 512), "KK_OP_Q4_1_BF16": (8 * 20, 512), "KK_OP_Q5_0_BF16": (8 * 22, 512), "KK_OP_Q5_1_BF16": (8 * 24, 512),
    "KK_OP_Q2K_BF16": (84, 512), "KK_OP_Q3K_BF16": (110, 512), "KK_OP_Q5K_BF16": (4 * 176, 2048),
    "KK_OP_IQ4NL_BF16": (8 * 18, 512), "KK_OP_MXFP4_BF16": (8 * 17, 512), "KK_OP_IQ4XS_BF16": (136, 512),
    "KK_OP_IQ2XXS_BF16": (66, 512), "KK_OP_IQ2XS_BF16": (74, 512), "KK_OP_IQ2S_BF16": (82, 512), "KK_OP_IQ3XXS_BF16": (98, 512),
    "KK_OP_IQ3S_BF16": (110, 512), "KK_OP_IQ1S_BF16": (50, 512), "KK_OP_IQ1M_BF16": (56, 512),
    # transposes: a warp iteration turns 256 elements (32 columns x 8 rows) into 32 16-byte stores (64 for the 4-byte verbatim form)
    "KK_OP_T_F32_BF16": (1024, 512), "KK_OP_T_F16_BF16": (512, 512), "KK_OP_T_B16": (512, 512), "KK_OP_T_B32": (1024, 1024),
    "KK_OP_TQ1_0_BF16": (54, 512), "KK_OP_TQ2_0_BF16": (66, 512), "KK_OP_NVFP4_BF16": (4 * 36, 512),
}

ITER_BYTES = {op: ((2 * v[0], 2 * v[1]) if op.startswith(("KK_OP_Q", "KK_OP_IQ", "KK_OP_TQ", "KK_OP_MXFP4", "KK_OP_NVFP4")) and op not in ("KK_OP_Q4K_BF16", "KK_OP_Q5K_BF16") else v)
              for op, v in _ITER_BYTES_1X.items()}

CLASSES = [("lds", r"^LDS"), ("ldg", r"^LDG"), ("stg", r"^STG"), ("prmt", r"^PRMT"), ("fadd/fmul", r"^(FADD|FMUL|FFMA)"), ("f2fp/cvt", r"^(F2FP|F2F|I2F|HADD2|HMUL2|HFMA2)"),
           ("lop/shf", r"^(LOP3|SHF|SHL|SHR|BFE|BFI|SGXT|POPC|LEA)"), ("imad/iadd", r"^(IMAD|IADD|VIADD|IABS|ISETP|IMNMX|VIMNMX|SEL|MOV|FSEL|PLOP3|FSETP)"),
           ("shfl", r"^SHFL"), ("branch/sync", r"^(BRA|BSSY|BSYNC|WARPSYNC|NANOSLEEP|SYNCS|BAR|EXIT|CALL|RET|BREAK|YIELD|NOP)")]


def fresh_object():
    """csrc/build/kk_kernels.o when the Makefile's last build is newer than every source it depends on (same flags: -O3 -lineinfo)."""
    obj = os.path.join(CSRC, "build", "kk_kernels.o")
    if not os.path.exists(obj):
        return None
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))]
    return obj if all(os.path.getmtime(x) <= os.path.getmtime(obj) for x in deps) else None


def disassemble(obj=None, resources=False):
    """nvdisasm -gi text of the kernels' object; with resources=True also {symbol: {"REG": n, "STACK": n, "LOCAL": n, ...}} from
    cuobjdump -res-usage of the same object."""
    with tempfile.TemporaryDirectory() as d:
        obj = obj or fresh_object()
        if obj is None:
            obj = os.path.join(d, "k.o")
            subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-I" + os.path.join(ROOT, "include"),
                                   "-c", KERNEL_CU, "-o", obj], cwd=CSRC, stderr=subprocess.DEVNULL)
        subprocess.check_call(["cuobjdump", "-xelf", "all", obj], cwd=d, stdout=subprocess.DEVNULL)
        cubin = [f for f in os.listdir(d) if f.endswith(".cubin")][0]
        text = subprocess.check_output(["nvdisasm", "-gi", "-c", os.path.join(d, cubin)], text=True)
        if not resources:
            return text
        res, fn = {}, None
        for l in subprocess.check_output(["cuobjdump", "-res-usage", obj], text=True).split("\n"):
            m = re.match(r"\s*Function (\S+):", l)
            if m:
                fn = m.group(1)
            elif fn and "REG:" in l:
                res[fn] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", l)}
                fn = None
        return text, res


def parse(text, kernel="kk_convert_kernel"):
    """-> list of dicts for the instructions of `kernel` (a substring of its symbol): idx, op (mnemonic), chain (the inline frames (file,
    line, inlined-at file, inlined-at line), innermost first), label index map."""
    lines = text.split("\n")
    start = next(i for i, l in enumerate(lines) if l.startswith(".text.") and kernel in l)
    ins, labels = [], {}
    chain, fresh = [], True
    ann = re.compile(r'//## File "([^"]+)", line (\d+)(?: inlined at "([^"]+)", line (\d+))?')
    for l in lines[start + 1:]:
        s = l.strip()
        if s.startswith(".text.") or s.startswith("//-----"):
            if ins:
                break
            continue
        m = ann.search(s)
        if m:
            if fresh:
                chain, fresh = [], False
            chain.append((m.group(1), int(m.group(2)), m.group(3), int(m.group(4)) if m.group(4) else None))
            continue
        if re.match(r"^\.L_x_\d+:", s):
            labels[s[:-1]] = len(ins)
            continue
        m = re.match(r"/\*([0-9a-f]+)\*/\s+(@!?U?P\d+\s+)?([A-Z0-9_.]+)\s*(.*);", s)
        if m:
            fresh = True
            ins.append({"i": len(ins), "pred": (m.group(2) or "").strip(), "mn": m.group(3), "args": m.group(4), "chain": chain})
    return ins, labels


def dispatch_lines():
    out = {}
    for n, l in enumerate(open(DISPATCH), 1):
        m = re.match(r"\s*case (KK_OP_\w+):", l)
        if m:
            out[n] = m.group(1)
    return out


def dispatch_op(chain, disp):
    """The op whose `case` line the instruction was inlined at: the frame inlined at a dispatch line, or code on that line itself."""
    for f, ln, f2, ln2 in reversed(chain):
        for ff, ll in ((f2, ln2), (f, ln)):
            if ff and ff.endswith(os.path.basename(DISPATCH)) and ll in disp:
                return disp[ll]
    return None


def loops_of(ins, labels):
    res = []
    for x in ins:
        if x["mn"].startswith("BRA"):
            m = re.search(r"`\((\.L_x_\d+)\)", x["args"])
            if m and m.group(1) in labels and labels[m.group(1)] <= x["i"]:
                res.append((labels[m.group(1)], x["i"]))
    return res


def successors(ins, labels, i, b):
    x = ins[i]
    succ = []
    is_bra = x["mn"].startswith("BRA")
    if is_bra and not x["mn"].startswith("BRA.DIV"):  # BRA.DIV: taken only when the warp has diverged (out-of-line handler)
        m = re.search(r"`\((\.L_x_\d+)\)", x["args"])
        tgt = labels.get(m.group(1)) if m else None
        if tgt is not None and i < tgt <= b:
            succ.append(tgt)
    conditional = bool(x["pred"]) or x["mn"].startswith("BRA.DIV")
    if conditional or not (is_bra or x["mn"] in ("EXIT", "RET")):
        succ.append(i + 1)
    return succ


def hot_path(ins, labels, a, b, mode="math"):
    """Instructions on the cheapest path from the loop head a to its back edge b that still performs the iteration's full work.

    The loop body without its backward branches is a DAG (edges: fall-through, forward branches inside the loop).  Predicated non-branch
    instructions count: they issue.
    mode "math": paths that skip the work (out-of-range lanes, ragged-tail variants) carry fewer conversion instructions, so the hot path is
    the one that maximises the count of F2FP (the bf16 packs: one per two outputs, the same in every arithmetic variant) and, among those,
    minimises the total — i.e. one destination pool (the n_dst > 1 ladder is a longer alternative), the cheapest of the alignment variants of
    the loads, and for Q4_K / Q5_K the FMA form that every quad with finite non-negative scales takes (the two-step form is the longer one).
    mode "vec" (the transposes, whose ragged path converts element by element and so carries MORE arithmetic than the vector path): the
    cheapest path that performs a 128-bit store."""
    if mode == "math":
        math = re.compile(r"^F2FP")
        best = {}
        for i in range(b, a - 1, -1):
            own = (1 if math.match(ins[i]["mn"]) else 0, -1)
            if i == b:
                best[i] = own
                continue
            opts = [best[j] for j in successors(ins, labels, i, b) if best.get(j) is not None]
            best[i] = (own[0] + max(opts)[0], own[1] + max(opts)[1]) if opts else None
        r = best.get(a)
        return (-r[1], r[0]) if r else (None, None)
    vec = re.compile(r"^STG\.E(\.NA)?\.128")
    inf = float("inf")
    f = {}  # f[i][seen] = fewest instructions from i to the back edge such that a 128-bit store lies on the whole path
    for i in range(b, a - 1, -1):
        here = bool(vec.match(ins[i]["mn"]))
        if i == b:
            f[i] = [1 if here else inf, 1]
            continue
        succ = [j for j in successors(ins, labels, i, b) if j in f]
        f[i] = [1 + min([f[j][1 if (s or here) else 0] for j in succ], default=inf) for s in (0, 1)]
    r = f.get(a, [inf])[0]
    return (int(r), 1) if r != inf else (None, None)


def classify(mn):
    base = mn.split(".")[0]
    for name, rx in CLASSES:
        if re.match(rx, base):
            return name
    return "other"


def analyse(kernel="kk_convert_kernel", text=None):
    """Per-op rows, total instructions and opcode counts of `kernel`; text: nvdisasm output to read (default: disassemble())."""
    ins, labels = parse(text if text is not None else disassemble(), kernel)
    disp = dispatch_lines()
    owner = [dispatch_op(x["chain"], disp) for x in ins]
    loops = loops_of(ins, labels)
    rows = []
    for op in dict.fromkeys(disp.values()):
        mine = [i for i, o in enumerate(owner) if o == op]
        if not mine:
            continue
        cand = []
        for a, b in loops:
            n = b - a + 1
            own = sum(1 for i in range(a, b + 1) if owner[i] == op)
            if own >= 0.5 * n:
                cand.append((n, a, b))
        if not cand:
            rows.append({"op": op, "static": len(mine), "loop": None})
            continue
        # main loop: the largest one that is not itself nested in a bigger candidate of the same op would double count the inner tail loops; the
        # consumers are one grid-stride loop each, so "largest" is that loop
        n, a, b = max(cand)
        mix = collections.Counter(classify(ins[i]["mn"]) for i in range(a, b + 1))
        inner = [(n2, a2, b2) for n2, a2, b2 in cand if a2 >= a and b2 <= b and (a2, b2) != (a, b)]
        hot, hot_math = hot_path(ins, labels, a, b, "vec" if op.startswith("KK_OP_T_") else "math")
        rows.append({"op": op, "static": len(mine), "loop": n, "hot": hot, "hot_math": hot_math, "mix": mix, "inner_loops": sorted(n2 for n2, _, _ in inner), "n_loops": len(cand)})
    return rows, len(ins), collections.Counter(x["mn"].split(".")[0] for x in ins)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kernel", default="kk_convert_kernel", help="substring of the kernel's symbol (kk_convert_f16_kernel: the fp16-output kernel)")
    ap.add_argument("--md")
    ap.add_argument("--json", help="write {op: {hot, bytes_in, bytes_out, issue_ceiling_GBps}} (read by tools/gpu_quick_types.py to print prediction next to measurement)")
    args = ap.parse_args()
    rows, total, _ = analyse(args.kernel)
    issue_rate = SM_COUNT * SM_GHZ * ISSUE_PER_CLK  # G warp instructions / s
    names = [c for c, _ in CLASSES] + ["other"]
    out = []
    out.append(f"{args.kernel}: {total} SASS instructions; issue rate {issue_rate:.0f} G warp-instr/s ({SM_COUNT} SMs x {SM_GHZ} GHz x {ISSUE_PER_CLK}/clk); "
               f"HBM copy peak {HBM_PEAK_GBS:.0f} GB/s\n")
    hdr = ["op", "SASS instr (whole op)", "main loop (static)", "hot path instr / warp iteration", "bytes in + out / iteration", "hot instr / KiB of traffic",
           "issue ceiling GB/s", "ceiling / HBM peak"] + names
    out.append("| " + " | ".join(hdr) + " |")
    out.append("|" + "---|" * len(hdr))
    for r in rows:
        if r["loop"] is None:
            out.append(f"| {r['op']} | {r['static']} | (no loop attributed) |" + " |" * (len(hdr) - 3))
            continue
        ib = ITER_BYTES.get(r["op"])
        hot = r.get("hot")
        if ib and hot:
            traffic = ib[0] + ib[1]
            per_kib = hot / traffic * 1024
            ceil = issue_rate / hot * traffic  # G instr/s / (instr/iter) * bytes/iter = GB/s
            cols = [str(hot), f"{ib[0]} + {ib[1]}", f"{per_kib:.0f}", f"{ceil:.0f}", f"{ceil / HBM_PEAK_GBS:.2f}"]
        else:
            cols = [str(hot or ""), "", "", "", ""]
        mix = [str(r["mix"].get(n, 0)) for n in names]
        extra = f" (+{len(r['inner_loops'])} inner: {r['inner_loops']})" if r["inner_loops"] else ""
        out.append(f"| {r['op']} | {r['static']} | {r['loop']}{extra} | " + " | ".join(cols + mix) + " |")
    if args.json:
        import json
        js = {}
        for r in rows:
            ib = ITER_BYTES.get(r["op"])
            if ib and r.get("hot"):
                js[r["op"]] = {"hot": r["hot"], "bytes_in": ib[0], "bytes_out": ib[1], "issue_ceiling_GBps": issue_rate / r["hot"] * (ib[0] + ib[1])}
        with open(args.json, "w") as f:
            json.dump({"issue_rate_Ginstr_s": issue_rate, "hbm_peak_GBps": HBM_PEAK_GBS, "ops": js}, f, indent=1)
    text = "\n".join(out) + "\n"
    sys.stdout.write(text)
    if args.md:
        with open(args.md, "w") as f:
            f.write("# Static SASS budget of the consumer loops (tools/sass_budget.py — an analysis of the compiled code, NOT a measurement)\n\n" + text)


if __name__ == "__main__":
    main()
