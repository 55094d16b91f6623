"""The compiled kernel itself, checked on the CPU tier: tools/sass_budget.py reads kk_convert_kernel's SASS (nvdisasm, no GPU) and this
pins what the round's tuning relied on — the instruction mix that proves the design (TMA bulk copies in and out, no tensor-core or
local-memory instructions, no spills) and an upper bound on every dequantiser's hot path, so that a change to the shared helpers
(byte_to_float, lds64_funnel, lut16x8, store16_all) that makes a loop heavier fails here, not in next round's profile."""
import shutil

import pytest

from tools import sass_budget

pytestmark = pytest.mark.skipif(shutil.which("nvcc") is None or shutil.which("nvdisasm") is None, reason="needs the CUDA toolkit (nvcc, nvdisasm)")

# hot-path warp instructions per ONE-block-group of work (one destination pool, aligned loads) of the loops before they were unrolled, + ~5 %; the
# loops are unrolled twice now (two independent chains per iteration), which tools/sass_budget.py folds into its bytes-per-iteration table —
# so the comparison is made per KiB of algorithmic traffic, the quantity the issue ceiling is computed from
# Q4_K / Q5_K: per four-block quad on the FMA form
HOT_MAX = {
    "KK_OP_COPY": 42, "KK_OP_F32_BF16": 84, "KK_OP_F16_BF16": 60, "KK_OP_F8E4M3_BF16": 53, "KK_OP_F8E5M2_BF16": 53,
    "KK_OP_Q4K_BF16": 250, "KK_OP_Q8_0_BF16": 67, "KK_OP_Q6K_BF16": 88, "KK_OP_Q4_0_BF16": 68, "KK_OP_Q4_1_BF16": 80, "KK_OP_Q5_0_BF16": 85,
    "KK_OP_Q5_1_BF16": 95, "KK_OP_Q2K_BF16": 84, "KK_OP_Q3K_BF16": 101, "KK_OP_Q5K_BF16": 288, "KK_OP_IQ4NL_BF16": 92, "KK_OP_IQ4XS_BF16": 99,
    "KK_OP_MXFP4_BF16": 92, "KK_OP_NVFP4_BF16": 99, "KK_OP_IQ2XXS_BF16": 88, "KK_OP_IQ2XS_BF16": 89, "KK_OP_IQ2S_BF16": 82,
    "KK_OP_IQ3XXS_BF16": 90, "KK_OP_IQ3S_BF16": 92, "KK_OP_IQ1S_BF16": 81, "KK_OP_IQ1M_BF16": 91, "KK_OP_TQ1_0_BF16": 84, "KK_OP_TQ2_0_BF16": 63,
}


@pytest.fixture(scope="module")
def analysis():
    return sass_budget.analyse()


def test_instruction_mix_proves_the_design(analysis):
    _, total, mix = analysis
    assert mix["UBLKCP"] >= 10, "TMA bulk copies (cp.async.bulk -> UBLKCP.S.G in, UBLKCP.G.S out x 8 destinations) must be in the kernel"
    assert mix["SYNCS"] >= 4, "mbarrier operations (SYNCS) pace the stage ring"
    assert not any(m in mix for m in ("STL", "LDL")), "local-memory traffic means the kernel spills"
    assert not any(m.startswith(("HMMA", "IMMA", "UTCHMMA", "UTCMMA", "UTCQMMA")) for m in mix), "byte work must not be shaped into tensor-core math"
    assert total < 20000


def test_hot_paths_stay_within_the_committed_budget(analysis):
    rows, _, _ = analysis
    got = {r["op"]: r.get("hot") for r in rows}
    found = [op for op in HOT_MAX if got.get(op)]
    assert len(found) >= len(HOT_MAX) - 4, f"hot paths found only for {found} (loop attribution changed?)"  # ptxas merges a few look-alike tails (IQ2_XS / IQ2_S / IQ3_S)
    per_kib = lambda op, n, table: n / (sum(table[op]) / 1024.0)  # noqa: E731
    over = {op: (round(per_kib(op, got[op], sass_budget.ITER_BYTES), 1), round(per_kib(op, HOT_MAX[op], sass_budget._ITER_BYTES_1X), 1)) for op in found
            if op not in ("KK_OP_F32_BF16", "KK_OP_F16_BF16") and per_kib(op, got[op], sass_budget.ITER_BYTES) > 1.08 * per_kib(op, HOT_MAX[op], sass_budget._ITER_BYTES_1X)}
    assert not over, f"hot paths grew past their budget (instructions per KiB: got, limit): {over}"


def test_issue_ceiling_of_every_dequantiser_clears_the_hbm_roofline(analysis):
    """The point of the budget: with one destination pool no consumer loop may saturate instruction issue before HBM saturates."""
    rows, _, _ = analysis
    rate = sass_budget.SM_COUNT * sass_budget.SM_GHZ * sass_budget.ISSUE_PER_CLK
    for r in rows:
        ib = sass_budget.ITER_BYTES.get(r["op"])
        if ib and r.get("hot"):
            ceiling = rate / r["hot"] * (ib[0] + ib[1])
            assert ceiling > 1.1 * sass_budget.HBM_PEAK_GBS, (r["op"], r["hot"], ceiling)
