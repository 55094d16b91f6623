"""The fp16-output kernel (kk_convert_f16_kernel, KK_LOAD_F16), checked on the CPU tier from its SASS like tests/test_sass_budget.py checks
the bf16 one: the same design (TMA bulk copies, mbarriers, no local memory, no spills), no more registers than the bf16 kernel, every op's
hot path within 5 % of the bf16 kernel's for that op in the same build, and every loop's issue ceiling above the HBM roofline."""
import shutil

import pytest

from tools import sass_budget

pytestmark = pytest.mark.skipif(shutil.which("nvcc") is None or shutil.which("nvdisasm") is None, reason="needs the CUDA toolkit (nvcc, nvdisasm)")

BF16, F16 = "kk_convert_kernel", "kk_convert_f16_kernel"


@pytest.fixture(scope="module")
def build():
    text, res = sass_budget.disassemble(resources=True)
    return text, res, sass_budget.analyse(BF16, text), sass_budget.analyse(F16, text)


def resources(res, kernel):
    hit = [v for k, v in res.items() if kernel + "E" in k]  # the mangled name ends "<len>kk_convert..._kernelE<params>"
    assert len(hit) == 1, (kernel, list(res))
    return hit[0]


def test_the_kernels_are_told_apart():
    assert BF16 not in F16, "tools/sass_budget.py finds the bf16 kernel by its name as a substring"


def test_instruction_mix_no_spills_no_local_memory(build):
    _, res, _, (_, total, mix) = build
    assert mix["UBLKCP"] >= 10 and mix["SYNCS"] >= 4
    assert not any(m in mix for m in ("STL", "LDL")), "local-memory traffic means the kernel spills"
    assert not any(m.startswith(("HMMA", "IMMA")) for m in mix)
    r = resources(res, F16)
    assert r["STACK"] == 0 and r["LOCAL"] == 0
    assert 0 < total < 20000


def test_no_more_registers_than_the_bf16_kernel(build):
    _, res, _, _ = build
    assert resources(res, F16)["REG"] <= resources(res, BF16)["REG"]


def test_every_hot_path_within_5_percent_of_the_bf16_kernel(build):
    _, _, (rows_b, _, _), (rows_h, _, _) = build
    hb = {r["op"]: r.get("hot") for r in rows_b if r.get("hot")}
    hh = {r["op"]: r.get("hot") for r in rows_h if r.get("hot")}
    assert len(hb) >= 25 and set(hb) <= set(hh), (sorted(hb), sorted(hh))
    over = {op: (hh[op], hb[op]) for op in hb if hh[op] > 1.05 * hb[op]}
    assert not over, f"f16 hot paths more than 5 % above the bf16 kernel's (f16, bf16): {over}"


def test_issue_ceiling_clears_the_hbm_roofline(build):
    _, _, _, (rows, _, _) = build
    rate = sass_budget.SM_COUNT * sass_budget.SM_GHZ * sass_budget.ISSUE_PER_CLK
    n = 0
    for r in rows:
        ib = sass_budget.ITER_BYTES.get(r["op"])
        if ib and r.get("hot"):
            assert rate / r["hot"] * (ib[0] + ib[1]) > 1.1 * sass_budget.HBM_PEAK_GBS, (r["op"], r["hot"])
            n += 1
    assert n >= 25
