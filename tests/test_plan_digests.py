"""Plans are pinned byte for byte: every plan of the corpus in tests/golden/make_plan_digests.py (golden and seeded synthetic checkpoints,
load shapes, flag sets, layer ranges, staging-chunk sizes) must hash to the digest tests/golden/plan_digests.json holds.  The other plan
tests check that plans produce the right pools; this one also pins where chunks are cut, how reads are laid out and how tiles are counted.
The corpus is checked to reach every plannable op, the row exchange, the four transposes, un-permuted Q/K pieces, split expert stacks
and a stage filter, so it cannot quietly shrink."""
import importlib.util
import json
import os

from kukeon_b200 import gpupool

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# every op code a plan can carry (kk_ops.h KKOp: 20-22 and 26-28 are unassigned)
PLANNABLE_OPS = set(range(0, 20)) | {23, 24, 25} | set(range(29, 39))
TRANSPOSES = {4, 5, 6, 7}
ROWSPLIT = 10


def _maker():
    spec = importlib.util.spec_from_file_location("make_plan_digests", os.path.join(G, "make_plan_digests.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _reached(plan: dict, flags: int, seen: dict) -> None:
    for part in plan["parts"]:
        for ch in part["chunks"]:
            seen["ops"].update(s["op"] for s in ch["segs"])
            # un-permuted Q/K rows: a (head, odd half) group reads file rows that lie before the even half's last row
            if flags & gpupool.LOAD_HF_LAYOUT and any(b[0] < a[0] for a, b in zip(ch["reads"], ch["reads"][1:])):
                seen["unpermuted"] = True
    seen["experts"] = seen["experts"] or any(".experts." in t["name"] for L in plan["layouts"] for t in L["tensors"])
    seen["stage"] = seen["stage"] or "layers" in plan


def test_plan_digests(tmp_path):
    mk = _maker()
    want = json.load(open(os.path.join(G, "plan_digests.json")))
    desc = mk.Describer(gpupool)
    seen = {"ops": set(), "unpermuted": False, "experts": False, "stage": False}
    ckpts = mk.corpus(str(tmp_path))
    assert sorted(name for name, _, _ in ckpts) == sorted(want)
    for name, path, root in ckpts:
        got = {}
        for (mode, n, fl), results in mk.plans(desc, path, root):
            key = mk.group_key(mode, n, fl)
            got[key] = mk.digest(results)
            assert got[key] == want[name].get(key), f"{name} {key}: the plans differ from the pinned ones"
            for _, _, r in results:
                if "json" in r:
                    _reached(json.loads(r["json"]), fl, seen)
        assert sorted(got) == sorted(want[name])
    assert PLANNABLE_OPS <= seen["ops"], f"ops the corpus does not reach: {sorted(PLANNABLE_OPS - seen['ops'])}"
    assert ROWSPLIT in seen["ops"] and TRANSPOSES <= seen["ops"]
    assert seen["unpermuted"], "no plan un-permutes Q/K rows"
    assert seen["experts"], "no plan splits an expert stack"
    assert seen["stage"], "no plan filters a layer range"
