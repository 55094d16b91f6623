"""CPU tier: the load-shape resolver (kk_plan.cpp resolve_load_shape) through tests/emul/kk_load_shape_test, over every combination of
mode, fan-out, part count, device count, peer access and the scatter exchange flag.  The expected table is the loader's rule as it stood
before the resolver existed: model_load's checks in their order, do_load's `replicas`, the fill_dsts ladder and the `loaded` rule.  On one
GPU this is the only check of the single-process multi-device orders (push, replicas, NVLS, RAW over >= 2 devices)."""
import itertools
import json
import os
import subprocess

import pytest

from kukeon_b200 import gpupool as g

_HERE = os.path.dirname(os.path.abspath(__file__))
BIN = os.path.join(_HERE, "emul", "_build", "kk_load_shape_test")
EINVAL, EUNSUPPORTED = -1, -7

MODES = [-1, g.MODE_SINGLE, g.MODE_BROADCAST, g.MODE_SCATTER, 3]
FANOUTS = [-1, g.FANOUT_P2P, g.FANOUT_NVLS, g.FANOUT_NONE, g.FANOUT_RAW, g.FANOUT_PULL, 5]
PARTS = [(0, 0), (3, 1), (0, 2), (2, 3), (3, 3), (-1, 2), (1, 9), (7, 8)]  # (part_index, part_count)
N_DEVICES = [1, 2, 8]
PEER_OK = [0, 1]
FLAGS = [0, g.LOAD_SCATTER_EXCHANGE]
CASES = list(itertools.product(MODES, FANOUTS, FLAGS, PARTS, N_DEVICES, PEER_OK))


def expected(mode, fanout, flags, part_index, part_count, n_devices, peer_ok):
    """model_load's option checks and the loader's per-stage predicates, as written before they were resolved in one place."""
    if part_count <= 1:
        part_count, part_index = 1, 0
    if part_index < 0 or part_index >= part_count or part_count > g.KK_MAX_DEVICES:
        return {"status": EINVAL, "error": f"part {part_index} of {part_count} out of range"}
    if not g.MODE_SINGLE <= mode <= g.MODE_SCATTER:
        return {"status": EINVAL, "error": f"unknown mode {mode}"}
    if not g.FANOUT_P2P <= fanout <= g.FANOUT_PULL:
        return {"status": EINVAL, "error": f"unknown fanout {fanout}"}
    if fanout == g.FANOUT_NVLS:
        if mode != g.MODE_BROADCAST:
            return {"status": EUNSUPPORTED, "error": "fan-out NVLS only applies to KK_MODE_BROADCAST"}
        if part_count > 1:
            return {"status": EUNSUPPORTED,
                    "error": "fan-out NVLS needs one process owning all devices (sharing a multicast object across processes is not implemented)"}
        if n_devices < 2:
            return {"status": EUNSUPPORTED, "error": "fan-out NVLS needs at least two devices in the context"}
    if fanout == g.FANOUT_RAW and mode != g.MODE_BROADCAST:
        return {"status": EINVAL, "error": "KK_FANOUT_RAW only applies to KK_MODE_BROADCAST"}
    multi = part_count > 1
    if fanout == g.FANOUT_PULL and mode != g.MODE_BROADCAST:
        return {"status": EINVAL, "error": "KK_FANOUT_PULL only applies to KK_MODE_BROADCAST"}
    if fanout == g.FANOUT_PULL and not multi:
        return {"status": EINVAL, "error": "KK_FANOUT_PULL is for one-process-per-GPU operation (part_count > 1); one process owning the GPUs "
                                           "fans out with P2P stores"}
    if multi and n_devices != 1:
        return {"status": EINVAL, "error": f"multi-process parts need a one-device context (got {n_devices} devices)"}
    if multi and mode == g.MODE_SINGLE:
        return {"status": EINVAL, "error": "KK_MODE_SINGLE cannot be split into parts"}

    n_parts = 1 if mode == g.MODE_SINGLE else part_count if multi else n_devices
    local_parts = [part_index] if multi else [0] if mode == g.MODE_SINGLE else list(range(n_devices))
    bcast = mode == g.MODE_BROADCAST
    is_raw, is_pull, is_nvls = (bcast and fanout == f for f in (g.FANOUT_RAW, g.FANOUT_PULL, g.FANOUT_NVLS))
    replicas = not multi and bcast and len(local_parts) > 1 and (fanout == g.FANOUT_NONE or not peer_ok)
    # fill_dsts: the multicast object, the slice buffer, the own pool alone, or the peers' pools too (attached ones, or the context's when
    # peer access is on); RAW stages through raw_stage1 instead
    if is_raw:
        order = "raw"
    elif is_nvls:
        order = "nvls"
    elif is_pull:
        order = "pull"
    elif bcast and fanout != g.FANOUT_NONE and (multi or (peer_ok and len(local_parts) > 1)):
        order = "push"
    else:
        order = "replicas" if replicas else "own"
    return {"status": 0, "order": order, "multi_proc": int(multi), "rank": part_index, "n_parts": n_parts, "local_parts": local_parts,
            "every_part": int(replicas and not is_raw),  # do_load: RAW's stage 1 came first, then `replicas`
            "xdst": int(mode == g.MODE_SCATTER and bool(flags & g.LOAD_SCATTER_EXCHANGE) and n_parts > 1),
            "peer_ok": peer_ok, "two_stage": int((is_raw or is_pull) and multi)}


@pytest.fixture(scope="module")
def resolved(native):
    subprocess.run(["make", "-C", os.path.join(_HERE, "emul"), "-s"], check=True)
    r = subprocess.run([BIN], input="".join(f"{m} {f} {x} {i} {n} {d} {p}\n" for m, f, x, (i, n), d, p in CASES),
                       capture_output=True, text=True, timeout=60, check=True)
    lines = r.stdout.splitlines()
    assert len(lines) == len(CASES), r.stderr[-500:]
    return {case: json.loads(line) for case, line in zip(CASES, lines)}


def test_every_combination_resolves_as_the_loader_decided(resolved):
    bad = []
    for case in CASES:
        mode, fanout, flags, (part_index, part_count), n_devices, peer_ok = case
        want = expected(mode, fanout, flags, part_index, part_count, n_devices, peer_ok)
        if resolved[case] != want:
            bad.append((case, resolved[case], want))
    assert not bad, f"{len(bad)} of {len(CASES)} cases differ, first: {bad[:3]}"


def test_the_grid_reaches_every_order_and_every_refusal(resolved):
    assert {r["order"] for r in resolved.values() if r["status"] == 0} == {"own", "replicas", "push", "nvls", "raw", "pull"}
    errors = {r["error"] for r in resolved.values() if r["status"] != 0}
    for what in ("out of range", "unknown mode", "unknown fanout", "NVLS only applies", "one process owning all devices", "at least two devices",
                 "KK_FANOUT_RAW only applies", "KK_FANOUT_PULL only applies", "one-process-per-GPU", "one-device context", "cannot be split"):
        assert any(what in e for e in errors), what


# (mode, fanout, flags, (part_index, part_count), n_devices, peer_ok) -> what the loader does with it
PINNED = [
    # NVLS in a context without peer access: every device converts every part, each through the multicast destination
    ((g.MODE_BROADCAST, g.FANOUT_NVLS, 0, (0, 0), 2, 0), {"order": "nvls", "every_part": 1, "two_stage": 0}),
    ((g.MODE_BROADCAST, g.FANOUT_NVLS, 0, (0, 0), 2, 1), {"order": "nvls", "every_part": 0, "two_stage": 0}),
    # single-process RAW converts in the same kk_load; one rank of a multi-process RAW or PULL load waits for kk_convert_local
    ((g.MODE_BROADCAST, g.FANOUT_RAW, 0, (0, 0), 2, 1), {"order": "raw", "every_part": 0, "two_stage": 0}),
    ((g.MODE_BROADCAST, g.FANOUT_RAW, 0, (0, 0), 2, 0), {"order": "raw", "every_part": 0, "two_stage": 0}),
    ((g.MODE_BROADCAST, g.FANOUT_RAW, 0, (2, 3), 1, 0), {"order": "raw", "two_stage": 1, "local_parts": [2]}),
    ((g.MODE_BROADCAST, g.FANOUT_PULL, 0, (2, 3), 1, 0), {"order": "pull", "two_stage": 1, "local_parts": [2]}),
    # multi-process KK_FANOUT_NONE broadcast: its own part only, loaded after kk_load_part
    ((g.MODE_BROADCAST, g.FANOUT_NONE, 0, (2, 3), 1, 0), {"order": "own", "every_part": 0, "two_stage": 0, "local_parts": [2]}),
    ((g.MODE_BROADCAST, g.FANOUT_P2P, 0, (0, 0), 8, 0), {"order": "replicas", "every_part": 1}),
    ((g.MODE_BROADCAST, g.FANOUT_P2P, 0, (0, 0), 8, 1), {"order": "push", "every_part": 0, "local_parts": list(range(8))}),
    # the scatter row exchange needs every rank's pool, with or without peer access (fill_dsts then reports it unreachable)
    ((g.MODE_SCATTER, g.FANOUT_P2P, g.LOAD_SCATTER_EXCHANGE, (0, 0), 2, 0), {"order": "own", "xdst": 1, "peer_ok": 0}),
    ((g.MODE_SCATTER, g.FANOUT_NONE, g.LOAD_SCATTER_EXCHANGE, (0, 0), 1, 0), {"order": "own", "xdst": 0, "n_parts": 1}),
]


@pytest.mark.parametrize("case,want", PINNED, ids=[str(c) for c, _ in PINNED])
def test_pinned_shapes(resolved, case, want):
    got = resolved[case]
    assert got["status"] == 0 and {k: got[k] for k in want} == want, (case, got)
