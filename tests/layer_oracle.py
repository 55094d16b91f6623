"""Independent restatement of the pipeline-stage rule (kk_load_opts.layer_begin / layer_end, include/kukeon_gpuload.h) over the
oracle's index records.  It shares no code with the library: the stage tests compare the library's selection against this, and then
apply oracle.plan_pool / oracle.expected_pool to what it keeps.  It sits here, next to the tests that use it, because oracle/ is the
suite's fixed reference and a new feature's rule is added beside it rather than into it."""
from __future__ import annotations

import re
from typing import List, Optional, Tuple

EINVAL, EUNSUPPORTED = -1, -7
# the first "<container>.<N>." whose container is a whole dotted component
LAYER_RE = re.compile(r"^((?:[^.]*\.)*?)(layers|h|blk)\.(\d+)\.")
EMBED = ("embed_tokens.weight", "token_embd.weight", "wte.weight")
HEAD = ("lm_head.weight", "lm_head.bias", "norm.weight", "norm.bias", "ln_f.weight", "ln_f.bias")


class StageError(ValueError):
    def __init__(self, code: int, msg: str):
        super().__init__(msg)
        self.code = code


def layer_of(name: str) -> Optional[Tuple[str, int]]:
    """(stack, N): stack is the name up to and including "<container>."; None for a tensor without a layer."""
    m = LAYER_RE.match(name)
    return (m.group(1) + m.group(2) + ".", int(m.group(3))) if m else None


def n_layers(recs: List[dict]) -> int:
    return 1 + max((lo[1] for lo in map(layer_of, (r["name"] for r in recs)) if lo), default=-1)


def select_layers(recs: List[dict], begin: int, end: int) -> List[dict]:
    """The records stage [begin, end) keeps, in index order; raises StageError with the kk_status the library returns."""
    if end == 0 and begin == 0:
        return list(recs)
    if end == 0 or begin >= end:
        raise StageError(EINVAL, f"bad range [{begin}, {end})")
    stacks = {lo[0] for lo in map(layer_of, (r["name"] for r in recs)) if lo}
    if len(stacks) > 1:
        raise StageError(EUNSUPPORTED, f"two stacks {sorted(stacks)}")
    if not stacks:
        raise StageError(EUNSUPPORTED, "no layered tensors")
    n = n_layers(recs)
    if end > n:
        raise StageError(EINVAL, f"end {end} > {n} layers")
    first, last = begin == 0, end == n
    tied = not any(r["name"].endswith("lm_head.weight") or r["name"] == "output.weight" for r in recs)
    out = []
    for r in recs:
        name = r["name"]
        lo = layer_of(name)
        if lo:
            keep = begin <= lo[1] < end
        elif name.endswith(EMBED):
            keep = first or (last and tied)
        elif name.endswith("wpe.weight"):
            keep = first
        elif name == "output.weight" or name.endswith(HEAD):
            keep = last
        else:
            keep = True
        if keep:
            out.append(r)
    return out
