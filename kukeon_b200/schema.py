""""next" row f3 of SURVEY.md §8(f): the manifest surface for GPU-resident weights, as a Python model of the Go code a kukeon
maintainer would add (Go is not installed here; INTEGRATION.md has the transliteration).

Proposed schema — `models[]` on a v1beta1 ContainerSpec, next to `volumes[]` (pkg/api/model/v1beta1/container.go:206-213):

    containers:
      - id: work
        models:
          - name: llama            # unique per container; becomes /run/kukeon/gpupool/<name> when more than one is mounted
            source: /models/llama-3-8b        # absolute host path: directory (index.json / *.safetensors / *.gguf) or one file
            mode: broadcast        # single | broadcast | scatter      (kk_mode; default single)
            devices: [0, 1]        # CUDA ordinals the agent may attach to (default: every device of the daemon's pool)
            layers: [0, 16]        # pipeline stage: only layers [begin, end) of the checkpoint (default: all of them)
            adapter: /models/llama-3-8b-lora  # absolute host path of a PEFT LoRA adapter merged into the pool on the GPU (default: none)
            target: /run/kukeon/gpupool       # absolute container path of the read-only manifest mount (default shown)
            options: {gpt2Conv1dTranspose: false, keepF32: false, f8ToBf16: false}

`validate_models` is the sibling of `validateVolumes` (internal/controller/create_container.go:284-380): same order of checks, same
error style — a sentinel (here: an attribute of `Err`, named as it would be in internal/errdefs/errdefs.go:131-144) wrapped with
the offending index and value, `"%w (model[%d] source %q)"`.  Nothing here touches a GPU.
"""
from __future__ import annotations

import os
import re
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

from . import gpupool

DEFAULT_TARGET = "/run/kukeon/gpupool"
MODES = {"": gpupool.MODE_SINGLE, "single": gpupool.MODE_SINGLE, "broadcast": gpupool.MODE_BROADCAST, "scatter": gpupool.MODE_SCATTER}
OPTION_FLAGS = {"gpt2Conv1dTranspose": gpupool.LOAD_GPT2_CONV1D_T, "keepF32": gpupool.LOAD_KEEP_F32, "f8ToBf16": gpupool.LOAD_F8_TO_BF16,
                "f16": gpupool.LOAD_F16, "hfLayout": gpupool.LOAD_HF_LAYOUT}


MODEL_NAME_RE = re.compile(r"^[A-Za-z0-9][A-Za-z0-9._-]*$")


class Err:
    """Sentinels, worded like internal/errdefs/errdefs.go's volume block."""
    ModelNameRequired = "model name is required"
    ModelNameDuplicate = "model name is declared more than once in the container"
    ModelNameInvalid = "model name must be one path component of letters, digits, '.', '_' or '-' (it becomes a directory and an env-name suffix)"
    ModelSourceRequired = "model source is required"
    ModelSourceNotAbsolute = "model source must be an absolute host path"
    ModelSourceNotFound = "model source does not exist on the host"
    ModelTargetNotAbsolute = "model target must be an absolute container path"
    ModelModeUnknown = 'model mode is not recognized; expected "", "single", "broadcast", or "scatter"'
    ModelDevicesInvalid = "model devices must be distinct non-negative CUDA ordinals"
    ModelLayersInvalid = "model layers must be [begin, end): two non-negative integers with begin < end"
    ModelOptionUnknown = "model option is not recognized"
    ModelRegistryNotSupported = "registry references are not supported; use an absolute host path as source"
    ModelAdapterNotAbsolute = "model adapter must be an absolute host path"
    ModelAdapterNotFound = "model adapter does not exist on the host"
    ModelAdapterRegistryNotSupported = "adapter registry references are not supported; use an absolute host path as adapter"


class SchemaError(ValueError):
    """`errors.Is(err, sentinel)` is `e.sentinel == Err.X`; str(e) is the wrapped message."""

    def __init__(self, sentinel: str, detail: str):
        super().__init__(f"{sentinel} ({detail})")
        self.sentinel = sentinel


@dataclass
class ModelSpec:
    name: str
    source: str
    mode: int = gpupool.MODE_SINGLE
    devices: List[int] = field(default_factory=list)
    target: str = DEFAULT_TARGET
    flags: int = 0
    layers: Optional[Tuple[int, int]] = None  # pipeline stage [begin, end); None: the whole checkpoint
    adapter: Optional[str] = None  # PEFT LoRA adapter merged on load (kk_load_adapter); None: the base checkpoint alone


def _q(s: str) -> str:
    return '"' + s.replace("\\", "\\\\").replace('"', '\\"') + '"'  # Go's %q for the strings that occur here


def validate_models(models: Optional[List[dict]], stat=os.stat) -> List[ModelSpec]:
    out: List[ModelSpec] = []
    seen = set()
    for i, m in enumerate(models or []):
        name = str(m.get("name") or "").strip()
        if not name:
            raise SchemaError(Err.ModelNameRequired, f"model[{i}]")
        if not MODEL_NAME_RE.match(name) or name in (".", ".."):
            # the name is joined into <cell dir>/gpupool/<name> on the host and into the mount target in the container: "../x", "a/b" or a NUL
            # would let a manifest write outside the cell directory.  Refused here, before anything is loaded or a refcount is taken.
            raise SchemaError(Err.ModelNameInvalid, f"model[{i}] name {_q(name)}")
        if name in seen:
            raise SchemaError(Err.ModelNameDuplicate, f"model[{i}] name {_q(name)}")
        seen.add(name)
        src = str(m.get("source") or "").strip()
        if not src:
            raise SchemaError(Err.ModelSourceRequired, f"model[{i}]")
        if not os.path.isabs(src):
            # "org/name" or "hf://..." look like registry references: point at the deferred feature, like ErrVolumeNamedNotSupported does
            if "://" in src or (os.sep in src and not src.startswith(".")):
                raise SchemaError(Err.ModelRegistryNotSupported, f"model[{i}] source {_q(src)}")
            raise SchemaError(Err.ModelSourceNotAbsolute, f"model[{i}] source {_q(src)}")
        try:
            stat(src)
        except FileNotFoundError:
            raise SchemaError(Err.ModelSourceNotFound, f"model[{i}] source {_q(src)}") from None
        except OSError as e:
            raise ValueError(f"failed to stat model[{i}] source {_q(src)}: {e}") from e
        adapter = m.get("adapter")
        if adapter is not None:
            adapter = str(adapter).strip()
            if not os.path.isabs(adapter):
                if "://" in adapter or (os.sep in adapter and not adapter.startswith(".")):
                    raise SchemaError(Err.ModelAdapterRegistryNotSupported, f"model[{i}] adapter {_q(adapter)}")
                raise SchemaError(Err.ModelAdapterNotAbsolute, f"model[{i}] adapter {_q(adapter)}")
            try:
                stat(adapter)
            except FileNotFoundError:
                raise SchemaError(Err.ModelAdapterNotFound, f"model[{i}] adapter {_q(adapter)}") from None
            except OSError as e:
                raise ValueError(f"failed to stat model[{i}] adapter {_q(adapter)}: {e}") from e
        target = str(m.get("target") or DEFAULT_TARGET).strip()
        if not os.path.isabs(target):
            raise SchemaError(Err.ModelTargetNotAbsolute, f"model[{i}] target {_q(target)}")
        mode = str(m.get("mode") or "").strip().lower()
        if mode not in MODES:
            raise SchemaError(Err.ModelModeUnknown, f"model[{i}] mode {_q(mode)}")
        devs = m.get("devices") or []
        if not isinstance(devs, list) or any(isinstance(d, bool) or not isinstance(d, int) or d < 0 for d in devs) or len(set(devs)) != len(devs) \
                or len(devs) > gpupool.KK_MAX_DEVICES:
            raise SchemaError(Err.ModelDevicesInvalid, f"model[{i}] devices {devs!r}")
        layers = m.get("layers")
        if layers is not None:
            if not isinstance(layers, list) or len(layers) != 2 or any(isinstance(v, bool) or not isinstance(v, int) or not 0 <= v < 2**32 for v in layers) \
                    or layers[0] >= layers[1]:
                raise SchemaError(Err.ModelLayersInvalid, f"model[{i}] layers {layers!r}")
            layers = (layers[0], layers[1])
        flags = 0
        for k, v in (m.get("options") or {}).items():
            if k not in OPTION_FLAGS:
                raise SchemaError(Err.ModelOptionUnknown, f"model[{i}] option {_q(str(k))}")
            if v:
                flags |= OPTION_FLAGS[k]
        out.append(ModelSpec(name=name, source=src, mode=MODES[mode], devices=list(devs), target=target, flags=flags, layers=layers,
                             adapter=adapter))
    return out


def models_of_cell(doc: dict, stat=os.stat) -> Dict[str, List[ModelSpec]]:
    """A parsed v1beta1 Cell manifest (docs/examples/claude-code/cell.yaml shape) -> {container id: validated models}."""
    if not isinstance(doc, dict) or doc.get("kind") != "Cell":
        raise ValueError(f"expected kind Cell, got {doc.get('kind') if isinstance(doc, dict) else type(doc).__name__!r}")
    out: Dict[str, List[ModelSpec]] = {}
    for c in (doc.get("spec") or {}).get("containers") or []:
        try:
            specs = validate_models(c.get("models"), stat)
        except SchemaError as e:
            raise SchemaError(e.sentinel, f"container {_q(str(c.get('id', '')))}: {str(e)[len(e.sentinel) + 2:-1]}") from None
        if specs:
            out[str(c.get("id", ""))] = specs
    return out
